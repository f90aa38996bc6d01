"""Caption-to-image retrieval evaluation on the device: the drop-in for the loop of eval_retrieval.py:253-358 (fine-tuned TASK7 /
TASK8 model) and of evaluation/eval_coco_retrieval.py:336-412 (zero-shot pre-trained model).

    from vilbert_b200.retrieval import RetrievalEvaluator, evaluate_retrieval, retrieval_metrics

    ev = RetrievalEvaluator(model, features, spatials, image_mask, chunk=500)   # gallery [G, Nv, 2048] / [G, Nv, 5] / [G, Nv]
    scores = ev.score(captions, input_mask, segment_ids, task_id=8)            # device f32 [C, G]
    ranks, topk = ev.rank(scores, target_image, k=20)                           # device int32 [C], [C, k]
    r1, r5, r10, medr, meanr = retrieval_metrics(ranks)

    r1, r5, r10, medr, meanr, results = evaluate_retrieval(model, dataset, task_id="TASK8")

Image-to-text retrieval (text retrieval) from the same score matrix: each image's rank is that of its best-placed ground-truth
caption (vb_retrieval_rank_sets), with the same tie and NaN order.

    ranks_i, topk_i = ev.rank_captions(scores, target_image, k=20)              # device int32 [G], [G, k]
    (r1, r5, r10, medr, meanr), n_without = i2t_metrics(ranks_i)
    out = evaluate_retrieval_both(model, dataset, task_id="TASK8")             # {"t2i", "i2t", "rsum", "images_without_caption"}

The reference scores every caption against the same gallery with one model call per caption and gallery half, so each call moves
the half's region features to the device and embeds them again. Here the work runs chunk outer, caption inner: a chunk of images
is loaded and embedded once (Plan(image_prefix=True).run_image_prefix()), then every caption costs a few device-to-device copies
from a caption bank uploaded once and one replay of a fast-mode forward (text batch 1 broadcast to the chunk) that builds only the
score head. Scores stay on the device; vb_retrieval_rank ranks them there, and one read-back returns ranks and top-k lists.
With pack=True (or engine.pack_padding) each pair runs on a plan that holds the chunk's valid regions and the caption's valid
tokens only (retrieval_pack_plan, DESIGN.md §4e).

Across GPUs (torchrun, one rank per GPU): pass group= (e.g. dist.group.WORLD) to score() / evaluate_retrieval*(). Each of the W
ranks scores its contiguous caption block (shard_bounds) against the whole gallery, the blocks are gathered into the same [C, G]
matrix on every rank (gather_rows), and every rank ranks it and returns the same metrics and lists. A fixed-length vector of the
shapes, options and exact checksums of the inputs and weights is compared first (check_agreement), so ranks called with other
data or weights raise ValueError instead of hanging or gathering a wrong matrix. group=None runs on one GPU with no
torch.distributed call.

    out = evaluate_retrieval_both(model, dataset, task_id="TASK8", group=dist.group.WORLD)     # same result on every rank

Differences from the reference: equal scores are ordered by image index (the reference's default argsort leaves their order
unspecified), and progress is logged once per chunk rather than after every caption (no caption has a full score row before the
last chunk).
"""
import logging
from collections import OrderedDict

import numpy as np
import torch
import torch.distributed as dist

from . import _lib as L
from .engine import PRECISIONS, pack_capacity

logger = logging.getLogger(__name__)

# the score head of each model kind (Engine heads): VILBertForVLTasks' vil_logit (eval_retrieval.py:299-310), the pre-training
# model's alignment logits, scored as softmax(logits, 1)[:, 0] (eval_coco_retrieval.py:357-363)
SCORE_HEAD = {"vl": "vil_logit", "pretraining": "seq_relationship_score"}
MAX_TOPK = 64            # vb_retrieval_rank[_sets]: k <= 64
MAX_GALLERY = 50000      # ... and at most 50,000 columns per row (images, or captions for rank_captions)


def retrieval_metrics(ranks):
    """(r1, r5, r10, medr, meanr) of 0-based target ranks with the reference's formulas (eval_retrieval.py:340-345). A rank of -1
    (the target is outside the gallery) raises IndexError, as the reference's np.where(...)[0][0] does."""
    r = ranks.detach().cpu().numpy() if torch.is_tensor(ranks) else np.asarray(ranks)
    r = r.astype(np.float64)
    if (r < 0).any():
        raise IndexError("retrieval_metrics: a caption's target image is not in the gallery")
    r1 = 100.0 * np.sum(r < 1) / len(r)
    r5 = 100.0 * np.sum(r < 5) / len(r)
    r10 = 100.0 * np.sum(r < 10) / len(r)
    medr = np.floor(np.median(r) + 1)
    meanr = np.mean(r) + 1
    return r1, r5, r10, medr, meanr


def _task_number(task_id):
    """eval_retrieval.py:269-271 fills the task tokens with int(task_id[4:]): "TASK8" -> 8; an int passes through."""
    if isinstance(task_id, str):
        return int(task_id[4:])
    return int(task_id)


def read_retrieval_dataset(dataset):
    """The reference's retrieval item protocol (RetreivalDatasetVal.__getitem__, retreival_dataset.py:430-468): item 2c + h is
    (features, spatials, image_mask, caption, input_mask, segment_ids, target, caption_idx, image_idx) of caption c against gallery
    half h. Returns the gallery (the two halves of items 0 and 1, concatenated), the captions in item order (int64 [C, Nt] each) and
    every caption's target: the first image whose target is 1 (np.where(...)[0][0]); a caption without one raises IndexError."""
    n = len(dataset)
    if n < 2 or n % 2:
        raise ValueError(f"retrieval dataset: {n} items; expected two gallery halves per caption")
    halves = [dataset[0], dataset[1]]
    feats = torch.cat([torch.as_tensor(h[0]) for h in halves])
    spats = torch.cat([torch.as_tensor(h[1]) for h in halves])
    imask = torch.cat([torch.as_tensor(h[2]) for h in halves])
    caps, masks, segs, targets = [], [], [], []
    for c in range(n // 2):
        a, b = (halves[0], halves[1]) if c == 0 else (dataset[2 * c], dataset[2 * c + 1])
        caps.append(torch.as_tensor(a[3]).reshape(-1))
        masks.append(torch.as_tensor(a[4]).reshape(-1))
        segs.append(torch.as_tensor(a[5]).reshape(-1))
        t = np.concatenate([np.asarray(torch.as_tensor(a[6]).reshape(-1).float()), np.asarray(torch.as_tensor(b[6]).reshape(-1).float())])
        hit = np.where(t == 1)[0]
        if len(hit) == 0:
            raise IndexError(f"retrieval dataset: caption {c} has no target image")
        targets.append(int(hit[0]))
    return (feats, spats, imask, torch.stack(caps).long(), torch.stack(masks).long(), torch.stack(segs).long(),
            torch.tensor(targets, dtype=torch.int64))


def _row_lengths(mask):
    """(valid entries per row, whether the row is prefix-valid and non-empty) of a 0/1 host mask [rows, N]."""
    m = mask.ne(0)
    n = m.sum(1)
    return n, (n >= 1) & m.eq(torch.arange(m.size(1)).unsqueeze(0) < n.unsqueeze(1)).all(1)


def retrieval_pack_plan(image_mask, caption_mask, chunk, has_task):
    """The host decision of a packed retrieval evaluation from the gallery's and the captions' host masks ([G, Nv], [C, Nt]):
    -> (chunks, fallback chunks, fallback captions). Each chunk is (first image, images n, rows_v, groups); groups maps the text
    capacity rows_t of a packed plan to its captions, in ascending order, after the padded group (key None) if there is one.
    A chunk packs its valid regions, rows_v = pack_capacity(valid regions, n * Nv); a caption of L valid rows (task token
    included) is broadcast to the n images as n * L rows, rows_t = pack_capacity(n * L, n * Nt). A chunk with an image row that
    is not prefix-valid or empty runs every caption padded (rows_v None); a caption whose mask is not prefix-valid runs padded on
    every chunk."""
    G, Nv = image_mask.shape
    Nt = caption_mask.shape[1] + has_task
    nv, ok_v = _row_lengths(image_mask)
    nt, ok_t = _row_lengths(caption_mask)
    lengths = (nt + has_task).tolist()
    ok_t = ok_t.tolist()
    chunks, bad_chunks = [], 0
    for lo in range(0, G, chunk):
        n = min(chunk, G - lo)
        if not bool(ok_v[lo:lo + n].all()):
            chunks.append((lo, n, None, {None: list(range(len(lengths)))}))
            bad_chunks += 1
            continue
        cap = {L: pack_capacity(n * L, n * Nt) for L in set(lengths)}
        groups = {}
        for c, (L, ok) in enumerate(zip(lengths, ok_t)):
            groups.setdefault(cap[L] if ok else None, []).append(c)
        order = sorted(groups, key=lambda k: -1 if k is None else k)
        chunks.append((lo, n, pack_capacity(int(nv[lo:lo + n].sum()), n * Nv), OrderedDict((k, groups[k]) for k in order)))
    return chunks, bad_chunks, ok_t.count(False)


# ------------------------------------------------------------------------------------------ across GPUs
# the fields of the vector every rank all-gathers before scoring (check_agreement), in order
AGREEMENT_FIELDS = ("captions", "caption length", "images", "regions", "chunk", "pack", "head", "task", "precision",
                    "deterministic", "caption ids", "caption masks", "segment ids", "image masks", "image features",
                    "image spatials", "parameters")


def shard_bounds(C, world):
    """Each rank's contiguous caption block [lo, hi): rank r scores [r·C // W, (r+1)·C // W). Every caption lands in exactly one
    block, in order, and block sizes differ by at most one; with C < W some blocks are empty."""
    return [(r * C // world, (r + 1) * C // world) for r in range(world)]


def checksum(t):
    """The int64 sum of t's bytes read as int32 bit patterns (zero-padded to a multiple of 4 bytes). Integer sums are exact, so
    the value does not depend on summation order or device: equal tensors give equal checksums on every rank."""
    b = t.detach().contiguous().reshape(-1).view(torch.uint8)
    if b.numel() % 4 or b.storage_offset() % 4:
        b = torch.cat((b, b.new_zeros(-b.numel() % 4)))
    return int(b.view(torch.int32).sum(dtype=torch.int64))


def _comm_device(group, device):
    """Where a collective's tensors live: `device` with NCCL, the host with gloo (or any other backend)."""
    return torch.device(device) if "nccl" in str(dist.get_backend(group)) else torch.device("cpu")


def check_agreement(fields, group, device="cpu"):
    """All-gathers {AGREEMENT_FIELDS name: int} over `group` (one fixed-length int64 vector per rank) and raises ValueError on
    every rank, naming each field on which the ranks differ. The vector's length does not depend on the inputs, so this
    collective is safe to enter with any arguments; the ones whose sizes do depend on them come after it."""
    mine = torch.tensor([int(fields[n]) for n in AGREEMENT_FIELDS], dtype=torch.int64, device=_comm_device(group, device))
    world = dist.get_world_size(group)
    every = torch.empty(world * mine.numel(), dtype=torch.int64, device=mine.device)
    dist.all_gather_into_tensor(every, mine, group=group)
    every = every.view(world, -1).cpu()
    bad = [f"{n} {every[:, i].tolist()}" for i, n in enumerate(AGREEMENT_FIELDS) if bool((every[:, i] != every[0, i]).any())]
    if bad:
        raise ValueError(f"retrieval across {world} ranks: every rank must call with the same data, options and weights; "
                         f"they differ in: {'; '.join(bad)} (per rank)")


def gather_rows(block, C, group):
    """The [C, G] matrix made of every rank's block of rows (shard_bounds(C, W), this rank's is `block`), in caption order, on
    every rank of `group`. The blocks are padded to ceil(C / W) rows and gathered with one all_gather_into_tensor on block's
    device."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    bounds = shard_bounds(C, world)
    lo, hi = bounds[rank]
    if block.shape[0] != hi - lo:
        raise ValueError(f"rank {rank}: a block of {block.shape[0]} rows; shard_bounds gives it {hi - lo}")
    per = -(-C // world)
    padded = block.new_zeros((per, block.shape[1]))
    padded[:hi - lo] = block
    every = block.new_empty((world * per, block.shape[1]))
    dist.all_gather_into_tensor(every, padded, group=group)
    return torch.cat([every[r * per:r * per + (b - a)] for r, (a, b) in enumerate(bounds)])


class RetrievalEvaluator:
    """Scores captions against a fixed image gallery on fast-mode forward-only plans with a precomputed image prefix.

    model: VILBertForVLTasks (scores = vil_logit) or BertForMultiModalPreTraining (zero shot: softmax(seq_relationship_score, 1)[:, 0]),
    in eval mode. features f32 [G, Nv, 2048], spatials f32 [G, Nv, 5], image_mask [G, Nv], on the host (staged through pinned memory
    one chunk at a time) or on the model's device. Chunks of `chunk` images share one plan; a smaller last chunk gets its own.
    recycle: build the plans with their buffers placed by lifetime (Plan(recycle=True)), which holds a fraction of the bytes at the
    same launches and scores; None takes engine.recycle_forward_only.

    pack: score each (caption, chunk) pair on a packed plan (Plan(packed=...), DESIGN.md §4g) that holds the chunk's valid regions and
    the caption's valid tokens only; None follows engine.pack_padding. The decision is taken on the host from the masks
    (retrieval_pack_plan): a chunk whose image mask is not prefix-valid or has an empty row, and a caption whose mask is not
    prefix-valid, run on the padded plan and are counted in engine.pack_fallbacks["mask"]."""

    def __init__(self, model, features, spatials, image_mask, chunk=500, recycle=None, pack=None):
        self.model = model
        heads = getattr(model, "_heads", None)
        if heads not in SCORE_HEAD:
            raise TypeError("RetrievalEvaluator scores with VILBertForVLTasks or BertForMultiModalPreTraining")
        if model.training:
            raise ValueError("RetrievalEvaluator runs forward-only plans: call model.eval() first")
        if features.dim() != 3 or spatials.shape[:2] != features.shape[:2] or tuple(image_mask.shape) != tuple(features.shape[:2]):
            raise ValueError("gallery: features [G, Nv, F], spatials [G, Nv, 5] and image_mask [G, Nv]")
        if torch.is_grad_enabled() and (features.requires_grad or spatials.requires_grad):
            raise ValueError("RetrievalEvaluator runs forward-only plans: it computes no gradient of the gallery's features or spatials")
        self.G, self.Nv = int(features.shape[0]), int(features.shape[1])
        if self.G > MAX_GALLERY:
            raise ValueError(f"gallery of {self.G} images: the device ranking supports at most {MAX_GALLERY}")
        if chunk < 1:
            raise ValueError("chunk must be positive")
        self.features, self.spatials, self.image_mask = features, spatials, image_mask
        self.chunk = min(int(chunk), self.G)
        self.heads = heads
        self.head = SCORE_HEAD[heads]
        self.recycle = recycle
        self.pack = pack

    def _plan(self, n, Nt, packed=None):
        return self.model.engine.plan(n, Nt, self.Nv, heads=self.heads, outputs=(self.head,), fast_mode=True, image_prefix=True,
                                      recycle=self.recycle, packed=packed)

    def _chunks(self, input_mask, has_task):
        """The chunks of a score() call as retrieval_pack_plan gives them; without packing every chunk has the padded group only.
        Packing counts its fallbacks in engine.pack_fallbacks["mask"]. Masks already on the device are copied to the host once
        here, never per caption."""
        eng = self.model.engine
        if not (self.pack if self.pack is not None else eng.pack_padding):
            C = int(input_mask.shape[0])
            return [(lo, min(self.chunk, self.G - lo), None, {None: range(C)}) for lo in range(0, self.G, self.chunk)]
        chunks, bad_chunks, bad_captions = retrieval_pack_plan(self.image_mask.cpu(), input_mask.cpu(), self.chunk, int(has_task))
        if bad_chunks + bad_captions:
            eng.pack_fallbacks["mask"] += bad_chunks + bad_captions
        return chunks

    def _load_chunk(self, plan, lo, n):
        dev = self.model.engine.device
        parts = []
        for t in (self.features, self.spatials, self.image_mask):
            x = t[lo:lo + n]
            if x.device.type == "cpu" and not x.is_pinned():
                x = x.pin_memory()          # asynchronous upload; the caching host allocator keeps it alive until the copy ran
            parts.append(x if x.device == dev or x.device.type == "cpu" else x.to(dev))
        plan.load_images(*parts)
        plan.run_image_prefix()

    def score(self, captions, input_mask, segment_ids, task_id=None, group=None):
        """Device f32 [C, G]: the score of every caption (int64 [C, Nt], with its mask and segment ids) against every image.
        task_id (int or "TASKn") sets the task tokens of a model with config.task_specific_tokens; the pre-training model takes
        none (TypeError, as its forward has no task_ids parameter).

        group: a torch.distributed process group. None, or a group of one rank, scores every caption here and makes no
        torch.distributed call. With W > 1 ranks, every rank must call with the same arguments (and evaluators built alike): the
        ranks first compare the shapes, options and checksums of the inputs and the weights (check_agreement, ValueError on
        every rank if they differ), rank r then scores its caption block shard_bounds(C, W)[r] against the whole gallery, and
        every rank returns the same gathered [C, G] (gather_rows). A rank with an empty block scores nothing but joins both
        collectives. Packing is decided per rank on its block, so engine.pack_fallbacks counts what this rank ran: a chunk that
        falls back is counted once on every rank with captions."""
        model, eng = self.model, self.model.engine
        if self.heads == "pretraining" and task_id is not None:
            raise TypeError("BertForMultiModalPreTraining.forward() takes no task_ids (vilbert.py:1471-1484): score without task_id")
        if model.training:
            raise ValueError("RetrievalEvaluator runs forward-only plans: call model.eval() first")
        has_task = bool(model.config.task_specific_tokens) and self.heads == "vl"
        if has_task and task_id is None:
            raise ValueError("config.task_specific_tokens is set: task_id is required")
        world = 1 if group is None else dist.get_world_size(group)
        if world == 1:
            return self._score_rows(captions, input_mask, segment_ids, task_id, has_task)
        C = int(captions.shape[0])
        check_agreement(self._agreement(captions, input_mask, segment_ids, task_id), group, eng.device)
        lo, hi = shard_bounds(C, world)[dist.get_rank(group)]
        if hi > lo:
            block = self._score_rows(captions[lo:hi], input_mask[lo:hi], segment_ids[lo:hi], task_id, has_task)
        else:
            block = torch.empty((0, self.G), dtype=torch.float32, device=eng.device)
        return gather_rows(block.to(_comm_device(group, eng.device)), C, group).to(eng.device)

    def _agreement(self, captions, input_mask, segment_ids, task_id):
        """This rank's check_agreement fields for a score() call."""
        eng = self.model.engine
        return dict(zip(AGREEMENT_FIELDS, (
            captions.shape[0], captions.shape[1], self.G, self.Nv, self.chunk,
            self.pack if self.pack is not None else eng.pack_padding, list(SCORE_HEAD).index(self.heads),
            -1 if task_id is None else _task_number(task_id), PRECISIONS.index(eng.precision),
            torch.are_deterministic_algorithms_enabled(),
            *(checksum(t) for t in (captions, input_mask, segment_ids, self.image_mask, self.features, self.spatials, eng.ps.flat)))))

    def _score_rows(self, captions, input_mask, segment_ids, task_id, has_task):
        """The scores of these captions against the whole gallery on this device: chunk outer, capacity group middle, caption
        inner."""
        model, eng = self.model, self.model.engine
        dev = eng.device
        C, Nt = int(captions.shape[0]), int(captions.shape[1])
        chunks = self._chunks(input_mask, has_task)
        # the caption bank: uploaded once, read row by row with device-to-device copies
        ids = captions.to(dev, torch.int64, non_blocking=True)
        mask = input_mask.to(dev, torch.int64, non_blocking=True)
        seg = segment_ids.to(dev, torch.int64, non_blocking=True)
        task = torch.full((1, 1), _task_number(task_id), dtype=torch.int64, device=dev) if has_task else None
        scores = torch.empty((C, self.G), dtype=torch.float32, device=dev)
        model._sync_weights()
        # chunk outer, plan (padded, or one packed capacity of the captions) middle, caption inner: each plan embeds the chunk
        # once in its prefix, and every caption lands at its own row
        for ci, (lo, n, rows_v, groups) in enumerate(chunks):
            for rows_t, group in groups.items():
                plan = self._plan(n, Nt, None if rows_t is None else (rows_t, rows_v))
                self._load_chunk(plan, lo, n)
                out = plan.outputs[self.head]
                for c in group:
                    plan.load_inputs(ids[c:c + 1], None, None, seg[c:c + 1], mask[c:c + 1], None, task)
                    if eng.auto_graph:
                        plan.maybe_capture_passes(after=1)
                    plan.run_forward()
                    if self.heads == "vl":
                        scores[c, lo:lo + n].copy_(out.view(-1))
                    else:
                        scores[c, lo:lo + n].copy_(torch.softmax(out, dim=1)[:, 0])
            logger.info("retrieval: chunk %d/%d (images %d-%d) scored against %d captions", ci + 1, len(chunks), lo, lo + n - 1, C)
        return scores

    @staticmethod
    def rank(scores, target_image, k=20):
        """(ranks int32 [C], topk int32 [C, k]) on the device: the 0-based position of each caption's target image in its row's stable
        descending order (ties by image index, NaN last), -1 for a target outside the gallery, and the first k images of that order
        (-1 past the gallery's end). k <= 64."""
        if scores.dim() != 2 or scores.dtype != torch.float32 or not scores.is_cuda or scores.stride(1) != 1:
            raise ValueError("scores: device f32 [C, G] with contiguous rows")
        C, G = scores.shape
        target = torch.as_tensor(target_image).to(scores.device, torch.int64).reshape(-1).contiguous()
        if target.numel() != C:
            raise ValueError(f"target_image: one per caption ({C}), got {target.numel()}")
        ranks = torch.empty(C, dtype=torch.int32, device=scores.device)
        topk = torch.empty((C, int(k)), dtype=torch.int32, device=scores.device)
        L.call(L.lib().vb_retrieval_rank, scores, scores.stride(0), C, G, target, int(k), ranks, topk,
               stream=torch.cuda.current_stream(scores.device).cuda_stream)
        return ranks, topk

    @staticmethod
    def rank_captions(scores, target_image, k=20):
        """Image-to-text ranks from the same score matrix: (ranks int32 [G], topk int32 [G, k]) on the device. ranks[g] is the
        0-based position of image g's best-placed ground-truth caption (the captions c with target_image[c] == g) in the stable
        descending order of column g of scores (ties by caption index, NaN last), -1 for an image without a caption; topk[g] is
        the first k captions of that order (-1 past the last caption). k <= 64, at most 50,000 captions."""
        if scores.dim() != 2 or scores.dtype != torch.float32 or not scores.is_cuda or scores.stride(1) != 1:
            raise ValueError("scores: device f32 [C, G] with contiguous rows")
        if not 1 <= int(k) <= MAX_TOPK:
            raise ValueError(f"k = {k}: the device ranking returns 1 to {MAX_TOPK} entries per image")
        C, G = scores.shape
        target = torch.as_tensor(target_image).to(scores.device, torch.int64).reshape(-1)
        if target.numel() != C:
            raise ValueError(f"target_image: one per caption ({C}), got {target.numel()}")
        set_off, set_idx = caption_sets(target, G)
        by_image = scores.t().contiguous()                              # [G, C]: one row per image
        ranks = torch.empty(G, dtype=torch.int32, device=scores.device)
        topk = torch.empty((G, int(k)), dtype=torch.int32, device=scores.device)
        L.call(L.lib().vb_retrieval_rank_sets, by_image, C, G, C, set_off, set_idx, int(k), ranks, topk,
               stream=torch.cuda.current_stream(scores.device).cuda_stream)
        return ranks, topk


def caption_sets(target_image, G):
    """Each image's ground-truth captions as CSR on target_image's device, with no host synchronisation: (set_off int64 [G + 1],
    set_idx int64) with image g's captions, in ascending order, at set_idx[set_off[g]:set_off[g + 1]]. A caption whose target is
    outside [0, G) belongs to no image; an image without a caption has an empty range."""
    target = torch.as_tensor(target_image).to(torch.int64).reshape(-1)
    sorted_target, set_idx = torch.sort(target, stable=True)
    set_off = torch.searchsorted(sorted_target, torch.arange(G + 1, dtype=torch.int64, device=target.device))
    return set_off, set_idx


def i2t_metrics(ranks):
    """((r1, r5, r10, medr, meanr), images without a caption) of image-to-text ranks (rank_captions): retrieval_metrics over the
    images with at least one caption; an image without one (rank -1) is counted, not ranked."""
    r = ranks.detach().cpu().numpy() if torch.is_tensor(ranks) else np.asarray(ranks)
    ranked = r[r >= 0]
    if len(ranked) == 0:
        raise ValueError("i2t_metrics: no image has a caption")
    return retrieval_metrics(ranked), int(len(r) - len(ranked))


def evaluate_retrieval(model, dataset, task_id=None, chunk=500, k=20, pack=None, group=None):
    """The loop of eval_retrieval.py:253-358 (and, with the pre-training model and task_id=None, of eval_coco_retrieval.py:336-412):
    (r1, r5, r10, medr, meanr, results), results being each caption's top-k image list (the reference dumps the top 20 into
    *_result.json). The dataset is read through the reference's item protocol (read_retrieval_dataset); metrics are taken over the
    captions evaluated, which with the reference's 5,000 x 1,000 sizes is exactly its number. Puts the model in eval mode, as the
    reference loop does. pack: score on packed plans (RetrievalEvaluator); None follows model.engine.pack_padding.
    group: a torch.distributed process group to shard the captions over (RetrievalEvaluator.score); every rank ranks the gathered
    scores and returns the same result."""
    model.eval()
    feats, spats, imask, caps, masks, segs, targets = read_retrieval_dataset(dataset)
    ev = RetrievalEvaluator(model, feats, spats, imask, chunk=chunk, pack=pack)
    scores = ev.score(caps, masks, segs, task_id=task_id, group=group)
    ranks, topk = ev.rank(scores, targets, k=k)
    both = torch.cat((ranks.view(-1, 1), topk), dim=1).cpu()       # the one read-back
    r1, r5, r10, medr, meanr = retrieval_metrics(both[:, 0])
    logger.info("Final r1:%.3f, r5:%.3f, r10:%.3f, mder:%.3f, meanr:%.3f", r1, r5, r10, medr, meanr)
    return r1, r5, r10, medr, meanr, both[:, 1:1 + min(k, ev.G)].tolist()


def evaluate_retrieval_both(model, dataset, task_id=None, chunk=500, k=20, pack=None, group=None):
    """Both retrieval directions from one scoring pass, with the arguments of evaluate_retrieval:
    {"t2i": (r1, r5, r10, medr, meanr, results), "i2t": (r1, r5, r10, medr, meanr, results), "rsum": float,
    "images_without_caption": n}. t2i (caption-to-image, image retrieval) is what evaluate_retrieval returns. i2t (image-to-text,
    text retrieval) ranks each image's best-placed ground-truth caption (rank_captions); its metrics are retrieval_metrics over the
    images with at least one caption (i2t_metrics), and its results are every image's top-k caption list. rsum is the sum of both
    directions' r1, r5 and r10. Both directions' ranks and top-k lists are read back in one copy. With group=, as for
    evaluate_retrieval, every rank returns the same dictionary."""
    model.eval()
    feats, spats, imask, caps, masks, segs, targets = read_retrieval_dataset(dataset)
    ev = RetrievalEvaluator(model, feats, spats, imask, chunk=chunk, pack=pack)
    scores = ev.score(caps, masks, segs, task_id=task_id, group=group)
    C, G = scores.shape
    ranks_t, topk_t = ev.rank(scores, targets, k=k)
    ranks_i, topk_i = ev.rank_captions(scores, targets, k=k)
    both = torch.cat((torch.cat((ranks_t.view(-1, 1), topk_t), 1), torch.cat((ranks_i.view(-1, 1), topk_i), 1))).cpu()
    t2i = retrieval_metrics(both[:C, 0])
    i2t, without = i2t_metrics(both[C:, 0])
    logger.info("Final t2i r1:%.3f, r5:%.3f, r10:%.3f, mder:%.3f, meanr:%.3f", *t2i)
    logger.info("Final i2t r1:%.3f, r5:%.3f, r10:%.3f, mder:%.3f, meanr:%.3f (%d images without a caption)", *i2t, without)
    return {"t2i": (*t2i, both[:C, 1:1 + min(k, G)].tolist()), "i2t": (*i2t, both[C:, 1:1 + min(k, C)].tolist()),
            "rsum": float(sum(t2i[:3]) + sum(i2t[:3])), "images_without_caption": without}
