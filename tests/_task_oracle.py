"""Restatement of the reference's per-task objectives and batch scores (vilbert/task_utils.py:31-376, 618-623) on the outputs of a
model with the reference's forward signature: what vilbert_b200.tasks.ForwardModelsTrain / ForwardModelsVal are checked against.
Also a float64 model of the fused V-logit-mc / soft-target BCE kernel (vb_bce_gather_loss) and of its argmax rule, used by the
CPU tests to pin the closed forms against torch autograd and torch.max."""
import math

import torch
import torch.nn.functional as F

MC_OFFSET = 101     # task_utils.py:353: vision_logit[:, 101:]


def bce(x, t):
    """nn.BCEWithLogitsLoss(reduction="mean") of LoadLosses (task_utils.py:25-28)."""
    return F.binary_cross_entropy_with_logits(x, t, reduction="mean")


def score_with_logits(logits, labels):
    """compute_score_with_logits (task_utils.py:618-623): the label mass at the argmax of each row. The one-hot has the labels'
    shape and the argmax is scattered along dim 1, so 1-D int labels (Foil) raise IndexError, as in the reference."""
    pick = torch.max(logits, 1)[1]
    onehot = torch.zeros(labels.size(), device=labels.device)
    onehot.scatter_(1, pick.view(-1, 1), 1)
    return onehot * labels


def objective(kind, heads, target, mc_ids=None, batch_size=None, num_options=None):
    """(loss, summed batch score) of the objective `kind` from the nine head outputs, formed as task_utils.py:121-162 / 325-374 do.
    binary_ce / tri_ce (CrossEntropyLoss on int labels) raise from the score, like the reference."""
    vil_prediction, vil_prediction_gqa, vil_logit, vil_binary, vil_tri, _, vision_logit, _, _ = heads[:9]
    if kind in ("vqa", "gqa"):                                     # :325-334, VL-classifier(-GQA): mean * answers
        lg = vil_prediction if kind == "vqa" else vil_prediction_gqa
        return bce(lg, target) * target.size(1), score_with_logits(lg, target).sum()
    if kind == "logit_ce":                                         # :336-340, VL-logit: CE over the options of each question
        lg = vil_logit.view(batch_size, num_options)
        return F.cross_entropy(lg, target), (torch.max(lg, 1)[1] == target).sum()
    if kind == "vlogit_bce":                                       # :342-347, V-logit: mean * regions, target at the argmax region
        loss = bce(vision_logit, target) * target.size(1)
        pick = torch.max(vision_logit, dim=1)[1]
        return loss, (target.squeeze(2).gather(1, pick.view(-1, 1)) > 0.5).sum()
    if kind == "vlogit_mc":                                        # :349-357, V-logit-mc: gathered choices, mean * choices
        lg = vision_logit[:, MC_OFFSET:].squeeze(2).gather(1, mc_ids).unsqueeze(2)
        loss = bce(lg, target) * target.size(1)
        return loss, (torch.max(lg, dim=1)[1] == torch.max(target, dim=1)[1]).sum()
    if kind in ("binary_bce", "tri_bce"):                          # :359-367, soft targets, plain mean
        lg = vil_binary if kind == "binary_bce" else vil_tri
        return bce(lg, target), score_with_logits(lg, target).sum()
    if kind in ("binary_ce", "tri_ce"):                            # the same lines with CrossEntropyLoss and int labels (Foil)
        lg = vil_binary if kind == "binary_ce" else vil_tri
        loss = F.cross_entropy(lg, target)
        return loss, score_with_logits(lg, target).sum()
    raise ValueError(kind)


def reshape_batch(process, batch_size, features, spatials, image_mask, question, input_mask, segment_ids, target):
    """The `process` reshapes of task_utils.py:198-310 restated with torch views. Returns the model inputs, the target and
    (batch_size, num_options) as the reference leaves them."""
    num_options = None
    if process == "dialog":
        nround, num_options = question.size(1), question.size(2)
        rep = lambda x: x.unsqueeze(1).unsqueeze(1).expand(batch_size, nround, num_options, *x.shape[1:]).reshape(-1, *x.shape[1:])
        features, spatials, image_mask = rep(features), rep(spatials), rep(image_mask)
        question, input_mask, segment_ids = (x.reshape(-1, x.size(3)) for x in (question, input_mask, segment_ids))
        target = target.view(-1)
        batch_size = batch_size * nround
    elif process == "expand":
        num_options = question.size(1)
        rep = lambda x: x.unsqueeze(1).expand(batch_size, num_options, *x.shape[1:]).reshape(-1, *x.shape[1:])
        features, spatials, image_mask = rep(features), rep(spatials), rep(image_mask)
        question, input_mask, segment_ids = (x.reshape(-1, x.size(2)) for x in (question, input_mask, segment_ids))
    elif process == "retrieval":
        num_options = question.size(1)
        features, spatials = features.reshape(-1, *features.shape[2:]), spatials.reshape(-1, *spatials.shape[2:])
        image_mask, question, input_mask, segment_ids = (x.reshape(-1, x.size(2)) for x in (image_mask, question, input_mask, segment_ids))
    elif process == "nlvr":
        B = batch_size
        features = features.view(B * 2, features.size(1) // 2, features.size(2))
        spatials = spatials.view(B * 2, spatials.size(1) // 2, spatials.size(2))
        image_mask = image_mask.view(B * 2, image_mask.size(1) // 2)
        question, input_mask, segment_ids = (x.repeat(1, 2).view(B * 2, x.size(1)) for x in (question, input_mask, segment_ids))
    return (features, spatials, image_mask, question, input_mask, segment_ids), target, batch_size, num_options


def reference_step(kind, process, task_id, batch, model):
    """ForwardModelsTrain's body (task_utils.py:186-376) on the module surface: (loss, summed batch score, batch_size)."""
    if task_id in ("TASK4", "TASK17"):
        features, spatials, image_mask, question, target, input_mask, segment_ids, mc_ids, co_mask, _ = batch
    else:
        features, spatials, image_mask, question, target, input_mask, segment_ids, co_mask, _ = batch
        mc_ids = None
    batch_size = features.size(0)
    (features, spatials, image_mask, question, input_mask, segment_ids), target, batch_size, num_options = reshape_batch(
        process, batch_size, features, spatials, image_mask, question, input_mask, segment_ids, target)
    task_tokens = question.new().resize_(question.size(0), 1).fill_(int(task_id[4:]))
    heads = model(question, features, spatials, segment_ids, input_mask, image_mask, None, task_tokens)
    loss, score = objective(kind, heads, target, mc_ids, batch_size, num_options)
    return loss, score, batch_size


# ------------------------------------------------------------------------------------------ synthetic task batches
# task id -> (type, loss, process) of vilbert_tasks.yml
TASK_CFG = {
    "TASK1": ("VL-classifier", "BCEWithLogitLoss", "normal"), "TASK3": ("VL-logit", "CrossEntropyLoss", "dialog"),
    "TASK4": ("V-logit-mc", "BCEWithLogitLoss", "normal"), "TASK5": ("VL-logit", "CrossEntropyLoss", "expand"),
    "TASK7": ("VL-logit", "CrossEntropyLoss", "retrieval"), "TASK9": ("V-logit", "BCEWithLogitLoss", "normal"),
    "TASK12": ("VL-binary-classifier", "BCEWithLogitLoss", "nlvr"), "TASK13": ("VL-tri-classifier", "BCEWithLogitLoss", "normal"),
    "TASK15": ("VL-classifier-GQA", "BCEWithLogitLoss", "normal"), "TASK16": ("VL-binary-classifier", "CrossEntropyLoss", "normal"),
    "TASK17": ("V-logit-mc", "BCEWithLogitLoss", "normal"),
    "TASK2": ("VL-classifier", "BCEWithLogitLoss", "normal"), "TASK8": ("VL-logit", "CrossEntropyLoss", "retrieval"),
    "TASK10": ("V-logit", "BCEWithLogitLoss", "normal"), "TASK11": ("V-logit", "BCEWithLogitLoss", "normal"),
}
TASK_CFG = {k: dict(type=t, loss=lo, process=p) for k, (t, lo, p) in TASK_CFG.items()}


def kind_of(task_id):
    """The fused objective kind of a task of TASK_CFG (vilbert_b200.tasks.TASK_KINDS)."""
    from vilbert_b200.tasks import task_kind
    return task_kind(TASK_CFG, task_id)


def make_batch(cfgj, task_id, B, Nv, Nt, options=3, C=4, nround=2, seed=0):
    """A batch in the layout the reference's dataset of `task_id` yields (CPU tensors)."""
    g = torch.Generator().manual_seed(seed)
    proc, kind = TASK_CFG[task_id]["process"], kind_of(task_id)
    Fv, V = cfgj["v_feature_size"], cfgj["vocab_size"]
    lead = {"retrieval": (B, options), "nlvr": (B,)}.get(proc, (B,))
    nv = 2 * Nv if proc == "nlvr" else Nv
    features = torch.relu(torch.randn(*lead, nv, Fv, generator=g))
    spatials = torch.rand(*lead, nv, 5, generator=g)
    n_valid = torch.randint(max(2, nv - 15), nv + 1, lead, generator=g)
    image_mask = (torch.arange(nv) < n_valid.unsqueeze(-1)).long()
    qlead = {"expand": (B, options), "retrieval": (B, options), "dialog": (B, nround, options)}.get(proc, (B,))
    question = torch.randint(0, V, (*qlead, Nt), generator=g)
    input_mask = (torch.arange(Nt) < torch.randint(3, Nt + 1, qlead, generator=g).unsqueeze(-1)).long()
    segment_ids = torch.zeros_like(question)
    co_mask = torch.zeros(*qlead, nv, Nt)
    mc = None
    if kind in ("vqa", "gqa"):
        n = 3129 if kind == "vqa" else 1533
        target = torch.zeros(B, n)
        target.scatter_(1, torch.randint(0, n, (B, 3), generator=g), torch.tensor([0.3, 0.6, 1.0]).expand(B, 3).contiguous())
    elif kind == "logit_ce":
        target = torch.randint(0, options, (B, nround) if proc == "dialog" else (B,), generator=g)
    elif kind == "vlogit_bce":
        target = (torch.rand(B, Nv, 1, generator=g) * (image_mask.unsqueeze(-1) > 0)).round() * 0.9
    elif kind == "vlogit_mc":
        n_real = torch.randint(1, C + 1, (B,), generator=g)
        mc = torch.randint(0, min(Nv - MC_OFFSET, 204), (B, C), generator=g)
        pad = torch.arange(C) >= n_real.unsqueeze(1)
        mc[pad] = min(Nv - MC_OFFSET - 1, 204)                  # GuessWhat-style padding: one region repeated
        target = (torch.rand(B, C, 1, generator=g) > 0.6).float() * (~pad).unsqueeze(-1)
        image_mask[:, Nv - 3:] = 0                                # the padding region is masked (vision_logit ~ -10000 there)
    elif kind == "binary_bce":
        target = torch.rand(B, 2, generator=g).round()
    elif kind == "tri_bce":
        target = torch.softmax(torch.randn(B, 3, generator=g) * 3, 1)
    else:
        target = torch.randint(0, 2, (B,), generator=g)
    qid = torch.arange(B)
    if mc is not None:
        return (features, spatials, image_mask, question, target, input_mask, segment_ids, mc, co_mask, qid)
    return (features, spatials, image_mask, question, target, input_mask, segment_ids, co_mask, qid)


# ------------------------------------------------------------------------------------------ models of the fused kernels
def bce_gather_closed_form(logits, off, ids, target, loss_mul):
    """What vb_bce_gather_loss computes, in float64: logits [rows, width], ids [rows, C] or None, target [rows, C]. Returns
    (loss, d loss / d logits [rows, width]); a duplicated id sums the gradients of its choices; an id outside [0, width - off)
    contributes nothing to the gradient and makes the loss NaN."""
    x64, t64 = logits.double(), target.double()
    rows, width = x64.shape
    C = t64.shape[1]
    cols = (torch.arange(C).expand(rows, C) if ids is None else ids.long()) + off
    ok = (cols >= off) & (cols < width)
    x = x64.gather(1, cols.clamp(0, width - 1))
    per = torch.clamp(x, min=0) - x * t64 + torch.log1p(torch.exp(-x.abs()))
    per = torch.where(ok, per, torch.full_like(per, math.nan))
    scale = loss_mul / (rows * C)
    g = torch.where(ok, (torch.sigmoid(x) - t64) * scale, torch.zeros_like(x))
    d = torch.zeros_like(x64).scatter_add_(1, cols.clamp(0, width - 1), g)
    return per.sum() * scale, d


def argmax_torch_rule(row):
    """The argmax rule of vb_task_score, written out: a NaN beats any number, and the first index wins among equals / NaNs."""
    best, bi = None, None
    for i, v in enumerate(row.tolist()):
        if bi is None:
            best, bi = v, i
            continue
        if math.isnan(best):
            continue
        if math.isnan(v) or v > best:
            best, bi = v, i
    return bi
