"""Execution engine of the H100 ViLBERT hot path.

Mirrors, operation for operation, what the reference's eager modules do in
VILBertForVLTasks.forward -> BertModel.forward -> BertEncoder.forward (vilbert/vilbert.py:1638-1708,
:1309-1406, :934-1107) and what autograd derives from them, but as a static *plan*: for a given
(B, Nt, Nv) shape every activation buffer is allocated once and the forward and backward passes
become flat lists of C-ABI calls into libvilbert_b200.so (wgmma GEMMs, fused attention, row-wise
kernels). A plan can be replayed eagerly (a tight loop of ctypes calls) or captured into one CUDA
graph per pass. PyTorch is used for device memory, streams and (optionally) graph capture only.

Numerics (DESIGN.md §6). Accumulation is always fp32 (registers); the residual stream, LayerNorm
statistics and outputs, softmax statistics, biases and every gradient accumulation are fp32; 16-bit copies of
activations and weights exist only as tensor-core operands. Three operand precisions (Engine(precision=...)):
  "fp16" (default)  forward operands (activations, weights) fp16 — 11 significant bits, the reference's own reduced
                    precision (model.half(), train_concap.py:504-505) — gradient operands (dy, dS, ...) bf16 for range.
                    wgmma takes one operand type for both inputs, so every forward operand the backward contracts with a
                    gradient (weights for dgrad, saved activations for wgrad) also has a bf16 copy, written by the kernel
                    that produces it (Operand.bw);
  "fp32"            split precision: every forward operand is stored as fp16 hi + lo and every forward contraction
                    runs as three tensor-core passes (hi.hi + lo.hi + hi.lo), ~fp32 accuracy (north_star 1e-3);
  "bf16"            every operand bf16 (round-1 arithmetic; kept for A/B measurements).
"""
import bisect
import dataclasses
import math
import warnings
import zlib
from collections import Counter, OrderedDict, namedtuple

import torch

from . import _lib as L

F32, BF16, F16, I64 = torch.float32, torch.bfloat16, torch.float16, torch.int64
PRECISIONS = ("fp16", "fp32", "bf16")
# the single-stream baseline hard-codes its region-feature width and region-class count (basebert.py:329, 613); v_feature_size and
# v_target_size do not apply to it
BASE_FEATURE_SIZE, BASE_REGION_CLASSES = 2048, 1601
# outputs of the baseline, in the order BaseBertForVLTasks.forward returns them (basebert.py:954-962), and of its BertModel
BASE_HEAD_NAMES = ("vil_prediction", "vil_logit", "vil_binary_prediction", "vision_prediction", "vision_logit", "linguisic_prediction",
                   "linguisic_logit")
BASE_BERT_OUT_NAMES = ("sequence_output", "pooled_output")
# the float inputs a plan can backpropagate into (Plan(input_grads=...)): the region features and their boxes
INPUT_GRAD_NAMES = ("input_imgs", "image_loc")
# heads a packed plan (Plan(packed=...)) can build: the pooled heads and the per-region logit, which it scatters back to the padded
# layout. The prediction heads of pre-training are packed only inside the fused objective (loss="pretraining", loss_in_forward=True):
# the masked-LM head compacts its labelled rows through the text row map, the region head scatters its rows to the padded layout
PACKED_HEADS = ("vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_binary_prediction", "vil_tri_prediction", "vision_logit")
# the score head a packed retrieval plan (fast_mode and image_prefix) builds, per model kind: VILBertForVLTasks' vil_logit, the
# pre-training model's alignment logits (zero-shot retrieval)
RETRIEVAL_SCORE_HEADS = {"vl": "vil_logit", "pretraining": "seq_relationship_score"}
# config options packed plans refuse: they reshape or export the padded streams
PACK_REFUSED_CONFIG = ("in_batch_pairs", "fast_mode", "dynamic_attention", "visualization")
# the value a masked region's logit takes in a packed plan: the reference's additive mask, which in fp32 is no further from it
# (BCE-with-logits at target 0 of either is 0.0 with gradient 0.0)
PACKED_MASKED_LOGIT = -10000.0


def pack_capacity(count, padded_rows):
    """Rows of a packed stream holding `count` valid rows of a padded [B, N] batch: count rounded up to a step of one sixteenth
    of the padded rows, itself a multiple of the GEMMs' 128-row tile, and never more than the padded rows. The valid-row sum of a
    64-256-sample batch moves by a few percent from batch to batch, less than one step, so a task settles on one or two
    capacities (plans), and the rows a capacity wastes are at most a sixteenth of the padded ones."""
    if count < 1:
        raise ValueError("a packed stream needs at least one valid row")
    step = max(128, -(-padded_rows // 16 // 128) * 128)
    return min(-(-count // step) * step, padded_rows)


def prefix_lengths(mask):
    """Valid length per row of a 0/1 host mask [rows, N], or None when some row is not prefix-valid (a 0 before a 1) or has no 1."""
    m = mask.ne(0)
    n = m.sum(1)
    ok = bool((n >= 1).all()) and bool(m.eq(torch.arange(m.size(1)).unsqueeze(0) < n.unsqueeze(1)).all())
    return n if ok else None


def check_pack_config(cfg):
    """engine.pack_padding with a config option packed plans refuse (PACK_REFUSED_CONFIG) raises NotImplementedError."""
    bad = [f for f in PACK_REFUSED_CONFIG if getattr(cfg, f, False)]
    if bad:
        raise NotImplementedError(f"engine.pack_padding does not support config.{bad[0]}")


def pretraining_pack_rows(attention_mask, image_attention_mask, masked_lm_labels, image_label, B, Nt, Nv):
    """Host decision of a packed pre-training step from host tensors (None: a mask of all ones, labels that select nothing), with
    no device read: (rows_t, rows_v) of the packed plan, or the reason the batch runs padded. "mask": a mask is not prefix-valid
    or has an empty row; "label": a token with masked_lm_labels != -1 sits where attention_mask == 0, or a region with
    image_label == 1 (image_label covers regions 1 .. Nv - 1) where image_attention_mask == 0 — the padded loss reads those rows."""
    mt = torch.ones(B, Nt, dtype=I64) if attention_mask is None else attention_mask.reshape(B, Nt)
    mv = torch.ones(B, Nv, dtype=I64) if image_attention_mask is None else image_attention_mask.reshape(B, Nv)
    lt, lv = prefix_lengths(mt), prefix_lengths(mv)
    if lt is None or lv is None:
        return "mask"
    if masked_lm_labels is not None and bool((masked_lm_labels.reshape(B, Nt).ne(-1) & mt.eq(0)).any()):
        return "label"
    if image_label is not None and bool((image_label.reshape(B, Nv - 1).eq(1) & mv[:, 1:].eq(0)).any()):
        return "label"
    return pack_capacity(int(lt.sum()), B * Nt), pack_capacity(int(lv.sum()), B * Nv)


def pack_summary(attention_mask, image_attention_mask, masked_lm_labels, image_label, B, Nt, Nv):
    """vb_pack_summary of device-resident masks and labels (None as in pretraining_pack_rows) on the current stream, read back with
    one device-to-host copy: the host waits for the stream here. -> int32 host tensor [2B + 5] (layout: include/vilbert_b200.h)."""
    dev = next(t.device for t in (attention_mask, image_attention_mask, masked_lm_labels, image_label) if t is not None and t.is_cuda)
    as_dev = lambda t: None if t is None else t.to(device=dev, dtype=I64, non_blocking=True).contiguous()
    ins = [as_dev(t) for t in (attention_mask, image_attention_mask, masked_lm_labels, image_label)]
    out = torch.empty(2 * B + 5, dtype=torch.int32, device=dev)
    L.call(L.lib().vb_pack_summary, ins[0], ins[1], B, Nt, Nv, ins[2], ins[3], out)
    return out.cpu()


def pretraining_pack_rows_from_summary(summary, B, Nt, Nv):
    """The decision of pretraining_pack_rows from a vb_pack_summary result (pack_summary)."""
    s = summary.tolist()
    if s[2 * B] or s[2 * B + 1]:
        return "mask"
    if s[2 * B + 2] or s[2 * B + 3]:
        return "label"
    return pack_capacity(sum(s[:B]), B * Nt), pack_capacity(sum(s[B:2 * B]), B * Nv)


def _pad8(n):
    return (n + 7) // 8 * 8


def dropout_site_id(name):
    """Stable 32-bit id of a dropout layer, shared with the oracle's mask generator (crc32 of its canonical name)."""
    return zlib.crc32(name.encode()) & 0xFFFFFFFF


class Operand:
    """A 16-bit tensor-core operand: `hi` in the engine's forward format (fp16, or bf16 with precision="bf16"), `lo` its
    split-precision low part (None unless precision="fp32"), `bw` the bf16 copy the backward GEMMs contract with (hi itself
    when hi is bf16, None when nothing in the backward reads it)."""
    __slots__ = ("hi", "lo", "bw")

    def __init__(self, hi, lo=None, bw=None):
        self.hi, self.lo, self.bw = hi, lo, bw

    @property
    def fp16(self):
        """Format flag of the C ABI (1 = fp16, 0 = bf16)."""
        return 1 if self.hi.dtype == F16 else 0

    @property
    def extra_bw(self):
        """The bf16 copy as a separate output of the kernel that writes hi: None when there is none or it is hi itself."""
        return None if self.bw is None or self.bw is self.hi else self.bw

    def _map(self, f):
        hi = f(self.hi)
        return Operand(hi, None if self.lo is None else f(self.lo), hi if self.bw is self.hi else (None if self.bw is None else f(self.bw)))

    def cols(self, a, b):
        """Columns [a, b) (the Q / K / V panels of a packed projection)."""
        return self._map(lambda t: t[:, a:b])

    def view(self, *shape):
        return self._map(lambda t: t.view(*shape))

    def ptrs(self, off=0):
        """(hi, lo, extra_bw) data pointers `off` elements in (None for a missing part): the 16-bit outputs of the cast and
        optimizer kernels."""
        return tuple(None if t is None else t.data_ptr() + t.element_size() * off for t in (self.hi, self.lo, self.extra_bw))


# ------------------------------------------------------------------------------------------ parameters
class ParamStore:
    """All parameters live in ONE flat fp32 buffer (reference state_dict names map to views of it), with a
    flat fp32 gradient buffer of the same layout (what the data-parallel all-reduce operates on) and a flat
    bf16 shadow used as GEMM operands. query/key/value weights of one attention are allocated contiguously
    so that the fused [3H, H] QKV GEMM reads them in place."""

    def __init__(self, cfg, device, heads="vl", op_dtype=F16, split=False, num_labels=None):
        """heads: "vl" = pre-training heads + the 7 task heads (VILBertForVLTasks), "pretraining" = cls.* only
        (BertForMultiModalPreTraining), "none" = bare BertModel; "base" = the single-stream baseline BaseBertForVLTasks with
        `num_labels` answers (vilbert/basebert.py), "base_none" = its bare BertModel. op_dtype: format of the 16-bit weight
        shadow; split: also keep the low parts (shadow_lo) for the split-precision mode."""
        assert heads in ("vl", "pretraining", "none", "base", "base_none")
        self.op_dtype, self.split = op_dtype, split
        self.heads = heads
        self.base = heads in ("base", "base_none")
        with_task_heads = heads == "vl"
        self.cfg = cfg
        self.device = device
        self.entries = OrderedDict()   # reference name -> (offset, shape)
        self.fused = {}                # fused qkv name -> (offset, shape)
        self.parts = {}                # fused qkv name -> the entry names it spans, in order
        self._off = 0
        c = cfg
        if self.base:
            self._base_layout(num_labels)
            self._alloc()
            return
        Ht, It, Hv, Iv, Hb = c.hidden_size, c.intermediate_size, c.v_hidden_size, c.v_intermediate_size, c.bi_hidden_size
        for h in (Ht, It, Hv, Iv, Hb, c.v_feature_size):
            if h % 8:
                raise ValueError("vilbert_b200: hidden sizes must be multiples of 8 (TMA row pitch)")
        add, lin, ln = self._add, self._lin, self._ln
        add("bert.embeddings.word_embeddings.weight", (c.vocab_size, Ht))
        add("bert.embeddings.position_embeddings.weight", (c.max_position_embeddings, Ht))
        add("bert.embeddings.token_type_embeddings.weight", (c.type_vocab_size, Ht))
        ln("bert.embeddings.LayerNorm", Ht)
        if c.task_specific_tokens:
            add("bert.embeddings.task_embeddings.weight", (20, Ht))
        lin("bert.v_embeddings.image_embeddings", Hv, c.v_feature_size)
        lin("bert.v_embeddings.image_location_embeddings", Hv, 5)
        ln("bert.v_embeddings.LayerNorm", Hv)
        # Encoder parameters are laid out in EXECUTION order (the interleaving schedule of BertEncoder.forward,
        # vilbert.py:960-1096): backward then finishes the flat gradient buffer from its end towards its start, so the
        # data-parallel all-reduce can start on finished tail ranges while earlier layers are still in backward.
        def block(kind, i, H, I):
            p = f"bert.encoder.{kind}.{i}"
            self._qkv(f"{p}.attention.self", ("query", "key", "value"), H, H)
            if kind == "v_layer" and getattr(c, "dynamic_attention", False):
                # BertImageSelfAttention.dyLinear_q / dyLinear_k (vilbert.py:561-563), contiguous so that one [2Hv, Ht] GEMM computes both gates
                self._qkv(f"{p}.attention.self", ("dyLinear_q", "dyLinear_k"), H, Ht, fused="dy")
            lin(f"{p}.attention.output.dense", H, H); ln(f"{p}.attention.output.LayerNorm", H)
            lin(f"{p}.intermediate.dense", I, H)
            lin(f"{p}.output.dense", H, I); ln(f"{p}.output.LayerNorm", H)

        def conn(i):
            p = f"bert.encoder.c_layer.{i}"
            self._qkv(f"{p}.biattention", ("query1", "key1", "value1"), Hb, Hv, fused="qkv1")
            self._qkv(f"{p}.biattention", ("query2", "key2", "value2"), Hb, Ht, fused="qkv2")
            lin(f"{p}.biOutput.dense1", Hv, Hb); ln(f"{p}.biOutput.LayerNorm1", Hv); lin(f"{p}.biOutput.q_dense1", Hv, Hb)
            lin(f"{p}.biOutput.dense2", Ht, Hb); ln(f"{p}.biOutput.LayerNorm2", Ht); lin(f"{p}.biOutput.q_dense2", Ht, Hb)
            lin(f"{p}.v_intermediate.dense", Iv, Hv); lin(f"{p}.v_output.dense", Hv, Iv); ln(f"{p}.v_output.LayerNorm", Hv)
            lin(f"{p}.t_intermediate.dense", It, Ht); lin(f"{p}.t_output.dense", Ht, It); ln(f"{p}.t_output.LayerNorm", Ht)

        t_start = v_start = 0
        for count, (v_end, t_end) in enumerate(zip(c.v_biattention_id, c.t_biattention_id)):
            for i in range(t_start, t_end):
                block("layer", i, Ht, It)
            for i in range(v_start, v_end):
                block("v_layer", i, Hv, Iv)
            conn(count)
            v_start, t_start = v_end, t_end
        for i in range(v_start, c.v_num_hidden_layers):
            block("v_layer", i, Hv, Iv)
        for i in range(t_start, c.num_hidden_layers):
            block("layer", i, Ht, It)
        lin("bert.t_pooler.dense", Hb, Ht); lin("bert.v_pooler.dense", Hb, Hv)
        if heads != "none":
            add("cls.predictions.bias", (c.vocab_size,))
            lin("cls.predictions.transform.dense", Ht, Ht); ln("cls.predictions.transform.LayerNorm", Ht)
            lin("cls.bi_seq_relationship", 2, Hb)
            lin("cls.imagePredictions.transform.dense", Hv, Hv); ln("cls.imagePredictions.transform.LayerNorm", Hv)
            lin("cls.imagePredictions.decoder", c.v_target_size, Hv)
        self.with_task_heads = with_task_heads
        if with_task_heads:
            for nm, i, o in (("vil_prediction", Hb, 3129), ("vil_prediction_gqa", Hb, 1533), ("vil_binary_prediction", 2 * Hb, 2)):
                lin(f"{nm}.logit_fc.0", 2 * Hb, i); ln(f"{nm}.logit_fc.2", 2 * Hb); lin(f"{nm}.logit_fc.3", o, 2 * Hb)
            lin("vil_logit", 1, Hb); lin("vil_tri_prediction", 3, Hb); lin("vision_logit", 1, Hv); lin("linguisic_logit", 1, Ht)
        self._alloc()

    def _base_layout(self, num_labels):
        """BaseBertForVLTasks' parameters (basebert.py:284-359, 507-519, 893-978) under the reference's state_dict names, in execution
        order: embeddings, layers, pooler, heads. SimpleClassifier's weight-normed linears keep weight_g (0-d) and weight_v."""
        c, add, lin, ln = self.cfg, self._add, self._lin, self._ln
        H, I = c.hidden_size, c.intermediate_size
        for h in (H, I):
            if h % 8:
                raise ValueError("vilbert_b200: hidden sizes must be multiples of 8 (TMA row pitch)")
        self.with_task_heads = False
        add("bert.embeddings.word_embeddings.weight", (c.vocab_size, H))
        add("bert.embeddings.position_embeddings.weight", (c.max_position_embeddings, H))
        add("bert.embeddings.token_type_embeddings.weight", (c.type_vocab_size, H))
        ln("bert.embeddings.LayerNorm", H)
        lin("bert.image_embeddings.image_embeddings", H, BASE_FEATURE_SIZE)
        add("bert.image_embeddings.token_type_embeddings.weight", (c.type_vocab_size, H))
        lin("bert.image_embeddings.image_location_embeddings", H, 5)
        ln("bert.image_embeddings.LayerNorm", H)
        for i in range(c.num_hidden_layers):
            p = f"bert.encoder.layer.{i}"
            self._qkv(f"{p}.attention.self", ("query", "key", "value"), H, H)
            lin(f"{p}.attention.output.dense", H, H); ln(f"{p}.attention.output.LayerNorm", H)
            lin(f"{p}.intermediate.dense", I, H)
            lin(f"{p}.output.dense", H, I); ln(f"{p}.output.LayerNorm", H)
        lin("bert.pooler.dense", H, H)
        if self.heads == "base_none":
            return
        if not num_labels or num_labels < 1:
            raise ValueError("BaseBertForVLTasks needs num_labels >= 1")
        self.num_labels = int(num_labels)
        add("cls.predictions.bias", (c.vocab_size,))
        lin("cls.predictions.transform.dense", H, H); ln("cls.predictions.transform.LayerNorm", H)
        lin("cls.seq_relationship", 2, H)
        lin("cls.imagePredictions.transform.dense", H, H); ln("cls.imagePredictions.transform.LayerNorm", H)
        lin("cls.imagePredictions.decoder", BASE_REGION_CLASSES, H)
        for i, (o, k) in ((0, (2 * H, H)), (3, (self.num_labels, 2 * H))):
            add(f"vil_prediction.main.{i}.weight_g", ())
            add(f"vil_prediction.main.{i}.weight_v", (o, k))
            add(f"vil_prediction.main.{i}.bias", (o,))
        lin("vil_logit", 1, H); lin("vision_logit", 1, H); lin("linguisic_logit", 1, H)

    def _alloc(self):
        device, op_dtype, split = self.device, self.op_dtype, self.split
        self.numel = self._off
        self.flat = torch.zeros(self.numel, dtype=F32, device=device)
        self.grad = torch.zeros(self.numel, dtype=F32, device=device)
        self.shadow = torch.zeros(self.numel, dtype=op_dtype, device=device)
        self.shadow_lo = torch.zeros(self.numel, dtype=op_dtype, device=device) if split else None
        # bf16 copy for the backward (dgrad: dy bf16 x W): the shadow itself when the operand format is already bf16
        self.shadow_b = self.shadow if op_dtype == BF16 else torch.zeros(self.numel, dtype=BF16, device=device)
        self.shadows = Operand(self.shadow, self.shadow_lo, self.shadow_b)
        self.shadow_version = None

    def _add(self, name, shape):
        self.entries[name] = (self._off, tuple(shape))
        self._off += _pad8(math.prod(shape))

    def _lin(self, name, o, i):
        self._add(name + ".weight", (o, i)); self._add(name + ".bias", (o,))

    def _ln(self, name, h):
        self._add(name + ".weight", (h,)); self._add(name + ".bias", (h,))

    def _qkv(self, prefix, names, o, i, fused="qkv"):
        assert (o * i) % 8 == 0 and o % 8 == 0
        w0 = self._off
        for nm in names:
            self._add(f"{prefix}.{nm}.weight", (o, i))
        b0 = self._off
        for nm in names:
            self._add(f"{prefix}.{nm}.bias", (o,))
        self.fused[f"{prefix}.{fused}.weight"] = (w0, (len(names) * o, i))
        self.fused[f"{prefix}.{fused}.bias"] = (b0, (len(names) * o,))
        self.parts[f"{prefix}.{fused}.weight"] = tuple(f"{prefix}.{nm}.weight" for nm in names)
        self.parts[f"{prefix}.{fused}.bias"] = tuple(f"{prefix}.{nm}.bias" for nm in names)

    def _layout(self, name):
        return self.entries[name] if name in self.entries else self.fused[name]

    def span(self, name):
        """(flat offset, numel) of an entry or a fused projection."""
        off, shape = self._layout(name)
        return off, math.prod(shape)

    def _view(self, flat, name):
        off, shape = self._layout(name)
        return flat[off:off + math.prod(shape)].view(shape)

    def p(self, name):
        return self._view(self.flat, name)

    def g(self, name):
        return self._view(self.grad, name)

    def w(self, name):
        """The 16-bit operand copies of one weight."""
        return self.shadows._map(lambda t: self._view(t, name))

    def cast_args(self, off, n):
        """Arguments (without the stream) of the vb_cast_f32_to_bf16 launch that refreshes elements [off, off + n) of the 16-bit
        copies from the fp32 parameters."""
        hi, lo, bw = self.shadows.ptrs(off)
        return (self.flat.data_ptr() + 4 * off, hi, n, self.shadows.fp16, lo, bw)

    def refresh_shadow(self):
        """16-bit operand copy (hi, and lo in split precision) of every parameter in one launch on the current stream (belongs
        with the optimizer step in training)."""
        L.call(L.lib().vb_cast_f32_to_bf16, *self.cast_args(0, self.numel))


# ------------------------------------------------------------------------------------------ plan
class Act:
    """A residual-stream activation: fp32 values, its tensor-core Operand, fp32 gradient (lazily allocated). Plan.act makes them.
    Three rules carry a gradient through a plan, each kept in one place:
    1. needs-grad (Plan.act): `rg` is set when the op that made the activation has a trainable parameter or an input that needs a
       gradient, as autograd's requires_grad; nothing made under the reference's torch.no_grad() (fixed_t_layer / fixed_v_layer) does.
    2. registration (Plan.push_bwd): a block whose output needs no gradient registers no backward emitter.
    3. first write (Plan.grad_zeroed / Plan.grad_acc): `gw` tells whether a backward op has written g32 yet. The first one
       overwrites it, or zeroes it and adds; every later one accumulates.
    The output of a residual LayerNorm (Plan.dense_res_ln) has one reader of its gradient, that LayerNorm's backward, which can add
    a second fp32 input as it reads (ln_reads). Its first writer may leave its residual-path part in g_add instead of adding it in a
    GEMM epilogue; a later writer adds g_add into g32 first (Plan._fold_g_add), so every sum keeps the order it has without it."""
    __slots__ = ("f32", "op", "g32", "gw", "M", "H", "rg", "ln_reads", "g_add", "mod")

    def __init__(self, f32, op, M, H, rg):
        self.f32, self.op, self.M, self.H, self.rg = f32, op, M, H, rg
        self.g32, self.gw = None, False
        self.ln_reads, self.g_add = False, None
        self.mod = None          # module path of the block whose output this is (anomaly labels of the gradient delivered into it)


# Objectives that can be fused into a plan, and the outputs each differentiates (task_utils.py:325-374, vilbert.py:1506-1590):
LOSS_HEADS = {
    "vqa": ("vil_prediction",),                 # VL-classifier: BCEWithLogits.mean() * 3129
    "gqa": ("vil_prediction_gqa",),             # VL-classifier-GQA: BCEWithLogits.mean() * 1533
    "vlogit_bce": ("vision_logit",),            # V-logit (refcoco*): BCEWithLogits(vision_logit [B,Nv,1], target).mean() * Nv
    "logit_ce": ("vil_logit",),                 # VL-logit (retrieval, VCR): CE over vil_logit.view(B / options, options)
    "binary_ce": ("vil_binary_prediction",),    # VL-binary-classifier with CrossEntropyLoss (Foil): CE over the 2-way head, int labels
    "tri_ce": ("vil_tri_prediction",),          # VL-tri-classifier with CrossEntropyLoss: CE over 3 classes, int labels
    "vlogit_mc": ("vision_logit",),             # V-logit-mc (Visual7w, GuessWhatPointing): BCE(vision_logit[:, 101:].gather(1, ids), target).mean() * C
    "binary_bce": ("vil_binary_prediction",),   # VL-binary-classifier with BCEWithLogitLoss (NLVR2): BCE over soft [B, 2] targets, mean()
    "tri_bce": ("vil_tri_prediction",),         # VL-tri-classifier with BCEWithLogitLoss (SNLI-VE): BCE over soft [B, 3] targets, mean()
    "pretraining": ("linguisic_prediction", "vision_prediction", "seq_relationship_score"),   # masked-LM CE + masked-region KL + alignment CE
}

# the fine-tuning objectives of the task table (everything but the pre-training objective): these can be placed at the end of the
# forward pass and given an on-device batch score (Plan(loss_in_forward=..., score=...))
TASK_KINDS = tuple(k for k in LOSS_HEADS if k != "pretraining")
# V-logit-mc scores the regions after the first 101 (task_utils.py:353: vision_logit[:, 101:])
MC_REGION_OFFSET = 101
# score of each task objective (task_utils.py:121-162, 618-623); binary_ce / tri_ce have none: with int labels the reference's
# compute_score_with_logits scatters into a 1-D tensor and raises (INTEGRATION.md)
SCORE_MODES = {"vqa": L.VB_SCORE_SOFT, "gqa": L.VB_SCORE_SOFT, "logit_ce": L.VB_SCORE_LABEL, "vlogit_bce": L.VB_SCORE_THRESHOLD,
               "vlogit_mc": L.VB_SCORE_CHOICE, "binary_bce": L.VB_SCORE_SOFT, "tri_bce": L.VB_SCORE_SOFT}

# slots of the three pre-training losses in Plan.objective_out / Plan.loss_grad (loss="pretraining", loss_in_forward=True)
PRETRAINING_SLOTS = {"linguisic_prediction": 0, "vision_prediction": 1, "seq_relationship_score": 2}


def nce_negative_count(cfg):
    """Negatives per masked region of visual_target == 2: int(0.7 N) from other samples + int(0.3 N) from the same sample
    (vilbert.py:1524-1557), N = config.num_negative."""
    return int(cfg.num_negative * 0.7) + int(cfg.num_negative * 0.3)


HEAD_NAMES = ("vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_binary_prediction", "vil_tri_prediction",
              "vision_prediction", "vision_logit", "linguisic_prediction", "linguisic_logit")
BERT_OUT_NAMES = ("sequence_output_t", "sequence_output_v", "pooled_output_t", "pooled_output_v")
# the heads of BertForMultiModalPreTraining (vilbert.py:1497), in the order its forward returns them
PRETRAINING_HEAD_NAMES = ("linguisic_prediction", "vision_prediction", "seq_relationship_score")

# per-row evaluation results of a task kind (EvaluatingModel, task_utils.py:777-847; Plan(results=...)): the head they read and the
# mode of vb_task_results. VL-classifier / GQA: the answer index; VL-logit: the option probabilities; V-logit: the region and its
# IoU; V-logit-mc: the chosen choice. The binary / tri types have no per-row results.
RESULT_MODES = {"vqa": ("vil_prediction", L.VB_RESULT_ARGMAX), "gqa": ("vil_prediction_gqa", L.VB_RESULT_ARGMAX),
                "logit_ce": ("vil_logit", L.VB_RESULT_SOFTMAX), "vlogit_bce": ("vision_logit", L.VB_RESULT_GATHER),
                "vlogit_mc": ("vision_logit", L.VB_RESULT_ARGMAX)}
# how the objective, score and results of a task kind address its head (Plan._head_layout): column c of row r is
# logits[r * ld + off + c], or with ids (the loss_inputs entry of the int64 [rows, cols] choice ids) logits[r * ld + off + ids[r, c]]
# with width the columns an id may reach; key is the loss_inputs entry of its labels (int64 [rows]) or targets (f32 [rows, cols])
HeadLayout = namedtuple("HeadLayout", "name logits rows cols ld off ids width key")


# deterministic plans (Plan(deterministic=True), DESIGN.md §4h): entry points whose float atomics make the summation order depend on
# scheduling, and the workspace floats their _det twin (same arguments + a trailing workspace) needs, from the arguments of the launch
# (_lib.launch_args: named after the parameters of the default entry point).
# vb_layernorm_bwd / vb_add_layernorm_bwd (Plan.ln_bwd) and the atomic GEMMs (Plan.gemm) are switched where they are emitted.
DET_WORKSPACE = {
    "vb_colsum": lambda a: L.VB_DET_SLICES * a.N,
    "vb_loc_proj_bwd": lambda a: L.VB_DET_SLICES * 6 * a.H,
    "vb_small_linear_bwd": lambda a: L.VB_DET_SLICES * (a.N * a.K + a.N),
    "vb_embed_text_bwd": None,
    "vb_ce_loss": lambda a: L.VB_DET_LOSS_SLICES,
    "vb_kl_masked_loss": lambda a: L.VB_DET_LOSS_SLICES,
    "vb_bce_logits_loss": lambda a: L.VB_DET_LOSS_SLICES,
}
# kernels of the single-stream baseline (BaseBertForVLTasks) with float atomics and no deterministic variant
DET_MISSING_BASELINE = ("vb_concat_embed_ln_bwd", "vb_embed_text_bwd_padded")
# streams an op list can name: main, vision, and the two weight-gradient side streams (Plan._run)
N_STREAMS = 4

# anomaly detection (Plan(anomaly=True), torch.autograd.set_detect_anomaly(True), DESIGN.md §4i): per entry point that runs in the
# backward role, the gradient values one launch writes, read by parameter name from the launch's own arguments (C values as
# emitted, _lib.launch_args) as (output name, pointer, rows, cols, ld in elements, VB_NAN_* dtype); a null pointer is an output the
# launch does not write. `p` is the plan, for the extents no argument carries: the rows of a packed stream (_attn_rows), of a
# scattered-into buffer (_buf_rows) and the ranges of parameter gradients (_param_numel). A _det twin shares the entry of its
# default entry point; the workspaces of the row-wise _det kernels are not listed: a launch writes only the slices it uses. An
# entry point emitted in the backward role without an entry fails when the plan is built.
_F32, _BF16 = L.VB_NAN_F32, L.VB_NAN_BF16


def _gemm_outputs(p, a):
    g = a[0]._obj
    rows = g.M * (g.split_k if g.atomic_out == L.VB_GEMM_PARTIALS else 1)     # deterministic split-K: one slice per split
    return [("out_f32", g.out_f32, rows, g.N, g.ld_out_f32, _F32),
            ("out_bf16", g.out_bf16, g.M, g.N, g.ld_out_bf16, L.VB_NAN_F16 if g.out_fp16 else _BF16),
            ("out_colsum", g.out_colsum, 1, g.N, g.N, _F32)]


def _attn_bwd_outputs(p, a):
    x = a[0]._obj
    hd, rq, rk = x.H * x.D, p._attn_rows(x.q_off, x.B, x.Nq), p._attn_rows(x.k_off, x.B, x.Nk)
    return [("dQ", x.dQ, rq, hd, x.lddq, _BF16), ("dK", x.dK, rk, hd, x.lddk, _BF16), ("dV", x.dV, rk, hd, x.lddv, _BF16),
            ("dbias_q", x.dbias_q, 1, hd, hd, _F32), ("dbias_k", x.dbias_k, 1, hd, hd, _F32), ("dbias_v", x.dbias_v, 1, hd, hd, _F32)]


def _vec(name, ptr, n, dt=_F32):
    return (name, ptr, 1, n, n, dt)


def _tables(*names):
    """Embedding-table gradients: whole parameter ranges."""
    return lambda p, a: [_vec(n, getattr(a, n), p._param_numel(getattr(a, n))) for n in names]


_ln_bwd = lambda p, a: [("dx_f32", a.dx_f32, a.M, a.H, a.lddx, _F32), ("dx_bf16", a.dx_bf16, a.M, a.H, a.lddx, _BF16),
                        _vec("dgamma", a.dgamma, a.H), _vec("dbeta", a.dbeta, a.H), _vec("dbias", a.dbias, a.H)]
_region_loss = lambda p, a: [("dscores_f32", a.dscores_f32, a.B * a.Nv, a.D, a.D, _F32)]
_scattered = lambda p, a: [("dst", a.dst, p._buf_rows[a.dst], a.cols, a.cols, _F32)]
ANOMALY_OUTPUTS = {
    "vb_gemm_bf16": _gemm_outputs,
    "vb_attention_bwd": _attn_bwd_outputs,
    "vb_layernorm_bwd": _ln_bwd,
    "vb_add_layernorm_bwd": _ln_bwd,
    "vb_colsum": lambda p, a: [_vec("out", a.out, a.N)],
    "vb_reduce_slices": lambda p, a: [_vec("dst", a.dst, a.n)],
    "vb_memset_zero": lambda p, a: [_vec("ptr", a.ptr, a.bytes // 4)],
    "vb_axpy_f32": lambda p, a: [_vec("y", a.y, a.n)],
    "vb_embed_text_bwd": _tables("dword", "dpos", "dtype", "dtask"),
    "vb_embed_text_bwd_padded": _tables("dword", "dpos", "dtype"),
    "vb_loc_proj_bwd": lambda p, a: [_vec("dW", a.dW, 5 * a.H), _vec("db", a.db, a.H)],
    "vb_loc_proj_dx": lambda p, a: [("dx", a.dx, a.M, 5, 5, _F32)],
    "vb_small_linear_bwd": lambda p, a: [("dx", a.dx, a.M, a.K, a.lddx, _F32), _vec("dW", a.dW, a.N * a.K), _vec("db", a.db, a.N)],
    "vb_fuse_pooled_bwd": lambda p, a: [_vec("da", a.da, a.n), _vec("db", a.db, a.n)],
    "vb_relu_bwd": lambda p, a: [_vec("dx_bf16", a.dx_bf16, a.n, _BF16), _vec("dx_f32", a.dx_f32, a.n)],
    "vb_sum_strided": lambda p, a: [_vec("dst", a.dst, a.count_k * a.n)],
    "vb_masked_mean_bwd": lambda p, a: [("dx", a.dx, a.B * a.N, a.H, a.H, _F32)],
    "vb_gate_scale_bwd": lambda p, a: [("dqk", a.dqk, a.B * a.N, a.cols, a.ldd, _BF16), ("dz", a.dz, a.B, a.cols, a.cols, _F32),
                                       ("dz16", a.dz16, a.B, a.cols, a.cols, _BF16)],
    "vb_scatter_rows_f32": _scattered,
    "vb_scatter_add_rows_f32": _scattered,
    "vb_pack_rows_f32": lambda p, a: [("dst", a.dst, a.rows, a.cols, a.cols, _F32)],
    "vb_unpack_rows_f32": lambda p, a: [("dst", a.dst, a.B * a.N, a.cols, a.cols, _F32)],
    "vb_zero_tail_rows": lambda p, a: [],      # zeros into the rows of no sample; the launch before it declared those buffers
    # packed retrieval (forward-only plans): int32 segments, and copies of rows some earlier launch wrote
    "vb_pack_segments": lambda p, a: [],
    "vb_broadcast_segment_rows": lambda p, a: [],
    "vb_cast2d_f32_to_bf16": lambda p, a: [("dst", a.dst, a.rows, a.cols, a.ldd, _BF16)],
    "vb_weight_norm_bwd": lambda p, a: [_vec("dg", a.dg, 1), _vec("dv", a.dv, a.n)],
    "vb_tanh_bwd": lambda p, a: [("dx_bf16", a.dx_bf16, a.M, a.N, a.N, _BF16), _vec("dbias", a.dbias, a.N)],
    "vb_concat_embed_ln_bwd": lambda p, a: [
        ("dxt", a.dxt, a.B * a.Nt, a.H, a.H, _F32), ("dxv", a.dxv, a.B * a.Nv, a.H, a.H, _F32),
        ("dxv_bf16", a.dxv_bf16, a.B * a.Nv, a.H, a.H, _BF16)] + [_vec(n, getattr(a, n), a.H) for n in (
            "dgamma_t", "dbeta_t", "dgamma_v", "dbeta_v", "dcol_v", "dcol_v2")],
    "vb_ce_loss": lambda p, a: [("dlogits_f32", a.dlogits_f32, a.rows, a.cols, a.ld_d32, _F32),
                                ("dlogits_bf16", a.dlogits_bf16, a.rows, a.cols, a.ld_d16, _BF16)],
    "vb_bce_logits_loss": lambda p, a: [("dlogits_f32", a.dlogits_f32, a.rows, a.cols, a.cols, _F32),
                                        ("dlogits_bf16", a.dlogits_bf16, a.rows, a.cols, a.ld_dlogits_bf16, _BF16)],
    "vb_bce_gather_loss": lambda p, a: [("dlogits_f32", a.dlogits_f32, a.rows, a.width, a.ld_d32, _F32),
                                        ("dlogits_bf16", a.dlogits_bf16, a.rows, a.width, a.ld_d16, _BF16)],
    "vb_kl_masked_loss": lambda p, a: [("dscores_f32", a.dscores_f32, a.B * a.Nv, a.C, a.C, _F32),
                                       ("dscores_bf16", a.dscores_bf16, a.B * a.Nv, a.C, a.ld_d16, _BF16)],
    "vb_mse_masked_loss": _region_loss,
    "vb_nce_region_loss": _region_loss,
    "vb_scale_by_device": lambda p, a: [_vec("dst", a.dst, a.n)],
}
# a _det twin takes its default entry point's parameters plus a trailing ws (vb_layernorm_bwd_det: those of vb_add_layernorm_bwd),
# so it shares that entry point's entry
ANOMALY_OUTPUTS.update({n: ANOMALY_OUTPUTS["vb_add_layernorm_bwd" if n == "vb_layernorm_bwd_det" else n[:-len("_det")]]
                        for n in L.FUNCTIONS if n.endswith("_det")})


# one checked region: its id (the index into Plan.nan_records) and where it comes from — the op (its index in Plan.fwd or Plan.bwd,
# `section`), the op's entry point and stream, the output (its index among the op's checked outputs and its name) and the module path
# of the block that emitted the op (a fused objective: its kind)
NanRecord = namedtuple("NanRecord", "region section op entry output name module stream")
C_SIZEOF_NAN_REGION = L.C.sizeof(L.NanRegion)
NAN_FLAG_CLEAR = 2 ** 31 - 1
# alignment of every buffer a plan places in a region of its own or in the shared arena
BUF_ALIGN = 256


def _struct_pointers(s):
    for cls in reversed(type(s).__mro__):
        for f, t in cls.__dict__.get("_fields_", ()):
            v = getattr(s, f)
            if t is L.C.c_void_p:
                if v:
                    yield v
            elif isinstance(t, type) and issubclass(t, L.C.Structure):
                yield from _struct_pointers(v)


def op_pointers(fn, args):
    """Every address one emitted launch passes: its void* arguments and the void* fields of the descriptor structs it passes by
    reference (nested ones included)."""
    for a, t in zip(args, fn.argtypes):
        if a is None:
            continue
        if hasattr(a, "_obj"):
            yield from _struct_pointers(a._obj)
        elif t is L.C.c_void_p:
            yield a


def happens_before_clocks(sections):
    """Vector clocks of the ops of `sections` (op lists run one after the other, every stream joined in between), from the stream
    markers Plan._run issues: -> [(op, stream, own count, clock before the op)]. An op x happens before an op y exactly when
    x's own count is at most y's clock-before entry for x's stream."""
    vc = [[0] * N_STREAMS for _ in range(N_STREAMS)]
    out, events = [], {}

    def join(dst, src):
        vc[dst] = [max(a, b) for a, b in zip(vc[dst], src)]
    for ops in sections:
        for s in range(N_STREAMS):              # a run starts after everything before it
            join(0, vc[s])
        for s in range(1, N_STREAMS):
            join(s, vc[0])
        for op in ops:
            fn, args, sid = op
            if fn is None:
                if not args:                    # text <-> vision barrier
                    join(1, vc[0]); join(0, vc[1])
                elif args[0] == "all":
                    for s in range(1, N_STREAMS):
                        join(s, vc[0])
                    for s in range(1, N_STREAMS):
                        join(0, vc[s])
                elif args[0] == "rec":
                    events[args[1]] = list(vc[sid])
                elif args[0] == "wait":
                    join(sid, events[args[1]])
                continue
            before = list(vc[sid])
            vc[sid][sid] += 1
            out.append((op, sid, vc[sid][sid], before))
    return out


def lifetime_layout(sections, spans, pinned):
    """First-fit placement by decreasing size of the byte ranges `spans` ((address, nbytes) of the buffers of a recording build,
    indexed) over their conflict graph. Two buffers conflict unless every use of one happens before every use of the other
    (happens_before_clocks) on the ops of `sections`; the buffers in `pinned` conflict with every used buffer (they live for the
    whole plan), and a buffer no op uses with none (it sits at offset 0, and the extent covers it). -> (offset per index, extent),
    offsets aligned to BUF_ALIGN."""
    n, S = len(spans), N_STREAMS
    big = 1 << 62
    last = [[0] * S for _ in range(n)]          # per stream: the latest own count of a use
    first = [[big] * S for _ in range(n)]       # per stream: the least clock-before entry over the uses
    used = [False] * n
    order = sorted((a, i) for i, (a, nb) in enumerate(spans) if nb > 0)
    starts = [a for a, _ in order]
    for op, s, own, before in happens_before_clocks(sections):
        fn, args, _ = op
        for p in op_pointers(fn, args):
            k = bisect.bisect_right(starts, p) - 1
            if k < 0:
                continue
            i = order[k][1]
            if p >= spans[i][0] + spans[i][1]:
                continue
            used[i] = True
            last[i][s] = max(last[i][s], own)
            first[i] = [min(a, b) for a, b in zip(first[i], before)]
    for i in pinned:
        last[i], first[i], used[i] = [big] * S, [0] * S, True

    def before(i, j):
        return all(a <= b for a, b in zip(last[i], first[j]))
    size = [-(-nb // BUF_ALIGN) * BUF_ALIGN for _, nb in spans]
    offset, placed = [0] * n, []
    extent = max([0] + [size[i] for i in range(n) if not used[i]])
    for i in sorted((i for i in range(n) if used[i] and size[i]), key=lambda i: (-size[i], i)):
        taken = sorted((offset[j], offset[j] + size[j]) for j in placed if not (before(i, j) or before(j, i)))
        off = 0
        for a, b in taken:
            if off + size[i] <= a:
                break
            off = max(off, b)
        offset[i] = off
        placed.append(i)
        extent = max(extent, off + size[i])
    return offset, extent


@dataclasses.dataclass(frozen=True)
class PlanSpec:
    """A plan's shape, options and the engine values its build reads (head_dropout_prob, bwd_gemm_max_ctas, the streams as the plan
    uses them), each in one normal form, so that one plan has exactly one spec: Engine.plan caches plans by it. PlanSpec.of makes it.

    grad_outputs: the outputs that will receive a gradient in backward (dead branches are not emitted). heads: "vl" | "pretraining"
    | "none" | the baseline's "base" | "base_none" (engine.ps.heads by default). train: nn.Dropout layers active (model.train()).

    loss fuses an objective of LOSS_HEADS into the plan (vqa_loss=True is the round-1 spelling of loss="vqa"): by default its
    kernel starts the backward, writes its scalar to self.loss and writes d loss / d head into the head's output-gradient buffer
    (loss="vqa", the round-1 objective of task_utils.py:325-327, also writes the head's bf16 backward operand, so no cast runs).
    Its labels and targets are static plan inputs (self.loss_inputs); the objective, score and results of a task kind address
    its head through one layout (_head_layout), and _objective_outputs sets up where their scalars land.

    Task objectives (TASK_KINDS) take three more options. loss_in_forward=True emits the objective at the END of the forward list
    (a forward-only plan yields the loss) and stores d loss / d head; the backward then starts with head gradient = stored gradient
    x self.loss_grad (a device scalar, 1 by default: what the caller's d(total)/d(loss) is copied into). score=True also emits the
    on-device batch score of the kind (self.score, device f32 [1]; self.preds, the per-row argmax). choices: answer options of
    logit_ce (engine.loss_options by default) and multiple-choice ids per sample of vlogit_mc; None for every other objective.

    loss="pretraining" with loss_in_forward=True keeps the three pre-training losses apart: self.objective_out (device f32 [3]) holds
    masked_lm, masked_img and next_sentence, self.loss is None, and self.loss_grad (f32 [3]) scales each head gradient by its own
    slot. A plan without grad_outputs computes the losses only and writes no gradient. pretraining: the engine and config values
    its build reads (engine.lm_compact, engine.lm_capacity, config.visual_target, nce_negative_count), None for other plans.

    outputs: the heads (names of HEAD_NAMES) the plan builds; None builds all of them. A head not named gets no kernel, no buffer
    and no entry in self.outputs (the four BertModel outputs are always there); what a kept head reads (the fused pooled vector,
    the alignment head of an odd batch, dropout sites) is built as in the all-heads plan, so a kept head is bitwise the same.
    results: a kind of RESULT_MODES; the forward ends with vb_task_results on that kind's head, and self.results_out packs
    objective_out (loss, score), the per-row argmax and the per-row values into one device buffer (fetch_results).
    With heads="pretraining", outputs= names heads of PRETRAINING_HEAD_NAMES: ("seq_relationship_score",) builds no masked-LM or
    region decoder.

    fast_mode: text batch 1 broadcast to the image batch (config.fast_mode by default). image_prefix=True (forward-only plans): the
    image embedding (feature cast, box projection, embedding GEMM, LayerNorm) and the additive image mask are emitted into
    self.prefix, run by run_image_prefix() on what load_images() loaded, and write private buffers that no op of the forward writes;
    the forward starts at the text embeddings and reads those image states as they are, so one image batch serves many text forwards.

    frozen: ParamStore entry names whose parameters take no gradient (requires_grad=False; the tied decoder is the word-embedding
    entry). While the forward is emitted every activation records whether it needs a gradient, as autograd does: it does when the
    op that produced it has a trainable parameter or an input that needs one (Act.rg, set by Plan.act). The forward is the
    same; the backward computes no gradient of a frozen parameter (no weight-gradient GEMM, bias column sum, LayerNorm gamma /
    beta sum or embedding scatter), no gradient of an activation that needs none, and registers nothing for a block with nothing
    to do. No range a frozen parameter owns appears in grad_touch. self.out_rg tells which outputs carry a gradient.

    input_grads: a subset of INPUT_GRAD_NAMES whose gradient the backward also computes. The image embedding's output then needs a
    gradient even with all of its parameters frozen, and the backward ends the image-embedding chain with d(input_imgs) = dy W (the
    feature GEMM's dgrad) and d(image_loc) = dy W_loc (vb_loc_proj_dx). They land in private buffers outside the arena and outside
    grad_touch; self.input_grad maps each input whose gradient the backward writes to its buffer ([B*Nv, Fv] / [B*Nv, 5] fp32). An
    input behind a no_grad layer (fixed_v_layer > 0) gets no entry, as it gets no gradient in torch.

    packed=(rows_t, rows_v): the two streams hold the valid rows only (DESIGN.md §4g). Refused with the options that reshape or
    export the padded streams, with input gradients (they are padded tensors) and with heads that are not packed: the heads of
    VILBertForVLTasks among PACKED_HEADS (outputs=), or the three heads of BertForMultiModalPreTraining under the fused objective
    with its losses in the forward (loss="pretraining", loss_in_forward=True, engine.lm_compact, all three heads). Retrieval
    (fast_mode and image_prefix together, forward-only) packs with the score head alone (RETRIEVAL_SCORE_HEADS): rows_t then counts
    the caption's rows after its broadcast to the B images.

    deterministic=True (torch.use_deterministic_algorithms(True), DESIGN.md §4h; None reads torch's flag at the call): every sum
    that float atomics would make order-dependent goes through the _det variant of its kernel (per-block partials in a workspace of
    the plan, then one ordered sum), the GEMM weight gradients that split K store their splits apart and add them in split order,
    and all launches go to one stream, so no two kernels add into the same range concurrently. Two runs give bitwise identical
    results on the same GPU model and build. self.det_ws_bytes: the workspace the plan allocated for it. The single-stream
    baseline has kernels without a deterministic variant: it raises RuntimeError, or with torch's warn_only=True warns and builds
    the default plan.

    recycle=True (forward-only plans: no train mode, no grad_outputs, no input_grads; DESIGN.md §3; None takes
    engine.recycle_forward_only for a forward-only plan): buffers whose lifetimes are disjoint share bytes. The plan is built twice
    in the same order. The first build records every buffer request in host memory that it does not fill (also under
    torch.use_deterministic_algorithms(True)); the vector clocks of its ops (happens_before_clocks) give each buffer its uses, and
    lifetime_layout places them. The second build emits the same launches with each buffer at its place, in one region of the
    plan or, with the shared arena, at the start of the arena (arena_bytes is the extent). Private buffers and the buffers the host
    reads after a run (_host_reads) keep bytes of their own. self.held_bytes: arena extent + the plan's own device buffers.

    anomaly=True (torch.autograd.set_detect_anomaly(True), DESIGN.md §4i; None reads torch.is_anomaly_enabled() and
    torch.is_anomaly_check_nan_enabled() at the call; a plan with no backward has nothing to check and is the unchecked plan):
    every op in the backward role — the backward list, the head-gradient writes of a forward-placed objective, vb_scale_by_device —
    is tagged with the module path of the block that emitted it, and after each block one vb_nan_check per stream the block used
    scans the gradients its ops wrote (ANOMALY_OUTPUTS) on that stream. Region ids follow op-list order and the flag (reset at the
    start of every forward) keeps the least id that held a NaN, so anomaly_report() names the first op whose outputs held one.
    Removing the checks and the reset leaves the unchecked plan's launches. The checks only read."""
    B: int
    Nt: int
    Nv: int
    grad_outputs: frozenset
    heads: str
    train: bool
    loss: str
    choices: int
    score: bool
    loss_in_forward: bool
    outputs: frozenset
    results: str
    fast_mode: bool
    image_prefix: bool
    frozen: frozenset
    input_grads: frozenset
    packed: tuple
    deterministic: bool
    recycle: bool
    anomaly: bool
    head_dropout_prob: float
    bwd_gemm_max_ctas: int
    two_streams: bool
    wgrad_streams: bool
    pretraining: tuple

    @classmethod
    def of(cls, engine, B, Nt, Nv, grad_outputs=(), vqa_loss=False, heads=None, train=False, loss=None, choices=None, score=False,
           loss_in_forward=False, outputs=None, results=None, fast_mode=None, image_prefix=False, frozen=frozenset(),
           input_grads=frozenset(), packed=None, deterministic=None, recycle=None, anomaly=None):
        """The spec of the plan of `engine` with this shape and these options; raises what the options ask that no plan does."""
        cfg, base = engine.cfg, engine.ps.base
        grad_outputs, frozen, input_grads = frozenset(grad_outputs), frozenset(frozen), frozenset(input_grads)
        outputs = None if outputs is None else frozenset(outputs)
        packed = None if packed is None else (int(packed[0]), int(packed[1]))
        train, score, loss_in_forward, image_prefix = bool(train), bool(score), bool(loss_in_forward), bool(image_prefix)
        loss = "vqa" if vqa_loss else loss
        backward = bool(grad_outputs or input_grads)
        recycle = bool(engine.recycle_forward_only and not (train or backward) if recycle is None else recycle)
        det = torch.are_deterministic_algorithms_enabled() if deterministic is None else bool(deterministic)
        if anomaly is None:
            anomaly = torch.is_anomaly_enabled() and torch.is_anomaly_check_nan_enabled()
        anomaly = bool(anomaly) and backward
        if det and base:
            msg = (f"{' and '.join(DET_MISSING_BASELINE)} (the backward of BaseBertForVLTasks' embeddings) add with float atomics and "
                   "have no deterministic implementation; build the plan without torch.use_deterministic_algorithms(True), or with "
                   "warn_only=True to run the default kernels")
            if not torch.is_deterministic_algorithms_warn_only_enabled():
                raise RuntimeError(msg)
            warnings.warn(msg)
            det = False
        if packed is not None and base:
            raise NotImplementedError("packed plans run the two-stream VILBertForVLTasks only")
        if base and (loss is not None or outputs is not None or results is not None or fast_mode or image_prefix or score
                     or loss_in_forward):
            raise ValueError("single-stream baseline plans support grad_outputs, train, frozen, input_grads and recycle only")
        if anomaly and recycle:
            raise ValueError("anomaly checks read the gradients of a backward: a recycled (forward-only) plan has none")
        if recycle and (train or backward):
            raise ValueError("recycle=True shares the bytes of buffers whose lifetimes are disjoint, which only a forward-only plan "
                             "has: no train mode, no grad_outputs, no input_grads (the backward reads the saved activations)")
        unknown = sorted(n for n in frozen if n not in engine.ps.entries)
        if unknown:
            raise ValueError(f"frozen: {unknown[:4]} are not parameter entries of this model")
        unknown = sorted(n for n in input_grads if n not in INPUT_GRAD_NAMES)
        if unknown:
            raise ValueError(f"input_grads: {unknown} are not among the differentiable inputs {INPUT_GRAD_NAMES}")

        # the two-stream options (Plan._stream_modes); the baseline has none of them
        pairs, viz, dyn = [not base and bool(getattr(cfg, f, False)) for f in ("in_batch_pairs", "visualization", "dynamic_attention")]
        fast = not base and bool(getattr(cfg, "fast_mode", False) if fast_mode is None else fast_mode)
        if viz and train:
            raise ValueError("visualization exports the undropped attention probabilities: eval mode only")
        if fast and (train or grad_outputs or loss):
            raise ValueError("fast_mode is an inference path (text batch 1 broadcast to the image batch): no train mode / gradients")
        if image_prefix and (train or grad_outputs):
            raise ValueError("image_prefix keeps the image states across forwards: forward-only plans (no train mode, no grad_outputs)")
        if image_prefix and pairs:
            raise ValueError("image_prefix: in_batch_pairs re-expands the image batch inside the forward")
        if input_grads and (fast or image_prefix):
            raise ValueError("fast_mode and image_prefix plans are inference paths: no input gradients")

        # the fused objective
        if loss is not None and loss not in LOSS_HEADS:
            raise ValueError(f"loss must be one of {sorted(LOSS_HEADS)}")
        if (loss_in_forward or score) and loss not in TASK_KINDS and not (loss == "pretraining" and not score):
            raise ValueError(f"loss_in_forward needs a task objective, one of {TASK_KINDS}, or 'pretraining'; score needs a task objective")
        if score and loss not in SCORE_MODES:
            raise ValueError(f"loss={loss!r} has no batch score: with int labels the reference's compute_score_with_logits "
                             "raises (task_utils.py:618-623)")
        if loss == "vlogit_mc" and not (choices and choices > 0):
            raise ValueError("loss='vlogit_mc' needs choices= (multiple-choice ids per sample)")
        if loss == "vlogit_mc" and Nv <= MC_REGION_OFFSET:
            raise ValueError(f"loss='vlogit_mc' scores the regions after the first {MC_REGION_OFFSET}: Nv must exceed it")

        # outputs= and results=: known head names, and every head the objective, a gradient or the results read is kept
        heads = engine.ps.heads if heads is None else heads
        if results is not None:
            if results not in RESULT_MODES:
                raise ValueError(f"results must be one of {sorted(RESULT_MODES)}, got {results!r}")
            if loss is not None and (loss != results or not loss_in_forward):
                raise ValueError(f"results={results!r} goes with loss=None or loss={results!r}, loss_in_forward=True (got loss={loss!r})")
            if results not in ("vqa", "gqa") and loss != results:
                raise ValueError(f"results={results!r} reads the inputs of its objective: build it with loss={results!r}, loss_in_forward=True")
        if outputs is not None:
            if heads == "pretraining" and all(n in HEAD_NAMES + PRETRAINING_HEAD_NAMES for n in outputs):
                other = sorted(n for n in outputs if n not in PRETRAINING_HEAD_NAMES)
                if other:
                    raise ValueError(f"outputs: {other} are heads of VILBertForVLTasks (heads='vl'); the heads of heads='pretraining' are "
                                     f"{PRETRAINING_HEAD_NAMES}")
            else:
                unknown = sorted(n for n in outputs if n not in HEAD_NAMES)
                if unknown:
                    raise ValueError(f"outputs: unknown head name(s) {unknown}; the heads are {HEAD_NAMES}")
                if heads != "vl":
                    raise ValueError(f"outputs= selects among the heads of VILBertForVLTasks (heads='vl') or of BertForMultiModalPreTraining "
                                     f"(heads='pretraining'), not heads={heads!r}")
            need = {n for n in grad_outputs if n in HEAD_NAMES + PRETRAINING_HEAD_NAMES}
            if loss is not None:
                need |= set(LOSS_HEADS[loss])
            if results is not None:
                need.add(RESULT_MODES[results][0])
            missing = sorted(need - outputs)
            if missing:
                raise ValueError(f"outputs={sorted(outputs)} misses {missing}, which the plan's objective, gradients or results read")

        # packed=: the rows of each stream at the batch and text length the streams run at
        if packed is not None:
            rows_t, rows_v = packed
            Bs, Nts = B * B if pairs else B, Nt + (1 if cfg.task_specific_tokens else 0)
            if rows_t < 1 or rows_v < 1 or rows_t > Bs * Nts or rows_v > Bs * Nv:
                raise ValueError(f"packed={packed}: the rows of each stream must lie in [1, B * N] = [1, {Bs * Nts}], [1, {Bs * Nv}]")
            retrieval = fast and image_prefix
            bad = [n for n, on in (("in_batch_pairs", pairs), ("fast_mode", fast and not retrieval), ("dynamic_attention", dyn),
                                   ("visualization", viz), ("image_prefix", image_prefix and not retrieval),
                                   ("input_grads", bool(input_grads)))
                   if on]
            if bad:
                raise NotImplementedError(f"packed plans do not support {', '.join(bad)}")
            if retrieval:
                head = RETRIEVAL_SCORE_HEADS.get(heads)
                if head is None or outputs != {head} or loss is not None or results:
                    raise NotImplementedError(f"packed retrieval plans build the score head alone: outputs=({head!r},), no objective, got "
                                              f"{None if outputs is None else sorted(outputs)}")
            elif heads == "pretraining":
                if not (loss == "pretraining" and loss_in_forward and engine.lm_compact and
                        (outputs is None or outputs == frozenset(PRETRAINING_HEAD_NAMES))):
                    raise NotImplementedError("packed pre-training plans run the fused objective only: loss='pretraining', "
                                              "loss_in_forward=True, engine.lm_compact and all three heads")
            elif engine.ps.heads != "vl" or outputs is None or any(n not in PACKED_HEADS for n in outputs):
                raise NotImplementedError(f"packed plans build heads of VILBertForVLTasks among {PACKED_HEADS} only (outputs=...), got "
                                          f"{None if outputs is None else sorted(outputs)}")

        # what the objective's head layout reads (_head_layout)
        if loss is not None and not loss_in_forward:      # a forward-placed objective also serves forward-only (eval) plans
            if any(n not in grad_outputs for n in LOSS_HEADS[loss]):
                raise ValueError(f"loss={loss!r} differentiates {LOSS_HEADS[loss]}: add them to grad_outputs")
        if loss == "logit_ce":        # vil_logit.view(B / options, options); results="logit_ce" goes with this loss
            choices = choices or engine.loss_options
            rows = B * B if pairs else B
            if rows % choices:
                raise ValueError(f"loss='logit_ce': batch {rows} is not a multiple of {choices} options")
        else:
            choices = int(choices) if loss == "vlogit_mc" else None
        pre = (engine.lm_compact, engine.lm_capacity, cfg.visual_target, nce_negative_count(cfg)) if loss == "pretraining" else None
        two = engine.two_streams and not det
        return cls(B, Nt, Nv, grad_outputs, heads, train, loss, choices, score, loss_in_forward, outputs, results, fast, image_prefix,
                   frozen, input_grads, packed, det, recycle, anomaly, engine.head_dropout_prob, engine.bwd_gemm_max_ctas, bool(two),
                   bool(engine.wgrad_streams and two), pre)


class Plan:
    """Static execution plan of one PlanSpec, which documents its options."""

    def __init__(self, engine, spec, _recording=False):
        self.spec = spec
        self.recycle, self.anomaly = spec.recycle, spec.anomaly
        self._requests = [] if _recording else None     # recording build: (tensor, bytes, private) per buffer request
        self._place, self._n_req, self._region = None, 0, None
        if self.recycle and not _recording:
            # the recording build's buffers are address ranges only: torch.use_deterministic_algorithms(True) would fill each
            # torch.empty with NaN, writing host memory as large as the plain plan
            fill = torch.utils.deterministic.fill_uninitialized_memory
            torch.utils.deterministic.fill_uninitialized_memory = False
            try:
                rec = type(self)(engine, spec, _recording=True)
            finally:
                torch.utils.deterministic.fill_uninitialized_memory = fill
            self._place = rec._lifetime_placement()
        self.e, self.cfg = engine, engine.cfg
        self.det, self.packed, self.frozen, self.input_grads = spec.deterministic, spec.packed, spec.frozen, spec.input_grads
        self.train, self.heads, self.keep, self.fast, self.image_prefix = spec.train, spec.heads, spec.outputs, spec.fast_mode, spec.image_prefix
        # objective fused into the step (LOSS_HEADS): its scalar lands in self.loss (device) and its gradient goes straight into the
        # backward of the head(s) it reads
        self.grad_outputs, self.loss_kind, self.choices, self.results = spec.grad_outputs, spec.loss, spec.choices, spec.results
        self.loss_in_forward, self.want_score = spec.loss_in_forward, spec.score
        self.head_dropout_prob, self.two_streams, self.wgrad_streams = spec.head_dropout_prob, spec.two_streams, spec.wgrad_streams
        self._det_ws, self.det_ws_bytes = None, 0
        self._det_bias = []      # deterministic plans: attention bias sums (bias, d(Q|K|V), pitch) left to det_bias_sums
        self.input_grad = {}          # input name -> the buffer its gradient lands in (written by the backward)
        self.out_rg = {}              # output name -> it carries a gradient (some trainable parameter lies upstream of it)
        self.grad_touch = {}           # (flat offset, numel) -> index of the last backward op writing that gradient range
        self.ps = engine.ps
        self.lib = L.lib()
        self.dev = engine.device
        self.Bin = spec.B
        self._stream_modes(spec.B, spec.Nt, spec.Nv)
        self.attn_t, self.attn_v, self.attn_c = [], [], []
        self.prefix = []         # image_prefix: the image embedding and mask, run by run_image_prefix()
        self._private = False    # while set, buf() allocates private buffers (the image states of image_prefix)
        self.task_objective = self.loss_in_forward or self.want_score     # the objective's scalars live in self.objective_out
        self.op_dtype, self.split = engine.op_dtype, engine.split   # format of the forward operands (activations, weights)
        self.fwd_id = 0
        self.fwd, self.bwd = [], []
        self.prologue = []       # optional per-step ops run before the forward (see enable_training_prologue)
        self.epilogue = []       # optional per-step ops run after the backward (the fused optimizer: enable_optimizer)
        self.cur = self.fwd
        self.sid = 0             # stream the next emitted op goes to: 0 = text/main stream, 1 = vision stream
        self._streams = None
        self._n_events = 0
        self._scratch_epoch = 0
        self._keep = []          # ctypes structs / tensors referenced by raw pointer
        self._scratch = {}
        self._bwd_emitters = []
        self._no_grad = False    # set while a layer under the reference's torch.no_grad() is built (fixed_t_layer / fixed_v_layer)
        self._last_attn = None   # visualization: the export of the attention emitted last
        self._scatter_ok = False          # the baseline's row heads may scatter straight into the stream gradient (base_rows)
        self._live_ranges_cache = {}      # (lo, hi) -> live_ranges(lo, hi), for run_step_overlapped
        self._bucket_schedules = {}       # bucket table -> bucket_schedule(table)
        self._step_schedules = {}         # (bucket table, allreduce) -> step_schedule(table, allreduce)
        self._piece_runs, self._piece_graphs = Counter(), {}     # schedule -> eager runs / its graphs (run_backward_pieces)
        self.n_kernels_fwd = self.n_kernels_bwd = 0
        self.graph_fwd = self.graph_bwd = self.graph_step = None
        self._eager_runs = [0, 0]      # eager forward / backward executions (maybe_capture_passes)
        self._arena_off = self.arena_bytes = 0
        if self._place is not None:
            self._open_region()
        self._label = None       # module path of the backward-role ops being emitted (role()); None: not the backward role
        self._pending = []       # anomaly: (op list, index, module path) of the backward-role ops since the last check
        self._buf_rows = {}      # anomaly: data pointer -> leading dimension of the plan's buffers (extents of scattered-into rows)
        self.nan_records, self._nan_checks = [], []
        self.nan_flag = None
        if self.anomaly:
            self.nan_flag = torch.full((1,), NAN_FLAG_CLEAR, dtype=torch.int32, device=self.dev)
            self.emit(self.lib.vb_nan_check, None, 0, self.nan_flag, 1)       # the reset: first launch of every forward
        self._build()
        if self.anomaly:
            self._nan_table()
        if self._place is not None and self._n_req != len(self._place[0]):
            raise L.VBError(f"recycled plan: the second build made {self._n_req} buffer requests, the first {len(self._place[0])}")

    def _stream_modes(self, B, Nt, Nv):
        """Shapes of the two-stream options: in_batch_pairs, the task token, visualization, dynamic_attention and fast_mode."""
        # in_batch_pairs (vilbert.py:1008-1040): at the first connection layer every (text i, image j) combination of the input
        # batch becomes one sample: the streams run at the input batch before it and at B^2 from there on
        self.pairs = bool(getattr(self.cfg, "in_batch_pairs", False))
        self.B, self.Nt_in, self.Nv = (B * B if self.pairs else B), Nt, Nv
        self.has_task = bool(self.cfg.task_specific_tokens)
        self.Nt = Nt + (1 if self.has_task else 0)
        # FAST_MODE (vilbert.py:1042-1053, eval_retrieval.py): one caption (text batch 1) against B images; inference only
        # config.visualization (vilbert.py:451-458, 610-617, 813-821): export attention probabilities, queries and keys per layer
        self.viz = bool(getattr(self.cfg, "visualization", False))
        self.dyn = bool(getattr(self.cfg, "dynamic_attention", False))
        self.Bt = 1 if self.fast else B

    def want(self, name):
        """Whether the head `name` is built (outputs=)."""
        return self.keep is None or name in self.keep

    # ------------------------------------------------------------------ frozen parameters
    def trainable(self, *names):
        """Whether any of the parameters `names` takes a gradient. A name is an entry, a fused projection, or a Linear / LayerNorm
        module, which stands for its .weight and .bias."""
        entries, parts = self.ps.entries, self.ps.parts
        names = [m for n in names for m in ((n,) if n in entries or n in parts else (n + ".weight", n + ".bias"))]
        return any(p not in self.frozen for n in names for p in parts.get(n, (n,)))

    def act(self, f32, op, M, H, inputs=(), params=(), rg=False):
        """The Act an op makes from the Acts `inputs` with the parameters `params` (names as for trainable). It needs a gradient when
        one of them does (rule 1 of Act); rg: whether an input that is not an Act does (an operand whose producer the caller tracks,
        a plan input of input_grads). Under torch.no_grad() nothing does."""
        rg = not self._no_grad and bool(rg or any(i.rg for i in inputs) or self.trainable(*params))
        return Act(f32, op, M, H, rg)

    def grad_view(self, name):
        """Gradient view of the entry or fused projection `name` for the next backward op to write. grad_touch keeps, per range,
        the index of the last backward op that writes it."""
        if self.cur is self.bwd:
            self.grad_touch[self.ps.span(name)] = len(self.bwd)
        return self.ps.g(name)

    def pg(self, name):
        """Gradient view of the entry `name` for a backward op to write, or None when it is frozen."""
        return None if name in self.frozen else self.grad_view(name)

    def gparts(self, name):
        """Gradient views of the parts of `name` (the entries of a fused projection, or the entry itself), None for a frozen part.
        With every part trainable they are slices of one view of the whole range."""
        parts = self.ps.parts.get(name)
        if parts is None:
            return [self.pg(name)]
        if not any(p in self.frozen for p in parts):
            g = self.grad_view(name)
            n = g.shape[0] // len(parts)
            return [g[i * n:(i + 1) * n] for i in range(len(parts))]
        return [self.pg(p) for p in parts]

    @staticmethod
    def _runs(parts):
        """Maximal runs [a, b) of consecutive non-None entries of `parts`."""
        runs, a = [], None
        for i, g in enumerate(list(parts) + [None]):
            if g is not None and a is None:
                a = i
            elif g is None and a is not None:
                runs.append((a, i))
                a = None
        return runs

    # ------------------------------------------------------------------ infrastructure
    def buf(self, shape, dtype=F32, zero=False):
        """A static buffer of the plan. With the engine's shared activation arena enabled (Engine.enable_activation_arena), buffers
        that hold no state between runs (activations, scratch: everything a run writes before reading) are sub-allocated from the
        arena at the same offsets in every plan, so the plans of different shapes overlay each other; buffers that are
        initialised at build time or loaded from outside a run (zero=True: inputs, labels, output gradients, zero-padded
        operands) stay private.

        A recycled plan (recycle=True) places the other buffers where its recording build's lifetimes put them (_place), in
        its region (_open_region); the recording build itself hands out host memory it does not fill."""
        arena = self.e.arena
        zero = zero or self._private
        n = math.prod(int(d) for d in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        if self._requests is not None:
            t = torch.empty(shape, dtype=dtype)
            self._requests.append((t, nbytes, zero))
            return t
        if self._place is not None:
            sigs, offsets, _ = self._place
            i = self._n_req
            self._n_req += 1
            if i >= len(sigs) or sigs[i] != (nbytes, zero):
                raise L.VBError(f"recycled plan: buffer request {i} ({nbytes} bytes, private={zero}) differs from the recording build's")
            if not zero:
                return self._region[offsets[i]:offsets[i] + nbytes].view(dtype).view(shape)
        if arena is None or zero:
            t = (torch.zeros if zero else torch.empty)(shape, dtype=dtype, device=self.dev)
            self._keep.append(t)
        else:
            off = self._arena_off
            if off + nbytes > arena.numel():
                raise L.VBError(f"activation arena of {arena.numel() / 2**30:.2f} GiB is too small for plan B={self.B} Nt={self.Nt} Nv={self.Nv} "
                                f"(needs more than {(off + nbytes) / 2**30:.2f} GiB): pass a larger size to Engine.enable_activation_arena")
            self._arena_off = (off + nbytes + 255) // 256 * 256
            self.arena_bytes = self._arena_off
            t = arena[off:off + nbytes].view(dtype).view(shape)
        if self.anomaly and t.dim():
            self._buf_rows[t.data_ptr()] = t.shape[0]
        return t

    def _host_reads(self):
        """The tensors the host may read after a run, besides the private buffers: the outputs, the encoded layers
        (output_all_encoded_layers) and the attention exports of config.visualization."""
        acts = getattr(self, "enc_t", []) + getattr(self, "enc_v", []) + getattr(self, "enc", [])
        attn = self.attn_t + self.attn_v + [d for pair in self.attn_c for d in pair]
        return list(self.outputs.values()) + [a.f32 for a in acts] + [d[k] for d in attn for k in ("attn", "q", "k")]

    def _lifetime_placement(self):
        """Of a recording build: (per request (bytes, private), per request its offset in the recycled region or None when
        private, the region's extent). The one rule of what is not recycled: a private buffer stays private, and a buffer the host
        reads after a run (_host_reads) lives for the whole plan."""
        reqs = self._requests
        spans = [(t.data_ptr(), 0 if zero else nb) for t, nb, zero in reqs]
        pinned = set()
        for t in self._host_reads():
            p = t.data_ptr()
            pinned.update(i for i, (a, nb) in enumerate(spans) if a <= p < a + nb)
        offsets, extent = lifetime_layout((self.prefix, self.fwd, self.bwd), spans, pinned)
        return ([(nb, zero) for _, nb, zero in reqs], [None if zero else off for (_, _, zero), off in zip(reqs, offsets)], extent)

    def _open_region(self):
        """The bytes a recycled plan places its buffers in: the start of the shared arena (its extent is arena_bytes), or one
        device buffer of its own."""
        extent, arena = max(self._place[2], 1), self.e.arena
        if arena is None:
            self._region = torch.empty(extent, dtype=torch.uint8, device=self.dev)
            self._keep.append(self._region)
            return
        if extent > arena.numel():
            raise L.VBError(f"activation arena of {arena.numel() / 2**30:.2f} GiB is too small for plan B={self.B} Nt={self.Nt} Nv={self.Nv} "
                            f"(needs {extent / 2**30:.2f} GiB): pass a larger size to Engine.enable_activation_arena")
        self._region = arena
        self.arena_bytes = extent

    @property
    def held_bytes(self):
        """Device bytes the plan holds: its extent of the shared arena and its own buffers."""
        return self.arena_bytes + sum(t.numel() * t.element_size() for t in self._keep if torch.is_tensor(t))

    def buf16(self, shape, bw=True):
        """Forward-operand buffer in the engine's operand format; bw=False: no bf16 copy (nothing in the backward reads it)."""
        hi = self.buf(shape, self.op_dtype)
        lo = self.buf(shape, self.op_dtype) if self.split else None
        return Operand(hi, lo, None if not bw else (hi if self.op_dtype == BF16 else self.buf(shape, BF16)))

    def scratch(self, tag, shape, dtype):
        # with asynchronous weight-gradient streams a temporary may still be read after its layer's backward has moved on:
        # temporaries are then unique per backward emitter instead of being recycled by the next layer
        key = (tag, tuple(shape), dtype, self._scratch_epoch if self.wgrad_streams else 0)
        if key not in self._scratch:
            self._scratch[key] = self.buf(shape, dtype)
        return self._scratch[key]

    def emit(self, fn, *args):
        """Appends a launch of `fn` to the pass being built. Tensors, None and descriptor structs are passed as they are: the
        arguments become C values here (_lib.launch_args), which also checks their count against fn's prototype. A deterministic
        plan launches the _det twin of an entry point of DET_WORKSPACE instead, with its workspace."""
        if self.det and fn.__name__ in DET_WORKSPACE:
            size = DET_WORKSPACE[fn.__name__]
            if size is not None:
                args = args + (self.det_ws(size(L.launch_args(fn, *args))),)
            fn = getattr(self.lib, fn.__name__ + "_det")
        self.cur.append((fn, L.launch_args(fn, *args), self.sid if self.two_streams else 0))
        if self.anomaly and self._label is not None:
            self._pending.append((self.cur, len(self.cur) - 1, self._label))
        elif self.anomaly and self.cur is self.bwd:
            raise L.VBError(f"{fn.__name__}: a launch of the backward list emitted outside a role() (anomaly checks need its module)")

    # ------------------------------------------------------------------ anomaly detection
    class _Role:
        def __init__(self, plan, label):
            self.plan, self.label = plan, label

        def __enter__(self):
            self.prev = self.plan._label
            self.plan._label = self.label

        def __exit__(self, *exc):
            self.plan._label = self.prev
            if self.prev is None and exc[0] is None:
                self.plan._emit_nan_checks()
            return False

    def role(self, label):
        """Context in which the emitted ops are backward-role ops of the module `label` (None: not backward-role ops). Leaving the
        outermost role ends a block: a checked plan emits its checks there (_emit_nan_checks)."""
        return Plan._Role(self, label)

    def _emit_nan_checks(self):
        """After a block: the checked outputs (ANOMALY_OUTPUTS) of its backward-role ops become regions with ids in op-list order,
        and one vb_nan_check per stream the block used scans that stream's regions, on that stream after the block's ops. The
        launch's arguments are set by _nan_table once every region is known."""
        pending, self._pending = self._pending, []
        streams = OrderedDict()
        for ops, i, label in pending:
            fn, args, sid = ops[i]
            spec = ANOMALY_OUTPUTS.get(fn.__name__)
            if spec is None:
                raise L.VBError(f"{fn.__name__} runs in the backward role ({label}) but has no entry in engine.ANOMALY_OUTPUTS")
            k, section = 0, "fwd" if ops is self.fwd else "bwd"
            for name, ptr, rows, cols, ld, dt in spec(self, args):
                if not ptr or rows <= 0 or cols <= 0:
                    continue
                rid = len(self.nan_records)
                self.nan_records.append(NanRecord(rid, section, i, fn.__name__, k, name, label, sid))
                streams.setdefault(sid, []).append((ptr, rows, cols, ld, dt, rid))
                k += 1
        for sid, regions in streams.items():
            self.cur.append((self.lib.vb_nan_check, None, sid))
            self._nan_checks.append((self.cur, len(self.cur) - 1, regions))

    def _nan_table(self):
        """The static device table of every check's regions (contiguous per launch) and the arguments of the check launches."""
        regions = [r for _, _, rs in self._nan_checks for r in rs]
        arr = (L.NanRegion * max(len(regions), 1))()
        for e, (ptr, rows, cols, ld, dt, rid) in zip(arr, regions):
            e.ptr, e.rows, e.cols, e.ld, e.dtype, e.id = ptr, rows, cols, ld, dt, rid
        raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
        self.nan_table = raw.to(self.dev) if self.dev.type == "cuda" else raw
        size, first = C_SIZEOF_NAN_REGION, 0
        for ops, i, rs in self._nan_checks:
            fn = self.lib.vb_nan_check
            ops[i] = (fn, L.launch_args(fn, self.nan_table.data_ptr() + size * first, len(rs), self.nan_flag, 0), ops[i][2])
            first += len(rs)
        self.nan_regions = regions

    def anomaly_report(self):
        """After a backward of a checked plan (anomaly=True): the NanRecord of the first region, in op-list order, that held a NaN,
        or None. One device-to-host read of the flag (the host waits for the current stream)."""
        if not self.anomaly:
            raise ValueError("anomaly_report: the plan was built without anomaly checks")
        v = int(self.nan_flag.item())
        return None if v == NAN_FLAG_CLEAR else self.nan_records[v]

    def _attn_rows(self, off, B, N):
        """Query or key rows of an attention launch: B * N, or the rows of the packed stream whose offsets `off` points at."""
        if not off:
            return B * N
        return next(self.packed[k] for k, s in enumerate(("t", "v")) if self.seg[s][0].data_ptr() == off)

    def _param_numel(self, ptr):
        """Elements of the parameter-gradient entry that starts at `ptr` (0 for a null pointer)."""
        if not ptr:
            return 0
        off = (ptr - self.ps.grad.data_ptr()) // 4
        return next(math.prod(shape) for o, shape in self.ps.entries.values() if o == off)

    def det_ws(self, n):
        """fp32 workspace of at least n floats for a deterministic launch. A deterministic plan runs on one stream, so launches share
        the current buffer: each partials kernel and the ordered sum after it are done before the next launch writes it. A request
        larger than the current buffer allocates a new one; the launches emitted before keep the old one, so the plan holds every
        size the workspace grew through (all counted in det_ws_bytes)."""
        if self._det_ws is None or self._det_ws.numel() < n:
            self._det_ws = torch.empty(max(int(n), 1), dtype=F32, device="cpu" if self._requests is not None else self.dev)
            self._keep.append(self._det_ws)
            self.det_ws_bytes += self._det_ws.numel() * 4
        return self._det_ws

    def det_bias_sums(self):
        """Deterministic plans: the attention bias gradients the backward kernels would have summed with atomics, as ordered column
        sums of d(Q|K|V) (after the packed tail rows are zeroed)."""
        pending, self._det_bias = self._det_bias, []
        for db, dx, ld in pending:
            self.colsum(dx, ld, db, dx.shape[0], dx.shape[1])

    def sync_streams(self, mirror=True):
        """Both streams wait for each other here. Between two connection layers the text and the vision segments are
        data-independent (vilbert.py:977-1006), so they run on two CUDA streams (and as parallel branches of the
        captured graph). mirror=True also places a barrier at the mirrored position of the backward pass."""
        if not self.two_streams:
            return
        self.cur.append((None, (), 0))
        if mirror and self.cur is self.fwd:
            self._bwd_emitters.append(None)

    class _On:
        def __init__(self, plan, sid):
            self.plan, self.sid = plan, sid

        def __enter__(self):
            self.prev = self.plan.sid
            self.plan.sid = self.sid

        def __exit__(self, *exc):
            self.plan.sid = self.prev
            return False

    def on(self, sid):
        return Plan._On(self, sid)

    def push_bwd(self, fn, rg, label):
        """Registers a block's backward emitter; it will emit on the stream that is current now. rg: whether the block's output needs
        a gradient (Act.rg); a block whose output needs none registers nothing (rule 2 of Act), so neither does a layer built
        under torch.no_grad(). The wide heads register with rg=True: their emitters decide when they run. label: the module path
        of the block (the reference's parameter-name prefix), which names its ops in an anomaly report."""
        if rg:
            self._bwd_emitters.append((self.sid, fn, label))

    def drop(self, name, p, rows=None):
        """The vb_dropout descriptor of the dropout layer `name` with probability p, or None when inactive. rows: the stream
        ("t" / "v") of a row-indexed site; a packed plan gives it the stream's packed-row -> padded-row map, so its rows draw the
        masks of the padded rows they hold."""
        if not self.train or p is None or p <= 0.0:
            return None
        d = L.Dropout()
        d.step, d.site, d.p = L.arg(self.e.drop_step), dropout_site_id(name), float(p)
        if self.packed and rows is not None:
            d.row_map = L.arg(self.map_t if rows == "t" else self.map_v)
        self._keep.append(d)
        return d

    def _check_operands(self, fwd_ops, bwd_ops):
        """The kernels are told a format flag, not typed pointers: a buffer of the other format would be read as its bits.
        So forward operands must be Operands in the engine's format and backward operands bf16 tensors (None = absent)."""
        if any(o is not None and (not isinstance(o, Operand) or o.hi.dtype != self.op_dtype) for o in fwd_ops):
            raise TypeError(f"forward tensor-core operands must be Operands in {self.op_dtype}, got {[type(o).__name__ for o in fwd_ops]}")
        if any(t is not None and (not torch.is_tensor(t) or t.dtype != BF16) for t in bwd_ops):
            raise TypeError(f"backward tensor-core operands must be bf16 tensors, got {[getattr(t, 'dtype', t) for t in bwd_ops]}")

    def gemm(self, M, N, K, A, lda, B, ldb, a_mn=0, b_mn=0, bias=None, residual=None, ld_res=0, aux=None, ld_aux=0, act=0,
             out_f32=None, ld_of=0, out_bf16=None, ld_ob=0, out_pre=None, ld_op=0, atomic=0, split_k=1, alpha=1.0, out_colsum=None,
             dropout=None):
        """Operand formats follow the pass being emitted: in the forward pass A, B and the 16-bit output (out_bf16) are
        Operands (engine format, + low parts in split precision, + the output's bf16 copy for the backward); in the backward
        pass they are bf16 tensors: A a gradient, B the bf16 copy of a weight (dgrad) or of a saved activation (wgrad),
        the 16-bit output a gradient."""
        g = L.GemmArgs()
        fwd = self.cur is not self.bwd          # the forward or the image prefix
        if fwd:
            self._check_operands((A, B, out_bf16), ())
            g.a_fp16 = g.b_fp16 = g.out_fp16 = A.fp16
            g.A_lo, g.B_lo = L.arg(A.lo), L.arg(B.lo)
            if out_bf16 is not None:
                g.out_lo, g.out_b16, out_bf16 = L.arg(out_bf16.lo), L.arg(out_bf16.extra_bw), out_bf16.hi
            A, B = A.hi, B.hi
        else:
            self._check_operands((), (A, B, out_bf16))      # the format flags stay 0 (bf16)
        g.M, g.N, g.K = M, N, K
        g.A, g.lda, g.a_mn_major = L.arg(A), lda, a_mn
        g.B, g.ldb, g.b_mn_major = L.arg(B), ldb, b_mn
        g.alpha = alpha
        g.bias = L.arg(bias)
        g.residual, g.ld_res = L.arg(residual), ld_res
        g.aux, g.ld_aux = L.arg(aux), ld_aux
        g.act = act
        g.out_f32, g.ld_out_f32 = L.arg(out_f32), ld_of
        g.out_bf16, g.ld_out_bf16 = L.arg(out_bf16), ld_ob
        g.out_pre, g.ld_out_pre = L.arg(out_pre), ld_op
        g.atomic_out, g.split_k, g.block_n, g.max_ctas = atomic, split_k, 0, (0 if fwd else self.spec.bwd_gemm_max_ctas)
        g.out_colsum = L.arg(None if self.det else out_colsum)
        if dropout is not None:
            g.dropout = dropout
        self._keep.append(g)
        if self.det and atomic:
            # split-K weight gradients: each split stores its tile into its own slice of the workspace, one ordered sum adds them
            g.atomic_out, g.split_k = L.VB_GEMM_PARTIALS, 0
            bn, sp = L.C.c_int32(), L.C.c_int32()
            L.check(self.lib.vb_gemm_plan(L.C.byref(g), 132 if self.dev.type != "cuda" else 0, L.C.byref(bn), L.C.byref(sp)),
                    "vb_gemm_plan")
            if sp.value == 1:
                g.atomic_out, g.split_k = 1, 1      # one CTA per output tile: a single add per element, in launch order
                self.emit(self.lib.vb_gemm_bf16, g)
                return
            if ld_of != N:
                raise L.VBError(f"deterministic split-K GEMM needs a dense output (ld {ld_of} != N {N})")
            ws = self.det_ws(sp.value * M * N)
            g.out_f32, g.split_k = L.arg(ws), sp.value
            self.emit(self.lib.vb_gemm_bf16, g)
            self.emit(self.lib.vb_reduce_slices, ws, M * N, sp.value, M * N, out_f32)
            return
        self.emit(self.lib.vb_gemm_bf16, g)
        if self.det and out_colsum is not None:
            # the bias gradient fused into the epilogue: an ordered column sum of the operand the GEMM stored
            self.colsum(out_bf16, ld_ob, out_colsum, M, N)

    def attention(self, bwd, B, H, Nq, Nk, D, Q, ldq, K, ldk, V, ldv, mask, O, ldo, lse, dO=None, lddo=0, dQ=None, lddq=0,
                  dK=None, lddk=0, dV=None, lddv=0, delta=None, dbq=None, dbk=None, dbv=None, dropout=None, segs=None):
        """Q, K, V and O are Operands (the forward's; the backward re-reads them), dO / dQ / dK / dV bf16 tensors. segs: the
        (offsets, lengths) of the query and of the key stream of a packed plan (mask is then None)."""
        self._check_operands((Q, K, V, O), (dO, dQ, dK, dV))
        a = L.AttnArgs()
        a.qkv_fp16 = Q.fp16
        a.O_b16 = L.arg(O.extra_bw)     # forward: written; backward: read for delta (consistent with the bf16 backward products)
        if not bwd:
            a.Q_lo, a.K_lo, a.V_lo, a.O_lo = L.arg(Q.lo), L.arg(K.lo), L.arg(V.lo), L.arg(O.lo)
        a.B, a.H, a.Nq, a.Nk, a.D = B, H, Nq, Nk, D
        a.Q, a.ldq, a.K, a.ldk, a.V, a.ldv = L.arg(Q.hi), ldq, L.arg(K.hi), ldk, L.arg(V.hi), ldv
        a.mask, a.scale = L.arg(mask), 1.0 / math.sqrt(D)
        a.O, a.ldo, a.lse = L.arg(O.hi), ldo, L.arg(lse)
        a.dO, a.lddo, a.dQ, a.lddq = L.arg(dO), lddo, L.arg(dQ), lddq
        a.dK, a.lddk, a.dV, a.lddv, a.delta = L.arg(dK), lddk, L.arg(dV), lddv, L.arg(delta)
        if self.det and bwd:     # no atomics in the kernel: det_bias_sums takes ordered column sums of dQ / dK / dV instead
            self._det_bias += [(db, dx, ld) for db, dx, ld in ((dbq, dQ, lddq), (dbk, dK, lddk), (dbv, dV, lddv)) if db is not None]
            dbq = dbk = dbv = None
        a.dbias_q, a.dbias_k, a.dbias_v = L.arg(dbq), L.arg(dbk), L.arg(dbv)
        if dropout is not None:
            a.dropout = dropout
        if segs is not None:
            (qo, ql), (ko, kl) = segs
            a.q_off, a.q_len, a.k_off, a.k_len = L.arg(qo), L.arg(ql), L.arg(ko), L.arg(kl)
        self._keep.append(a)
        self.emit(self.lib.vb_attention_bwd if bwd else self.lib.vb_attention_fwd, a)
        if not bwd and self.viz:
            # config.visualization: the probabilities (fp32 [B, heads, Nq, Nk]) and views of the queries / keys the reference returns
            probs = self.buf((B, H, Nq, Nk), F32)
            self.emit(self.lib.vb_attention_probs, a, probs)
            self._last_attn = dict(attn=probs, q=Q.hi, k=K.hi, B=B, H=H, Nq=Nq, Nk=Nk, D=D)

    def zero_tail(self, stream, *ts):
        """Packed plans: rows of no sample (past off[B] of the stream "t" / "v") of the 2-D tensors `ts` (same shape and pitch; None
        entries skipped) set to zero. The attention kernels do not write them, and every later op reads them: a GEMM's weight
        gradient multiplies them by a zero gradient, which garbage would turn into NaN."""
        ts = [t for t in ts if t is not None]
        off = self.seg[stream][0]
        self.emit(self.lib.vb_zero_tail_rows, *ts, *([None] * (3 - len(ts))), ts[0].stride(0) * ts[0].element_size(),
                  ts[0].shape[1] * ts[0].element_size(), off.data_ptr() + 4 * self.n_seg[stream], ts[0].shape[0])

    def ln_fwd(self, x, gamma, beta, M, H, want_f32=True, out_drop=None, res=None, in_drop=None):
        """-> (fp32 output or None, Operand output, mean, rstd). res: LayerNorm of dropout_in(x) + res instead (the residual add is
        fused here rather than into the GEMM that wrote x); that sum is written over x, where the backward reads it."""
        y32 = self.buf((M, H), F32) if want_f32 else None
        y = self.buf16((M, H))
        mean, rstd = self.buf((M,), F32), self.buf((M,), F32)
        hi, lo, bw = y.ptrs()
        if res is not None:
            self.emit(self.lib.vb_add_layernorm_fwd, x, res, H, in_drop, x, gamma, beta, 1e-12, y32, hi, H, mean, rstd, M, H, y.fp16, lo, bw)
        else:
            self.emit(self.lib.vb_layernorm_fwd, x, H, gamma, beta, 1e-12, y32, hi, H, mean, rstd, M, H, out_drop, y.fp16, lo, bw)
        return y32, y, mean, rstd

    def ln_bwd(self, dy, x, gamma, mean, rstd, dx32, dx16, M, H, ggamma, gbeta, pre=None, gbias=None, out_drop=None, in_drop=None, dy2=None):
        """gbias: bias gradient of the Linear feeding this LayerNorm (column sums of dx), fused into the same pass. dy2: a second
        part of the output gradient (Act.g_add), added to dy as it is read."""
        tail = (x, H, gamma, mean, rstd, dx32, dx16, H, pre, H, ggamma, gbeta, gbias, M, H, out_drop, in_drop)
        if self.det:
            sums = any(g is not None for g in (ggamma, gbeta, gbias))
            self.emit(self.lib.vb_layernorm_bwd_det, dy, dy2, H, *tail, self.det_ws(3 * L.VB_DET_LN_SLICES * H) if sums else None)
        elif dy2 is not None:
            self.emit(self.lib.vb_add_layernorm_bwd, dy, dy2, H, *tail)
        else:
            self.emit(self.lib.vb_layernorm_bwd, dy, H, *tail)

    def colsum(self, X, ld, out, M, N):
        self.emit(self.lib.vb_colsum, X, 1 if X.dtype == BF16 else 0, ld, out, M, N)

    def grad_of(self, act):
        if act.g32 is None:
            act.g32 = self.buf((act.M, act.H), F32)
        return act.g32

    def grad_zeroed(self, act):
        """The gradient buffer of `act` for a backward op that adds to it: its first writer zeroes it first (rule 3 of Act)."""
        g = self.grad_of(act)
        if not act.gw:
            self.emit(self.lib.vb_memset_zero, g, g.numel() * 4)
            act.gw = True
        self._fold_g_add(act)
        return g

    def grad_acc(self, act):
        """-> (gradient buffer of `act`, accumulate flag) for a backward op that can overwrite or add: 0, overwrite, for its first
        writer (rule 3 of Act)."""
        g, acc = self.grad_of(act), 1 if act.gw else 0
        act.gw = True
        self._fold_g_add(act)
        return g, acc

    def _fold_g_add(self, act):
        """A later writer of g32 adds to it: the first writer's deferred part goes in first, so the sums keep their order."""
        if act.g_add is not None:
            self.emit(self.lib.vb_axpy_f32, act.g_add, act.g32, act.M * act.H, 1.0)
            act.g_add = None

    # dW, db of y = x W^T + b given dy (bf16 operand copy)
    def linear_wgrad(self, dy16, ld_dy, x16, ld_x, M, N_out, K_in, wname, gw=None, bias_from=(None, 0)):
        """dW += dy^T x (split-K, atomics). Nothing on the critical chain depends on it, so with wgrad_streams it is issued on
        a side stream (2 = text chain, 3 = vision chain) right after an event marking that dy is ready; the side streams are
        joined at the data-parallel segment cuts and at the end of the backward pass. Frozen parameters (parts of a fused
        projection) get no column sum and no GEMM: each run of trainable parts gets its own on its columns of dy.
        bias_from: (dy, its row pitch) to take db as column sums of, where no kernel upstream has fused them into its pass."""
        dy_bias, ld_dyb = bias_from
        if dy_bias is not None:
            gb = self.gparts(wname + ".bias")
            nb = N_out // len(gb)
            for a, b in self._runs(gb):
                self.colsum(dy_bias[:, a * nb:b * nb], ld_dyb, gb[a], M, (b - a) * nb)
        if gw is not None:
            self._wgrad(dy16, ld_dy, x16, ld_x, M, N_out, K_in, gw)
            return
        gws = self.gparts(wname + ".weight")
        nw = N_out // len(gws)
        for a, b in self._runs(gws):
            self._wgrad(dy16[:, a * nw:b * nw], ld_dy, x16, ld_x, M, (b - a) * nw, K_in, gws[a])

    def _wgrad(self, dy16, ld_dy, x16, ld_x, M, N_out, K_in, out):
        if not self.wgrad_streams:
            self.gemm(N_out, K_in, M, dy16, ld_dy, x16, ld_x, a_mn=1, b_mn=1, out_f32=out, ld_of=K_in, atomic=1, split_k=0)
            return
        ev = self._n_events
        self._n_events += 1
        chain = self.sid
        self.cur.append((None, ("rec", ev), chain))
        self.sid = 2 + chain
        self.cur.append((None, ("wait", ev), self.sid))
        self.gemm(N_out, K_in, M, dy16, ld_dy, x16, ld_x, a_mn=1, b_mn=1, out_f32=out, ld_of=K_in, atomic=1, split_k=0)
        self.sid = chain

    # act.g32 (+)= dy16 @ W (+ extra32)
    def dgrad_into(self, act, dy16, ld_dy, W16, M, N_out, K_in, extra32=None):
        if not act.rg:      # the activation needs no gradient (frozen producer, or fixed_*_layer's no_grad): it stops here
            return
        g, acc = self.grad_acc(act)
        if not acc and extra32 is not None and act.ln_reads:
            act.g_add, extra32 = extra32, None      # added by the LayerNorm backward that reads g32: the GEMM reads no residual
        if acc and extra32 is not None:
            self.emit(self.lib.vb_axpy_f32, extra32, g, M * K_in, 1.0)
        self.gemm(M, K_in, N_out, dy16, ld_dy, W16, K_in, b_mn=1, residual=g if acc else extra32, ld_res=K_in, out_f32=g, ld_of=K_in)

    def add_grad(self, act, src32):
        if not act.rg:
            return
        g = self.grad_zeroed(act)
        self.emit(self.lib.vb_axpy_f32, src32, g, g.numel(), 1.0)

    # ------------------------------------------------------------------ blocks
    def dense_res_ln(self, a, K_in, res, wname, lnname, tag, drop=None, a_rg=True):
        """LN(dense(a) + residual)  — BertSelfOutput / BertOutput / BertBiOutput halves (vilbert.py:470-474, 513-517, 844-855).
        a_rg: whether `a` needs a gradient (the caller's backward takes the returned dy16 into it)."""
        ps, M, H = self.ps, res.M, res.H
        y = self.buf((M, H), F32)
        # the GEMM stores dense(a) only; dropout and the residual add are fused into the LayerNorm that reads it anyway
        self.gemm(M, H, K_in, a, K_in, ps.w(wname + ".weight"), K_in, bias=ps.p(wname + ".bias"), out_f32=y, ld_of=H)
        o32, o, mean, rstd = self.ln_fwd(y, ps.p(lnname + ".weight"), ps.p(lnname + ".bias"), M, H, res=res.f32, in_drop=drop)
        out = self.act(o32, o, M, H, inputs=(res,), params=(wname, lnname), rg=a_rg)
        out.ln_reads = True
        out.mod = lnname.rsplit(".", 1)[0]

        def bwd():
            """returns (dy16, dy32) of the dense output (== grad of the LN input); adds dy32 to res."""
            if not out.gw:
                return None
            dy32 = self.scratch(tag + ".dy32", (M, H), F32)
            dy16 = self.scratch(tag + ".dy16", (M, H), BF16)
            self.ln_bwd(out.g32, y, ps.p(lnname + ".weight"), mean, rstd, dy32, dy16, M, H, self.pg(lnname + ".weight"), self.pg(lnname + ".bias"),
                        gbias=self.pg(wname + ".bias"), in_drop=drop, dy2=out.g_add)
            out.g_add = None
            self.linear_wgrad(dy16, H, a.bw, K_in, M, H, K_in, wname)
            return dy16, dy32
        return out, bwd

    def ffn(self, x, I, w1, w2, lnname, tag, drop=None):
        """LN(dense2(gelu(dense1(x))) + x) — BertIntermediate + BertOutput (vilbert.py:500-503, 513-517)."""
        ps, M, H = self.ps, x.M, x.H
        pre16 = self.buf((M, I), BF16)          # gelu'(pre), bf16 in every mode (only the backward reads it)
        f = self.buf16((M, I))
        self.gemm(M, I, H, x.op, H, ps.w(w1 + ".weight"), H, bias=ps.p(w1 + ".bias"), act=L.VB_ACT_GELU, out_bf16=f, ld_ob=I,
                  out_pre=pre16, ld_op=I)
        f_rg = x.rg or self.trainable(w1)
        out, out_bwd = self.dense_res_ln(f, I, x, w2, lnname, tag + ".o", drop=drop, a_rg=f_rg)

        def bwd():
            r = out_bwd()
            if r is None or not f_rg:
                return
            dy16, dy32 = r
            dpre16 = self.scratch(tag + ".dpre16", (M, I), BF16)
            # d pre = (dy W2) * gelu'(pre)
            self.gemm(M, I, H, dy16, H, ps.w(w2 + ".weight").bw, I, b_mn=1, aux=pre16, ld_aux=I, act=L.VB_ACT_DGELU, out_bf16=dpre16, ld_ob=I,
                      out_colsum=self.pg(w1 + ".bias"))
            self.linear_wgrad(dpre16, I, x.op.bw, H, M, I, H, w1)
            self.dgrad_into(x, dpre16, I, ps.w(w1 + ".weight").bw, M, I, H, extra32=dy32)
        self.push_bwd(bwd, out.rg, out.mod)
        return out

    def self_attention_block(self, x, B, N, nh, mask, prefix, tag, p_attn=0.0, p_hidden=0.0, pool=None):
        """BertAttention (self-attention + output), text or image stream (vilbert.py:424-474, 571-633). pool: the pooled text states
        (text_pool) when config.dynamic_attention gates this image layer's queries and keys (:577-586)."""
        ps, M, H = self.ps, x.M, x.H
        D = H // nh
        qkv = self.buf16((M, 3 * H), bw=False)     # the attention backward converts its Q/K/V panels in shared memory
        self.gemm(M, 3 * H, H, x.op, H, ps.w(prefix + ".self.qkv.weight"), H, bias=ps.p(prefix + ".self.qkv.bias"), out_bf16=qkv, ld_ob=3 * H)
        if pool is not None:
            # z = dyLinear_q | dyLinear_k (pool) as one [B, 2H] GEMM; Q and K are scaled in place by 1 + sigmoid(z)
            Kp = pool.H
            z = self.buf((B, 2 * H), F32)
            self.gemm(B, 2 * H, Kp, pool.op, Kp, ps.w(prefix + ".self.dy.weight"), Kp, bias=ps.p(prefix + ".self.dy.bias"), out_f32=z, ld_of=2 * H)
            self.emit(self.lib.vb_gate_scale_fwd, qkv.hi, qkv.lo, 3 * H, z, B, N, 2 * H, qkv.fp16)
        ctx = self.buf16((M, H))
        lse = self.buf((B, nh, N), F32)
        q, k, v = qkv.cols(0, H), qkv.cols(H, 2 * H), qkv.cols(2 * H, 3 * H)
        adrop = self.drop(prefix + ".self.dropout", p_attn)
        segs = (self.seg[tag], self.seg[tag]) if self.packed else None
        self.attention(False, B, nh, N, N, D, q, 3 * H, k, 3 * H, v, 3 * H, mask, ctx, H, lse, dropout=adrop, segs=segs)
        if self.packed:
            self.zero_tail(tag, ctx.hi, ctx.lo, ctx.extra_bw)
        if self.viz:
            (self.attn_t if tag == "t" else self.attn_v).append(self._last_attn)
        qkv_rg = x.rg or self.trainable(prefix + ".self.qkv")
        gate_rg = pool is not None and (pool.rg or self.trainable(prefix + ".self.dy"))
        ctx_rg = qkv_rg or gate_rg
        out, out_bwd = self.dense_res_ln(ctx, H, x, prefix + ".output.dense", prefix + ".output.LayerNorm", tag + ".ao",
                                         drop=self.drop(prefix + ".output.dropout", p_hidden, tag), a_rg=ctx_rg)

        def bwd():
            r = out_bwd()
            if r is None or not ctx_rg:
                return
            dy16, dy32 = r
            dctx = self.scratch(tag + ".dctx", (M, H), BF16)
            self.gemm(M, H, H, dy16, H, ps.w(prefix + ".output.dense.weight").bw, H, b_mn=1, out_bf16=dctx, ld_ob=H)
            dqkv = self.scratch(tag + ".dqkv", (M, 3 * H), BF16)
            delta = self.scratch(tag + ".delta", (B, nh, N), F32)
            # bias gradients = column sums of dQ|dK|dV, fused into the attention backward
            gq, gk, gv = self.gparts(prefix + ".self.qkv.bias")
            gated = pool is not None                 # ... except under the gate, where the biases sit before the scaling
            self.attention(True, B, nh, N, N, D, q, 3 * H, k, 3 * H, v, 3 * H, mask, ctx, H, lse, dO=dctx, lddo=H,
                           dQ=dqkv[:, 0:H], lddq=3 * H, dK=dqkv[:, H:2 * H], lddk=3 * H, dV=dqkv[:, 2 * H:], lddv=3 * H, delta=delta,
                           dbq=None if gated else gq, dbk=None if gated else gk, dbv=gv, dropout=adrop, segs=segs)
            if self.packed:
                self.zero_tail(tag, dqkv)
            self.det_bias_sums()
            if gated:
                # the gate Linear needs dz32 for its bias sum, dz16 for its weight gradient and for d pool
                dyw_rg = self.trainable(prefix + ".self.dy.weight") or pool.rg
                dz32 = self.scratch(tag + ".dz32", (B, 2 * H), F32) if self.trainable(prefix + ".self.dy.bias") else None
                dz16 = self.scratch(tag + ".dz16", (B, 2 * H), BF16) if dyw_rg else None
                self.emit(self.lib.vb_gate_scale_bwd, dqkv, 3 * H, qkv.hi, qkv.lo, 3 * H, z, dz32, dz16, B, N, 2 * H, qkv.fp16)
                for (a, b) in self._runs((gq, gk)):      # the parts of one range are adjacent in the flat buffer
                    self.colsum(dqkv[:, a * H:b * H], 3 * H, (gq, gk)[a], M, (b - a) * H)
                if dz32 is not None or dz16 is not None:
                    self.linear_wgrad(dz16, 2 * H, pool.op.bw, pool.H, B, 2 * H, pool.H, prefix + ".self.dy", bias_from=(dz32, 2 * H))
                    self.dgrad_into(pool, dz16, 2 * H, ps.w(prefix + ".self.dy.weight").bw, B, 2 * H, pool.H)
            self.linear_wgrad(dqkv, 3 * H, x.op.bw, H, M, 3 * H, H, prefix + ".self.qkv")
            self.dgrad_into(x, dqkv, 3 * H, ps.w(prefix + ".self.qkv.weight").bw, M, 3 * H, H, extra32=dy32)
        self.push_bwd(bwd, out.rg, prefix)
        return out

    def connection_layer(self, v, t, idx):
        """BertConnectionLayer.forward (vilbert.py:871-900): co-attention both ways + dual FFN."""
        ps, c, B = self.ps, self.cfg, self.B
        p = f"bert.encoder.c_layer.{idx}"
        Hb, nh = c.bi_hidden_size, c.bi_num_attention_heads
        D = Hb // nh
        Mv, Mt, Hv, Ht, Nv, Nt = v.M, t.M, v.H, t.H, self.Nv, self.Nt
        qkv1 = self.buf16((Mv, 3 * Hb), bw=False)
        qkv2 = self.buf16((Mt, 3 * Hb), bw=False)
        with self.on(1):
            self.gemm(Mv, 3 * Hb, Hv, v.op, Hv, ps.w(p + ".biattention.qkv1.weight"), Hv, bias=ps.p(p + ".biattention.qkv1.bias"), out_bf16=qkv1, ld_ob=3 * Hb)
        self.gemm(Mt, 3 * Hb, Ht, t.op, Ht, ps.w(p + ".biattention.qkv2.weight"), Ht, bias=ps.p(p + ".biattention.qkv2.bias"), out_bf16=qkv2, ld_ob=3 * Hb)
        self.sync_streams()      # each direction needs the other stream's keys / values
        q1, k1, v1 = qkv1.cols(0, Hb), qkv1.cols(Hb, 2 * Hb), qkv1.cols(2 * Hb, 3 * Hb)
        q2, k2, v2 = qkv2.cols(0, Hb), qkv2.cols(Hb, 2 * Hb), qkv2.cols(2 * Hb, 3 * Hb)
        ctx1 = self.buf16((Mt, Hb)); lse1 = self.buf((B, nh, Nt), F32)   # text queries over vision keys/values
        ctx2 = self.buf16((Mv, Hb)); lse2 = self.buf((B, nh, Nv), F32)   # vision queries over text keys/values
        L3 = 3 * Hb
        # dropout1 acts on attention_probs1 (text queries over regions), dropout2 on attention_probs2 (vilbert.py:730, 738, 778, 800)
        adrop1 = self.drop(p + ".biattention.dropout1", c.v_attention_probs_dropout_prob)
        adrop2 = self.drop(p + ".biattention.dropout2", c.attention_probs_dropout_prob)
        seg_tv = (self.seg["t"], self.seg["v"]) if self.packed else None
        seg_vt = (self.seg["v"], self.seg["t"]) if self.packed else None
        self.attention(False, B, nh, Nt, Nv, D, q2, L3, k1, L3, v1, L3, self.mask_v, ctx1, Hb, lse1, dropout=adrop1, segs=seg_tv)
        if self.packed:
            self.zero_tail("t", ctx1.hi, ctx1.lo, ctx1.extra_bw)
        a1 = self._last_attn if self.viz else None
        with self.on(1):
            self.attention(False, B, nh, Nv, Nt, D, q1, L3, k2, L3, v2, L3, self.mask_t, ctx2, Hb, lse2, dropout=adrop2, segs=seg_vt)
            if self.packed:
                self.zero_tail("v", ctx2.hi, ctx2.lo, ctx2.extra_bw)
            a2 = self._last_attn if self.viz else None
        if self.viz:
            self.attn_c.append((a1, a2))
        # biOutput: ctx2 -> vision stream (dense1 / LayerNorm1), ctx1 -> text stream (dense2 / LayerNorm2) (:890-892)
        # a side whose projections are frozen and whose input needs no gradient takes no gradient: dQ of its queries' direction
        # and dK / dV of the other are not computed
        need1 = v.rg or self.trainable(p + ".biattention.qkv1")
        need2 = t.rg or self.trainable(p + ".biattention.qkv2")
        ctx_rg = need1 or need2
        with self.on(1):
            v1o, v1_bwd = self.dense_res_ln(ctx2, Hb, v, p + ".biOutput.dense1", p + ".biOutput.LayerNorm1", "c.v.bo",
                                            drop=self.drop(p + ".biOutput.dropout1", c.v_hidden_dropout_prob, "v"), a_rg=ctx_rg)
        t1o, t1_bwd = self.dense_res_ln(ctx1, Hb, t, p + ".biOutput.dense2", p + ".biOutput.LayerNorm2", "c.t.bo",
                                        drop=self.drop(p + ".biOutput.dropout2", c.hidden_dropout_prob, "t"), a_rg=ctx_rg)

        def bwd():
            if not (v1o.gw or t1o.gw):
                return
            for a in (v1o, t1o):   # a stream without downstream gradient contributes zeros
                if a.rg and not a.gw:
                    self.grad_zeroed(a)
            rv, rt = v1_bwd(), t1_bwd()
            if not ctx_rg:
                return
            dqkv1 = self.scratch("c.dqkv1", (Mv, L3), BF16)
            dqkv2 = self.scratch("c.dqkv2", (Mt, L3), BF16)
            dctx2 = self.scratch("c.dctx2", (Mv, Hb), BF16)
            dctx1 = self.scratch("c.dctx1", (Mt, Hb), BF16)
            dyv16, dyv32 = rv
            dyt16, dyt32 = rt
            self.gemm(Mv, Hb, Hv, dyv16, Hv, ps.w(p + ".biOutput.dense1.weight").bw, Hb, b_mn=1, out_bf16=dctx2, ld_ob=Hb)
            self.gemm(Mt, Hb, Ht, dyt16, Ht, ps.w(p + ".biOutput.dense2.weight").bw, Hb, b_mn=1, out_bf16=dctx1, ld_ob=Hb)
            gq1, gk1, gv1 = self.gparts(p + ".biattention.qkv1.bias") if need1 else (None,) * 3
            gq2, gk2, gv2 = self.gparts(p + ".biattention.qkv2.bias") if need2 else (None,) * 3
            d1 = self.scratch("c.delta1", (B, nh, Nt), F32)
            d2 = self.scratch("c.delta2", (B, nh, Nv), F32)
            part1 = (lambda a, b: dqkv1[:, a:b]) if need1 else (lambda a, b: None)
            part2 = (lambda a, b: dqkv2[:, a:b]) if need2 else (lambda a, b: None)
            self.attention(True, B, nh, Nt, Nv, D, q2, L3, k1, L3, v1, L3, self.mask_v, ctx1, Hb, lse1, dO=dctx1, lddo=Hb,
                           dQ=part2(0, Hb), lddq=L3, dK=part1(Hb, 2 * Hb), lddk=L3, dV=part1(2 * Hb, L3), lddv=L3, delta=d1,
                           dbq=gq2, dbk=gk1, dbv=gv1, dropout=adrop1, segs=seg_tv)
            self.attention(True, B, nh, Nv, Nt, D, q1, L3, k2, L3, v2, L3, self.mask_t, ctx2, Hb, lse2, dO=dctx2, lddo=Hb,
                           dQ=part1(0, Hb), lddq=L3, dK=part2(Hb, 2 * Hb), lddk=L3, dV=part2(2 * Hb, L3), lddv=L3, delta=d2,
                           dbq=gq1, dbk=gk2, dbv=gv2, dropout=adrop2, segs=seg_vt)
            if self.packed:
                for stream, need, d in (("v", need1, dqkv1), ("t", need2, dqkv2)):
                    if need:
                        self.zero_tail(stream, d)
            self.det_bias_sums()
            if need1:
                self.linear_wgrad(dqkv1, L3, v.op.bw, Hv, Mv, L3, Hv, p + ".biattention.qkv1")
            if need2:
                self.linear_wgrad(dqkv2, L3, t.op.bw, Ht, Mt, L3, Ht, p + ".biattention.qkv2")
            self.dgrad_into(v, dqkv1, L3, ps.w(p + ".biattention.qkv1.weight").bw, Mv, L3, Hv, extra32=dyv32)
            self.dgrad_into(t, dqkv2, L3, ps.w(p + ".biattention.qkv2.weight").bw, Mt, L3, Ht, extra32=dyt32)
        # the cross-modal backward touches both streams' tensors: it runs on the main stream between two barriers
        self._bwd_emitters.append(None)
        self.push_bwd(bwd, v1o.rg or t1o.rg, p + ".biOutput")
        self._bwd_emitters.append(None)
        with self.on(1):
            v2o = self.ffn(v1o, c.v_intermediate_size, p + ".v_intermediate.dense", p + ".v_output.dense", p + ".v_output.LayerNorm", "c.v.ffn",
                           drop=self.drop(p + ".v_output.dropout", c.v_hidden_dropout_prob, "v"))
        t2o = self.ffn(t1o, c.intermediate_size, p + ".t_intermediate.dense", p + ".t_output.dense", p + ".t_output.LayerNorm", "c.t.ffn",
                       drop=self.drop(p + ".t_output.dropout", c.hidden_dropout_prob, "t"))
        return v2o, t2o

    def broadcast_text(self, t):
        """FAST_MODE: t [1*Nt, H] -> [B*Nt, H] (fp32 values and operand copies), and the text mask [1, Nt] -> [B, Nt]. Packed
        (retrieval): the caption's L valid rows -> B contiguous segments (b*L, L) of the rows_t rows, zeros after B*L, with the B
        segments written from the broadcast mask; L is read on the device."""
        B, M1, H = self.B, t.M, t.H
        if self.packed:
            rows, it = self.packed[0], torch.int32
            seg = (self.buf((B + 1,), it), self.buf((B,), it))
            self.map_t = self.buf((rows,), it)
            self.emit(self.lib.vb_pack_segments, self.in_amask_b, self.Nt_in, 1 if self.has_task else 0, B, rows, *seg, self.map_t)
            f32 = self.buf((rows, H), F32)
            op = self.buf16((rows, H), bw=False)
            for src, dst in ((t.f32, f32), (t.op.hi, op.hi), (t.op.lo, op.lo)):
                if dst is not None:
                    self.emit(self.lib.vb_broadcast_segment_rows, src, dst, H * dst.element_size(), self.seg["t"][1], B, rows)
            self.seg["t"], self.n_seg["t"] = seg, B
            return self.act(f32, op, rows, H, inputs=(t,))
        f32 = self.buf((B * M1, H), F32)
        op = self.buf16((B * M1, H), bw=False)      # FAST_MODE is inference only: no backward copy
        for src, dst in ((t.f32, f32), (t.op.hi, op.hi), (t.op.lo, op.lo)):
            if dst is not None:
                self.emit(self.lib.vb_broadcast_rows, src, dst, M1 * H * dst.element_size(), B)
        nt4 = (self.Nt * 4 + 15) // 16 * 16           # the mask row is padded to 16 bytes for the broadcast kernel
        if nt4 == self.Nt * 4:
            m = self.buf((B, self.Nt), F32)
            self.emit(self.lib.vb_broadcast_rows, self.mask_t, m, self.Nt * 4, B)
        else:
            m = self.mask_t.new_empty((B, self.Nt)); self._keep.append(m)
            self.emit(self.lib.vb_mask_to_additive, self.in_amask_b, m, B, self.Nt_in, 1 if self.has_task else 0)
        self.mask_t = m
        return self.act(f32, op, B * M1, H, inputs=(t,))

    def expand_pairs(self, t, v):
        """in_batch_pairs (vilbert.py:1008-1040): sample p = i * b + j of the expanded batch pairs text i with image j —
        txt.unsqueeze(1).expand(b, b, ...) (every text repeated b times) and img.unsqueeze(0).expand(b, b, ...) (the image batch
        tiled b times). Backward: the gradient of an item is the sum over its b copies (vb_sum_strided)."""
        b, lib = self.Bin, self.lib
        outs = []
        self.sync_streams()      # the image stream's tensors are expanded on the main stream
        for act, N, is_text in ((t, self.Nt, True), (v, self.Nv, False)):
            n = N * act.H
            f32 = self.buf((b * b * N, act.H), F32)
            op = self.buf16((b * b * N, act.H))
            for src, dst in zip((act.f32, act.op.hi, act.op.lo, act.op.extra_bw), (f32, op.hi, op.lo, op.extra_bw)):
                if dst is None:
                    continue
                if is_text:
                    self.emit(lib.vb_repeat_rows, src, dst, n * dst.element_size(), b, b)
                else:
                    self.emit(lib.vb_broadcast_rows, src, dst, b * n * dst.element_size(), b)
            out = self.act(f32, op, b * b * N, act.H, inputs=(act,))
            outs.append(out)

            def bwd(act=act, out=out, n=n, is_text=is_text):
                if not out.gw:
                    return
                g, acc = self.grad_acc(act)
                if is_text:   # g[i] = sum_j out.g32[i * b + j]
                    self.emit(lib.vb_sum_strided, out.g32, g, n, b, b * n, b, n, acc)
                else:         # g[j] = sum_i out.g32[i * b + j]
                    self.emit(lib.vb_sum_strided, out.g32, g, n, b, n, b, b * n, acc)
            self._bwd_emitters.append(None)
            self.push_bwd(bwd, out.rg, "bert.encoder")
            self._bwd_emitters.append(None)
        # masks: text mask rows repeated, image mask tiled (4-byte rows: plain torch-free kernels need 16-byte items -> host-side views)
        mt = self.buf((b * b, self.Nt), F32); mv = self.buf((b * b, self.Nv), F32)
        self.emit(lib.vb_mask_to_additive, self.in_amask_pairs, mt, b * b, self.Nt_in, 1 if self.has_task else 0)
        self.emit(lib.vb_mask_to_additive, self.in_imask_pairs, mv, b * b, self.Nv, 0)
        self.mask_t, self.mask_v = mt, mv
        self.sync_streams()
        return outs[0], outs[1]

    def text_layer(self, x, i):
        p = f"bert.encoder.layer.{i}"
        c = self.cfg
        h1 = self.self_attention_block(x, self.n_seg["t"] if self.packed else x.M // self.Nt, self.Nt, c.num_attention_heads, self.mask_t, p + ".attention", "t",
                                       p_attn=c.attention_probs_dropout_prob, p_hidden=c.hidden_dropout_prob)
        return self.ffn(h1, c.intermediate_size, p + ".intermediate.dense", p + ".output.dense", p + ".output.LayerNorm", "t.ffn",
                        drop=self.drop(p + ".output.dropout", c.hidden_dropout_prob, "t"))

    def text_pool(self, t):
        """dynamic_attention: masked mean of the text states over the tokens (vilbert.py:578-579) as an Act [B, Ht] with GEMM operand
        copies; its backward adds d pool to the gradient of the text states. Emitted on the text stream; the caller places a
        barrier before the image layers that read it (their backward accumulates d pool, mirrored barrier, then this backward)."""
        B, Ht, lib = self.B, t.H, self.lib
        p32 = self.buf((B, Ht), F32)
        p = self.buf16((B, Ht))
        self.emit(lib.vb_masked_mean_fwd, t.f32, self.mask_t, p32, *p.ptrs(), p.fp16, B, self.Nt, Ht)
        pool = self.act(p32, p, B, Ht, inputs=(t,))
        mask = self.mask_t

        def bwd():
            if not pool.gw:
                return
            g, acc = self.grad_acc(t)
            self.emit(lib.vb_masked_mean_bwd, pool.g32, mask, g, acc, B, self.Nt, Ht)
        self.push_bwd(bwd, pool.rg, "bert.encoder")
        return pool

    def image_layer(self, x, i, pool=None):
        p = f"bert.encoder.v_layer.{i}"
        c = self.cfg
        h1 = self.self_attention_block(x, self.B if self.packed else x.M // self.Nv, self.Nv, c.v_num_attention_heads, self.mask_v, p + ".attention", "v",
                                       p_attn=c.v_attention_probs_dropout_prob, p_hidden=c.v_hidden_dropout_prob, pool=pool)
        return self.ffn(h1, c.v_intermediate_size, p + ".intermediate.dense", p + ".output.dense", p + ".output.LayerNorm", "v.ffn",
                        drop=self.drop(p + ".output.dropout", c.v_hidden_dropout_prob, "v"))

    # ------------------------------------------------------------------ embeddings
    def embeddings(self):
        ps, c, B, lib = self.ps, self.cfg, self.Bin, self.lib     # the embeddings run at the INPUT batch
        Ht, Hv, Nt, Nv, Fv = c.hidden_size, c.v_hidden_size, self.Nt, self.Nv, c.v_feature_size
        Bt = self.Bt
        Mt, Mv = Bt * Nt, B * Nv
        # static inputs (the text side has batch 1 in FAST_MODE)
        self.in_ids = self.buf((Bt, self.Nt_in), I64, zero=True)
        self.in_tt = self.buf((Bt, self.Nt_in), I64, zero=True)
        self.in_task = self.buf((Bt,), I64, zero=True) if self.has_task else None
        self.in_amask = self.buf((Bt, self.Nt_in), I64, zero=True)
        self.in_amask_b = self.in_amask.expand(B, self.Nt_in).contiguous() if self.fast else self.in_amask   # refreshed in load_inputs
        if self.pairs:   # 0/1 masks of the expanded batch (text rows repeated, image rows tiled); refreshed in load_inputs
            self.in_amask_pairs = self.buf((B * B, self.Nt_in), I64, zero=True)
            self.in_imask_pairs = self.buf((B * B, Nv), I64, zero=True)
        self.in_imask = self.buf((B, Nv), I64, zero=True)
        self.in_feat = self.buf((B, Nv, Fv), F32, zero=True)
        self.in_loc = self.buf((B, Nv, 5), F32, zero=True)
        self.seg = {}
        if self.packed:
            # the rows of each stream and their padded rows, from the loaded masks (one kernel; the lengths exclude every masked key,
            # so no additive mask exists)
            (Mt, Mv), self.mask_t, self.mask_v = self.packed, None, None
            it = torch.int32
            self.n_seg = {"t": Bt, "v": B}       # samples of each stream (the text has one until broadcast_text)
            if self.fast:
                # retrieval: the caption is one segment of the Nt rows until broadcast_text; the image segments are written by the
                # prefix into private buffers, so they outlive every caption forward like the image states
                Mt = Nt
                self.seg["t"], self.map_t = (self.buf((2,), it), self.buf((1,), it)), self.buf((Mt,), it)
                self.emit(lib.vb_pack_segments, self.in_amask, self.Nt_in, 1 if self.has_task else 0, 1, Mt, *self.seg["t"], self.map_t)
                self.seg["v"], self.map_v = (self.buf((B + 1,), it, zero=True), self.buf((B,), it, zero=True)), self.buf((Mv,), it, zero=True)
                self.cur = self.prefix
                self.emit(lib.vb_pack_segments, self.in_imask, Nv, 0, B, Mv, *self.seg["v"], self.map_v)
                self.cur = self.fwd
            else:
                self.seg = {"t": (self.buf((B + 1,), it), self.buf((B,), it)), "v": (self.buf((B + 1,), it), self.buf((B,), it))}
                self.map_t, self.map_v = self.buf((Mt,), it), self.buf((Mv,), it)
                self.emit(lib.vb_pack_build, self.in_amask, self.Nt_in, 1 if self.has_task else 0, self.in_imask, Nv, B, Mt, Mv,
                          self.seg["t"][0], self.seg["t"][1], self.map_t, self.seg["v"][0], self.seg["v"][1], self.map_v)
        else:
            self.mask_t = self.buf((Bt, Nt), F32)
            self.mask_v = self.buf((B, Nv), F32, zero=self.image_prefix)
            self.emit(lib.vb_mask_to_additive, self.in_amask, self.mask_t, Bt, self.Nt_in, 1 if self.has_task else 0)
            if self.image_prefix:
                self.cur = self.prefix
            self.emit(lib.vb_mask_to_additive, self.in_imask, self.mask_v, B, Nv, 0)
            self.cur = self.fwd
        self.sync_streams()
        # text: gather-sum (+ task row) then LayerNorm (vilbert.py:346-367). Packed: the sums of the padded rows (cheap), their valid
        # rows gathered, and the LayerNorm on those
        xe = xe_pad = self.buf((Bt * Nt, Ht), F32)
        e = "bert.embeddings"
        self.emit(lib.vb_embed_text_fwd, self.in_ids, self.in_tt, self.in_task, ps.p(e + ".word_embeddings.weight"),
                  ps.p(e + ".position_embeddings.weight"), ps.p(e + ".token_type_embeddings.weight"),
                  ps.p(e + ".task_embeddings.weight") if self.has_task else None, xe, Bt, self.Nt_in, Ht)
        if self.packed:
            xe = self.buf((Mt, Ht), F32)
            self.emit(lib.vb_pack_rows_f32, xe_pad, xe, self.map_t, Mt, Ht)
        tdrop = self.drop(e + ".dropout", c.hidden_dropout_prob, "t")
        t32, top, tmean, trstd = self.ln_fwd(xe, ps.p(e + ".LayerNorm.weight"), ps.p(e + ".LayerNorm.bias"), Mt, Ht, out_drop=tdrop)
        tables = [e + n for n in (".word_embeddings.weight", ".position_embeddings.weight", ".token_type_embeddings.weight")]
        tables.append(e + ".task_embeddings.weight" if self.has_task else None)
        t = self.act(t32, top, Mt, Ht, params=(e + ".LayerNorm", *[n for n in tables if n is not None]))

        def bwd_text():
            if t.gw:
                dxe = self.scratch("emb.dxe", (Mt, Ht), F32)
                self.ln_bwd(t.g32, xe, ps.p(e + ".LayerNorm.weight"), tmean, trstd, dxe, None, Mt, Ht, self.pg(e + ".LayerNorm.weight"),
                            self.pg(e + ".LayerNorm.bias"), out_drop=tdrop)
                if self.packed:     # back to the padded rows the embedding sums were gathered from (zeros on the masked ones)
                    dxe_pad = self.scratch("emb.dxe_pad", (B * Nt, Ht), F32)
                    self.emit(lib.vb_unpack_rows_f32, dxe, dxe_pad, self.seg["t"][0], self.seg["t"][1], B, Nt, Ht, 0.0)
                    dxe = dxe_pad
                gt = [None if n is None else self.pg(n) for n in tables]
                if any(g is not None for g in gt):
                    self.emit(lib.vb_embed_text_bwd, dxe, self.in_ids, self.in_tt, self.in_task, *gt, B, self.Nt_in, Ht)
        self.push_bwd(bwd_text, t.rg, e)
        # image: region features fp32 -> bf16 ingest, 2048 -> Hv GEMM with the 5 -> Hv box projection as residual, LayerNorm (:1421-1432).
        # image_prefix: the same launches go to self.prefix on the main stream, and the LayerNorm's outputs (the image states the
        # forward reads) are private buffers
        ve = "bert.v_embeddings"
        if self.image_prefix:
            self.cur = self.prefix
        with self.on(0 if self.image_prefix else 1):
            yv, feat = self.image_embedding(ve, Hv)
            vdrop = self.drop(ve + ".dropout", c.hidden_dropout_prob, "v")     # BertImageEmbeddings uses hidden_dropout_prob (vilbert.py:1419)
            self._private = self.image_prefix
            v32, vop, vmean, vrstd = self.ln_fwd(yv, ps.p(ve + ".LayerNorm.weight"), ps.p(ve + ".LayerNorm.bias"), Mv, Hv, out_drop=vdrop)
            self._private = False
            self.cur = self.fwd
            v = self.act(v32, vop, Mv, Hv, params=(ve + ".image_embeddings", ve + ".image_location_embeddings", ve + ".LayerNorm"),
                         rg=self.input_grads)
            if self.image_prefix:
                self.image_states = (v32, vop.hi, vop.lo, self.mask_v) + ((*self.seg["v"], self.map_v) if self.packed else ())

            def bwd_image():
                if v.gw:
                    dyv32 = self.scratch("emb.dyv32", (Mv, Hv), F32)
                    dyv16 = self.scratch("emb.dyv16", (Mv, Hv), BF16)
                    self.ln_bwd(v.g32, yv, ps.p(ve + ".LayerNorm.weight"), vmean, vrstd, dyv32, dyv16, Mv, Hv, self.pg(ve + ".LayerNorm.weight"),
                                self.pg(ve + ".LayerNorm.bias"), gbias=self.pg(ve + ".image_embeddings.bias"), out_drop=vdrop)
                    self.image_embedding_bwd(ve, Hv, feat, dyv16, dyv32)
            self.push_bwd(bwd_image, v.rg, ve)
        return t, v

    def image_embedding(self, prefix, H):
        """The image embedding up to its LayerNorm (vilbert.py:1421-1432, basebert.py:324-359) on the loaded regions: feature cast to
        an operand, the 5 -> H box projection, and the region-feature GEMM with the box term as its residual. -> (fp32 output
        [regions, H], the feature Operand)."""
        ps, lib = self.ps, self.lib
        B, Nv, Fv = self.in_feat.shape
        M = self.packed[1] if self.packed else B * Nv
        feat = self.buf16((M, Fv))
        hi, lo, bw = feat.ptrs()
        self.loc_rows = self.in_loc
        if self.packed:     # the valid regions' features cast straight into packed operand rows, and their boxes
            self.emit(lib.vb_pack_regions, self.in_feat, self.map_v, M, Fv, feat.fp16, hi, lo, bw)
            self.loc_rows = self.buf((M, 5), F32)
            self.emit(lib.vb_pack_rows_f32, self.in_loc, self.loc_rows, self.map_v, M, 5)
        else:
            self.emit(lib.vb_cast_f32_to_bf16, self.in_feat, hi, M * Fv, feat.fp16, lo, bw)
        locp = self.buf((M, H), F32)
        self.emit(lib.vb_loc_proj_fwd, self.loc_rows, ps.p(prefix + ".image_location_embeddings.weight"),
                  ps.p(prefix + ".image_location_embeddings.bias"), locp, M, H)
        y = self.buf((M, H), F32)
        self.gemm(M, H, Fv, feat, Fv, ps.w(prefix + ".image_embeddings.weight"), Fv, bias=ps.p(prefix + ".image_embeddings.bias"),
                  residual=locp, ld_res=H, out_f32=y, ld_of=H)
        return y, feat

    def image_embedding_bwd(self, prefix, H, feat, dy16, dy32):
        """Gradients of image_embedding from d(output): the region-feature GEMM's weight from its bf16 copy dy16, the box
        projection from the fp32 dy32 (either None: no gradient wanted), then the input gradients of input_grads: the features
        by the dgrad GEMM dy16 W, the boxes by vb_loc_proj_dx on dy32."""
        ps = self.ps
        M, Fv = feat.hi.shape
        if dy16 is not None:
            self.linear_wgrad(dy16, H, feat.bw, Fv, M, H, Fv, prefix + ".image_embeddings")
        if dy32 is not None:
            gw, gb = self.pg(prefix + ".image_location_embeddings.weight"), self.pg(prefix + ".image_location_embeddings.bias")
            if gw is not None or gb is not None:
                self.emit(self.lib.vb_loc_proj_bwd, dy32, self.loc_rows, gw, gb, M, H)
        if dy16 is not None and "input_imgs" in self.input_grads:
            g = self.input_grad["input_imgs"] = self.buf((M, Fv), F32, zero=True)
            self.gemm(M, Fv, H, dy16, H, ps.w(prefix + ".image_embeddings.weight").bw, Fv, b_mn=1, out_f32=g, ld_of=Fv)
        if dy32 is not None and "image_loc" in self.input_grads:
            g = self.input_grad["image_loc"] = self.buf((M, 5), F32, zero=True)
            self.emit(self.lib.vb_loc_proj_dx, dy32, ps.p(prefix + ".image_location_embeddings.weight"), g, M, H)

    # ------------------------------------------------------------------ poolers and heads
    def pooler(self, seq, N, wname):
        """Linear + ReLU on token 0 (vilbert.py:1116-1122, 1131-1137); A is read with row pitch N*H."""
        ps, B, H, Hb = self.ps, self.B, seq.H, self.cfg.bi_hidden_size
        p32 = self.buf((B, Hb), F32)
        p = self.buf16((B, Hb), bw=False)
        x, ldx = seq.op, N * H
        if self.packed:      # each sample's first row, through the stream's offsets
            first = self.seg["t" if wname == "bert.t_pooler.dense" else "v"][0][:B]
            x, ldx = self.gather_rows(seq.op, first, B, H), H
        self.gemm(B, Hb, H, x, ldx, ps.w(wname + ".weight"), H, bias=ps.p(wname + ".bias"), act=L.VB_ACT_RELU, out_f32=p32, ld_of=Hb,
                  out_bf16=p, ld_ob=Hb)
        pooled = self.act(p32, p, B, Hb, inputs=(seq,), params=(wname,))
        pooled.mod = wname.rsplit(".", 1)[0]

        def bwd():
            if not pooled.gw:
                return
            dpre = self.scratch("pool.dpre", (B, Hb), BF16)
            dpre32 = self.scratch("pool.dpre32", (B, Hb), F32)
            self.emit(self.lib.vb_relu_bwd, pooled.g32, p32, dpre, dpre32, B * Hb)
            self.linear_wgrad(dpre, Hb, x.bw, ldx, B, Hb, H, wname, bias_from=(dpre32, Hb))
            self.pooler_dgrad(seq, N, dpre, wname, first if self.packed else None)
        self.push_bwd(bwd, pooled.rg, pooled.mod)
        return pooled

    def pooler_dgrad(self, seq, N, dpre, wname, rows=None):
        """Backward of a pooler's Linear into its input: rows b*N (token 0 of every sample; packed: the rows `rows`) of the sequence
        gradient += dpre @ W, with the sequence gradient zeroed on its first write."""
        if not seq.rg:
            return
        g = self.grad_zeroed(seq)
        B, K = dpre.shape
        if rows is not None:
            d = self.scratch("pool.dx", (B, seq.H), F32)
            self.gemm(B, seq.H, K, dpre, K, self.ps.w(wname + ".weight").bw, seq.H, b_mn=1, out_f32=d, ld_of=seq.H)
            self.emit(self.lib.vb_scatter_add_rows_f32, d, g, rows, B, seq.H)
            return
        self.gemm(B, seq.H, K, dpre, K, self.ps.w(wname + ".weight").bw, seq.H, b_mn=1, residual=g, ld_res=N * seq.H, out_f32=g,
                  ld_of=N * seq.H)

    def out_grad_buffer(self, name, shape):
        """Static fp32 buffer the caller's d(loss)/d(output) is copied into before backward."""
        if name not in self.gout:
            self.gout[name] = self.buf(shape, F32, zero=True)
        return self.gout[name]

    def big_head(self, name, x, ld_x, M, K_in, N_out, wname, bias_name, w=None, gw_name=None, dl32=None):
        """Wide linear head (N_out in the thousands): logits = x W^T + b as fp32 [M, N_out]; backward from a
        caller-supplied fp32 d(logits), cast to a bf16 operand with an 8-padded row pitch unless the objective registered one it
        writes itself (self.head_dl16). w / gw_name: a weight and the entry of
        its gradient not named by `wname` (the decoder tied to the word embeddings). dl32: the buffer the backward reads d(logits)
        from when it is not the output-gradient buffer of `name` (a packed head, whose output is the padded layout). The backward
        returns None when nothing below the logits takes a gradient."""
        ps = self.ps
        W = w if w is not None else ps.w(wname + ".weight")
        wkey = gw_name if gw_name is not None else wname + ".weight"
        logits = self.buf((M, N_out), F32)
        self.gemm(M, N_out, K_in, x.op, ld_x, W, K_in, bias=ps.p(bias_name), out_f32=logits, ld_of=N_out)
        self.outputs[name] = logits
        self.out_rg[name] = x.rg or self.trainable(wkey, bias_name)

        def bwd():
            if name not in self.grad_outputs or not self.out_rg[name]:
                return None
            ldp = _pad8(N_out)
            dl, dl16 = self.out_grad_buffer(name, (M, N_out)) if dl32 is None else dl32, self.head_dl16.get(name)
            if dl16 is None:
                dl16 = self.scratch("head.dl16." + name, (M, ldp), BF16)
                self.emit(self.lib.vb_cast2d_f32_to_bf16, dl, N_out, dl16, ldp, M, N_out, 1.0)
            gb = self.pg(bias_name)
            if gb is not None:
                self.colsum(dl, N_out, gb, M, N_out)
            if gw_name is None:
                self.linear_wgrad(dl16, ldp, x.op.bw, ld_x, M, N_out, K_in, wname)
            elif self.trainable(gw_name):
                self.linear_wgrad(dl16, ldp, x.op.bw, ld_x, M, N_out, K_in, None, gw=self.grad_view(gw_name))
            return (dl16, ldp, W.bw) if x.rg else None
        return bwd

    def _wide_bwd(self, head_bwd, hn, tr_bwd, K, N_out):
        """Backward of a transform + wide decoder head: d(transform output) = d(logits) W, then the transform's backward."""
        def f():
            r = head_bwd()
            if r is None:
                return
            dl16, ldp, W16 = r
            g, _ = self.grad_acc(hn)      # the head is the transform's only reader: always the first write
            self.gemm(hn.M, K, N_out, dl16, ldp, W16, K, b_mn=1, out_f32=g, ld_of=K)
            tr_bwd()
        return f

    def lm_head_compact(self, ht, ht_bwd):
        """Masked-LM head of the fused pre-training objective without the [tokens, vocab] logits: the rows with a label
        (masked_lm_labels != -1, 15 % of the tokens; vilbert.py:1578-1583) are compacted on the device into a fixed-capacity
        operand (engine.lm_capacity of the rows), the tied decoder GEMM, the cross-entropy and both backward GEMMs run on those
        rows, and the gradient is scattered back to the token rows. More labelled rows than the capacity poison the loss (NaN).
        Packed: the labels stay in the padded layout, the labelled packed rows are found through the text row map (in the order of
        their padded rows), and the capacity is that of the padded rows, so both plans poison the loss under the same condition."""
        ps, c, lib = self.ps, self.cfg, self.lib
        M, Ht, V = ht.M, ht.H, c.vocab_size
        M_pad = self.B * self.Nt if self.packed else M
        cap = min(_pad8(M_pad), _pad8(max(64, int(math.ceil(self.e.lm_capacity * M_pad)))))
        labels = self.buf((M_pad,), I64, zero=True)      # a plan input (loaded from outside a run): private, never in the shared arena
        labels.fill_(-1)
        self.loss_inputs["masked_lm_labels"] = labels
        idx, cnt, lab_c = self.buf((cap,), torch.int32), self.buf((1,), torch.int32, zero=True), self.buf((cap,), I64)
        if self.packed:
            self.emit(lib.vb_compact_rows_mapped, labels, -1, self.map_t, M, cap, idx, cnt, lab_c)
        else:
            self.emit(lib.vb_compact_rows, labels, -1, M, cap, idx, cnt, lab_c)
        hc = self.gather_rows(ht.op, idx, cap, Ht)
        wn = "bert.embeddings.word_embeddings.weight"
        logits = self.buf((cap, V), F32)
        self.gemm(cap, V, Ht, hc, Ht, ps.w(wn), Ht, bias=ps.p("cls.predictions.bias"), out_f32=logits, ld_of=V)
        ldp = _pad8(V)
        self.lm_c = dict(cap=cap, idx=idx, count=cnt, labels=lab_c, logits=logits, dl32=self.buf((cap, V), F32),
                         dl16=self.buf((cap, ldp), BF16, zero=True), ldp=ldp)
        self.out_rg["linguisic_prediction"] = ht.rg or self.trainable(wn, "cls.predictions.bias")

        def bwd():
            if "linguisic_prediction" not in self.grad_outputs:     # a forward-only plan of the forward-placed objective
                return
            lc = self.lm_c
            gb = self.pg("cls.predictions.bias")
            if gb is not None:
                self.colsum(lc["dl32"], V, gb, cap, V)
            if self.trainable(wn):
                self.linear_wgrad(lc["dl16"], ldp, hc.bw, Ht, cap, V, Ht, None, gw=self.grad_view(wn))
            if not ht.rg:
                return
            gc = self.scratch("lm.gc", (cap, Ht), F32)
            self.gemm(cap, Ht, V, lc["dl16"], ldp, ps.w(wn).bw, Ht, b_mn=1, out_f32=gc, ld_of=Ht)
            g = self.grad_zeroed(ht)
            self.emit(lib.vb_scatter_rows_f32, gc, g, idx, cap, Ht, cnt, self.loss_slots[0])
            ht_bwd()
        return bwd

    def gather_rows(self, src, idx, rows, H):
        """The rows `idx` (int32 [rows]) of the Operand `src` as a compact Operand: hi with its bf16 copy, and lo."""
        op = self.buf16((rows, H))
        self.emit(self.lib.vb_gather_rows16, src.hi, op.hi, src.extra_bw, op.extra_bw, idx, rows, H)
        if op.lo is not None:
            self.emit(self.lib.vb_gather_rows16, src.lo, op.lo, None, None, idx, rows, H)
        return op

    def lm_rows(self):
        """(labelled rows of the last step, capacity) of the compacted masked-LM head (device sync)."""
        return int(self.lm_c["count"].item()), self.lm_c["cap"]

    def transform(self, x, wdense, lnname, tag):
        """Linear -> GELU -> LayerNorm (BertPredictionHeadTransform / BertImgPredictionHeadTransform / the first three
        stages of SimpleClassifier; vilbert.py:1152-1156, 1172-1176, 1714-1718)."""
        ps = self.ps
        M, K = x.M, x.H
        Hh = ps.p(wdense + ".weight").shape[0]
        g32, pre16 = self.buf((M, Hh), F32), self.buf((M, Hh), BF16)
        self.gemm(M, Hh, K, x.op, K, ps.w(wdense + ".weight"), K, bias=ps.p(wdense + ".bias"), act=L.VB_ACT_GELU, out_f32=g32, ld_of=Hh,
                  out_pre=pre16, ld_op=Hh)
        _, h, mean, rstd = self.ln_fwd(g32, ps.p(lnname + ".weight"), ps.p(lnname + ".bias"), M, Hh, want_f32=False)
        hn = self.act(None, h, M, Hh, inputs=(x,), params=(wdense, lnname))

        def bwd():
            if not hn.gw:
                return
            dpre16 = self.scratch(tag + ".dpre16", (M, Hh), BF16)
            self.ln_bwd(hn.g32, g32, ps.p(lnname + ".weight"), mean, rstd, None, dpre16, M, Hh, self.pg(lnname + ".weight"), self.pg(lnname + ".bias"),
                        pre=pre16, gbias=self.pg(wdense + ".bias"))
            self.linear_wgrad(dpre16, Hh, x.op.bw, K, M, Hh, K, wdense)
            self.dgrad_into(x, dpre16, Hh, ps.w(wdense + ".weight").bw, M, Hh, K)
        return hn, bwd

    def small_head(self, name, x, wname, N_out, addend=None, x32=None, M=None, K=None, in_drop=None):
        ps = self.ps
        M = x.M if M is None else M
        K = x.H if K is None else K
        xin = x.f32 if x32 is None else x32
        y = self.buf((M, N_out), F32)
        self.emit(self.lib.vb_small_linear_fwd, xin, K, ps.p(wname + ".weight"), ps.p(wname + ".bias"), addend, y, M, K, N_out, in_drop)
        self.outputs[name] = y
        self.out_rg[name] = x.rg or self.trainable(wname)

        def bwd():
            if name not in self.grad_outputs:
                return
            dy = self.out_grad_buffer(name, (M, N_out))
            g, acc = self.grad_acc(x) if x.rg else (None, 0)
            self.emit(self.lib.vb_small_linear_bwd, dy, xin, K, ps.p(wname + ".weight"), g, K, acc,
                      self.pg(wname + ".weight"), self.pg(wname + ".bias"), M, K, N_out, in_drop)
        self.push_bwd(bwd, self.out_rg[name], wname)

    def packed_vision_logit(self, seq_v, in_drop):
        """vision_logit of a packed plan: the Linear on the packed region rows, scattered to the padded [B * Nv, 1] layout with
        PACKED_MASKED_LOGIT on the masked regions, so the objective, score and results read it as in the padded plan. The backward
        gathers the padded gradient back to the packed rows."""
        ps, lib, B, Nv, name = self.ps, self.lib, self.B, self.Nv, "vision_logit"
        M, K = seq_v.M, seq_v.H
        off, ln = self.seg["v"]
        y = self.buf((M, 1), F32)
        self.emit(lib.vb_small_linear_fwd, seq_v.f32, K, ps.p(name + ".weight"), ps.p(name + ".bias"), None, y, M, K, 1, in_drop)
        out = self.buf((B * Nv, 1), F32)
        self.emit(lib.vb_unpack_rows_f32, y, out, off, ln, B, Nv, 1, PACKED_MASKED_LOGIT)
        self.outputs[name] = out
        self.out_rg[name] = seq_v.rg or self.trainable(name)

        def bwd():
            if name not in self.grad_outputs:
                return
            dy = self.scratch("vlogit.dy", (M, 1), F32)
            self.emit(lib.vb_pack_rows_f32, self.out_grad_buffer(name, (B * Nv, 1)), dy, self.map_v, M, 1)
            g, acc = self.grad_acc(seq_v) if seq_v.rg else (None, 0)
            self.emit(lib.vb_small_linear_bwd, dy, seq_v.f32, K, ps.p(name + ".weight"), g, K, acc,
                      self.pg(name + ".weight"), self.pg(name + ".bias"), M, K, 1, in_drop)
        self.push_bwd(bwd, self.out_rg[name], name)

    def packed_vision_prediction(self, hv):
        """The region decoder of a packed plan: the [rows_v, C] logits of the packed region rows, scattered to the padded
        [B * Nv, C] layout (0 on the masked regions, which no region objective reads), so the KL / MSE / NCE kernels run as in the
        padded plan. Its backward gathers the padded gradient back to the packed rows before the decoder's backward (big_head)."""
        lib, B, Nv, C_, name = self.lib, self.B, self.Nv, self.cfg.v_target_size, "vision_prediction"
        M, K = hv.M, hv.H
        dl = self.buf((M, C_), F32) if name in self.grad_outputs else None
        head_bwd = self.big_head(name, hv, K, M, K, C_, "cls.imagePredictions.decoder", "cls.imagePredictions.decoder.bias", dl32=dl)
        off, ln = self.seg["v"]
        out = self.buf((B * Nv, C_), F32)
        self.emit(lib.vb_unpack_rows_f32, self.outputs[name], out, off, ln, B, Nv, C_, 0.0)
        self.outputs[name] = out

        def bwd():
            if name in self.grad_outputs and self.out_rg[name]:
                self.emit(lib.vb_pack_rows_f32, self.out_grad_buffer(name, (B * Nv, C_)), dl, self.map_v, M, C_)
            return head_bwd()
        return bwd

    def build_heads(self, seq_t, seq_v, pooled_t, pooled_v):
        """VILBertForVLTasks.forward after self.bert (vilbert.py:1673-1708) + BertPreTrainingHeads (:1228-1243).
        Dropout layers are identity (eval-mode / p = 0 parity protocol)."""
        ps, c, B, lib = self.ps, self.cfg, self.B, self.lib
        Hb, Ht, Hv, Nt, Nv = c.bi_hidden_size, c.hidden_size, c.v_hidden_size, self.Nt, self.Nv
        mul = 1 if c.fusion_method == "mul" else 0
        def fuse(drop, label):
            f32 = self.buf((B, Hb), F32)
            f = self.buf16((B, Hb))
            hi, lo, bw = f.ptrs()
            self.emit(lib.vb_fuse_pooled_fwd, pooled_t.f32, pooled_v.f32, f32, hi, B * Hb, mul, drop, f.fp16, lo, bw)
            act = self.act(f32, f, B, Hb, inputs=(pooled_t, pooled_v))

            def fuse_bwd():
                if not act.gw:
                    return
                for a in (pooled_t, pooled_v):
                    if a.rg:
                        self.grad_zeroed(a)
                self.emit(lib.vb_fuse_pooled_bwd, act.g32, pooled_t.f32, pooled_v.f32, pooled_t.g32, pooled_v.g32, B * Hb, mul, drop)
            self.push_bwd(fuse_bwd, act.rg, label)
            return act
        # VILBertForVLTasks.dropout on the fused vector (vilbert.py:1677-1682); BertPreTrainingHeads has its own nn.Dropout(0.1)
        # on its own fused vector (:1233-1241) — a different mask, needed only where the alignment score is an output
        # outputs=: the fused vector feeds the vil_* heads (the binary one only at even B), the alignment head the binary one at odd B
        want = self.want
        need_fused = any(want(n) for n in ("vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_tri_prediction")) or (
            want("vil_binary_prediction") and B % 2 == 0)
        fused = fuse(self.drop("dropout.pooled", self.head_dropout_prob), "dropout") if self.heads == "vl" and need_fused else None
        need_cls_fused = (self.heads == "pretraining" and want("seq_relationship_score")) or (B % 2 == 1 and want("vil_binary_prediction"))
        cls_drop = self.drop("cls.dropout", 0.1)
        if need_cls_fused:
            fused_cls = fuse(cls_drop, "cls.dropout") if (cls_drop is not None or fused is None) else fused
        else:
            fused_cls = None

        # --- cls: masked-LM head (decoder tied to the word embeddings), image-region head, alignment head
        self.lm_c = None
        if want("linguisic_prediction"):
            ht, ht_bwd = self.transform(seq_t, "cls.predictions.transform.dense", "cls.predictions.transform.LayerNorm", "lm.tr")
            # fused pre-training objective: only the masked rows enter the LM cross-entropy, so the tied decoder runs on those alone
            if self.loss_kind == "pretraining" and self.e.lm_compact:
                lm_bwd = None
                lm_compact_bwd = self.lm_head_compact(ht, ht_bwd)
            else:
                lm_bwd = self.big_head("linguisic_prediction", ht, Ht, B * Nt, Ht, c.vocab_size, None, "cls.predictions.bias",
                                       w=ps.w("bert.embeddings.word_embeddings.weight"), gw_name="bert.embeddings.word_embeddings.weight")
        if want("vision_prediction"):
            hv, hv_bwd = self.transform(seq_v, "cls.imagePredictions.transform.dense", "cls.imagePredictions.transform.LayerNorm", "im.tr")
            if self.packed:
                im_bwd = self.packed_vision_prediction(hv)
            else:
                im_bwd = self.big_head("vision_prediction", hv, Hv, B * Nv, Hv, c.v_target_size, "cls.imagePredictions.decoder",
                                       "cls.imagePredictions.decoder.bias")
        if want("linguisic_prediction"):
            self.push_bwd(self._wide_bwd(lm_bwd, ht, ht_bwd, Ht, c.vocab_size) if lm_bwd is not None else lm_compact_bwd, True,
                          "cls.predictions")
        if want("vision_prediction"):
            self.push_bwd(self._wide_bwd(im_bwd, hv, hv_bwd, Hv, c.v_target_size), True, "cls.imagePredictions")

        if self.heads == "pretraining":
            # BertForMultiModalPreTraining returns the alignment score of self.cls (vilbert.py:1497)
            if want("seq_relationship_score"):
                self.small_head("seq_relationship_score", fused_cls, "cls.bi_seq_relationship", 2)
            return
        if want("vil_binary_prediction") and B % 2 == 0:
            # vil_binary_prediction pairs consecutive samples: pooled.view(-1, 2*Hb) (:1686-1689)
            pair = self.act(fused.f32.view(B // 2, 2 * Hb), fused.op.view(B // 2, 2 * Hb), B // 2, 2 * Hb, inputs=(fused,))
            hb, hb_bwd = self.transform(pair, "vil_binary_prediction.logit_fc.0", "vil_binary_prediction.logit_fc.2", "bin.tr")
            # LayerNorm output is needed in fp32 for the 2-way linear: recompute it from the bf16 copy is lossy, so run the small
            # linear on an fp32 LayerNorm output
            hb32 = self.buf((B // 2, 2 * Hb), F32)
            # re-emit LN with an fp32 output (cheap: B/2 rows)
            fwd_fn, fwd_args, fwd_sid = self.fwd[-1]
            self.fwd[-1] = (fwd_fn, fwd_args._replace(y_f32=L.arg(hb32)), fwd_sid)
            hb.f32 = hb32

            def bin_bwd():
                if not hb.gw:
                    return
                hb_bwd()
                if pair.gw:   # gradient landed in pair.g32 [B/2, 2Hb] == [B, Hb]
                    self.add_grad(fused, pair.g32.view(B, Hb))
            self.push_bwd(bin_bwd, hb.rg, "vil_binary_prediction.logit_fc")   # registered first => runs after the 2-way linear's backward
            self.small_head("vil_binary_prediction", hb, "vil_binary_prediction.logit_fc.3", 2)
        elif want("vil_binary_prediction"):
            # odd batch: the reference returns the [B, 2] alignment output of self.cls here (:1673, 1686)
            self.small_head("vil_binary_prediction", fused_cls, "cls.bi_seq_relationship", 2)

        for nm in ("vil_prediction", "vil_prediction_gqa"):
            if not want(nm):
                continue
            n_out = ps.p(nm + ".logit_fc.3.weight").shape[0]     # the answer vocabulary
            hh, hh_bwd = self.transform(fused, nm + ".logit_fc.0", nm + ".logit_fc.2", nm + ".tr")
            head_bwd = self.big_head(nm, hh, 2 * Hb, B, 2 * Hb, n_out, nm + ".logit_fc.3", nm + ".logit_fc.3.bias")
            self.push_bwd(self._wide_bwd(head_bwd, hh, hh_bwd, 2 * Hb, n_out), True, nm + ".logit_fc")
        if want("vil_logit"):
            self.small_head("vil_logit", fused, "vil_logit", 1)
        if want("vil_tri_prediction"):
            self.small_head("vil_tri_prediction", fused, "vil_tri_prediction", 3)
        if want("vision_logit") and self.packed:
            self.packed_vision_logit(seq_v, self.drop("dropout.seq_v", self.head_dropout_prob, "v"))
        elif want("vision_logit"):
            self.small_head("vision_logit", seq_v, "vision_logit", 1, addend=self.mask_v,
                            in_drop=self.drop("dropout.seq_v", self.head_dropout_prob))
        if want("linguisic_logit"):
            self.small_head("linguisic_logit", seq_t, "linguisic_logit", 1, in_drop=self.drop("dropout.seq_t", self.head_dropout_prob))

    # ------------------------------------------------------------------ whole model
    def _build(self):
        c, B = self.cfg, self.B
        self.outputs, self.gout = OrderedDict(), {}
        self._objective_outputs()
        self.enc_t, self.enc_v = [], []
        t, v = self.embeddings()
        # BertEncoder.forward interleaving schedule (vilbert.py:960-1096)
        t_start = v_start = 0
        for count, (v_end, t_end) in enumerate(zip(c.v_biattention_id, c.t_biattention_id)):
            # fixed_t_layer / fixed_v_layer (vilbert.py:968-1003): the first layers of a stream run under no_grad — what they make
            # needs no gradient (Plan.act), so their backward is not emitted and their output stops the gradient (embeddings and
            # the frozen layers' parameters receive none)
            for i in range(t_start, t_end):
                self._no_grad = i < getattr(c, "fixed_t_layer", 0)
                t = self.text_layer(t, i)
                self._no_grad = False
            pool = None
            if self.dyn and v_end > v_start:
                # dynamic_attention: this segment's image layers read the pooled text states of the segment's END (the text layers
                # run first in the reference, vilbert.py:977-1004), so the two streams cannot overlap here
                pool = self.text_pool(t)
                self.sync_streams()
            with self.on(1):
                for i in range(v_start, v_end):
                    self._no_grad = i < getattr(c, "fixed_v_layer", 0)
                    v = self.image_layer(v, i, pool)
                    self._no_grad = False
            if count == 0 and self.fast:
                t = self.broadcast_text(t)
            if count == 0 and self.pairs:
                t, v = self.expand_pairs(t, v)
            if c.with_coattention:
                v, t = self.connection_layer(v, t, count)
            v_start, t_start = v_end, t_end
            self.enc_t.append(t); self.enc_v.append(v)     # output_all_encoded_layers: one entry per connection layer (:1075-1077)
        pool = None
        if self.dyn and c.v_num_hidden_layers > v_start:
            pool = self.text_pool(t)      # the trailing image layers see the text states BEFORE the trailing text layers (:1079-1092)
            self.sync_streams()
        with self.on(1):
            for i in range(v_start, c.v_num_hidden_layers):
                v = self.image_layer(v, i, pool)
        for i in range(t_start, c.num_hidden_layers):
            t = self.text_layer(t, i)
        self.sync_streams()      # poolers and heads read both streams; they run on the main stream
        self.seq_t, self.seq_v = t, v
        self.pooled_t = self.pooler(t, self.Nt, "bert.t_pooler.dense")
        self.pooled_v = self.pooler(v, self.Nv, "bert.v_pooler.dense")
        # packed: the sequence outputs are the packed rows [rows, H] (map_t / map_v give their padded rows)
        self.outputs["sequence_output_t"] = t.f32 if self.packed else t.f32.view(B, self.Nt, -1)
        self.outputs["sequence_output_v"] = v.f32 if self.packed else v.f32.view(B, self.Nv, -1)
        self.outputs["pooled_output_t"] = self.pooled_t.f32
        self.outputs["pooled_output_v"] = self.pooled_v.f32
        for nm, act in (("sequence_output_t", t), ("sequence_output_v", v), ("pooled_output_t", self.pooled_t), ("pooled_output_v", self.pooled_v)):
            self.out_rg[nm] = act.rg
        if self.heads != "none":
            self.build_heads(t, v, self.pooled_t, self.pooled_v)
            for nm in ("vision_prediction", "vision_logit"):
                if nm in self.outputs:
                    self.outputs[nm] = self.outputs[nm].view(B, self.Nv, -1)
            for nm in ("linguisic_prediction", "linguisic_logit"):
                if nm in self.outputs:
                    self.outputs[nm] = self.outputs[nm].view(B, self.Nt, -1)
        self.sync_streams(mirror=False)
        if self.loss_in_forward:
            with self.role(self.loss_kind):      # its head-gradient writes stand for torch's loss node
                self._emit_loss()
        if self.results is not None:
            self._emit_results()
        self.n_kernels_fwd = sum(1 for op in self.fwd if op[0] is not None)

        # ---------------- backward
        self.cur = self.bwd
        with self.role(self.loss_kind):
            if self.loss_in_forward:
                self._emit_grad_scale()
            elif self.loss_kind is not None:
                self._emit_loss()
        self._emit_backward((("sequence_output_t", self.seq_t), ("sequence_output_v", self.seq_v), ("pooled_output_t", self.pooled_t),
                             ("pooled_output_v", self.pooled_v)))

    def _emit_backward(self, bert_outputs):
        """The rest of the backward list: the caller's gradients into the BertModel outputs ((name, Act) pairs), the registered
        emitters in reverse order, and a join of every stream."""
        for nm, act in bert_outputs:
            if nm in self.grad_outputs:
                with self.role(act.mod or "bert"):
                    self.add_grad(act, self.out_grad_buffer(nm, (act.M, act.H)))
        self.sync_streams()
        for entry in reversed(self._bwd_emitters):
            if entry is None:
                self.sync_streams()
            else:
                self.sid, emitter, label = entry
                self._scratch_epoch += 1
                with self.role(label):
                    emitter()
        self.sid = 0
        self.cur.append((None, ("all",), 0))     # join every stream (incl. the weight-gradient side streams)
        self.n_kernels_bwd = sum(1 for op in self.bwd if op[0] is not None)
        self.cur = self.fwd

    def attention_export(self):
        """The reference's all_attention_mask triple (BertEncoder.forward, vilbert.py:1098-1107) for config.visualization: lists of
        attn_data dicts in layer order — text / image: {"attn", "queries", "keys"}; connection layers: {"attn1", "queries1",
        "keys1", "attn2", "querues2" (the reference's spelling), "keys2"}. Tensors are fp32 [B, heads, N, ...] copies."""
        def qk(d, which, N):
            x = d[which]
            return x.float().reshape(d["B"], N, d["H"], d["D"]).permute(0, 2, 1, 3).contiguous()
        def one(d):
            return {"attn": d["attn"].clone(), "queries": qk(d, "q", d["Nq"]), "keys": qk(d, "k", d["Nk"])}
        ts, vs = [one(d) for d in self.attn_t], [one(d) for d in self.attn_v]
        cs = [{"attn1": a1["attn"].clone(), "queries1": qk(a1, "q", a1["Nq"]), "keys1": qk(a1, "k", a1["Nk"]),
               "attn2": a2["attn"].clone(), "querues2": qk(a2, "q", a2["Nq"]), "keys2": qk(a2, "k", a2["Nk"])} for a1, a2 in self.attn_c]
        return ts, vs, cs

    def _objective_outputs(self):
        """Where the fused objective's scalars land, for every kind of plan (all None without an objective):
        - summed (loss= without loss_in_forward or score): self.loss, a private device f32 [1];
        - forward-placed task objective: self.objective_out f32 [2] holds (loss, score), read with one copy; self.loss and self.score
          (None without score=True) are its slots;
        - forward-placed pre-training: self.objective_out f32 [3] holds (masked_lm, masked_img, next_sentence); self.loss is None;
        - results=: self.results_out, one private byte buffer, holds objective_out (loss, score), the per-row argmax
          (self.results_argmax, int64) and values (self.results_values, f32), read with one copy (fetch_results). VL-logit has a row
          per question and a value per option, V-logit one value (the IoU) per row.
        self.loss_slots are the three scalars the pre-training losses land in (the summed loss three times). self.preds (sized by the
        head) and self.loss_grad (read by the backward) are created by _emit_score and _emit_grad_scale."""
        k, r = self.loss_kind, self.results
        self.loss_inputs = {}
        self.head_grad = {}     # loss_in_forward: d loss / d head, written by the forward-placed objective
        self.head_dl16 = {}     # head name -> the bf16 gradient operand the objective writes for big_head
        self.loss = self.score = self.preds = self.loss_grad = self.objective_out = self.results_out = None
        if r is not None:
            opts = self.choices
            rows = self.B // opts if r == "logit_ce" else self.B
            nval = {L.VB_RESULT_SOFTMAX: opts, L.VB_RESULT_GATHER: 1}.get(RESULT_MODES[r][1], 0)
            self.results_out = self.buf((8 + 8 * rows + 4 * rows * nval,), torch.uint8, zero=True)
            self.objective_out = self.results_out[:8].view(F32)
            self.results_argmax = self.results_out[8:8 + 8 * rows].view(I64)
            self.results_values = self.results_out[8 + 8 * rows:].view(F32).view(rows, nval) if nval else None
        elif self.task_objective:
            self.objective_out = self.buf((3 if k == "pretraining" else 2,), F32, zero=True)
        elif k is not None:
            self.loss = self.buf((1,), F32, zero=True)
        if self.task_objective and k != "pretraining":
            self.loss = self.objective_out[0:1]
        if self.want_score:
            self.score = self.objective_out[1:2]
        pre = self.task_objective and k == "pretraining"
        self.loss_slots = [self.objective_out[i:i + 1] for i in range(3)] if pre else [self.loss] * 3

    def _head_layout(self, k):
        """The HeadLayout of task kind k. A classifier head is read whole, a row per sample (per sample pair for the binary head at
        even B); VL-logit has a row per question over its answer options; V-logit-mc gathers its choices from the regions after
        the first MC_REGION_OFFSET. Describes only: the objective creates the loss_inputs entries (_emit_loss)."""
        name = LOSS_HEADS[k][0]
        lg = self.outputs[name]
        rows, cols = lg.shape[0], lg.shape[1]
        key = "labels" if k in ("logit_ce", "binary_ce", "tri_ce") else "target"
        if k == "logit_ce":       # vil_logit.view(B / options, options)
            opts = self.choices
            return HeadLayout(name, lg, rows // opts, opts, opts, 0, None, 0, key)
        if k == "vlogit_mc":      # vision_logit[:, 101:].gather(1, ids)
            return HeadLayout(name, lg, rows, self.choices, cols, MC_REGION_OFFSET, "multiple_choice_ids", cols, key)
        return HeadLayout(name, lg, rows, cols, cols, 0, None, 0, key)

    def _emit_loss(self):
        """The fused objective: one loss kernel per head writes the scalar (self.loss, fp32 device) and the fp32 d(loss)/d(head
        output) into the plan's output-gradient buffer, from where the head's backward proceeds as for a caller-supplied gradient
        (loss_in_forward: into a buffer of its own, _head_grad). Labels / targets are static plan inputs (self.loss_inputs), laid
        out as the head is (_head_layout)."""
        lib, k, li = self.lib, self.loss_kind, self.loss_inputs
        if k == "pretraining":
            self._emit_pretraining_loss()
            return
        h = self._head_layout(k)
        if h.ids is not None:
            li[h.ids] = self.buf((h.rows, h.cols), I64, zero=True)
        li[h.key] = self.buf((h.rows,), I64, zero=True) if h.key == "labels" else self.buf((h.rows, h.cols), F32, zero=True)
        lg, inp, loss = h.logits, li[h.key], self.loss
        if k == "vqa":
            self.vqa_target = li["target"]      # the VQA soft target under its round-1 name
        if h.key == "labels":
            d = self._head_grad(h.name, tuple(h.logits.shape))
            self.emit(lib.vb_ce_loss, lg, h.ld, inp, -1, loss, d, h.ld, None, 0, h.rows, h.cols, 1.0, 0)
        elif k in ("vqa", "gqa", "vlogit_bce"):
            if k == "vqa" and not self.task_objective:
                # the summed VQA objective (the round-1 training step) also writes the bf16 operand of the wide head's backward GEMMs
                # (8-padded rows), registered for big_head so that no cast follows; its fp32 gradient is rewritten every backward
                d = self.gout[h.name] = self.buf(tuple(h.logits.shape), F32)
                d16 = self.head_dl16[h.name] = self.buf((h.rows, _pad8(h.cols)), BF16, zero=True)
            else:
                d, d16 = self._head_grad(h.name, tuple(h.logits.shape)), None
            self.emit(lib.vb_bce_logits_loss, lg, inp, loss, d, d16, 0 if d16 is None else d16.shape[1], h.rows, h.cols, 1.0)
        else:   # V-logit-mc: BCE mean x C over the gathered choices; the soft-target binary / tri heads: BCE mean
            d = self._head_grad(h.name, tuple(h.logits.shape))
            row_loss = self.buf((h.rows,), F32)
            self.emit(lib.vb_bce_gather_loss, lg, h.ld, h.off, h.ld, li.get(h.ids), inp, h.rows, h.cols,
                      float(h.cols if k == "vlogit_mc" else 1.0), row_loss, loss, 0, d, h.ld, None, 0)
        if self.want_score:
            with self.role(None):
                self._emit_score()

    def _emit_pretraining_loss(self):
        """vilbert.py:1578-1590: masked-LM CE (ignore_index -1), the masked-region objective of config.visual_target (0: KL to the
        class distribution, 1: masked MSE, 2: NCE against the negatives in loss_inputs["neg_index"]) and the alignment CE
        (ignore_index -1, :1450). The summed plan adds all three into self.loss (train_concap.py's masked_loss_t + masked_loss_v +
        next_sentence_loss) and writes the gradients into the heads' output-gradient buffers; with loss_in_forward each loss gets
        its slot of self.objective_out and each gradient a buffer of its own (none in a forward-only plan)."""
        lib, B, Nv, li, c = self.lib, self.B, self.Nv, self.loss_inputs, self.cfg
        V, C, R = c.vocab_size, c.v_target_size, Nv - 1
        sep, slot = self.loss_in_forward, self.loss_slots
        acc = 0 if sep else 1           # the summed plan adds the region and alignment losses to the masked-LM loss

        def grad(name, shape):
            if not sep:
                return self.out_grad_buffer(name, shape)
            return self._head_grad(name, shape) if name in self.grad_outputs else None

        if self.lm_c is not None:
            lc = self.lm_c
            d32 = grad("linguisic_prediction", (lc["cap"], V)) if sep else lc["dl32"]
            d16 = None if sep else lc["dl16"]      # loss_in_forward: the backward scales d32, then casts it into dl16
            self.emit(lib.vb_ce_loss, lc["logits"], V, lc["labels"], -1, slot[0], d32, V, d16, lc["ldp"], lc["cap"], V, 1.0, 0)
            if sep:
                # more labelled rows than the capacity must already show in the forward (eval plans have no backward): the scatter
                # kernel's count check poisons the masked-LM slot; the rows it moves are a 4-column dummy
                src = self.scratch("lm.cap.src", (lc["cap"], 4), F32)
                dst = self.scratch("lm.cap.dst", (B * self.Nt, 4), F32)
                with self.role(None):
                    self.emit(lib.vb_scatter_rows_f32, src, dst, lc["idx"], lc["cap"], 4, lc["count"], slot[0])
        else:
            lg, rows = self.outputs["linguisic_prediction"], B * self.Nt
            li["masked_lm_labels"] = self.buf((rows,), I64, zero=True)
            d = grad("linguisic_prediction", tuple(lg.shape))
            self.emit(lib.vb_ce_loss, lg, V, li["masked_lm_labels"], -1, slot[0], d, V, None, 0, rows, V, 1.0, 0)
        sv = self.outputs["vision_prediction"]
        li["image_target"] = self.buf((B, R, C), F32, zero=True)
        li["image_label"] = self.buf((B, R), I64, zero=True)
        dv = grad("vision_prediction", tuple(sv.shape))
        vt = c.visual_target
        if vt == 0:
            self.emit(lib.vb_kl_masked_loss, sv, li["image_target"], li["image_label"], slot[1], dv, None, 0, B, Nv, C, 1.0, acc)
        elif vt == 1:
            row_loss = self.buf((B * Nv,), F32)
            self.emit(lib.vb_mse_masked_loss, sv, li["image_target"], li["image_label"], B, Nv, C, 1.0, row_loss, slot[1], acc, dv)
        elif vt == 2:
            n = nce_negative_count(c)
            li["neg_index"] = self.buf((B, R, n), I64, zero=True)
            row_loss = self.buf((B * Nv,), F32)
            self.emit(lib.vb_nce_region_loss, sv, li["image_target"], li["image_label"], li["neg_index"],
                      B, Nv, C, n, 1.0, row_loss, slot[1], acc, dv)
        else:
            raise ValueError(f"visual_target must be 0, 1 or 2, got {vt!r}")
        ns = self.outputs["seq_relationship_score"]
        li["next_sentence_label"] = self.buf((B,), I64, zero=True)
        d = grad("seq_relationship_score", tuple(ns.shape))
        self.emit(lib.vb_ce_loss, ns, 2, li["next_sentence_label"], -1, slot[2], d, 2, None, 0, B, 2, 1.0, acc)

    def _head_grad(self, name, shape):
        """Where the objective writes d loss / d head: the head's output-gradient buffer, or with loss_in_forward a buffer of its own
        that the backward scales into it (_emit_grad_scale)."""
        if not self.loss_in_forward:
            return self.out_grad_buffer(name, shape)
        self.head_grad[name] = self.buf(shape, F32, zero=True)
        return self.head_grad[name]

    def _emit_score(self):
        """The batch score of the task objective (task_utils.py:121-162, 325-374, 618-623) into self.score, argmax per row into
        self.preds, from the head logits and the objective's own labels or targets."""
        h, li = self._head_layout(self.loss_kind), self.loss_inputs
        labels, target = (li["labels"], None) if h.key == "labels" else (None, li["target"])
        self.preds = self.buf((h.rows,), I64, zero=True)
        self.emit(self.lib.vb_task_score, SCORE_MODES[self.loss_kind], h.logits, h.ld, h.off, h.cols, li.get(h.ids), h.width, target,
                  h.cols if target is not None else 0, labels, h.rows, self.score, 0, self.preds)

    def _emit_results(self):
        """vb_task_results on the head of self.results (RESULT_MODES), addressed as the objective and the score address it; the
        V-logit results read the target at the chosen region (its IoU)."""
        h, mode = self._head_layout(self.results), RESULT_MODES[self.results][1]
        target = self.loss_inputs["target"] if mode == L.VB_RESULT_GATHER else None
        vals = self.results_values
        self.emit(self.lib.vb_task_results, mode, h.logits, h.ld, h.off, h.cols, self.loss_inputs.get(h.ids), h.width, target,
                  h.cols if target is not None else 0, h.rows, self.results_argmax, vals, 1 if vals is None else vals.shape[1])

    def fetch_results(self):
        """Reads results_out with one device-to-host copy: (loss, score, argmax int64 [rows], values f32 [rows, n] or None) on the
        host. loss and score are 0 where the plan has no objective / score."""
        raw = self.results_out.cpu()
        rows, vals = self.results_argmax.numel(), self.results_values
        loss, score = raw[:8].view(F32).tolist()
        if vals is not None:
            vals = raw[8 + 8 * rows:].view(F32).view(vals.shape)
        return loss, score, raw[8:8 + 8 * rows].view(I64), vals

    def _emit_grad_scale(self):
        """Backward of a forward-placed objective: head gradient = stored d loss / d head x self.loss_grad (device scalar). The
        pre-training objective has one scalar per loss (PRETRAINING_SLOTS); its compacted masked-LM gradient is scaled into
        lm_c["dl32"] and cast from there into its bf16 operand lm_c["dl16"]."""
        pre = self.loss_kind == "pretraining"
        self.loss_grad = self.buf((3 if pre else 1,), F32, zero=True)
        self.loss_grad.fill_(1.0)
        for name, d in self.head_grad.items():
            if name in self.grad_outputs:
                s = self.loss_grad[PRETRAINING_SLOTS[name]] if pre else self.loss_grad
                if name == "linguisic_prediction" and self.lm_c is not None:
                    lc = self.lm_c
                    V = self.cfg.vocab_size
                    self.emit(self.lib.vb_scale_by_device, d, lc["dl32"], d.numel(), s)
                    self.emit(self.lib.vb_cast2d_f32_to_bf16, lc["dl32"], V, lc["dl16"], lc["ldp"], lc["cap"], V, 1.0)
                    continue
                g = self.out_grad_buffer(name, tuple(d.shape))
                self.emit(self.lib.vb_scale_by_device, d, g, d.numel(), s)

    # ------------------------------------------------------------------ execution
    def load_inputs(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                    task_ids=None, non_blocking=True):
        """Host (ideally pinned) or device tensors -> the plan's static input buffers. An image_prefix plan loads the text side only:
        its images come from load_images(), and input_imgs / image_loc / image_attention_mask must be None."""
        if self.image_prefix and not (input_imgs is None and image_loc is None and image_attention_mask is None):
            raise ValueError("image_prefix plan: load the images with load_images() (load_inputs loads the text side only)")
        self.in_ids.copy_(input_txt, non_blocking=non_blocking)
        if token_type_ids is None:
            self.in_tt.zero_()
        else:
            self.in_tt.copy_(token_type_ids, non_blocking=non_blocking)
        if attention_mask is None:
            self.in_amask.fill_(1)
        else:
            self.in_amask.copy_(attention_mask, non_blocking=non_blocking)
        if self.fast:
            self.in_amask_b.copy_(self.in_amask.expand_as(self.in_amask_b))
        if not self.image_prefix:
            self.load_images(input_imgs, image_loc, image_attention_mask, non_blocking)
        if self.pairs:
            b = self.Bin
            self.in_amask_pairs.view(b, b, -1).copy_(self.in_amask.unsqueeze(1).expand(b, b, -1))
            self.in_imask_pairs.view(b, b, -1).copy_(self.in_imask.unsqueeze(0).expand(b, b, -1))
        if self.has_task:
            if task_ids is None:
                raise ValueError("task_specific_tokens is set: task_ids is required")
            self.in_task.copy_(task_ids.reshape(-1), non_blocking=non_blocking)

    def load_images(self, input_imgs, image_loc, image_attention_mask=None, non_blocking=True):
        """Region features [B, Nv, 2048], boxes [B, Nv, 5] and the 0/1 image mask [B, Nv] (None: all ones) -> the plan's image inputs.
        An image_prefix plan then runs run_image_prefix(); any other plan reads them in its forward (load_inputs calls this)."""
        if image_attention_mask is None:
            self.in_imask.fill_(1)
        else:
            self.in_imask.copy_(image_attention_mask, non_blocking=non_blocking)
        self.in_feat.copy_(input_imgs, non_blocking=non_blocking)
        self.in_loc.copy_(image_loc, non_blocking=non_blocking)

    def run_image_prefix(self):
        """image_prefix: the image embedding and the additive image mask from the loaded images into the plan's private image
        states, which every later run_forward() reads until the next call. Its intermediates may live in the shared arena, so it
        counts as a forward of this plan there."""
        if not self.image_prefix:
            raise ValueError("run_image_prefix: the plan was built without image_prefix=True")
        self._claim_forward(writes_grad=False)
        self._run(self.prefix)

    def _claim_forward(self, writes_grad):
        """Every run of forward ops starts here: a new forward id, whose activations the shared arena now holds (holds_forward),
        and with writes_grad (the run includes the backward) a flat gradient buffer that is no longer known to be zero."""
        self.fwd_id += 1
        self.e.arena_owner = (self, self.fwd_id)
        if writes_grad:
            self.e.grad_clean = False

    def _run(self, ops):
        """Issues the ops on their streams. Markers: (None, ()) = barrier between the text and vision streams;
        (None, ("all",)) = join of every stream; (None, ("rec"|"wait", id)) = event edge to a weight-gradient side stream."""
        main = torch.cuda.current_stream()
        if self._streams is None:
            n = 4 if self.wgrad_streams else (2 if self.two_streams else 1)
            self._streams = [torch.cuda.Stream(device=self.dev) for _ in range(n - 1)]
        streams = [main] + self._streams
        handles = [st.cuda_stream for st in streams]
        check = L.check
        events = {}
        for fn, args, sid in ops:
            if fn is None:
                if not args:                      # text <-> vision barrier
                    if len(streams) > 1:
                        aux = streams[1]
                        e1 = torch.cuda.Event(); e1.record(main); aux.wait_event(e1)
                        e2 = torch.cuda.Event(); e2.record(aux); main.wait_event(e2)
                elif args[0] == "all":
                    # full barrier over every stream. Fork first (main -> side streams), then join (side -> main): inside a
                    # graph capture a side stream only belongs to the capture once it has waited on a captured event
                    e = torch.cuda.Event(); e.record(main)
                    for st in streams[1:]:
                        st.wait_event(e)
                    for st in streams[1:]:
                        e2 = torch.cuda.Event(); e2.record(st); main.wait_event(e2)
                elif args[0] == "rec":
                    e = torch.cuda.Event(); e.record(streams[sid]); events[args[1]] = e
                elif args[0] == "wait":
                    streams[sid].wait_event(events[args[1]])
                continue
            st = fn(*args, handles[sid] if sid < len(handles) else handles[0])
            if st:
                check(st, fn.__name__)

    def run_forward(self):
        self._claim_forward(writes_grad=False)
        if self.graph_fwd is not None:
            self.graph_fwd.replay()
        else:
            self._run(self.fwd)
            self._eager_runs[0] += 1

    def holds_forward(self, fwd_id):
        """The activations are still those of this plan's forward `fwd_id`: no later forward of this plan ran and, with the shared
        arena, no other plan's forward overwrote them."""
        return self.fwd_id == fwd_id and (self.e.arena is None or self.e.arena_owner == (self, fwd_id))

    def run_backward(self):
        if not self.holds_forward(self.fwd_id):
            raise L.VBError("shared activation arena: another plan's forward ran between this plan's forward and backward "
                            "(its saved activations are gone); run forward + backward per batch, or disable the arena")
        self.e.grad_clean = False
        if self.graph_bwd is not None:
            self.graph_bwd.replay()
        else:
            self._run(self.bwd)
            self._eager_runs[1] += 1

    def maybe_capture_passes(self, after=2):
        """Module-surface path: once a pass of this plan has run eagerly `after` times (kernels loaded, attributes set), capture
        it into its own CUDA graph — without a warm-up run, which would accumulate into the gradient buffer — so that the
        ~600 ctypes launches of a step become two graph replays."""
        if self.graph_fwd is None and self._eager_runs[0] >= after:
            torch.cuda.synchronize()
            self.graph_fwd = self._record(self.fwd)
        if self.graph_bwd is None and self._eager_runs[1] >= after:
            torch.cuda.synchronize()
            self.graph_bwd = self._record(self.bwd)

    def _record(self, *op_lists):
        """One CUDA graph of the op lists, issued one after the other."""
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for ops in op_lists:
                self._run(ops)
        return g

    def _warm_up(self, *op_lists):
        """Runs the op lists once on a side stream before a capture (module load, shared-memory attributes). It runs the forward
        and the backward: a step of this plan."""
        self._claim_forward(writes_grad=True)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for ops in op_lists:
                self._run(ops)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()

    def enable_training_prologue(self, zero_grad=True, refresh_weights=True):
        """Makes run_step a complete training-step body: bump the dropout step counter (train mode), zero the flat
        gradient buffer and refresh the bf16 weight shadow from the fp32 master parameters (what an optimizer step
        invalidates) before the forward. With two streams only the weights the first text layers need (everything laid out
        before the first connection layer) are cast on the main stream; the rest of the cast and the gradient memset run on
        the vision stream underneath those text layers (the vision stream's own first consumer, the image embedding, is
        queued behind them and is not needed before the first connection layer)."""
        ps, lib = self.ps, self.lib
        self.prologue = self.cur = []
        if self.train:
            self.emit(lib.vb_step_counter_bump, self.e.drop_step)
        n = ps.numel
        first_c = [off for name, (off, _) in ps.entries.items() if ".c_layer." in name]
        split = min(first_c) if (self.two_streams and first_c) else n
        if refresh_weights and split > 0:
            self.emit(lib.vb_cast_f32_to_bf16, *ps.cast_args(0, split))
        self.sync_streams(mirror=False)       # the vision stream starts after the main-stream part
        with self.on(1):
            if zero_grad:
                self.emit(lib.vb_memset_zero, ps.grad, ps.grad.numel() * 4)
            if refresh_weights and split < n:
                self.emit(lib.vb_cast_f32_to_bf16, *ps.cast_args(split, n - split))
        self.cur = self.fwd
        self.graph_step = None

    def enable_optimizer(self, opt, dropout_bump=True):
        """Training step with the fused optimizer (optim.FusedAdamW): the step body becomes [dropout step bump] + forward + loss +
        backward + ONE AdamW launch that also rewrites the 16-bit weight copy and zeroes the gradients — no weight cast and no
        gradient memset in the step. (The host-side lr table of `opt` is refreshed by opt.step(); here the launch alone is
        replayed, e.g. inside the step graph, with the table currently on the device.) With `max_grad_norm` the gradient-norm
        launch precedes it, so every replay clips and skips a non-finite step on the device. A plan with anomaly checks refuses:
        the step would apply a NaN gradient before the host could raise."""
        if getattr(opt, "shard_state", False):
            raise ValueError("enable_optimizer: a sharded optimizer (shard_state=True) exchanges gradients and weights with collectives "
                             "around its launches; a step captured in the plan would need them inside the capture. Use "
                             "loss.backward(); optimizer.step()")
        if self.anomaly:
            raise ValueError("enable_optimizer: a plan with anomaly checks (torch.autograd.set_detect_anomaly(True)) reports a NaN "
                             "gradient on the host after the backward; a step placed in the plan would apply it first")
        self.prologue = self.cur = []
        if self.train and dropout_bump:
            self.emit(self.lib.vb_step_counter_bump, self.e.drop_step)
        self.cur = self.fwd
        self.epilogue = [(fn, args, 0) for fn, args in opt.ops()]
        self.graph_step = None

    @property
    def n_launches_step(self):
        return sum(1 for op in self.prologue + self.epilogue if op[0] is not None) + self.n_kernels_fwd + self.n_kernels_bwd

    def run_step(self):
        """(prologue) + forward + (loss) + backward (+ epilogue); gradients accumulate into ParamStore.grad."""
        self._claim_forward(writes_grad=True)
        if self.graph_step is not None:
            self.graph_step.replay()
        else:
            self._run(self.prologue)
            self._run(self.fwd)
            self._run(self.bwd)
            self._run(self.epilogue)

    def _straddled(self):
        """Per position i of the backward list (a cut before bwd[i], 0..len): how many side-stream event edges it straddles. A piece
        ends with a join of every stream and the next one starts with a fork, so any position works as long as no event recorded
        in one piece is waited for in a later one (rec/wait markers of the side streams): a legal cut straddles none."""
        rec_pos, last_wait = {}, {}
        for i, op in enumerate(self.bwd):
            if op[0] is None and len(op[1]) == 2:
                if op[1][0] == "rec": rec_pos[op[1][1]] = i
                elif op[1][0] == "wait": last_wait[op[1][1]] = i
        straddle = [0] * (len(self.bwd) + 1)
        for ev, r in rec_pos.items():
            for i in range(r + 1, last_wait.get(ev, r) + 1):
                straddle[i] += 1
        return straddle

    def ddp_segments(self, n_segments=4, tail_cut=True):
        """Cuts the backward op list at stream barriers into `n_segments` pieces and returns
        [(bwd_op_lo, bwd_op_hi, grad_lo, grad_hi)]: after piece i has run, the flat gradient range [grad_lo, grad_hi) is
        final (no later op writes it) and may be all-reduced while the remaining pieces execute. The ranges tile the
        whole flat buffer from its end (heads, last layers) to its start (embeddings). With `tail_cut` one extra piece holds
        only the last few kernels, so up to n_segments + 1 pieces are returned."""
        n_ops = len(self.bwd)
        straddle = self._straddled()
        n_kern = [0] * (n_ops + 1)                      # kernels in bwd[:i]
        for i, op in enumerate(self.bwd):
            n_kern[i + 1] = n_kern[i] + (op[0] is not None)
        cand = [i for i in range(1, n_ops) if straddle[i] == 0 and self.bwd[i - 1][0] is not None or
                (straddle[i] == 0 and self.bwd[i - 1][0] is None and not self.bwd[i - 1][1])]
        cuts = []
        for k in range(1, n_segments):
            want = n_kern[n_ops] * k // n_segments     # equal kernel counts per piece
            free = [c for c in cand if c not in cuts]
            if not free:
                break
            cuts.append(min(free, key=lambda c: abs(n_kern[c] - want)))
        if tail_cut and cand:
            # one more cut just before the last kernels (the embedding backward): everything except the embedding tables, whose
            # gradients only the very last kernels produce, leaves the exposed final all-reduce
            late = [c for c in cand if n_kern[n_ops] - n_kern[c] >= 3]
            if late and (not cuts or late[-1] > max(cuts)):
                cuts.append(late[-1])
        cuts = sorted(set(cuts)) + [n_ops]
        # every piece must contain at least one kernel (an empty CUDA graph is legal but pointless)
        kept, prev = [], 0
        for cpos in cuts:
            if n_kern[cpos] > n_kern[prev]:
                kept.append(cpos)
                prev = cpos
        if not kept or kept[-1] != n_ops:               # trailing markers join the last piece that has kernels
            if kept: kept[-1] = n_ops
            else: kept = [n_ops]
        cuts = kept
        ranges = sorted(self.grad_touch.items())          # by flat offset
        numel = self.e.ps.numel
        segs, lo_op, hi_grad = [], 0, numel
        for cut in cuts:
            ready_lo = 0 if cut == n_ops else hi_grad
            if cut != n_ops:
                for (off, n), touch in reversed(ranges):
                    if off >= hi_grad:
                        continue
                    if touch >= cut:
                        break
                    ready_lo = off
            segs.append((lo_op, cut, ready_lo, hi_grad))
            lo_op, hi_grad = cut, ready_lo
        return segs

    def capture_segments(self, n_segments=4, tail_cut=True):
        """Captures the step as CUDA graphs, one per backward piece of ddp_segments (graph 0 = prologue + forward + first
        backward piece), for the data-parallel step: see run_step_overlapped."""
        self.segments = self.ddp_segments(n_segments, tail_cut=tail_cut)
        self._warm_up(self.prologue, self.fwd, self.bwd)
        barrier = [(None, ("all",), 0)]
        self.segment_graphs = [self._record(*([self.prologue, self.fwd] if i == 0 else []), barrier + self.bwd[lo:hi] + barrier)
                               for i, (lo, hi, _, _) in enumerate(self.segments)]
        torch.cuda.synchronize()

    def live_ranges(self, lo, hi):
        """Sub-ranges of the flat gradient range [lo, hi) that the backward of THIS plan writes (coalesced, 1024-element
        granularity): parameters whose gradient is identically zero for this plan (heads outside the objective, the never-called
        q_dense1/2 of BertBiOutput, vilbert.py:834,841) are not exchanged — zeros average to zeros on every rank."""
        spans = sorted((off, off + n) for (off, n) in self.grad_touch if off + n > lo and off < hi)
        out = []
        for a, b in spans:
            a, b = max(a, lo) // 1024 * 1024, min(-(-min(b, hi) // 1024) * 1024, hi)
            a = max(a, lo)
            if out and a <= out[-1][1] + 4096:
                out[-1][1] = max(out[-1][1], b)
            else:
                out.append([a, b])
        return [(a, b) for a, b in out if b > a]

    def capture_step_ddp(self, allreduce_range, n_segments=8, tail_cut=True, skip_dead=True):
        """Data-parallel step as ONE CUDA graph: prologue + forward + the backward pieces of ddp_segments, with the all-reduce of
        each finished gradient range captured on a communication stream inside the same graph (NCCL collectives are capturable),
        forked after its piece and joined at the end. Compared with capture_segments / run_step_overlapped there is a single
        graph launch per step and no host-side event bookkeeping between pieces. `allreduce_range(lo, hi)` must enqueue the
        collective on the current stream (async_op=False semantics). The epilogue (enable_optimizer) runs after the
        communication stream has joined, so a clipping optimizer takes the norm of the averaged gradient."""
        self.segments = self.ddp_segments(n_segments, tail_cut=tail_cut)
        torch.cuda.synchronize()
        barrier = [(None, ("all",), 0)]
        g = torch.cuda.CUDAGraph()
        comm = torch.cuda.Stream(device=self.dev)
        self._ddp_comm = comm
        with torch.cuda.graph(g):
            main = torch.cuda.current_stream()
            self._run(self.prologue); self._run(self.fwd)
            for (lo_op, hi_op, lo, hi) in self.segments:
                self._run(barrier + self.bwd[lo_op:hi_op] + barrier)
                if hi > lo:
                    ev = torch.cuda.Event(); ev.record(main)
                    comm.wait_event(ev)
                    with torch.cuda.stream(comm):
                        for (a, b) in (self.live_ranges(lo, hi) if skip_dead else [(lo, hi)]):
                            allreduce_range(a, b)
            ev = torch.cuda.Event(); ev.record(comm)
            main.wait_event(ev)
            self._run(self.epilogue)
        self.graph_step_ddp = g
        torch.cuda.synchronize()

    def run_step_ddp(self):
        self._claim_forward(writes_grad=True)
        self.graph_step_ddp.replay()

    def run_step_overlapped(self, allreduce_range, comm_stream, skip_dead=True):
        """Replays the segment graphs; after each one the finished tail range of the flat gradient buffer is handed to
        `allreduce_range(lo, hi)` (issued under `comm_stream`, which first waits for that segment) so the collective
        overlaps the rest of the backward. Ranges no backward op of this plan writes (live_ranges) are not exchanged.
        Returns the list of whatever allreduce_range returned (async work handles). No epilogue runs here: a caller that
        launches the optimizer afterwards must first wait for these collectives, and with max_grad_norm so must the gradient
        norm, which is to be taken of the averaged gradient."""
        self._claim_forward(writes_grad=True)
        main = torch.cuda.current_stream()
        works = []
        for g, (_, _, lo, hi) in zip(self.segment_graphs, self.segments):
            g.replay()
            if hi > lo:
                ev = torch.cuda.Event()
                ev.record(main)
                with torch.cuda.stream(comm_stream):
                    comm_stream.wait_event(ev)
                    for (a, b) in (self._live_cache(lo, hi) if skip_dead else [(lo, hi)]):
                        works.append(allreduce_range(a, b))
        return works

    def _live_cache(self, lo, hi):
        c = self._live_ranges_cache
        if (lo, hi) not in c:
            c[(lo, hi)] = self.live_ranges(lo, hi)
        return c[(lo, hi)]

    def _bucket_ready(self, key, weights=False):
        """Per bucket (lo, hi) of `key`: one past the last backward op that passes an address inside the bucket's range of the flat
        gradient buffer (0 when none does). The launches themselves are read (op_pointers), so side-stream event markers and, in
        deterministic plans, the ordered sums of split-K and bias gradients are seen where they run. An address stands for the
        span from it to the end of the outermost range containing it (ranges nest: a fused projection holds its parts): the
        gradient ranges of grad_touch, which records when a gradient view was taken.

        weights=True: the readiness of a step, which rewrites the weights as well. The addresses inside the fp32 parameters
        (ps.flat: LayerNorm gammas, the baseline's weight-norm v and g) and inside every 16-bit copy (ps.shadows: the dgrad GEMMs'
        operands, the tied decoder's word-embedding copy) count too, and any entry or fused projection is such a range."""
        ps = self.ps
        spans = sorted(set(self.grad_touch) | ({ps.span(n) for n in list(ps.entries) + list(ps.fused)} if weights else set()))
        starts = [off for off, _ in spans]
        outer_end, m = [], 0
        for off, n in spans:          # the end of the outermost range so far
            m = max(m, off + n)
            outer_end.append(m)
        bufs = [ps.grad] + ([ps.flat] + [t for t in (ps.shadow, ps.shadow_lo, ps.shadows.extra_bw) if t is not None] if weights else [])
        bases = [(t.data_ptr(), t.data_ptr() + t.element_size() * ps.numel, t.element_size()) for t in bufs]
        ready = [0] * len(key)
        for i, (fn, args, _) in enumerate(self.bwd):
            if fn is None:
                continue
            for p in op_pointers(fn, args):
                for base, end, es in bases:
                    if base <= p < end:
                        break
                else:
                    continue
                o = (p - base) // es
                j = bisect.bisect_right(starts, o) - 1
                if j < 0 or outer_end[j] <= o:
                    continue
                for k, (lo, hi) in enumerate(key):
                    if lo < outer_end[j] and o < hi:
                        ready[k] = i + 1
        return ready

    @staticmethod
    def _check_buckets(key, what):
        if any(b[0] >= b[1] for b in key) or any(a[1] > b[0] for a, b in zip(key, key[1:])):
            raise ValueError(f"{what}: the buckets must be non-empty, disjoint and in ascending order")

    def bucket_schedule(self, buckets):
        """The backward of the module surface's overlapped data parallelism (ddp.DistributedDataParallel(delay_allreduce=False)) cut
        into pieces: -> ((op_lo, op_hi, ranges), ...), where `ranges` are the buckets to all-reduce once bwd[op_lo:op_hi] has run.

        `buckets` is the reducer's table, the same on every rank: (lo, hi) ranges of the flat gradient buffer in ascending order.
        They are handed over in descending order, each exactly once, whatever this plan is, so ranks whose plans differ (packed
        capacities, a padded fallback, frozen or deterministic variants) issue the same collectives in the same order; only where
        the backward pauses for them depends on the plan. A bucket is ready once no later backward op writes its gradient
        (_bucket_ready). The cut of bucket k is the latest readiness of the buckets at or above it, moved forward to the next
        position that straddles no side-stream event edge (_straddled). Cached per table: ddp.trainable_ranges changes it with
        requires_grad."""
        key = tuple((int(lo), int(hi)) for lo, hi in buckets)
        sched = self._bucket_schedules.get(key)
        if sched is not None:
            return sched
        if self.anomaly:
            raise ValueError("bucket_schedule: the NaN checks of an anomaly plan read the gradients after the backward, and their "
                             "report comes before any collective; such plans all-reduce after the backward")
        self._check_buckets(key, "bucket_schedule")
        ready = self._bucket_ready(key)
        straddle = self._straddled()
        pieces, op_lo, cut, pending = [], 0, 0, []
        for k in reversed(range(len(key))):
            c = max(cut, ready[k])
            while straddle[c]:
                c += 1
            if c != cut and pending:
                pieces.append((op_lo, cut, tuple(pending)))
                op_lo, pending = cut, []
            cut = c
            pending.append(key[k])
        pieces.append((op_lo, cut, tuple(pending)))
        if any(op[0] is not None for op in self.bwd[cut:]):     # kernels that write no bucket (input gradients): a last piece
            pieces.append((cut, len(self.bwd), ()))
        sched = self._bucket_schedules[key] = tuple(pieces)
        return sched

    def step_schedule(self, buckets, allreduce):
        """The backward cut into pieces for an optimizer step that runs while it does (optim step_in_backward):
        -> ((op_lo, op_hi, ranges, steps), ...), where once bwd[op_lo:op_hi] has run `ranges` are the buckets to all-reduce and
        `steps` the indexes (into `buckets`, descending) of the buckets whose step may start.

        A bucket may be stepped once no later backward op reads or writes its weights, 16-bit copies or gradient
        (_bucket_ready(weights=True)), moved forward past side-stream event edges as in bucket_schedule. With `allreduce` (data
        parallel, delay_allreduce=False) the collectives keep bucket_schedule's pieces, order and cut points exactly, the step of
        a bucket comes no earlier than its collective's handover, and a step point between two of those cuts is one more join of
        the streams: nothing here depends on more than the plan and the table, so ranks issue the same collectives. Without it
        `ranges` are empty. Cached per (table, allreduce)."""
        key = tuple((int(lo), int(hi)) for lo, hi in buckets)
        sched = self._step_schedules.get((key, allreduce))
        if sched is not None:
            return sched
        if self.anomaly:
            raise ValueError("step_schedule: the NaN report of an anomaly plan comes after the backward; its step runs after it")
        self._check_buckets(key, "step_schedule")
        straddle = self._straddled()
        floor, hand, cuts = [0] * len(key), {}, set()
        if allreduce:
            index = {b: k for k, b in enumerate(key)}
            for _, hi, ranges in self.bucket_schedule(key):
                cuts.add(hi)
                hand[hi] = ranges
                for r in ranges:
                    floor[index[r]] = hi
        step_at = []
        for k, r in enumerate(self._bucket_ready(key, weights=True)):
            c = max(floor[k], r)
            while straddle[c]:
                c += 1
            step_at.append(c)
        cuts.update(step_at)
        last = max(cuts, default=0)
        if any(op[0] is not None for op in self.bwd[last:]):     # kernels that touch no bucket (input gradients): a last piece
            cuts.add(len(self.bwd))
        pieces, op_lo = [], 0
        for c in sorted(cuts):
            pieces.append((op_lo, c, hand.get(c, ()), tuple(k for k in reversed(range(len(key))) if step_at[k] == c)))
            op_lo = c
        sched = self._step_schedules[(key, allreduce)] = tuple(pieces)
        return sched

    def _piece(self, lo, hi):
        """bwd[lo:hi] between two joins of every stream: a piece starts with a fork, so that in a graph capture every side stream it
        uses joins the capture, and ends with a join, so that everything it wrote is done when the main stream's event fires."""
        barrier = [(None, ("all",), 0)]
        return barrier + self.bwd[lo:hi] + barrier

    def _schedule(self, buckets, step, allreduce):
        return self.step_schedule(buckets, allreduce) if step is not None else self.bucket_schedule(buckets)

    def run_backward_pieces(self, buckets, handover, comm_stream, step=None, step_stream=None):
        """The backward as the pieces of bucket_schedule(buckets). After each piece that finished buckets, `comm_stream` waits for an
        event recorded on the current stream and handover(ranges) is called under comm_stream with them; it enqueues the
        collectives, which stay outside any graph (DESIGN.md §4c). Pieces run eagerly, or as one CUDA graph each once
        maybe_capture_pieces captured them. The caller makes the current stream wait for the collectives before reading the buffer.

        With `step`, the pieces of step_schedule(buckets, allreduce=handover is not None): after each piece with step points,
        `step_stream` waits for the same event and step(bucket indexes) is called under step_stream (after that piece's handover);
        the caller makes the current stream wait for step_stream too."""
        if not self.holds_forward(self.fwd_id):
            raise L.VBError("shared activation arena: another plan's forward ran between this plan's forward and backward "
                            "(its saved activations are gone); run forward + backward per batch, or disable the arena")
        self.e.grad_clean = False
        sched = self._schedule(buckets, step, handover is not None)
        sinks = ((handover, comm_stream), (step, step_stream))
        graphs = self._piece_graphs.get(sched)
        main = torch.cuda.current_stream()
        for i, (lo, hi, *items) in enumerate(sched):
            if hi > lo:
                if graphs is not None:
                    graphs[i].replay()
                else:
                    self._run(self._piece(lo, hi))
            ev = None
            for (fn, stream), it in zip(sinks, items):
                if it:
                    if ev is None:
                        ev = torch.cuda.Event()
                        ev.record(main)
                    stream.wait_event(ev)
                    with torch.cuda.stream(stream):
                        fn(it)
        if graphs is None:
            self._piece_runs[sched] += 1

    def maybe_capture_pieces(self, buckets, after=2, step=False, allreduce=True):
        """maybe_capture_passes for the pieces of bucket_schedule(buckets) (with `step`: of step_schedule(buckets, allreduce)): once
        they have run eagerly `after` times, one CUDA graph per non-empty piece, captured without a warm-up run (it would accumulate
        into the gradient buffer)."""
        sched = self._schedule(buckets, True if step else None, allreduce)
        if sched not in self._piece_graphs and self._piece_runs[sched] >= after:
            torch.cuda.synchronize()
            self._piece_graphs[sched] = [self._record(self._piece(lo, hi)) if hi > lo else None for lo, hi, *_ in sched]

    def capture(self, separate=False):
        """Captures the plan into CUDA graphs (one for the whole step, or one per pass)."""
        self._warm_up(self.prologue, self.fwd, self.bwd, self.epilogue)
        if separate:
            self.graph_fwd, self.graph_bwd = self._record(self.fwd), self._record(self.bwd)
        else:
            self.graph_step = self._record(self.prologue, self.fwd, self.bwd, self.epilogue)
        torch.cuda.synchronize()


class BasePlan(Plan):
    """Plan of the single-stream baseline BaseBertForVLTasks (heads "base" / "base_none"; vilbert/basebert.py). It has none of the
    two-stream options (batch pairs, task token, fast mode, gate, attention export), and its plans take grad_outputs, train,
    frozen, input_grads and recycle only: no fused objective, outputs= selection or image prefix (PlanSpec.of)."""

    def _stream_modes(self, B, Nt, Nv):
        self.pairs = self.has_task = self.viz = self.dyn = False
        self.B, self.Nt_in, self.Nt, self.Nv, self.Bt = B, Nt, Nt, Nv, B

    def _build(self):
        """basebert.BertModel.forward + BaseBertForVLTasks.forward (basebert.py:706-774, 923-962): both embeddings LayerNormed into one
        [B, Nt+Nv, H] stream under the concatenated mask, num_hidden_layers BERT layers over it, the tanh pooler on row 0 and the seven
        heads. The wide heads (masked-LM, region classes) read their rows gathered into compact operands and scatter their gradient
        back; the 1-output heads run over the whole stream with a zero output gradient on the rows they do not return."""
        c, B = self.cfg, self.B
        self.outputs, self.gout = OrderedDict(), {}
        self._objective_outputs()
        self.N = self.Nt + self.Nv
        x = self.base_embeddings()
        self.enc = []
        for i in range(c.num_hidden_layers):
            x = self.base_layer(x, i)
            self.enc.append(x)
        self.seq = x
        self.pooled = self.base_pooler(x)
        self.outputs["sequence_output"] = x.f32.view(B, self.N, -1)
        self.outputs["pooled_output"] = self.pooled.f32
        self.out_rg["sequence_output"] = x.rg
        self.out_rg["pooled_output"] = self.pooled.rg
        views = self.build_base_heads(x, self.pooled) if self.heads == "base" else {}
        self.n_kernels_fwd = sum(1 for op in self.fwd if op[0] is not None)

        self.cur = self.bwd
        self._emit_backward((("sequence_output", self.seq), ("pooled_output", self.pooled)))
        self.gout.update(views)      # the 1-output heads take their caller's gradient into their rows of the whole-stream buffer

    def base_embeddings(self):
        """BertEmbeddings + BertImageEmbeddings + torch.cat (basebert.py:284-359, 718-747). The region side (feature cast, box
        projection, 2048 -> H GEMM) runs on the second stream under the text gather; vb_concat_embed_ln_fwd adds the image token-type
        row, applies both LayerNorms and dropouts and writes the stream with its operand copies."""
        ps, c, B, lib = self.ps, self.cfg, self.B, self.lib
        H, Nt, Nv, Fv = c.hidden_size, self.Nt, self.Nv, BASE_FEATURE_SIZE
        Mt, Mv, M = B * Nt, B * Nv, B * self.N
        self.in_ids = self.buf((B, Nt), I64, zero=True)
        self.in_tt = self.buf((B, Nt), I64, zero=True)
        self.in_task = None
        self.in_amask = self.buf((B, Nt), I64, zero=True)
        self.in_imask = self.buf((B, Nv), I64, zero=True)
        self.in_feat = self.buf((B, Nv, Fv), F32, zero=True)
        self.in_loc = self.buf((B, Nv, 5), F32, zero=True)
        self.mask = self.buf((B, self.N), F32)
        self.emit(lib.vb_mask_concat_additive, self.in_amask, self.in_imask, self.mask, B, Nt, Nv)
        self.sync_streams()      # the second stream reads the inputs that load_inputs copied on the main stream
        e, ie = "bert.embeddings", "bert.image_embeddings"
        t_tables = [e + n for n in (".word_embeddings.weight", ".position_embeddings.weight", ".token_type_embeddings.weight")]
        xt = self.buf((Mt, H), F32)
        self.emit(lib.vb_embed_text_fwd, self.in_ids, self.in_tt, None, *[ps.p(n) for n in t_tables], None, xt, B, Nt, H)
        with self.on(1):
            xv, feat = self.image_embedding(ie, H)
        self.sync_streams()
        trow = ps.p(ie + ".token_type_embeddings.weight")[1]
        tdrop = self.drop(e + ".dropout", c.hidden_dropout_prob)
        vdrop = self.drop(ie + ".dropout", c.hidden_dropout_prob)
        y32, y = self.buf((M, H), F32), self.buf16((M, H))
        mean, rstd = self.buf((M,), F32), self.buf((M,), F32)
        lnt, lnv = e + ".LayerNorm", ie + ".LayerNorm"
        self.emit(lib.vb_concat_embed_ln_fwd, xt, xv, trow, ps.p(lnt + ".weight"), ps.p(lnt + ".bias"), ps.p(lnv + ".weight"), ps.p(lnv + ".bias"),
                  y32, *y.ptrs(), y.fp16, mean, rstd, B, Nt, Nv, H, tdrop, vdrop)
        img = [ie + n for n in (".image_embeddings.weight", ".image_embeddings.bias", ".token_type_embeddings.weight",
                                ".image_location_embeddings.weight", ".image_location_embeddings.bias")]
        lns = [lnt + ".weight", lnt + ".bias", lnv + ".weight", lnv + ".bias"]
        x = self.act(y32, y, M, H, params=(*t_tables, *img, *lns), rg=self.input_grads)

        def bwd():
            if not x.gw:
                return
            gt = [self.pg(n) for n in t_tables]
            dxt = self.scratch("emb.dxt", (Mt, H), F32) if any(g is not None for g in gt) else None
            want32 = self.trainable(img[3], img[4]) or "image_loc" in self.input_grads
            want16 = self.trainable(img[0]) or "input_imgs" in self.input_grads
            dxv32 = self.scratch("emb.dxv32", (Mv, H), F32) if want32 else None
            dxv16 = self.scratch("emb.dxv16", (Mv, H), BF16) if want16 else None
            gtype = self.pg(img[2])
            self.emit(lib.vb_concat_embed_ln_bwd, x.g32, xt, xv, trow, ps.p(lnt + ".weight"), ps.p(lnv + ".weight"), mean, rstd, dxt, dxv32, dxv16,
                      *[self.pg(n) for n in lns], self.pg(img[1]), None if gtype is None else gtype[1], B, Nt, Nv, H, tdrop, vdrop)
            if dxt is not None:
                self.emit(lib.vb_embed_text_bwd_padded, dxt, self.in_ids, self.in_tt, *gt, B, Nt, H)
            self.image_embedding_bwd(ie, H, feat, dxv16, dxv32)
        self.push_bwd(bwd, x.rg, e)
        return x

    def base_layer(self, x, i):
        """basebert.BertLayer over the whole stream at N = Nt + Nv with the concatenated mask (basebert.py:480-485)."""
        p, c = f"bert.encoder.layer.{i}", self.cfg
        h1 = self.self_attention_block(x, self.B, self.N, c.num_attention_heads, self.mask, p + ".attention", "t",
                                       p_attn=c.attention_probs_dropout_prob, p_hidden=c.hidden_dropout_prob)
        return self.ffn(h1, c.intermediate_size, p + ".intermediate.dense", p + ".output.dense", p + ".output.LayerNorm", "t.ffn",
                        drop=self.drop(p + ".output.dropout", c.hidden_dropout_prob))

    def base_pooler(self, seq):
        """BertPooler (basebert.py:507-519): Linear on row 0 of every sample (A read with row pitch N*H), then tanh."""
        ps, B, H, N, w = self.ps, self.B, seq.H, self.N, "bert.pooler.dense"
        pre = self.buf((B, H), F32)
        self.gemm(B, H, H, seq.op, N * H, ps.w(w + ".weight"), H, bias=ps.p(w + ".bias"), out_f32=pre, ld_of=H)
        y32, y = self.buf((B, H), F32), self.buf16((B, H))
        self.emit(self.lib.vb_tanh_fwd, pre, y32, *y.ptrs(), y.fp16, B * H)
        pooled = self.act(y32, y, B, H, inputs=(seq,), params=(w,))
        pooled.mod = "bert.pooler"

        def bwd():
            if not pooled.gw:
                return
            dpre = self.scratch("pool.dpre", (B, H), BF16)
            self.emit(self.lib.vb_tanh_bwd, pooled.g32, y32, dpre, self.pg(w + ".bias"), B, H)
            self.linear_wgrad(dpre, H, seq.op.bw, N * H, B, H, H, w)
            self.pooler_dgrad(seq, N, dpre, w)
        self.push_bwd(bwd, pooled.rg, pooled.mod)
        return pooled

    def base_rows(self, seq, a, b, tag, label):
        """Rows [a, b) of every sample of the stream as a compact Act (operand copies: the head transform reads nothing else). Its
        backward scatters the compact gradient into those rows of the stream gradient."""
        lib, B, N, H = self.lib, self.B, self.N, seq.H
        n = b - a
        idx = self.buf((B * n,), torch.int32, zero=True)
        idx.copy_((torch.arange(B).view(B, 1) * N + torch.arange(a, b).view(1, n)).reshape(-1).to(torch.int32))
        rows = self.act(None, self.gather_rows(seq.op, idx, B * n, H), B * n, H, inputs=(seq,))

        def bwd():
            if not rows.gw:
                return
            if not seq.gw:      # the gathered heads' backward runs first: zero the stream gradient once, then scatter disjoint rows
                self._scatter_ok = True
            g = self.grad_zeroed(seq)
            if self._scatter_ok:
                self.emit(lib.vb_scatter_rows_f32, rows.g32, g, idx, B * n, H, None, None)
                return
            full = self.scratch(tag + ".full", (B * N, H), F32)      # the stream gradient already holds other contributions
            self.emit(lib.vb_memset_zero, full, full.numel() * 4)
            self.emit(lib.vb_scatter_rows_f32, rows.g32, full, idx, B * n, H, None, None)
            self.emit(lib.vb_axpy_f32, full, g, full.numel(), 1.0)
        self.push_bwd(bwd, rows.rg, label)
        return rows

    def base_simple_classifier(self, x):
        """vil_prediction = SimpleClassifier (basebert.py:965-978): weight_norm(Linear(H, 2H), dim=None) -> ReLU -> Dropout(0.5) ->
        weight_norm(Linear(2H, num_labels), dim=None) on the pooled output. Like the reference's weight_norm pre-forward hook, every
        forward first derives both weights from (g, v) (vb_weight_norm_fwd: fp32 and the operand copies), so a parameter update by
        any optimizer is picked up without a separate refresh. The dropout sits in the first GEMM's epilogue after the ReLU; its
        backward folds the 1 / (1 - p) scale into the dgrad GEMM and gates by the dropped output."""
        ps, lib, B, H, Lb = self.ps, self.lib, self.B, x.H, self.ps.num_labels
        H2 = 2 * H
        W, self.wn_weights = {}, {}
        for i in (0, 3):
            nm = f"vil_prediction.main.{i}"
            v, g = ps.p(nm + ".weight_v"), ps.p(nm + ".weight_g")
            w32, op = self.buf(tuple(v.shape), F32), self.buf16(tuple(v.shape))
            scr = self.buf((L.VB_WEIGHT_NORM_SCRATCH // 8,), torch.float64)
            self.emit(lib.vb_weight_norm_fwd, v, g, v.numel(), w32, *op.ptrs(), op.fp16, scr)
            W[i] = (nm, v, g, op, scr)
            self.wn_weights[nm] = w32
        p_drop = 0.5
        drop = self.drop("vil_prediction.main.2", p_drop)
        h32, h = self.buf((B, H2), F32), self.buf16((B, H2))
        self.gemm(B, H2, H, x.op, H, W[0][3], H, bias=ps.p("vil_prediction.main.0.bias"), act=L.VB_ACT_RELU, out_f32=h32, ld_of=H2,
                  out_bf16=h, ld_ob=H2, dropout=drop)
        logits = self.buf((B, Lb), F32)
        self.gemm(B, Lb, H2, h, H2, W[3][3], H2, bias=ps.p("vil_prediction.main.3.bias"), out_f32=logits, ld_of=Lb)
        self.outputs["vil_prediction"] = logits
        part = lambda i: [f"vil_prediction.main.{i}.{s}" for s in ("weight_g", "weight_v", "bias")]
        h_rg = x.rg or self.trainable(*part(0))
        self.out_rg["vil_prediction"] = h_rg or self.trainable(*part(3))
        scale = 1.0 / (1.0 - p_drop) if drop is not None else 1.0

        def wn_wgrad(i, dy16, ld_dy, x16, ld_x, M, N_out, K_in):
            nm, v, g, _, scr = W[i]
            gg, gv = self.pg(nm + ".weight_g"), self.pg(nm + ".weight_v")
            if gg is None and gv is None:
                return
            dw = self.scratch(f"vilp.dw{i}", (N_out, K_in), F32)
            self.emit(lib.vb_memset_zero, dw, dw.numel() * 4)
            self.gemm(N_out, K_in, M, dy16, ld_dy, x16, ld_x, a_mn=1, b_mn=1, out_f32=dw, ld_of=K_in, atomic=1, split_k=0)
            self.emit(lib.vb_weight_norm_bwd, dw, v, g, v.numel(), gg, gv, scr)

        def bwd():
            if "vil_prediction" not in self.grad_outputs:
                return
            ldp = _pad8(Lb)
            dl32 = self.out_grad_buffer("vil_prediction", (B, Lb))
            dl16 = self.scratch("vilp.dl16", (B, ldp), BF16)
            self.emit(lib.vb_cast2d_f32_to_bf16, dl32, Lb, dl16, ldp, B, Lb, 1.0)
            gb = self.pg("vil_prediction.main.3.bias")
            if gb is not None:
                self.colsum(dl32, Lb, gb, B, Lb)
            wn_wgrad(3, dl16, ldp, h.bw, H2, B, Lb, H2)
            if not h_rg:
                return
            dh = self.scratch("vilp.dh32", (B, H2), F32)
            self.gemm(B, H2, Lb, dl16, ldp, W[3][3].bw, H2, b_mn=1, out_f32=dh, ld_of=H2, alpha=scale)
            dpre16, dpre32 = self.scratch("vilp.dpre16", (B, H2), BF16), self.scratch("vilp.dpre32", (B, H2), F32)
            self.emit(lib.vb_relu_bwd, dh, h32, dpre16, dpre32, B * H2)
            gb = self.pg("vil_prediction.main.0.bias")
            if gb is not None:
                self.colsum(dpre32, H2, gb, B, H2)
            wn_wgrad(0, dpre16, H2, x.op.bw, H, B, H2, H)
            self.dgrad_into(x, dpre16, H2, W[0][3].bw, B, H2, H)
        self.push_bwd(bwd, self.out_rg["vil_prediction"], "vil_prediction")

    def build_base_heads(self, seq, pooled):
        """The seven outputs of BaseBertForVLTasks.forward (basebert.py:929-962). Returns the views of the whole-stream output-gradient
        buffers that the caller's gradients of the 1-output heads go into. Emission order is chosen for the backward, which runs it
        in reverse: the gathered heads first (their scatters are the first writes to the stream gradient), then the 1-output heads
        over the stream and the pooled heads (which accumulate), then the pooler."""
        ps, c, B = self.ps, self.cfg, self.B
        H, Nt, Nv, N = seq.H, self.Nt, self.Nv, self.N
        self.base_simple_classifier(pooled)
        self.small_head("vil_logit", pooled, "vil_logit", 1)
        self.small_head("vil_binary_prediction", pooled, "cls.seq_relationship", 2)
        views = {}
        # self.dropout is one nn.Dropout called twice (basebert.py:949-952): two sites, each a mask over the whole stream
        for name, site, a, b in (("vision_logit", "dropout.seq_v", Nt, N), ("linguisic_logit", "dropout.seq_t", 0, Nt)):
            full = self.out_grad_buffer(name, (B * N, 1))
            self.small_head(name, seq, name, 1, addend=self.mask if name == "vision_logit" else None,
                            in_drop=self.drop(site, self.head_dropout_prob))
            self.outputs[name] = self.outputs[name].view(B, N, 1)[:, a:b]
            views[name] = full.view(B, N, 1)[:, a:b]
        rows_t = self.base_rows(seq, 0, Nt, "rows.t", "cls.predictions")
        rows_v = self.base_rows(seq, Nt, N, "rows.v", "cls.imagePredictions")
        wn = "bert.embeddings.word_embeddings.weight"
        ht, ht_bwd = self.transform(rows_t, "cls.predictions.transform.dense", "cls.predictions.transform.LayerNorm", "lm.tr")
        lm_bwd = self.big_head("linguisic_prediction", ht, H, B * Nt, H, c.vocab_size, None, "cls.predictions.bias", w=ps.w(wn), gw_name=wn)
        hv, hv_bwd = self.transform(rows_v, "cls.imagePredictions.transform.dense", "cls.imagePredictions.transform.LayerNorm", "im.tr")
        im_bwd = self.big_head("vision_prediction", hv, H, B * Nv, H, BASE_REGION_CLASSES, "cls.imagePredictions.decoder",
                               "cls.imagePredictions.decoder.bias")
        self.push_bwd(self._wide_bwd(lm_bwd, ht, ht_bwd, H, c.vocab_size), True, "cls.predictions")
        self.push_bwd(self._wide_bwd(im_bwd, hv, hv_bwd, H, BASE_REGION_CLASSES), True, "cls.imagePredictions")
        self.outputs["linguisic_prediction"] = self.outputs["linguisic_prediction"].view(B, Nt, -1)
        self.outputs["vision_prediction"] = self.outputs["vision_prediction"].view(B, Nv, -1)
        return views


class Engine:
    """Owns the parameters and the per-shape plans."""

    def __init__(self, cfg, device="cuda", heads="vl", _build_only=False, two_streams=True, wgrad_streams=True, precision="fp16",
                 num_labels=None):
        """_build_only=True (tests) allows a CPU device: plans can be constructed and inspected but never run.
        precision: "fp16" | "fp32" | "bf16" (module docstring). num_labels: answers of the baseline's vil_prediction (heads="base")."""
        cfg.check_supported()
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {PRECISIONS}")
        self.precision = precision
        self.op_dtype = BF16 if precision == "bf16" else F16
        self.split = precision == "fp32"
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda" and not _build_only:
            raise L.VBError("vilbert_b200 runs on sm_90a GPUs only; there is no CPU path (device=%s)" % device)
        L.lib()  # fail loudly now if the extension is missing
        self.ps = ParamStore(cfg, self.device, heads, self.op_dtype, self.split, num_labels=num_labels)
        self.two_streams = two_streams   # text / vision segments on two CUDA streams (parallel graph branches)
        self.wgrad_streams = wgrad_streams   # weight-gradient GEMMs on two more side streams (off the backward critical chain)
        self.plans = OrderedDict()       # LRU cache of per-shape plans (each owns its activation buffers)
        self.max_plans = 16              # a 12-in-1 mix has ~12 shapes x {train} x one gradient set in steady state
        self.head_dropout_prob = 0.1     # VILBertForVLTasks(dropout_prob=0.1), vilbert.py:1601
        self.drop_step = torch.zeros(1, dtype=torch.int32, device=self.device)   # dropout step counter (uint32 on the device)
        self.drop_step_host = 0          # host mirror of the counter for the eager module path (bump / set below)
        self.shadow_clean = False        # the 16-bit weight copy matches the fp32 master parameters
        self.shadow_trusted = False      # True while the engine's own fused optimizer is the only writer of the parameters
        self.grad_clean = False          # the flat gradient buffer is all zeros (set by zero_grad / the fused optimizer)
        self.loss_options = 4            # answer options per question of the VL-logit objective (retrieval / VCR: 4)
        # forward-only plans (no train mode, no grad_outputs, no input_grads) share the bytes of buffers with disjoint lifetimes
        # (Plan(recycle=True)); the default of Engine.plan(recycle=None)
        self.recycle_forward_only = False
        self.auto_graph = True           # module surface: capture a plan's passes into CUDA graphs after two eager runs
        self.arena = None                # optional shared activation arena (enable_activation_arena)
        self.arena_owner = None          # (plan, forward id) whose activations the arena currently holds
        self.bwd_gemm_max_ctas = 0       # persistent CTAs of the backward GEMMs (0 = one per SM); data parallel: leave SMs to NCCL (DESIGN §4c)
        self.lm_compact = True           # fused pre-training objective: masked-LM decoder + CE on the labelled rows only (Plan.lm_head_compact)
        self.lm_capacity = 0.25          # ... with room for this fraction of the token rows (15 % are masked; more poisons the loss with NaN)
        # task steps (vilbert_b200.tasks) on packed plans: the valid text tokens and image regions only (Plan(packed=...)), batches
        # that cannot be packed run padded and are counted by reason in pack_fallbacks; plan_builds counts plans built per
        # (B, Nt, Nv). A packed task holds one or two capacities (pack_capacity) per shape: the plan cache keeps room for them
        self.pack_padding = False
        self.pack_fallbacks = Counter()
        self.plan_builds = Counter()

    def plan(self, B, Nt, Nv, **options):
        """The cached plan of this shape and these options (the arguments of PlanSpec.of, which resolves and checks them). A call
        the spec refuses leaves the cache as it was."""
        spec = PlanSpec.of(self, B, Nt, Nv, **options)
        plan = self.plans.get(spec)
        if plan is not None:
            self.plans.move_to_end(spec)
            return plan
        # packed task steps add up to two capacities per task shape: a 12-task mix then holds ~36 plans in steady state
        while len(self.plans) >= self.max_plans * (3 if self.pack_padding else 1):   # evict the least recently used plan
            self.plans.popitem(last=False)
        plan = self.plans[spec] = (BasePlan if self.ps.base else Plan)(self, spec)
        self.plan_builds[(B, Nt, Nv)] += 1
        return plan

    def enable_activation_arena(self, nbytes):
        """One activation arena shared by all plans built afterwards (12-in-1 training holds a plan per task shape, but runs one
        forward + backward at a time, vilbert/task_utils.py:313-374 + train_tasks.py:545-551): their activation / scratch buffers
        overlay each other in `nbytes` of device memory instead of adding up. A plan's outputs must be consumed (the module
        surface copies the ones it returns) before another plan runs; run_backward refuses to run on clobbered activations."""
        if self.plans:
            raise L.VBError("enable_activation_arena must be called before the first plan is built")
        self.arena = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)

    def release_plans(self):
        """Drops every cached plan (and its activation / scratch buffers)."""
        self.plans.clear()

    def bump_dropout_step(self):
        """New dropout masks for the next forward (plans with a training prologue do this inside their graph)."""
        L.call(L.lib().vb_step_counter_bump, self.drop_step)
        self.drop_step_host = (self.drop_step_host + 1) & 0xFFFFFFFF

    def set_dropout_step(self, step):
        self.drop_step_host = int(step) & 0xFFFFFFFF
        self.drop_step.fill_(self.drop_step_host if self.drop_step_host < 2 ** 31 else self.drop_step_host - 2 ** 32)

    def refresh_weights(self):
        self.ps.refresh_shadow()
        self.shadow_clean = True

    def zero_grad(self, force=False):
        """Zeroes the flat gradient buffer unless it is known to be clean (the fused optimizer zeroes it in its own pass)."""
        if self.grad_clean and not force:
            return
        L.call(L.lib().vb_memset_zero, self.ps.grad, self.ps.grad.numel() * 4)
        self.grad_clean = True
