"""Packed pre-training steps on the host and on CPU-built plans: the host decision (capacities, the "mask" and "label" fallbacks,
the refusals), and that a packed pre-training plan launches the padded plan's ops at packed row counts plus its pack, unpack and
compaction launches, while a call without engine.pack_padding decides nothing."""
import json
import os
from collections import Counter

import pytest
import torch

from vilbert_b200.config import BertConfig
from vilbert_b200.engine import LOSS_HEADS, Engine, pack_capacity, pretraining_pack_rows

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
B, NT, NV = 4, 9, 11


def _cfgj(**over):
    return dict(json.load(open(os.path.join(GOLDEN, "tiny_b4.json")))["config"], **over)


def _engine(**over):
    return Engine(BertConfig.from_dict(_cfgj(**over)), "cpu", heads="pretraining", _build_only=True)


def _prefix(lens, n):
    return (torch.arange(n) < torch.tensor(lens).unsqueeze(1)).long()


def _batch():
    """Prefix-valid masks, masked-LM labels on valid tokens only and region labels on valid regions only."""
    mt, mv = _prefix([9, 3, 1, 6], NT), _prefix([11, 2, 5, 8], NV)
    lm = torch.full((B, NT), -1, dtype=torch.long)
    lm[0, 4], lm[1, 2], lm[3, 5] = 7, 9, 11
    il = torch.full((B, NV - 1), -1, dtype=torch.long)
    il[0, 9], il[1, 0], il[3, 6] = 1, 1, 1        # regions 10, 1 and 7
    return mt, mv, lm, il


def test_host_decision_capacities():
    mt, mv, lm, il = _batch()
    assert pretraining_pack_rows(mt, mv, lm, il, B, NT, NV) == (pack_capacity(19, B * NT), pack_capacity(26, B * NV))
    # no masks: every row valid
    assert pretraining_pack_rows(None, None, lm, il, B, NT, NV) == (B * NT, B * NV)
    # a region label of -1 or 0 on a masked region is not read by the loss
    il2 = il.clone(); il2[1, 5] = 0
    assert pretraining_pack_rows(mt, mv, lm, il2, B, NT, NV) == (pack_capacity(19, B * NT), pack_capacity(26, B * NV))


def test_host_decision_fallback_reasons():
    mt, mv, lm, il = _batch()
    bad = mt.clone(); bad[1, 0] = 0                       # a 0 before a 1
    assert pretraining_pack_rows(bad, mv, lm, il, B, NT, NV) == "mask"
    empty = mv.clone(); empty[2] = 0                      # an image row without any valid region
    assert pretraining_pack_rows(mt, empty, lm, il, B, NT, NV) == "mask"
    lm2 = lm.clone(); lm2[2, 3] = 5                       # a labelled token on a masked position
    assert pretraining_pack_rows(mt, mv, lm2, il, B, NT, NV) == "label"
    il2 = il.clone(); il2[1, 4] = 1                       # region 5 of sample 1 is masked (2 valid regions)
    assert pretraining_pack_rows(mt, mv, lm, il2, B, NT, NV) == "label"
    il3 = il.clone(); il3[1, 1] = 1                       # region 2 of sample 1 is the first masked one
    assert pretraining_pack_rows(mt, mv, lm, il3, B, NT, NV) == "label"


class _Model:
    """What BertForMultiModalPreTraining._packed_rows reads of a model."""

    def __init__(self, **over):
        self.engine = _engine(**over)
        self.config = self.engine.cfg
        self.engine.pack_padding = True


def _packed_rows(m, *a, input_grads=frozenset()):
    from vilbert_b200.modeling import BertForMultiModalPreTraining
    return BertForMultiModalPreTraining._packed_rows(m, *a, B, NT, NV, input_grads)


def test_module_decision_counts_fallbacks_and_refuses():
    mt, mv, lm, il = _batch()
    m = _Model()
    assert _packed_rows(m, mt, mv, lm, il) == pretraining_pack_rows(mt, mv, lm, il, B, NT, NV)
    lm2 = lm.clone(); lm2[2, 3] = 5
    assert _packed_rows(m, mt, mv, lm2, il) is None
    bad = mt.clone(); bad[1, 0] = 0
    assert _packed_rows(m, bad, mv, lm, il) is None
    assert m.engine.pack_fallbacks == Counter(label=1, mask=1)
    m.engine.pack_padding = False
    assert _packed_rows(m, bad, mv, lm2, il) is None and m.engine.pack_fallbacks == Counter(label=1, mask=1)
    m.engine.pack_padding = True
    with pytest.raises(NotImplementedError):
        _packed_rows(m, mt, mv, lm, il, input_grads=frozenset({"input_imgs"}))
    m.engine.lm_compact = False
    with pytest.raises(NotImplementedError):
        _packed_rows(m, mt, mv, lm, il)
    for flag in ("in_batch_pairs", "dynamic_attention", "visualization", "fast_mode"):
        mm = _Model(**{flag: True})
        with pytest.raises(NotImplementedError):
            _packed_rows(mm, mt, mv, lm, il)


FUSED = dict(loss="pretraining", loss_in_forward=True)


def test_plan_refusals():
    eng = _engine()
    rows = (24, 32)
    eng.plan(B, NT, NV, grad_outputs=LOSS_HEADS["pretraining"], packed=rows, **FUSED)
    eng.plan(B, NT, NV, outputs=LOSS_HEADS["pretraining"], packed=rows, **FUSED)
    with pytest.raises(NotImplementedError):      # the summed objective
        eng.plan(B, NT, NV, grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining", packed=rows)
    with pytest.raises(NotImplementedError):      # head outputs without the objective
        eng.plan(B, NT, NV, grad_outputs=LOSS_HEADS["pretraining"], packed=rows)
    with pytest.raises(NotImplementedError):
        eng.plan(B, NT, NV, packed=rows, input_grads={"input_imgs"}, **FUSED)
    eng.lm_compact = False
    with pytest.raises(NotImplementedError):
        eng.plan(B, NT, NV, packed=rows, **FUSED)
    with pytest.raises(NotImplementedError):
        _engine(dynamic_attention=True).plan(B, NT, NV, packed=rows, **FUSED)


def _ops(plan, which):
    return [op[0].__name__ for op in getattr(plan, which) if op[0] is not None]


PACK_OPS = {"vb_pack_build", "vb_pack_rows_f32", "vb_pack_regions", "vb_unpack_rows_f32", "vb_gather_rows16", "vb_zero_tail_rows",
            "vb_scatter_add_rows_f32"}


@pytest.mark.parametrize("vt,train", [(0, True), (1, True), (2, True), (0, False)])
def test_packed_plan_launches_the_padded_ops_at_packed_rows(vt, train):
    over = {} if vt == 0 else dict(visual_target=vt, v_target_size=48)
    eng = _engine(**over)
    kw = dict(grad_outputs=LOSS_HEADS["pretraining"] if train else (), train=train, **FUSED)
    rows_t, rows_v = 24, 32
    a, b = eng.plan(B, NT, NV, **kw), eng.plan(B, NT, NV, packed=(rows_t, rows_v), **kw)
    for which in ("fwd", "bwd"):
        pa = [n for n in _ops(a, which) if n not in ("vb_mask_to_additive", "vb_cast_f32_to_bf16", "vb_gather_rows16")]
        pb = [("vb_compact_rows" if n == "vb_compact_rows_mapped" else n) for n in _ops(b, which) if n not in PACK_OPS]
        assert pa == pb, which
    # the named launches of the packed heads: the labelled rows compacted through the text map, the region decoder's rows
    # scattered to the padded layout (and, with a backward, its padded gradient gathered back)
    fwd = [op for op in b.fwd if op[0] is not None]
    comp = [args for fn, args, _ in fwd if fn.__name__ == "vb_compact_rows_mapped"]
    assert len(comp) == 1 and comp[0].map == b.map_t.data_ptr() and comp[0].rows == rows_t
    assert comp[0].cap == a.lm_c["cap"] == b.lm_c["cap"]      # the capacity of the padded token rows
    C_ = eng.cfg.v_target_size
    unpack = [args for fn, args, _ in fwd if fn.__name__ == "vb_unpack_rows_f32" and args.cols == C_]
    assert len(unpack) == 1 and unpack[0].dst == b.outputs["vision_prediction"].data_ptr()
    gathers = [args for fn, args, _ in b.bwd if fn is not None and fn.__name__ == "vb_pack_rows_f32" and args.cols == C_]
    assert len(gathers) == (1 if train else 0)
    assert b.outputs["vision_prediction"].shape == a.outputs["vision_prediction"].shape == (B, NV, C_)
    assert b.loss_inputs["masked_lm_labels"].shape == a.loss_inputs["masked_lm_labels"].shape == (B * NT,)
    # every GEMM of the encoder and of the two transforms runs at the packed row counts; the region decoder at rows_v
    gm = [op[1][0]._obj for op in fwd if op[0].__name__ == "vb_gemm_bf16"]
    assert {g.M for g in gm} >= {rows_t, rows_v} and max(g.M for g in gm) <= max(rows_v, a.lm_c["cap"])
    assert any(g.M == rows_v and g.N == C_ for g in gm)


def test_pack_padding_off_changes_nothing():
    eng = _engine()
    p = eng.plan(B, NT, NV, grad_outputs=LOSS_HEADS["pretraining"], train=True, **FUSED)
    names = set(_ops(p, "fwd") + _ops(p, "bwd"))
    # the padded plan's masked-LM head gathers its labelled rows too (vb_gather_rows16)
    assert p.packed is None and not (PACK_OPS - {"vb_gather_rows16"}) & names
    assert "vb_compact_rows_mapped" not in names and "vb_compact_rows" in names
