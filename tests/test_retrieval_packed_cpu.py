"""Packed retrieval evaluation without a GPU: the host decision (capacities, capacity groups, fallbacks and their count, pack=None
following engine.pack_padding), the structure of packed fast-mode image-prefix plans against the padded ones, their refusals, and
the two new entry points as the header binds them."""
import json
import os
from collections import Counter

import pytest
import torch

from vilbert_b200 import _lib as L
from vilbert_b200 import engine as E
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import Engine, pack_capacity
from vilbert_b200.retrieval import RetrievalEvaluator, retrieval_pack_plan

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NT, NV = 9, 11
NEW_OPS = {"vb_pack_segments", "vb_broadcast_segment_rows"}
PACK_OPS = {"vb_pack_build", "vb_pack_rows_f32", "vb_pack_regions", "vb_unpack_rows_f32", "vb_gather_rows16", "vb_zero_tail_rows",
            "vb_scatter_add_rows_f32"} | NEW_OPS


def _prefix(lens, n):
    return (torch.arange(n) < torch.tensor(lens).unsqueeze(1)).long()


def _engine(heads="vl", **over):
    cfg = dict(json.load(open(os.path.join(GOLDEN, "tiny_b4.json")))["config"], **over)
    return Engine(BertConfig.from_dict(cfg), "cpu", heads=heads, _build_only=True)


def test_host_decision_capacities_groups_and_fallbacks():
    im = _prefix([3, 11, 1, 7, 5, 11, 2], NV)               # 7 images, chunks of 3: 3 + 3 + 1
    cm = _prefix([1, 9, 4, 4, 9, 2], NT)
    for has_task in (0, 1):
        chunks, bad_ch, bad_c = retrieval_pack_plan(im, cm, 3, has_task)
        assert (bad_ch, bad_c) == (0, 0) and [(lo, n) for lo, n, _, _ in chunks] == [(0, 3), (3, 3), (6, 1)]
        Nt = NT + has_task
        for lo, n, rows_v, groups in chunks:
            assert rows_v == pack_capacity(int(im[lo:lo + n].sum()), n * NV)
            assert None not in groups and list(groups) == sorted(groups)
            assert sorted(c for g in groups.values() for c in g) == list(range(6))
            for rows_t, caps in groups.items():
                assert all(rows_t == pack_capacity(n * (int(cm[c].sum()) + has_task), n * Nt) for c in caps)
                assert caps == sorted(caps)
    # a chunk with an empty image row or a hole runs padded, and so does a caption with a hole, on every chunk
    bad_im = im.clone(); bad_im[1] = 0; bad_im[4, 0] = 0
    bad_cm = cm.clone(); bad_cm[2, 0] = 0
    chunks, bad_ch, bad_c = retrieval_pack_plan(bad_im, bad_cm, 3, 1)
    assert (bad_ch, bad_c) == (2, 1)
    assert [rows_v for _, _, rows_v, _ in chunks] == [None, None, pack_capacity(2, NV)]
    assert chunks[0][3] == {None: list(range(6))}
    last = chunks[2][3]
    assert list(last)[0] is None and last[None] == [2] and all(2 not in g for k, g in last.items() if k is not None)


class _Model:
    """What RetrievalEvaluator reads of a model outside score()'s device work."""
    _heads = "vl"
    training = False

    def __init__(self):
        self.engine = _engine(task_specific_tokens=True)


def test_pack_argument_follows_the_engine_and_counts_fallbacks():
    m = _Model()
    im = _prefix([3, 11, 1, 7], NV)
    im[3, 0] = 0                                              # the second chunk (images 2, 3) falls back
    cm = _prefix([1, 9, 4], NT)
    cm[1, 3] = 0                                              # ... and caption 1
    feats, locs = torch.zeros(4, NV, 48), torch.zeros(4, NV, 5)
    padded = [(0, 2, None, {None: range(3)}), (2, 2, None, {None: range(3)})]

    def norm(chunks):
        return [(lo, n, rv, {k: list(g) for k, g in groups.items()}) for lo, n, rv, groups in chunks]
    ev = RetrievalEvaluator(m, feats, locs, im, chunk=2)
    assert norm(ev._chunks(cm, True)) == norm(padded) and not m.engine.pack_fallbacks
    m.engine.pack_padding = True
    got = ev._chunks(cm, True)
    assert got[0][2] is not None and got[1][2] is None and m.engine.pack_fallbacks == Counter(mask=2)
    assert norm(got) == norm(retrieval_pack_plan(im, cm, 2, 1)[0])
    assert norm(RetrievalEvaluator(m, feats, locs, im, chunk=2, pack=False)._chunks(cm, True)) == norm(padded)
    m.engine.pack_padding = False
    assert norm(RetrievalEvaluator(m, feats, locs, im, chunk=2, pack=True)._chunks(cm, True)) == norm(got)
    assert m.engine.pack_fallbacks == Counter(mask=4)


def _names(ops):
    return [fn.__name__ for fn, _, _ in ops if fn is not None]


@pytest.mark.parametrize("heads,head,task", [("vl", "vil_logit", False), ("vl", "vil_logit", True),
                                             ("pretraining", "seq_relationship_score", False)])
def test_packed_retrieval_plan_launches_the_padded_ops_at_packed_shapes(heads, head, task):
    eng = _engine(heads, task_specific_tokens=task)
    B = 4
    kw = dict(outputs=(head,), fast_mode=True, image_prefix=True)
    rows_t, rows_v = 20, 24
    a, b = eng.plan(B, NT, NV, **kw), eng.plan(B, NT, NV, packed=(rows_t, rows_v), **kw)
    for which in ("prefix", "fwd"):
        pa = [n for n in _names(getattr(a, which)) if n not in ("vb_mask_to_additive", "vb_cast_f32_to_bf16", "vb_broadcast_rows")]
        pb = [n for n in _names(getattr(b, which)) if n not in PACK_OPS]
        assert pa == pb, which
    assert _names(b.prefix)[:2] == ["vb_pack_segments", "vb_pack_regions"]
    Nt = NT + task
    # the image stream at rows_v in the prefix, the text at Nt rows (one sample) before the broadcast and rows_t after it
    gp = [args[0]._obj for fn, args, _ in b.prefix if fn is not None and fn.__name__ == "vb_gemm_bf16"]
    assert [g.M for g in gp] == [rows_v]
    gm = [args[0]._obj for fn, args, _ in b.fwd if fn is not None and fn.__name__ == "vb_gemm_bf16"]
    assert {g.M for g in gm} - {B} == {Nt, rows_t, rows_v}
    att = [args[0]._obj for fn, args, _ in b.fwd if fn is not None and fn.__name__ == "vb_attention_fwd"]
    assert att and all(x.q_off and x.k_len and not x.mask for x in att)
    assert {x.B for x in att} == {1, B}
    bc = [args for fn, args, _ in b.fwd if fn is not None and fn.__name__ == "vb_broadcast_segment_rows"]
    assert bc and all(x.rows == rows_t and x.repeats == B for x in bc)
    # no op touches a vocabulary- or region-class-wide head
    c = eng.cfg
    ns = {args[0]._obj.N for fn, args, _ in b.prefix + b.fwd if fn is not None and fn.__name__ == "vb_gemm_bf16"}
    assert not {c.vocab_size, c.v_target_size} & ns
    assert list(b.outputs)[-1] == head and tuple(b.outputs[head].shape) == tuple(a.outputs[head].shape)
    # the image segments are private: the prefix writes them once per chunk, every caption forward reads them
    for t in b.image_states[4:]:
        assert any(t is k for k in b._keep)
    assert eng.plan_builds[(B, NT, NV)] == 2


def test_packed_retrieval_plan_with_recycle_and_arena():
    eng = _engine(task_specific_tokens=True)
    eng.enable_activation_arena(64 << 20)
    kw = dict(outputs=("vil_logit",), fast_mode=True, image_prefix=True, packed=(20, 24))
    p, r = eng.plan(4, NT, NV, **kw), eng.plan(4, NT, NV, recycle=True, **kw)
    assert _names(p.prefix) == _names(r.prefix) and _names(p.fwd) == _names(r.fwd)
    assert r.held_bytes < p.held_bytes
    arena = eng.arena.untyped_storage().data_ptr()
    for plan in (p, r):
        assert all(t.untyped_storage().data_ptr() != arena for t in plan.image_states if t is not None)


def test_packed_retrieval_plan_is_deterministic_by_construction():
    eng = _engine(task_specific_tokens=True)
    plan = eng.plan(4, NT, NV, outputs=("vil_logit",), fast_mode=True, image_prefix=True, packed=(20, 24), deterministic=True)
    atomic = set(E.DET_WORKSPACE) | {"vb_layernorm_bwd", "vb_add_layernorm_bwd"}
    ops = [(fn, args, sid) for fn, args, sid in plan.prefix + plan.fwd if fn is not None]
    assert not [fn.__name__ for fn, _, _ in ops if fn.__name__ in atomic]
    assert all(not a[0]._obj.out_colsum for fn, a, _ in ops if fn.__name__ == "vb_gemm_bf16")
    assert {sid for _, _, sid in ops} == {0}


def test_refusals():
    eng = _engine()
    rows = (20, 24)
    with pytest.raises(NotImplementedError):          # fast_mode without the image prefix
        eng.plan(4, NT, NV, outputs=("vil_logit",), fast_mode=True, packed=rows)
    with pytest.raises(NotImplementedError):          # the image prefix without fast_mode
        eng.plan(4, NT, NV, outputs=("vil_logit",), image_prefix=True, packed=rows)
    with pytest.raises(NotImplementedError):          # another head than the score head
        eng.plan(4, NT, NV, outputs=("vil_logit", "vil_prediction"), fast_mode=True, image_prefix=True, packed=rows)
    with pytest.raises(NotImplementedError):
        eng.plan(4, NT, NV, fast_mode=True, image_prefix=True, packed=rows)
    with pytest.raises(NotImplementedError):
        _engine(visualization=True).plan(4, NT, NV, outputs=("vil_logit",), fast_mode=True, image_prefix=True, packed=rows)
    with pytest.raises(NotImplementedError):
        _engine(dynamic_attention=True).plan(4, NT, NV, outputs=("vil_logit",), fast_mode=True, image_prefix=True, packed=rows)
    pre = _engine("pretraining")
    with pytest.raises(NotImplementedError):
        pre.plan(4, NT, NV, outputs=("linguisic_prediction", "seq_relationship_score"), fast_mode=True, image_prefix=True, packed=rows)
    with pytest.raises(ValueError):                   # more text rows than B * Nt
        eng.plan(4, NT, NV, outputs=("vil_logit",), fast_mode=True, image_prefix=True, packed=(4 * NT + 1, 24))


def test_new_entry_points_are_bound_from_the_header():
    assert L.ARGS["vb_pack_segments"]._fields == ("mask", "N_in", "has_task", "B", "rows", "off", "len", "map")
    assert L.ARGS["vb_broadcast_segment_rows"]._fields == ("src", "dst", "row_bytes", "len", "repeats", "rows")
    lib = L.lib()
    for name in NEW_OPS:
        fn = getattr(lib, name)
        assert len(fn.argtypes) == len(L.ARGS[name]._fields) + 1 and name in E.ANOMALY_OUTPUTS
        with pytest.raises(TypeError, match=name):
            L.launch_args(fn, *([0] * len(fn.argtypes)))
