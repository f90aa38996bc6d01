"""Packed task steps on the host and on CPU-built plans: the capacity ladder, the packability check under every `process`, the
refusals, and that a packed plan launches the padded plan's ops at packed shapes while pack_padding=False changes nothing."""
import json
import os

import pytest
import torch

import _task_oracle as T
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import LOSS_HEADS, Engine, pack_capacity

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cfgj(**over):
    return dict(json.load(open(os.path.join(GOLDEN, "tiny_b4.json")))["config"], task_specific_tokens=True, max_position_embeddings=300,
                **over)


class _M:
    """What tasks.packed_rows reads of a model."""

    def __init__(self, **over):
        self.engine = Engine(BertConfig.from_dict(_cfgj(**over)), "cpu", _build_only=True)
        self.engine.pack_padding = True
        self.training = False


def test_capacity_ladder():
    assert pack_capacity(1, 40) == 40 and pack_capacity(14200, 256 * 101) == 9 * 1664   # step 1664 = 13 tiles
    for padded in (40, 1000, 25856, 78336):
        step = max(128, -(-padded // 16 // 128) * 128)
        for n in (1, padded // 3, padded // 2 + 7, padded):
            c = pack_capacity(n, padded)
            assert n <= c <= padded and (c == padded or c % step == 0) and c - n < step
    with pytest.raises(ValueError):
        pack_capacity(0, 10)


def _rows_np(mask_t, mask_v, has_task):
    import numpy as np
    lt = mask_t.numpy().sum(1) + (1 if has_task else 0)
    lv = mask_v.numpy().sum(1)
    return int(lt.sum()), int(lv.sum()), np.concatenate([[0], np.cumsum(lt)]), np.concatenate([[0], np.cumsum(lv)])


@pytest.mark.parametrize("task_id", ["TASK1", "TASK3", "TASK5", "TASK7", "TASK9", "TASK12", "TASK13"])
def test_packability_under_each_process(task_id):
    from vilbert_b200.data import expand_batch
    from vilbert_b200.tasks import packed_rows
    m = _M()
    cfgj = _cfgj()
    b = T.make_batch(cfgj, task_id, 4, 11 if task_id != "TASK4" else 110, 9)
    proc = T.TASK_CFG[task_id]["process"]
    if proc == "nlvr":      # each image's half of the mask must be prefix-valid
        nv = b[2].size(1) // 2
        b = list(b); b[2] = torch.cat([b[2][:, :nv], b[2][:, :nv]], 1); b = tuple(b)
    got = packed_rows(m, T.TASK_CFG, task_id, b, ("dialog", "expand", "retrieval", "nlvr"))
    _, _, im, _, am, _, _, _, _ = expand_batch(proc, b[0], b[1], b[2], b[3], b[5], b[6])
    nt, nv, _, _ = _rows_np(am, im, True)
    B = am.size(0)
    assert got == (pack_capacity(nt, B * (am.size(1) + 1)), pack_capacity(nv, B * im.size(1)))
    assert not m.engine.pack_fallbacks


def test_fallbacks_and_refusals():
    from vilbert_b200.tasks import packed_rows
    m = _M()
    b = list(T.make_batch(_cfgj(), "TASK1", 4, 11, 9))
    b[5] = b[5].clone(); b[5][2, 0] = 0
    assert packed_rows(m, T.TASK_CFG, "TASK1", tuple(b), ()) is None and m.engine.pack_fallbacks["mask"] == 1
    b = list(T.make_batch(_cfgj(), "TASK9", 4, 11, 9))
    b[4] = b[4].clone(); b[2] = b[2].clone(); b[2][0, -1] = 0; b[4][0, -1, 0] = 1.0
    assert packed_rows(m, T.TASK_CFG, "TASK9", tuple(b), ()) is None and m.engine.pack_fallbacks["target"] == 1
    m.training = True      # train mode packs: the packed plan draws the padded plan's dropout masks
    assert packed_rows(m, T.TASK_CFG, "TASK1", T.make_batch(_cfgj(), "TASK1", 4, 11, 9), ()) is not None
    assert sum(m.engine.pack_fallbacks.values()) == 2
    b = list(T.make_batch(_cfgj(), "TASK4", 2, 110, 9))      # every choice of sample 0 on a masked region, all targets 0
    b[4] = torch.zeros_like(b[4]); b[7] = torch.full_like(b[7], 5); b[2] = b[2].clone(); b[2][0, 100:] = 0
    assert packed_rows(m, T.TASK_CFG, "TASK4", tuple(b), ()) is None and m.engine.pack_fallbacks["choice"] == 1
    for flag in ("in_batch_pairs", "dynamic_attention", "visualization", "fast_mode"):
        mm = _M(**{flag: True}) if flag != "fast_mode" else _M()
        if flag == "fast_mode":
            mm.engine.cfg.fast_mode = True
        with pytest.raises(NotImplementedError):
            packed_rows(mm, T.TASK_CFG, "TASK1", T.make_batch(_cfgj(), "TASK1", 4, 11, 9), ())
    eng = _M().engine
    with pytest.raises(NotImplementedError):      # heads that are not packed
        eng.plan(4, 9, 11, loss="vqa", loss_in_forward=True, packed=(20, 30))


def _ops(plan, which):
    return [op[0].__name__ for op in getattr(plan, which) if op[0] is not None]


PACK_OPS = {"vb_pack_build", "vb_pack_rows_f32", "vb_pack_regions", "vb_unpack_rows_f32", "vb_gather_rows16", "vb_zero_tail_rows",
            "vb_scatter_add_rows_f32"}


@pytest.mark.parametrize("kind", ["vqa", "vlogit_bce", "logit_ce", "binary_bce"])
def test_packed_plan_launches_the_same_ops_at_packed_shapes(kind):
    eng = Engine(BertConfig.from_dict(_cfgj()), "cpu", _build_only=True)
    kw = dict(grad_outputs=LOSS_HEADS[kind], loss=kind, score=True, loss_in_forward=True, outputs=LOSS_HEADS[kind])
    a, b = eng.plan(4, 9, 11, **kw), eng.plan(4, 9, 11, packed=(24, 32), **kw)
    for which in ("fwd", "bwd"):
        pa = [n for n in _ops(a, which) if n not in ("vb_mask_to_additive", "vb_cast_f32_to_bf16")]
        pb = [n for n in _ops(b, which) if n not in PACK_OPS]
        assert pa == pb, which
    gm = [op[1][0]._obj for op in b.fwd if op[0] is not None and op[0].__name__ == "vb_gemm_bf16"]
    assert {g.M for g in gm} >= {24, 32} and max(g.M for g in gm) <= 32
    att = [op[1][0]._obj for op in b.fwd if op[0] is not None and op[0].__name__ == "vb_attention_fwd"]
    assert att and all(x.q_off and x.k_len and not x.mask for x in att)
    assert eng.plan_builds[(4, 9, 11)] == 2


def test_pack_padding_off_changes_no_launch():
    from vilbert_b200.tasks import packed_rows
    m = _M()
    m.engine.pack_padding = False
    assert packed_rows(m, T.TASK_CFG, "TASK1", T.make_batch(_cfgj(), "TASK1", 4, 11, 9), ()) is None and not m.engine.pack_fallbacks
    eng = Engine(BertConfig.from_dict(_cfgj()), "cpu", _build_only=True)
    p = eng.plan(4, 9, 11, grad_outputs=LOSS_HEADS["vqa"], loss="vqa", score=True, loss_in_forward=True)
    assert p.packed is None and not PACK_OPS & set(_ops(p, "fwd") + _ops(p, "bwd"))
    assert all(op[1][0]._obj.q_off is None for op in p.fwd if op[0] is not None and op[0].__name__ == "vb_attention_fwd")


def test_train_mode_row_indexed_dropout_sites_carry_the_row_map():
    """In a packed train-mode plan every row-indexed dropout site (residual LayerNorms, embedding LayerNorms, the vision_logit
    input) gets its stream's packed-row -> padded-row map, so it draws the padded plan's masks; the attention probabilities and
    the pooled vector keep their own (padded-coordinate / per-sample) indices; a padded plan passes no map."""
    import ctypes as C
    from vilbert_b200 import _lib as L
    eng = Engine(BertConfig.from_dict(_cfgj()), "cpu", _build_only=True)
    kw = dict(grad_outputs=LOSS_HEADS["vlogit_bce"], loss="vlogit_bce", score=True, loss_in_forward=True, outputs=LOSS_HEADS["vlogit_bce"],
              train=True)
    p, q = eng.plan(4, 9, 11, packed=(24, 32), **kw), eng.plan(4, 9, 11, **kw)
    maps = {p.map_t.data_ptr(), p.map_v.data_ptr()}

    def sites(plan):
        out = []
        for fn, args, _ in plan.fwd + plan.bwd:
            if fn is None or fn.__name__.startswith("vb_fuse_pooled"):
                continue
            for a in args:
                if type(a).__name__ == "CArgObject" and isinstance(a._obj, L.Dropout):
                    out.append((fn.__name__, a._obj.row_map))
        return out
    ps = sites(p)
    names = {n for n, _ in ps}
    assert {"vb_add_layernorm_fwd", "vb_add_layernorm_bwd", "vb_layernorm_fwd", "vb_layernorm_bwd", "vb_small_linear_fwd",
            "vb_small_linear_bwd"} <= names
    assert all(m in maps for _, m in ps), [x for x in ps if x[1] not in maps][:3]
    assert {m for _, m in ps} == maps
    assert all(not m for _, m in sites(q))
    att = [a[0]._obj for fn, a, _ in p.fwd if fn is not None and fn.__name__ == "vb_attention_fwd"]
    assert att and all(x.dropout.step and x.q_off for x in att)
    assert C.sizeof(L.DropoutSite) == 16 and C.sizeof(L.Dropout) == 24
