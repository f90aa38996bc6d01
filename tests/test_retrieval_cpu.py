"""Caption-to-image retrieval without a GPU: the metrics and the rank rule against what the reference's evaluate() returned
(tests/golden/retrieval_reference.json, written by tools/make_retrieval_golden.py), the reference's item protocol, the stable
tie / NaN order of vb_retrieval_rank restated in numpy, and the structure of image_prefix and zero-shot scoring plans."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

NT, NV = 9, 11
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden_tool():
    spec = importlib.util.spec_from_file_location("make_retrieval_golden", os.path.join(ROOT, "tools", "make_retrieval_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def stable_desc(s):
    """np.argsort(-s, kind="stable"): the order vb_retrieval_rank works in."""
    return np.argsort(-np.asarray(s, dtype=np.float32), kind="stable")


def key_order(s):
    """The kernel's rule restated: 64-bit keys (float mapped to an order-preserving uint32, -0.0 folded onto +0.0, NaN to 0; low
    word ~column), sorted descending."""
    u = np.asarray(s, dtype=np.float32).view(np.uint32).astype(np.uint64)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    u = np.where(u == 0x80000000, 0, u)
    hi = np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000)
    hi = np.where(nan, 0, hi)
    j = np.arange(len(u), dtype=np.uint64)
    keys = (hi << np.uint64(32)) | ((~j) & np.uint64(0xFFFFFFFF))
    return np.argsort(keys)[::-1]          # the keys are distinct


@pytest.mark.parametrize("zero_shot", [False, True])
def test_metrics_reproduce_the_reference(golden_dir, zero_shot):
    from vilbert_b200.retrieval import retrieval_metrics
    g = json.load(open(os.path.join(golden_dir, "retrieval_reference.json")))
    case = next(c for c in g["cases"] if c["zero_shot"] == zero_shot)
    scores, _ = _golden_tool().seeded_scores(case["seed"], zero_shot)
    assert scores[0, :4].tolist() == case["scores_row0_head"]
    target = np.arange(g["captions"]) // g["captions_per_image"]
    ranks = np.array([int(np.where(stable_desc(row) == t)[0][0]) for row, t in zip(scores.astype(np.float32), target)])
    assert list(retrieval_metrics(ranks)) == case["metrics"]
    assert list(retrieval_metrics(torch.from_numpy(ranks).int())) == case["metrics"]
    with pytest.raises(IndexError):
        retrieval_metrics(np.concatenate([ranks, [-1]]))


def test_stable_order_ties_nans_and_signed_zeros():
    rng = np.random.default_rng(0)
    rows = [np.array([1.0, np.nan, 1.0, -0.0, 0.0, np.nan, -np.inf, np.inf, 1e-45, -1e-45, 0.0], np.float32),
            np.full(7, np.nan, np.float32), np.zeros(5, np.float32), np.array([-0.0, 0.0, -0.0], np.float32),
            rng.integers(-3, 4, 500).astype(np.float32)]
    r = rng.normal(size=1000).astype(np.float32)
    r[rng.integers(0, 1000, 50)] = np.nan
    rows.append(r)
    for s in rows:
        assert np.array_equal(key_order(s), stable_desc(s)), s[:12]


class _FakeDataset:
    """The reference's RetreivalDatasetVal item layout over a gallery of 2H images and C captions (caption c -> image img[c])."""

    def __init__(self, C, H, img, Nv=3, Nt=4, F=2048):
        g = torch.Generator().manual_seed(3)
        self.H, self.img = H, img
        self.feat = torch.rand(2 * H, Nv, F, generator=g)
        self.loc = torch.rand(2 * H, Nv, 5, generator=g)
        self.mask = torch.ones(2 * H, Nv, dtype=torch.long)
        self.cap = torch.randint(0, 100, (C, Nt), generator=g)

    def __len__(self):
        return 2 * len(self.cap)

    def __getitem__(self, i):
        c, h = i // 2, i % 2
        sl = slice(h * self.H, (h + 1) * self.H)
        target = torch.zeros(self.H)
        for t in self.img[c]:
            if h * self.H <= t < (h + 1) * self.H:
                target[t - h * self.H] = 1
        return (self.feat[sl], self.loc[sl], self.mask[sl], self.cap[c], torch.ones_like(self.cap[c]), torch.zeros_like(self.cap[c]),
                target, c, h)


def test_item_protocol_reader():
    from vilbert_b200.retrieval import read_retrieval_dataset
    ds = _FakeDataset(4, 3, [[0], [5], [4, 1], [3]])
    f, s, m, cap, im, seg, tgt = read_retrieval_dataset(ds)
    assert torch.equal(f, ds.feat) and torch.equal(s, ds.loc) and torch.equal(m, ds.mask)
    assert torch.equal(cap, ds.cap) and cap.dtype == torch.int64 and im.shape == cap.shape and seg.shape == cap.shape
    assert tgt.tolist() == [0, 5, 1, 3]          # the first image with target 1
    with pytest.raises(IndexError):
        read_retrieval_dataset(_FakeDataset(2, 3, [[0], []]))


def _engine(golden_dir, heads="vl", **over):
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    cfg = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over)
    return Engine(BertConfig.from_dict(cfg), "cpu", heads=heads, _build_only=True)


def _names(ops):
    return [fn.__name__ for fn, _, _ in ops if fn is not None]


@pytest.mark.parametrize("arena", [False, True])
def test_image_prefix_plan_structure(golden_dir, arena):
    eng = _engine(golden_dir, task_specific_tokens=True)
    if arena:
        eng.enable_activation_arena(64 << 20)
    kw = dict(outputs=("vil_logit",), fast_mode=True)
    plan = eng.plan(4, NT, NV, image_prefix=True, **kw)
    ordinary = eng.plan(4, NT, NV, **kw)
    assert plan is not ordinary and eng.plan(4, NT, NV, image_prefix=True, **kw) is plan
    assert plan.fast and plan.Bt == 1
    assert _names(plan.prefix) == ["vb_mask_to_additive", "vb_cast_f32_to_bf16", "vb_loc_proj_fwd", "vb_gemm_bf16", "vb_layernorm_fwd"]
    assert all(sid == 0 for _, _, sid in plan.prefix)
    # the forward is the ordinary one without those five launches
    full = _names(ordinary.fwd)
    for n in _names(plan.prefix):
        full.remove(n)
    assert _names(plan.fwd) == full
    # the image states are private buffers, and no forward launch is handed one of them as a non-input pointer other than reads
    states = [t for t in plan.image_states if t is not None]
    for t in states:
        assert any(t is k for k in plan._keep)
        if arena:
            assert t.untyped_storage().data_ptr() != eng.arena.untyped_storage().data_ptr()
    ln = plan.prefix[-1][1]
    assert ln[5] == states[0].data_ptr() and ln[6] == states[1].data_ptr()


def test_image_prefix_build_errors(golden_dir):
    eng = _engine(golden_dir)
    with pytest.raises(ValueError, match="forward-only"):
        eng.plan(4, NT, NV, train=True, image_prefix=True)
    with pytest.raises(ValueError, match="forward-only"):
        eng.plan(4, NT, NV, grad_outputs=("vil_logit",), image_prefix=True)
    with pytest.raises(ValueError, match="in_batch_pairs"):
        _engine(golden_dir, in_batch_pairs=True).plan(4, NT, NV, image_prefix=True)
    plan = eng.plan(4, NT, NV, outputs=("vil_logit",), fast_mode=True, image_prefix=True)
    with pytest.raises(ValueError, match="load_images"):
        plan.load_inputs(torch.zeros(1, NT, dtype=torch.long), torch.zeros(4, NV, 2048), torch.zeros(4, NV, 5))
    with pytest.raises(ValueError, match="image_prefix"):
        eng.plan(4, NT, NV).run_image_prefix()


def test_zero_shot_plan_builds_only_the_alignment_head(golden_dir):
    eng = _engine(golden_dir, heads="pretraining")
    plan = eng.plan(4, NT, NV, outputs=("seq_relationship_score",), fast_mode=True, image_prefix=True)
    assert list(plan.outputs)[-1] == "seq_relationship_score" and "linguisic_prediction" not in plan.outputs
    assert "vision_prediction" not in plan.outputs
    c = eng.cfg
    ns = [args[0]._obj.N for fn, args, _ in plan.fwd + plan.prefix if fn is not None and fn.__name__ == "vb_gemm_bf16"]
    assert not {c.vocab_size, c.v_target_size} & set(ns)
    with pytest.raises(ValueError, match="heads='vl'"):
        eng.plan(4, NT, NV, outputs=("vil_logit",))
    with pytest.raises(ValueError, match="misses"):         # the pre-training objective reads all three heads
        eng.plan(4, NT, NV, loss="pretraining", loss_in_forward=True, outputs=("seq_relationship_score",))
    assert _engine(golden_dir, heads="pretraining").plan(4, NT, NV, outputs=("linguisic_prediction", "vision_prediction",
                                                                               "seq_relationship_score")) is not None


def test_evaluator_refusals_without_a_gpu():
    from vilbert_b200.retrieval import RetrievalEvaluator

    class M:
        _heads = "none"
        training = False
    with pytest.raises(TypeError):
        RetrievalEvaluator(M(), torch.zeros(2, 3, 8), torch.zeros(2, 3, 5), torch.ones(2, 3))
    M._heads, M.training = "vl", True
    with pytest.raises(ValueError, match="eval"):
        RetrievalEvaluator(M(), torch.zeros(2, 3, 8), torch.zeros(2, 3, 5), torch.ones(2, 3))
