"""Input gradients (Plan(input_grads=...); `features.grad` / `spatials.grad` on the module surface), checked without a GPU: the
oracles against the reference's fixtures, the launch lists of CPU-built plans, and the refusals."""
import json
import os
import re
import sys
import types

import pytest
import torch

from oracle import basebert_oracle as BO
from oracle import vilbert_oracle as O
from vilbert_b200 import _lib as L
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import BASE_HEAD_NAMES, INPUT_GRAD_NAMES, LOSS_HEADS, Engine
from vilbert_b200.modeling import BertPreTrainedModel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_input_grad_golden as MG  # noqa: E402
import plan_dump as PD  # noqa: E402

NT, NV = 9, 11
BOTH = frozenset(INPUT_GRAD_NAMES)
TRAIN = dict(grad_outputs=O.HEAD_NAMES, train=True)


def _fixture(golden_dir):
    meta = json.load(open(os.path.join(golden_dir, "tiny_input_grads.json")))
    return meta["cases"], torch.load(os.path.join(golden_dir, "tiny_input_grads.pt"))


def oracle_input_grads(name, meta, device="cpu"):
    """(d input_imgs, d image_loc) of a fixture case from the fp32 oracle (None where the input gets no gradient)."""
    if meta["kind"] == "baseline":
        cfg = O.make_config(meta["config"])
        P = BO.synth_params(cfg, meta["num_labels"], meta["seed"], device=device)
        inp = BO.synth_inputs(cfg, meta["B"], meta["Nt"], meta["Nv"], meta["input_seed"], device=device)
        R = BO.probe_weights(meta["B"], meta["Nt"], meta["Nv"], meta["num_labels"], cfg["vocab_size"], meta["probe_seed"], device=device)
        fn = lambda a: (lambda o: sum((o[k] * R[k]).sum() for k in BO.OUT_NAMES))(BO.base_bert_for_vl_tasks(P, cfg, *a))
    elif meta["kind"] == "pretraining":
        cfg = O.make_config(meta["config"])
        P = O.synth_params(cfg, seed=meta["seed"], with_task_heads=False, device=device)
        inp = O.synth_inputs(cfg, meta["B"], meta["Nv"], meta["Nt"], seed=meta["input_seed"], device=device)
        labels = tuple(t.to(device) for t in MG.pretraining_targets(cfg, meta["B"], meta["Nv"], meta["Nt"]))
        fn = lambda a: sum(w * x.sum() for w, x in zip(meta["loss_weights"], O.pretraining_losses(P, cfg, *a, *labels)))
    else:
        cfg = O.make_config(meta["config"])
        P = O.synth_params(cfg, seed=meta["seed"], device=device)
        inp = O.synth_inputs(cfg, meta["B"], meta["Nv"], meta["Nt"], seed=meta["input_seed"], device=device)
        drop = O.DropMasks(meta["train_step"], head_p=meta["head_dropout_prob"]) if meta["train_step"] is not None else None
        if meta["objective"] == "bert":
            fn = lambda a: MG.bert_objective(O.bert_model(P, cfg, *a, drop=drop))
        else:
            fn = lambda a: MG.heads_objective(O.vilbert_for_vl_tasks(P, cfg, *a, task_ids=inp["task_ids"], drop=drop)[1], meta["B"])
    feat = inp["input_imgs"].clone().requires_grad_(True)
    loc = inp["image_loc"].clone().requires_grad_(True)
    obj = fn((inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"]))
    if obj.requires_grad:
        obj.backward()
    return feat.grad, loc.grad


def _cfg(golden_dir, **over):
    return BertConfig.from_dict(dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over))


def _base_engine(golden_dir, **kw):
    tb = json.load(open(os.path.join(golden_dir, "tiny_basebert.json")))
    return Engine(BertConfig.from_dict(tb["config"]), "cpu", heads="base", _build_only=True, num_labels=tb["num_labels"], **kw)


def _names(ops):
    return [(fn.__name__ if fn is not None else ("MARK",) + tuple(args), sid) for fn, args, sid in ops]


# ------------------------------------------------------------------------------------------ oracle vs the reference's fixtures
@pytest.mark.parametrize("name", ["eval", "train", "tasktok_odd_b3", "in_batch_pairs", "dynamic_attention", "fixed_v_layer", "pretraining",
                                  "baseline"])
def test_oracle_input_grads_match_reference_fixture(golden_dir, name):
    cases, tensors = _fixture(golden_dir)
    meta, want = cases[name], tensors[name]
    got = oracle_input_grads(name, meta)
    for what, g in zip(INPUT_GRAD_NAMES, got):
        w = want[what]
        assert (g is None) == (w is None), (name, what)
        if w is None:
            continue
        if isinstance(w, dict):
            assert max(BO.digest_errors(g, w)) < 1e-5, (name, what)
        else:
            assert g.shape == w.shape and ((g - w).abs().max() / w.abs().max()).item() < 1e-5, (name, what)
            assert w.abs().max() > 0


def test_fixed_v_layer_gives_no_input_gradient(golden_dir):
    """fixed_v_layer: the first image layer runs under no_grad ahead of the first connection layer, so nothing below it gets a
    gradient. The plan differentiates neither input and adds no launch to the plain plan's backward."""
    cases, tensors = _fixture(golden_dir)
    assert tensors["fixed_v_layer"]["input_imgs"] is None and tensors["fixed_v_layer"]["image_loc"] is None
    over = {k: v for k, v in cases["fixed_v_layer"]["config"].items() if k in ("fixed_v_layer", "v_biattention_id", "t_biattention_id")}
    plain = Engine(_cfg(golden_dir, **over), "cpu", _build_only=True).plan(4, NT, NV, **TRAIN)
    plan = Engine(_cfg(golden_dir, **over), "cpu", _build_only=True).plan(4, NT, NV, input_grads=BOTH, **TRAIN)
    assert plan.input_grad == {}
    assert _names(plan.bwd) == _names(plain.bwd)


# ------------------------------------------------------------------------------------------ launch lists
def _extra_ops(plain, plan):
    """The backward ops of `plan` beyond those of `plain`, checking that removing them leaves the plain plan's list."""
    a, b = _names(plain.bwd), _names(plan.bwd)
    extra = [i for i, (fn, args, sid) in enumerate(plan.bwd) if fn is not None and fn.__name__ == "vb_loc_proj_dx"]
    assert len(extra) == 1
    gemm = [i for i, (fn, args, sid) in enumerate(plan.bwd)
            if fn is not None and fn.__name__ == "vb_gemm_bf16" and args[0]._obj.out_f32 == plan.input_grad["input_imgs"].data_ptr()]
    assert len(gemm) == 1
    rest = [x for i, x in enumerate(b) if i not in (extra[0], gemm[0])]
    assert rest == a
    return plan.bwd[gemm[0]], plan.bwd[extra[0]]


def _outside_arena(eng, t):
    a = eng.arena
    lo, hi = a.data_ptr(), a.data_ptr() + a.numel()
    return not (lo <= t.data_ptr() < hi)


@pytest.mark.parametrize("kind", ["two_stream", "in_batch_pairs", "baseline", "pretraining"])
def test_input_grad_plan_adds_exactly_two_launches(golden_dir, kind):
    """All parameters trainable: the input-gradient plan's backward is the plain plan's plus the feature dgrad GEMM and
    vb_loc_proj_dx; its gradient buffers are private (outside the activation arena) and outside grad_touch."""
    def build(**extra):
        if kind == "baseline":
            eng = _base_engine(golden_dir)
            eng.enable_activation_arena(64 << 20)
            return eng, eng.plan(3, NT, NV, grad_outputs=BASE_HEAD_NAMES, train=True, **extra)
        cfg = _cfg(golden_dir, in_batch_pairs=kind == "in_batch_pairs")
        eng = Engine(cfg, "cpu", heads="pretraining" if kind == "pretraining" else "vl", _build_only=True)
        eng.enable_activation_arena(64 << 20)
        if kind == "pretraining":
            return eng, eng.plan(4, NT, NV, grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining", loss_in_forward=True, train=True,
                                 **extra)
        return eng, eng.plan(4, NT, NV, **TRAIN, **extra)
    _, plain = build()
    eng, plan = build(input_grads=BOTH)
    gemm, dx = _extra_ops(plain, plan)
    B = 3 if kind == "baseline" else 4
    Fv = plan.in_feat.shape[-1]
    g = gemm[1][0]._obj
    assert (g.M, g.N, g.b_mn_major, g.atomic_out, g.residual) == (B * NV, Fv, 1, 0, None)
    assert dx[1].dx == plan.input_grad["image_loc"].data_ptr() and dx[1].M == B * NV
    assert tuple(plan.input_grad["input_imgs"].shape) == (B * NV, Fv) and tuple(plan.input_grad["image_loc"].shape) == (B * NV, 5)
    for t in plan.input_grad.values():
        assert _outside_arena(eng, t)
    assert set(plan.grad_touch) == set(plain.grad_touch)
    assert _names(plan.fwd) == _names(plain.fwd)


@pytest.mark.parametrize("kind", ["two_stream", "baseline"])
def test_all_frozen_input_grad_plan_writes_no_parameter_gradient(golden_dir, kind):
    """Every parameter frozen, only the inputs differentiated (the saliency setup): the outputs carry a gradient, the backward
    computes the input gradients and touches nothing of the flat gradient buffer."""
    if kind == "baseline":
        eng = _base_engine(golden_dir)
        plan = eng.plan(3, NT, NV, grad_outputs=("vil_prediction",), frozen=frozenset(eng.ps.entries), input_grads=BOTH)
    else:
        eng = Engine(_cfg(golden_dir), "cpu", _build_only=True)
        plan = eng.plan(4, NT, NV, grad_outputs=("vil_prediction",), frozen=frozenset(eng.ps.entries), input_grads=BOTH)
    assert plan.out_rg["vil_prediction"] and set(plan.input_grad) == BOTH
    assert plan.grad_touch == {}
    lines = []
    PD.dump_plan(lines, "plan", plan)
    assert not [x for x in lines if x.startswith("bwd ") and re.search(r"\bgrad\+\d+", x)]
    frozen_only = eng.plan(3 if kind == "baseline" else 4, NT, NV, grad_outputs=("vil_prediction",), frozen=frozenset(eng.ps.entries))
    assert not frozen_only.out_rg["vil_prediction"]


# ------------------------------------------------------------------------------------------ refusals and defaults
def test_inference_plans_refuse_input_grads(golden_dir):
    eng = Engine(_cfg(golden_dir), "cpu", _build_only=True)
    with pytest.raises(ValueError):
        eng.plan(4, NT, NV, fast_mode=True, input_grads=BOTH)
    with pytest.raises(ValueError):
        eng.plan(4, NT, NV, outputs=("vil_logit",), fast_mode=True, image_prefix=True, input_grads=frozenset({"input_imgs"}))
    with pytest.raises(ValueError):
        eng.plan(4, NT, NV, input_grads=frozenset({"input_txt"}))


def test_retrieval_evaluator_refuses_gallery_that_requires_grad():
    from vilbert_b200.retrieval import RetrievalEvaluator
    model = types.SimpleNamespace(_heads="vl", training=False)
    feat, loc, mask = torch.rand(3, 5, 8, requires_grad=True), torch.rand(3, 5, 5), torch.ones(3, 5, dtype=torch.long)
    with pytest.raises(ValueError):
        RetrievalEvaluator(model, feat, loc, mask)
    with torch.no_grad():
        RetrievalEvaluator(model, feat, loc, mask)


def test_which_inputs_a_call_differentiates():
    pick = BertPreTrainedModel._input_grads
    feat, loc = torch.rand(2, 3, 8), torch.rand(2, 3, 5)
    inputs = dict(input_txt=torch.zeros(2, 4, dtype=torch.long), input_imgs=feat, image_loc=loc, attention_mask=None,
                  image_attention_mask=None)
    assert pick(inputs) == frozenset()
    feat.requires_grad_(True)
    assert pick(inputs) == frozenset({"input_imgs"})
    loc.requires_grad_(True)
    assert pick(inputs) == BOTH
    with torch.no_grad():
        assert pick(inputs) == frozenset()
    for k in ("attention_mask", "image_attention_mask"):
        with pytest.raises(NotImplementedError):
            pick(dict(inputs, **{k: torch.ones(2, 3, requires_grad=True)}))
    assert pick(dict(inputs, image_attention_mask=torch.ones(2, 3))) == BOTH


def test_loc_proj_dx_is_exported():
    assert "vb_loc_proj_dx" in L.exported_symbols()
    assert hasattr(L.lib(), "vb_loc_proj_dx")
