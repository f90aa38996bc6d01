"""The fused pre-training objective without a GPU: structure of Plan(loss="pretraining", loss_in_forward=True), the visual_target
dispatch of the pre-training plans, and the closed forms of the masked-MSE and NCE region objectives against torch autograd."""
import json
import math
import os

import pytest
import torch

import _pretraining_oracle as P

NT, NV = 9, 11
NEW_OPS = {"vb_mse_masked_loss", "vb_nce_region_loss"}
HEADS = ("linguisic_prediction", "vision_prediction", "seq_relationship_score")


def _engine(golden_dir, precision="fp16", **over):
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    cfg = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over)
    if over.get("visual_target", 0):
        cfg["v_target_size"] = cfg["v_feature_size"]          # regression / NCE targets are region features
    return Engine(BertConfig.from_dict(cfg), "cpu", heads="pretraining", _build_only=True, precision=precision)


def _names(ops):
    return [fn.__name__ for fn, _, _ in ops if fn is not None]


def _kernels(ops):
    return [op for op in ops if op[0] is not None]


REGION_FN = {0: "vb_kl_masked_loss", 1: "vb_mse_masked_loss", 2: "vb_nce_region_loss"}


@pytest.mark.parametrize("vt", [0, 1, 2])
def test_three_slot_plan_structure(golden_dir, vt):
    """The objective is the end of the forward, its three kernels write the three consecutive slots of objective_out, and the backward
    starts by scaling each stored head gradient by its own slot of loss_grad (the compacted masked-LM gradient is then cast into its
    bf16 operand)."""
    eng = _engine(golden_dir, visual_target=vt)
    plan = eng.plan(4, NT, NV, grad_outputs=HEADS, train=True, loss="pretraining", loss_in_forward=True)
    f = _kernels(plan.fwd)
    out = plan.objective_out
    assert plan.loss is None and tuple(out.shape) == (3,) and tuple(plan.loss_grad.shape) == (3,)
    assert plan.loss_grad.tolist() == [1.0, 1.0, 1.0]
    lm, cap, region, ns = f[-4:]
    assert [op[0].__name__ for op in (lm, cap, region, ns)] == ["vb_ce_loss", "vb_scatter_rows_f32", REGION_FN[vt], "vb_ce_loss"]
    assert lm[1].loss == out.data_ptr() and cap[1].poison == out.data_ptr()      # the capacity check poisons the masked-LM slot
    assert region[1].loss == out.data_ptr() + 4 and ns[1].loss == out.data_ptr() + 8
    b = _kernels(plan.bwd)
    assert [op[0].__name__ for op in b[:4]] == ["vb_scale_by_device", "vb_cast2d_f32_to_bf16", "vb_scale_by_device", "vb_scale_by_device"]
    lg = plan.loss_grad.data_ptr()
    assert (b[0][1].scale, b[2][1].scale, b[3][1].scale) == (lg, lg + 4, lg + 8)
    assert b[0][1].src == plan.head_grad["linguisic_prediction"].data_ptr() and b[0][1].dst == plan.lm_c["dl32"].data_ptr()
    assert b[1][1].dst == plan.lm_c["dl16"].data_ptr()
    assert b[2][1].dst == plan.gout["vision_prediction"].data_ptr() and b[3][1].dst == plan.gout["seq_relationship_score"].data_ptr()
    # the objective is computed in the forward only
    assert not {REGION_FN[vt], "vb_ce_loss"} & set(_names(plan.bwd))


@pytest.mark.parametrize("vt", [0, 1, 2])
def test_eval_plan_has_no_backward_and_writes_no_gradient(golden_dir, vt):
    eng = _engine(golden_dir, visual_target=vt)
    plan = eng.plan(4, NT, NV, loss="pretraining", loss_in_forward=True)
    assert _names(plan.bwd) == [] and not plan.head_grad
    lm, cap, region, ns = _kernels(plan.fwd)[-4:]
    assert lm[1].dlogits_f32 is None and lm[1].dlogits_bf16 is None and ns[1].dlogits_f32 is None    # CE: no f32 / bf16 gradient
    assert region[1].dscores_f32 is None


def test_new_inputs_and_loss_grad_are_private(golden_dir):
    eng = _engine(golden_dir, visual_target=2)
    eng.enable_activation_arena(64 << 20)
    p = eng.plan(4, NT, NV, grad_outputs=HEADS, train=True, loss="pretraining", loss_in_forward=True)
    assert p.arena_bytes > 0
    a0, a1 = eng.arena.data_ptr(), eng.arena.data_ptr() + eng.arena.numel()
    for t in (p.objective_out, p.loss_grad, *p.loss_inputs.values(), *p.head_grad.values()):
        assert not (a0 <= t.data_ptr() < a1)
    assert set(p.loss_inputs) == {"masked_lm_labels", "image_target", "image_label", "next_sentence_label", "neg_index"}


def test_score_is_refused(golden_dir):
    eng = _engine(golden_dir)
    with pytest.raises(ValueError):
        eng.plan(4, NT, NV, loss="pretraining", score=True, loss_in_forward=True)
    with pytest.raises(ValueError):
        eng.plan(4, NT, NV, loss="pretraining", score=True)


@pytest.mark.parametrize("loss_in_forward", [False, True])
@pytest.mark.parametrize("vt", [1, 2])
def test_visual_target_dispatch(golden_dir, vt, loss_in_forward):
    """visual_target 1 / 2 emit their own region kernel, never the KL (which the summed plan used to emit for every visual_target)."""
    eng = _engine(golden_dir, visual_target=vt, num_negative=255)
    plan = eng.plan(4, NT, NV, grad_outputs=HEADS, train=True, loss="pretraining", loss_in_forward=loss_in_forward)
    names = _names(plan.fwd + plan.bwd)
    assert REGION_FN[vt] in names and "vb_kl_masked_loss" not in names and not (NEW_OPS - {REGION_FN[vt]}) & set(names)
    if vt == 2:
        assert tuple(plan.loss_inputs["neg_index"].shape) == (4, NV - 1, 254) and plan.loss_inputs["neg_index"].dtype == torch.int64
    else:
        assert "neg_index" not in plan.loss_inputs


def test_plan_key_separates_visual_target_and_negatives(golden_dir):
    eng = _engine(golden_dir, visual_target=2, num_negative=128)
    kw = dict(grad_outputs=HEADS, train=True, loss="pretraining", loss_in_forward=True)
    p = eng.plan(4, NT, NV, **kw)
    assert p.loss_inputs["neg_index"].shape[2] == 127 and eng.plan(4, NT, NV, **kw) is p
    eng.cfg.num_negative = 255
    q = eng.plan(4, NT, NV, **kw)
    assert q is not p and q.loss_inputs["neg_index"].shape[2] == 254
    eng.cfg.visual_target = 1
    r = eng.plan(4, NT, NV, **kw)
    assert r is not q and "vb_mse_masked_loss" in _names(r.fwd)


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_plans_without_the_new_option_launch_no_new_op(golden_dir, precision):
    from oracle import vilbert_oracle as O
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine, LOSS_HEADS
    eng = _engine(golden_dir, precision)
    vl = Engine(BertConfig.from_dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]), "cpu", _build_only=True,
                precision=precision)
    plans = [eng.plan(4, NT, NV, grad_outputs=HEADS, loss="pretraining", train=True), eng.plan(4, NT, NV, grad_outputs=HEADS, train=True),
             vl.plan(4, NT, NV, grad_outputs=O.HEAD_NAMES, train=True)]
    plans += [vl.plan(4, NT, NV, grad_outputs=LOSS_HEADS[k], loss=k, train=True, score=True, loss_in_forward=True) for k in ("vqa", "logit_ce")]
    for p in plans:
        p.enable_training_prologue()
        assert not NEW_OPS & set(_names(p.prologue + p.fwd + p.bwd))
    summed = plans[0]
    assert summed.loss is not None and not summed.head_grad and "vb_scale_by_device" not in _names(summed.bwd)


# ------------------------------------------------------------------------------------------ closed forms vs autograd (float64)
def _region_case(B, Nv, D, frac, seed):
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(B, Nv, D, generator=g, dtype=torch.float64)
    t = torch.randn(B, Nv - 1, D, generator=g, dtype=torch.float64)
    lab = torch.where(torch.rand(B, Nv - 1, generator=g) < frac, 1, -1)
    lab[0, 0] = 1 if frac > 0 else -1
    lab[1, 2] = 0 if B > 1 else lab[1 % B, 2]            # label 0 is not masked either
    return s, t, lab, g


@pytest.mark.parametrize("frac", [0.0, 0.15, 1.0])
def test_mse_closed_form_matches_autograd(frac):
    s, t, lab, _ = _region_case(3, 7, 16, frac, 1)
    sa = s.clone().requires_grad_(True)
    ref = P.mse_reference(sa, t, lab)
    ref.backward()
    loss, d = P.mse_closed_form(s, t, lab)
    assert abs(loss.item() - ref.item()) <= 1e-12 * max(1.0, abs(ref.item()))
    assert torch.allclose(d, sa.grad, rtol=1e-12, atol=1e-15)
    if frac == 0.0:
        assert loss.item() == 0.0 and d.abs().max() == 0        # max(n * D, 1): 0, not NaN
    assert d[:, 0].abs().max() == 0


@pytest.mark.parametrize("frac,n", [(0.15, 7), (1.0, 12)])
def test_nce_closed_form_matches_autograd_with_duplicates(frac, n):
    B, Nv, D = 3, 6, 8
    s, t, lab, g = _region_case(B, Nv, D, frac, 2)
    R = Nv - 1
    neg = torch.randint(0, B * R, (B, R, n), generator=g)
    neg[0, 0, :3] = neg[0, 0, 0]                           # duplicates
    neg[0, 0, 3] = 0                                       # the positive's own row as a negative
    sa = s.clone().requires_grad_(True)
    ref = P.nce_reference(sa, t, lab, neg)
    ref.backward()
    loss, d = P.nce_closed_form(s, t, lab, neg)
    assert abs(loss.item() - ref.item()) <= 1e-12 * abs(ref.item())
    assert torch.allclose(d, sa.grad, rtol=1e-10, atol=1e-14)


def test_nce_closed_form_edges():
    s, t, lab, g = _region_case(2, 5, 4, 0.0, 3)
    neg = torch.zeros(2, 4, 3, dtype=torch.long)
    loss, d = P.nce_closed_form(s, t, torch.full_like(lab, -1), neg)
    assert math.isnan(loss.item()) and d.abs().max() == 0        # F.cross_entropy over no rows
    lab = torch.full_like(lab, -1); lab[1, 2] = 1
    neg[1, 2, 1] = 8                                             # B * R: out of range
    loss, d = P.nce_closed_form(s, t, lab, neg)
    assert math.isnan(loss.item()) and torch.isfinite(d).all()
    assert P.negative_count(128) == 127 and P.negative_count(255) == 254
