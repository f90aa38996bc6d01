"""Gradient-norm clipping and non-finite step skipping of the fused optimizers (`max_grad_norm=`) on the GPU: the norm kernel
against a float64 norm, the clipped steps against torch.nn.utils.clip_grad_norm_ + the unclipped fused step and against the
float64 restatements (tests/_clip_oracle.py with oracle/adamw_oracle.py and tests/_radam_oracle.py), skipped steps, frozen
parameters and captured plan steps."""
import json
import os

import numpy as np
import pytest
import torch

import _clip_oracle as CO
import _radam_oracle as RO
from oracle import adamw_oracle as AO
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu


def _tiny_model(golden_dir, precision="fp16"):
    import vilbert_b200
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    cfg = O.make_config(cfgj)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1, precision=precision)
    model.load_state_dict(O.synth_params(cfg, seed=0, device="cuda"), strict=True)
    return model, cfg


def _make_opt(kind, model, **kw):
    from vilbert_b200.optim import FusedAdamW, FusedRAdam
    groups = AO.reference_param_groups(model.named_parameters(), base_lr=1e-3)
    if kind == "adamw":
        return FusedAdamW(groups, lr=1e-3, correct_bias=False, model=model, **kw)
    return FusedRAdam(groups, lr=1e-3, model=model, **kw)


def _fill_grad(eng, seed, scale=1e-2):
    eng.ps.grad.copy_(torch.randn(eng.ps.numel, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed)) * scale)


def _elem(model, name="bert.encoder.layer.0.attention.self.query.weight", k=5):
    """Flat index of element k of a parameter (padding between tensors belongs to none)."""
    p = dict(model.named_parameters())[name]
    return (p.data_ptr() - model.engine.ps.flat.data_ptr()) // 4 + k


def _trainable_grads(model):
    return [p.grad.detach() for p in model.parameters() if p.requires_grad]


def _rel(a, b, floor):
    return ((a.double() - b.double()).abs().max() / max(b.abs().max().item(), floor)).item()


def _f32(x):
    return float(np.float32(x))


def _state(opt):
    ps = opt.engine.ps
    return [t.clone() for t in (ps.flat, opt.exp_avg, opt.exp_avg_sq, ps.shadow, ps.shadow_b, opt._step_dev)]


# ---------------------------------------------------------------------------------------------------- the norm
@pytest.mark.parametrize("chunk", [32768, 1024])
@pytest.mark.parametrize("grad_scale", [1.0, 0.25])
def test_norm_matches_float64_and_is_bitwise_reproducible(golden_dir, chunk, grad_scale):
    """grad_norm = ||grad_scale g||_2 over the trainable tensors (tied decoder once) to 1e-6 relative; repeated launches and a
    CUDA-graph replay of the same launch give the same bits."""
    model, _ = _tiny_model(golden_dir)
    opt = _make_opt("adamw", model, zero_grad=False, chunk=chunk, max_grad_norm=1e9)
    opt.grad_scale = grad_scale
    eng = model.engine
    _fill_grad(eng, 3)
    ref = CO.global_norm(_trainable_grads(model), grad_scale)
    opt.launch()
    torch.cuda.synchronize()
    first = opt.grad_norm.clone()
    assert abs(first.item() - ref) <= 1e-6 * ref, (first.item(), ref)
    assert opt._clip_record[1].view(torch.float32).item() == 1.0 and opt.skipped_steps.item() == 0
    for _ in range(3):
        opt.launch()
        torch.cuda.synchronize()
        assert torch.equal(opt.grad_norm, first)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        opt.launch()
    opt._clip_record[0] = 0
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(opt.grad_norm, first)


# ---------------------------------------------------------------------------------------------------- clipped steps
def _clipped_step_case(golden_dir, kind, ratio):
    """FusedX(max_grad_norm=c) == clip_grad_norm_(c) over the trainable parameters followed by FusedX(), with c below (ratio 0.3:
    clipped) and above (3.0: coefficient 1) the norm, over four steps with the reference grouping; both match the float64
    restatement, which takes the betas as the Python floats the user passes (the kernels use fp32(1 - beta), as the reference's
    fp32 torch ops do)."""
    model_a, _ = _tiny_model(golden_dir)
    model_b, _ = _tiny_model(golden_dir)
    _fill_grad(model_a.engine, 10)
    c = ratio * CO.global_norm(_trainable_grads(model_a))
    opt_a = _make_opt(kind, model_a, max_grad_norm=c)
    opt_b = _make_opt(kind, model_b)
    named = list(model_b.named_parameters())
    groups = AO.reference_param_groups(named, base_lr=1e-3)
    ref = [p.detach().clone().double() for _, p in named]
    mom = [(torch.zeros_like(r), torch.zeros_like(r)) for r in ref]
    ora = RO.RAdamOracle([dict(gr, params=[torch.nn.Parameter(r)], lr=_f32(gr["lr"])) for gr, r in zip(groups, ref)], lr=_f32(1e-3),
                         betas=(0.9, 0.999), eps=_f32(1e-8)) if kind == "radam" else None
    for t in range(1, 5):
        for m in (model_a, model_b):
            _fill_grad(m.engine, 10 + t)
        grads = [p.grad.detach().clone() for _, p in named]
        opt_a.step()
        total = torch.nn.utils.clip_grad_norm_([p for _, p in named], c)
        opt_b.step()
        torch.cuda.synchronize()
        assert abs(opt_a.grad_norm.item() - total.item()) <= 1e-6 * total.item()
        cg = CO.clipped_grads(grads, c)
        if kind == "adamw":
            for r, (m1, m2), g, gr in zip(ref, mom, cg, groups):
                AO.adamw_step(r, g, m1, m2, t, _f32(gr["lr"]), beta1=0.9, beta2=0.999, eps=_f32(1e-6),
                              weight_decay=_f32(gr["weight_decay"]), correct_bias=False)
        else:
            for grp, g in zip(ora.param_groups, cg):
                grp["params"][0].grad = g
            ora.step()
    assert opt_a.skipped_steps.item() == 0 and opt_a.state_dict()["state"][0]["step"] == 4
    for (k, pa), (_, pb), r in zip(model_a.named_parameters(), named, ref):
        assert _rel(pa.detach(), pb.detach(), 1e-6) < 1e-6, k
        assert _rel(pa.detach(), r, 1e-6) < 2e-6, k
    ps = model_a.engine.ps
    assert torch.equal(ps.shadow, ps.flat.to(ps.op_dtype)) and model_a.engine.grad_clean and model_a.engine.shadow_clean


@pytest.mark.parametrize("kind", ["radam"])
@pytest.mark.parametrize("ratio", [0.3, 3.0])
def test_clipped_step_matches_torch_clip_then_fused_step(golden_dir, kind, ratio):
    _clipped_step_case(golden_dir, kind, ratio)


@pytest.mark.parametrize("ratio", [0.3, 3.0])
def test_clipped_adamw_step_matches_clip_then_step_with_python_betas(golden_dir, ratio):
    """AdamW's float64 restatement with betas (0.9, 0.999), not their fp32 neighbours: with fp32 betas it would form
    1 - fp32(0.999) = 0.00099998713 and sit 6e-6 relative off every update of a step from fresh moments."""
    _clipped_step_case(golden_dir, "adamw", ratio)


# ---------------------------------------------------------------------------------------------------- skipped steps
@pytest.mark.parametrize("kind", ["adamw", "radam"])
@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
def test_non_finite_gradient_skips_the_step(golden_dir, kind, bad):
    """One NaN / inf gradient element: p, m, v, both 16-bit copies, the device step counter and state_dict()["step"] stay as they
    were, skipped_steps is 1 and the gradient is zeroed. The finite steps after it end bitwise equal to a run that never saw
    the bad step."""
    model_a, _ = _tiny_model(golden_dir)
    model_b, _ = _tiny_model(golden_dir)
    opt_a = _make_opt(kind, model_a, max_grad_norm=1.0)
    opt_b = _make_opt(kind, model_b, max_grad_norm=1.0)
    for t in (1, 2):
        for m, o in ((model_a, opt_a), (model_b, opt_b)):
            _fill_grad(m.engine, 20 + t)
            o.step()
    torch.cuda.synchronize()
    before = _state(opt_a)
    step_before = opt_a.state_dict()["state"][0]["step"]
    _fill_grad(model_a.engine, 99)
    model_a.engine.ps.grad[_elem(model_a)] = bad
    opt_a.step()
    torch.cuda.synchronize()
    assert opt_a.skipped_steps.item() == 1 and not np.isfinite(opt_a.grad_norm.item())
    for x, y in zip(before, _state(opt_a)):
        assert torch.equal(x, y)
    assert opt_a.state_dict()["state"][0]["step"] == step_before == 2
    # every parameter's gradient is zeroed (padding between tensors belongs to none and is not touched)
    assert all(p.grad.abs().max().item() == 0 for p in model_a.parameters())
    assert model_a.engine.grad_clean and model_a.engine.shadow_clean
    for t in (3, 4, 5, 6, 7):             # RAdam crosses the rectification switch at t = 6 on both runs
        for m, o in ((model_a, opt_a), (model_b, opt_b)):
            _fill_grad(m.engine, 20 + t)
            o.step()
    torch.cuda.synchronize()
    for x, y in zip(_state(opt_a), _state(opt_b)):
        assert torch.equal(x, y)
    assert opt_a.state_dict()["state"][0]["step"] == 7 and opt_b.skipped_steps.item() == 0


def test_inf_max_grad_norm_skips_without_clipping(golden_dir):
    """max_grad_norm=inf: finite steps are bitwise the unclipped FusedAdamW's, a non-finite one is skipped."""
    model_a, _ = _tiny_model(golden_dir)
    model_b, _ = _tiny_model(golden_dir)
    opt_a = _make_opt("adamw", model_a, max_grad_norm=float("inf"))
    opt_b = _make_opt("adamw", model_b)
    for t in (1, 2, 3):
        for m, o in ((model_a, opt_a), (model_b, opt_b)):
            _fill_grad(m.engine, 40 + t, scale=10.0)
            if t == 2 and o is opt_a:
                m.engine.ps.grad[_elem(m, "bert.v_embeddings.image_embeddings.bias", 1)] = float("nan")
            if t != 2 or o is opt_a:
                o.step()
    torch.cuda.synchronize()
    assert opt_a.skipped_steps.item() == 1
    for x, y in zip(_state(opt_a), _state(opt_b)):
        assert torch.equal(x, y)


# ---------------------------------------------------------------------------------------------------- frozen parameters
@pytest.mark.parametrize("when", ["before", "after"])
def test_frozen_parameters_are_not_in_the_norm(golden_dir, when):
    """A parameter frozen before the optimizer is built, or after (the chunk table is rebuilt at the next step()), is left out of
    the norm: a NaN in its gradient range neither counts nor skips the step."""
    model, _ = _tiny_model(golden_dir)
    named = dict(model.named_parameters())
    frozen = [named[k] for k in ("bert.embeddings.word_embeddings.weight", "bert.encoder.layer.0.attention.self.query.weight")]
    if when == "before":
        for p in frozen:
            p.requires_grad_(False)
    opt = _make_opt("radam", model, zero_grad=False, max_grad_norm=1.0)
    if when == "after":
        for p in frozen:
            p.requires_grad_(False)
    eng = model.engine
    _fill_grad(eng, 7)
    flat = eng.ps.flat.data_ptr()
    for p in frozen:
        off = (p.data_ptr() - flat) // 4
        eng.ps.grad[off:off + p.numel()] = float("nan")
    trainable = [eng.ps.grad[(p.data_ptr() - flat) // 4:(p.data_ptr() - flat) // 4 + p.numel()] for p in model.parameters() if p.requires_grad]
    ref = CO.global_norm(trainable)
    w = [p.detach().clone() for p in frozen]
    opt.step()
    torch.cuda.synchronize()
    assert opt.skipped_steps.item() == 0 and abs(opt.grad_norm.item() - ref) <= 1e-6 * ref
    assert all(torch.equal(a, p.detach()) for a, p in zip(w, frozen))


# ---------------------------------------------------------------------------------------------------- captured steps
@pytest.mark.parametrize("kind", ["adamw", "radam"])
def test_captured_plan_step_equals_eager_steps_with_a_skip(golden_dir, kind):
    """Plan.enable_optimizer(FusedX(max_grad_norm=c)) captured and replayed 8 times == 8 eager step() calls on the same gradients,
    one of them holding a NaN: weights, moments, copies, step counter, norms and skip count bitwise equal. (The plan has no
    backward, so the gradient buffer is what the test wrote; zero_grad=False keeps it for the next step.)"""
    model, cfg = _tiny_model(golden_dir)
    eng, ps = model.engine, model.engine.ps
    opt = _make_opt(kind, model, zero_grad=False, max_grad_norm=0.05)
    _fill_grad(eng, 5)
    g0, p0 = ps.grad.clone(), ps.flat.clone()
    bad_at, bad_idx = 4, _elem(model, "bert.encoder.c_layer.0.biattention.query1.weight", 7)

    def reset():
        ps.flat.copy_(p0); ps.grad.copy_(g0); opt.exp_avg.zero_(); opt.exp_avg_sq.zero_(); opt._step_dev.zero_()
        opt._clip_record.zero_(); eng.refresh_weights()
        torch.cuda.synchronize()

    def run(step):
        norms = []
        for i in range(8):
            if i == bad_at:
                ps.grad[bad_idx] = float("nan")
            step()
            norms.append(opt.grad_norm.clone())
            if i == bad_at:
                ps.grad[bad_idx] = g0[bad_idx]
        torch.cuda.synchronize()
        return [t.clone() for t in (ps.flat, opt.exp_avg, opt.exp_avg_sq, ps.shadow, ps.shadow_b, opt._step_dev, opt._clip_record)], norms

    reset()
    eager, eager_norms = run(opt.step)
    assert opt.skipped_steps.item() == 1 and opt._step_dev.item() == 7
    reset()
    inp = O.synth_inputs(cfg, 4, 11, 9, seed=1234, device="cuda")
    plan = eng.plan(4, 9, 11)
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    plan.enable_optimizer(opt)
    assert len(plan.epilogue) == 2
    plan.capture()                                    # its warm-up run steps once: start again from the initial state
    reset()
    captured, captured_norms = run(plan.run_step)
    for a, b in zip(eager, captured):
        assert torch.equal(a, b)
    for a, b in zip(eager_norms, captured_norms):
        assert torch.equal(a, b) or (a.isnan().item() and b.isnan().item())
    assert opt.state_dict()["state"][0]["step"] == 7
