"""Fused RAdam (csrc/vb_optim.cu radam_kernel, optim.FusedRAdam) vs the restatement of the reference's RAdam
(tests/_radam_oracle.py, pinned bit-exactly against vilbert/optimization.py by tests/golden/radam_reference_steps.pt)."""
import io
import json
import os

import numpy as np
import pytest
import torch

import _radam_oracle as RO
from oracle import adamw_oracle as AO
from oracle import vilbert_oracle as O


# ---------------------------------------------------------------------------------------------------- CPU: the oracle
def test_oracle_reproduces_the_reference_fixture_bit_exactly(golden_dir):
    gold = torch.load(os.path.join(golden_dir, "radam_reference_steps.pt"))
    ps = [torch.nn.Parameter(p.clone()) for p in gold["params"]]
    opt = RO.RAdamOracle([{"params": [p], "lr": lr, "weight_decay": wd, "betas": b} for p, (lr, wd, b) in zip(ps, gold["hyper"])])
    for t, scale in enumerate(gold["lr_scale"], 1):
        for grp, (lr, _, _) in zip(opt.param_groups, gold["hyper"]):
            grp["lr"] = lr * scale
        for p, g in zip(ps, gold["grads"][t - 1]):
            p.grad = g.clone()
        opt.step()
        for p, ref in zip(ps, gold["trajectory"][t - 1]):
            assert torch.equal(p.detach(), ref), t
    for p, m, v in zip(ps, gold["exp_avg"], gold["exp_avg_sq"]):
        assert torch.equal(opt.state[p]["exp_avg"], m) and torch.equal(opt.state[p]["exp_avg_sq"], v)
        assert opt.state[p]["step"] == len(gold["lr_scale"])


def test_oracle_decay_is_applied_first_on_the_old_weights():
    p = torch.tensor([2.0], dtype=torch.float64); m = torch.zeros_like(p); v = torch.zeros_like(p)
    RO.radam_step(p, torch.tensor([0.5], dtype=torch.float64), m, v, 1, lr=0.1, weight_decay=0.5)
    # t = 1 is unrectified: step_size = lr / (1 - b1) = 1, m = 0.05. Decay first: 2 - 0.1 * 0.5 * 2 = 1.9, then 1.9 - 0.05
    assert abs(p.item() - 1.85) < 1e-12          # decay after the update would give (2 - 0.05) * 0.95 = 1.8525


def test_oracle_rectification_switches_on_at_step_6():
    n = [RO.rectification(t, 1e-3, 0.9, 0.999)[0] for t in range(1, 8)]
    assert all(x < 5 for x in n[:5]) and all(x >= 5 for x in n[5:])
    assert abs(n[4] - 4.996) < 1e-3 and abs(n[5] - 5.994) < 1e-3
    # unrectified steps are un-normalised: p -= lr / (1 - b1^t) * m
    p = torch.zeros(1, dtype=torch.float64); m = torch.zeros_like(p); v = torch.zeros_like(p)
    RO.radam_step(p, torch.tensor([3.0], dtype=torch.float64), m, v, 1, lr=1e-3)
    assert abs(p.item() + 1e-3 / 0.1 * 0.3) < 1e-15
    # rectified at t = 6: normalised by sqrt(v) + eps
    m.fill_(0.3); v.fill_(0.04); p.zero_()
    n6, ss6 = RO.rectification(6, 1e-3, 0.9, 0.999)
    RO.apply_update(p, torch.zeros(1, dtype=torch.float64), m, v, n6, ss6, 1e-3, 0.9, 0.999, 1e-8, 0.0)
    expected = -ss6 * 0.27 / ((0.04 * 0.999) ** 0.5 + 1e-8)
    assert abs(p.item() - expected) < 1e-12 * abs(expected)


def test_oracle_leader_group_lr_drives_every_tensor():
    """The first group's lr / betas set the step size of all tensors; a later group's own lr only reaches its weight decay."""
    a = torch.nn.Parameter(torch.ones(3, dtype=torch.float64)); b = torch.nn.Parameter(torch.ones(3, dtype=torch.float64))
    opt = RO.RAdamOracle([{"params": [a], "lr": 1e-3}, {"params": [b], "lr": 1e-1, "weight_decay": 0.5}])
    g = torch.tensor([0.2, -0.1, 0.4], dtype=torch.float64)
    a.grad = g.clone(); b.grad = g.clone()
    opt.step()
    # t = 1: step_size = 1e-3 / 0.1 from the leader; b: decay with its own lr first, then the leader's step
    assert torch.allclose(a.detach(), 1 - 1e-2 * 0.1 * g, rtol=0, atol=1e-15)
    assert torch.allclose(b.detach(), (1 - 0.5 * 1e-1) - 1e-2 * 0.1 * g, rtol=0, atol=1e-15)


# ---------------------------------------------------------------------------------------------------- CPU: host logic
def _cpu_engine_and_groups(golden_dir, base_lr=4e-5):
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    eng = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True)
    named = [(name, torch.nn.Parameter(eng.ps.p(name))) for name in eng.ps.entries]
    return eng, named, AO.reference_param_groups(named, base_lr=base_lr)


def test_fused_radam_host_state_uses_build_chunks_and_the_reference_layout(golden_dir):
    from vilbert_b200.optim import FusedRAdam, build_chunks
    eng, named, groups = _cpu_engine_and_groups(golden_dir)
    named[0][1].requires_grad_(False)                  # a frozen first tensor: the leader is the first TRAINABLE group
    opt = FusedRAdam(groups, lr=4e-5, engine=eng)
    assert opt.defaults == dict(lr=4e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0)
    assert opt.leader_group == 1
    base = eng.ps.flat.data_ptr()
    ranges = [((p.data_ptr() - base) // 4, p.numel(), gi) for gi, (_, p) in enumerate(named) if p.requires_grad]
    st, cn, gr = build_chunks(ranges)
    assert opt._chunk_start.tolist() == st.tolist() and opt._chunk_count.tolist() == cn.tolist() and opt._chunk_group.tolist() == gr.tolist()
    # the group table carries the reference's per-tensor lr / weight decay; correct_bias is unused (0)
    row = opt._groups_np[gr[-1]]
    assert row["lr"] == pytest.approx(groups[gr[-1]]["lr"]) and row["correct_bias"] == 0
    # state entries are views of the flat moment buffers
    p = named[3][1]
    opt.state[p]["exp_avg"].fill_(0.25)
    off = (p.data_ptr() - base) // 4
    assert opt.exp_avg[off:off + p.numel()].eq(0.25).all()
    with pytest.raises(ValueError):
        FusedRAdam([torch.nn.Parameter(torch.zeros(4))], engine=eng)


def test_fused_radam_loads_a_reference_layout_checkpoint_on_cpu(golden_dir):
    """A state dict in the reference's RAdam layout ({step, exp_avg, exp_avg_sq} per parameter index) lands in the flat
    buffers and sets the device step counter; tensors without an entry keep zero moments; state_dict() reports it back."""
    from vilbert_b200.optim import FusedRAdam
    eng, named, groups = _cpu_engine_and_groups(golden_dir)
    shadow = [torch.nn.Parameter(p.detach().clone().double()) for _, p in named]
    ora = RO.RAdamOracle([dict(g, params=[s]) for g, s in zip(groups, shadow)], lr=4e-5)
    gen = torch.Generator().manual_seed(3)
    for _ in range(3):
        for s in shadow[1:]:                           # the first tensor never gets a gradient: no state entry
            s.grad = torch.randn(s.shape, generator=gen, dtype=torch.float64) * 1e-2
        ora.step()
    sd = ora.state_dict()
    assert 0 not in sd["state"] and sd["state"][1]["step"] == 3
    opt = FusedRAdam(groups, lr=4e-5, engine=eng)
    opt.load_state_dict(sd)
    assert opt._step_dev.item() == 3
    assert opt.state[named[0][1]]["exp_avg"].abs().max() == 0
    for i in (1, 5, len(named) - 1):
        p = named[i][1]
        assert torch.equal(opt.state[p]["exp_avg"], sd["state"][i]["exp_avg"].float())
        assert torch.equal(opt.state[p]["exp_avg_sq"], sd["state"][i]["exp_avg_sq"].float())
    back = opt.state_dict()
    assert set(back["state"][1]) == {"step", "exp_avg", "exp_avg_sq"} and back["state"][1]["step"] == 3
    assert back["param_groups"][0].keys() == sd["param_groups"][0].keys()


# ---------------------------------------------------------------------------------------------------- GPU
def _tiny_model(golden_dir, precision="fp16", **over):
    import vilbert_b200
    cfgj = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over)
    cfg = O.make_config(cfgj)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1, precision=precision)
    model.load_state_dict(O.synth_params(cfg, seed=0, device="cuda"), strict=True)
    return model, cfg


def _rel(a, b, floor):
    return ((a.double() - b.double()).abs().max() / max(b.abs().max().item(), floor)).item()


def _f32(x):
    """A learning rate as the kernel's fp32 group table holds it: the oracle computes in float64 from the same value, so the
    comparison measures the kernel's arithmetic, not the table's storage precision. The betas stay the Python floats: the table
    carries fp32(1 - beta) beside them, and the kernel's rectification and moments follow the Python values."""
    return float(np.float32(x))


def _oracle_for(groups, params, lr):
    return RO.RAdamOracle([dict(g, params=[p], lr=_f32(g["lr"])) for g, p in zip(groups, params)], lr=_f32(lr),
                          betas=(0.9, 0.999), eps=1e-8)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_fused_radam_matches_float64_oracle_over_steps(golden_dir, precision):
    """Nine steps (unrectified 1-5, rectified from 6) with the reference's grouping and a changing lr: parameters, moments, the
    zeroed gradient, the 16-bit weight copies (hi + lo in split precision) and the engine's shadow flags."""
    from vilbert_b200.optim import FusedRAdam
    model, _ = _tiny_model(golden_dir, precision)
    named = list(model.named_parameters())
    groups = AO.reference_param_groups(named, base_lr=4e-5)
    opt = FusedRAdam(groups, lr=4e-5, model=model)
    ref = [torch.nn.Parameter(p.detach().clone().double()) for _, p in named]
    ora = _oracle_for(groups, ref, 4e-5)
    base = [g["lr"] for g in groups]
    gen = torch.Generator(device="cuda").manual_seed(1)
    eng = model.engine
    for t in range(1, 10):
        scale = min(1.0, t / 3) * (1.0 - 0.05 * t)       # warm-up then linear decay: the scheduler mutates group["lr"]
        for g, go, b in zip(opt.param_groups, ora.param_groups, base):
            g["lr"], go["lr"] = b * scale, _f32(b * scale)
        eng.ps.grad.copy_(torch.randn(eng.ps.numel, device="cuda", generator=gen) * 1e-2)
        for r, (_, p) in zip(ref, named):
            r.grad = p.grad.detach().double()
        opt.step()
        ora.step()
        torch.cuda.synchronize()
        assert all(p.grad.abs().max().item() == 0 for _, p in named) and eng.grad_clean
    assert opt.state_dict()["state"][0]["step"] == 9
    for r, (k, p) in zip(ref, named):
        assert _rel(p.detach(), r.detach(), 1e-6) < 2e-6, k
        assert _rel(opt.state[p]["exp_avg"], ora.state[r]["exp_avg"], 1e-12) < 1e-5, k
        assert _rel(opt.state[p]["exp_avg_sq"], ora.state[r]["exp_avg_sq"], 1e-12) < 2e-6, k
    ps = eng.ps
    assert torch.equal(ps.shadow, ps.flat.to(ps.op_dtype)) and torch.equal(ps.shadow_b, ps.flat.to(torch.bfloat16))
    if precision == "fp32":
        assert torch.equal(ps.shadow_lo, (ps.flat - ps.shadow.float()).to(ps.op_dtype))
    assert eng.shadow_clean and eng.shadow_trusted


@pytest.mark.gpu
def test_captured_plan_step_advances_the_rectification_schedule(golden_dir):
    """Plan.enable_optimizer(FusedRAdam) captured as one graph and replayed 7 times == 7 eager step() calls (each replay
    advances the device step counter, so it crosses the t = 6 switch). The gradient is held fixed (zero_grad=False) so that
    both runs see identical inputs."""
    from vilbert_b200.optim import FusedRAdam
    model, cfg = _tiny_model(golden_dir)
    eng, ps = model.engine, model.engine.ps
    opt = FusedRAdam(AO.reference_param_groups(model.named_parameters(), base_lr=1e-3), lr=1e-3, model=model, zero_grad=False)
    ps.grad.copy_(torch.randn(ps.numel, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)) * 1e-2)
    p0 = ps.flat.clone()

    def reset():
        ps.flat.copy_(p0); opt.exp_avg.zero_(); opt.exp_avg_sq.zero_(); opt._step_dev.zero_(); eng.refresh_weights()
        torch.cuda.synchronize()

    for _ in range(7):
        opt.step()
    torch.cuda.synchronize()
    eager = [t.clone() for t in (ps.flat, opt.exp_avg, opt.exp_avg_sq, ps.shadow, ps.shadow_b)]
    reset()
    inp = O.synth_inputs(cfg, 4, 11, 9, seed=1234, device="cuda")
    plan = eng.plan(4, 9, 11)
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    plan.enable_optimizer(opt)
    plan.capture()                                    # its warm-up run steps once: start again from the initial state
    reset()
    for _ in range(7):
        plan.run_step()
    torch.cuda.synchronize()
    assert opt._step_dev.item() == 7 and opt.state_dict()["state"][0]["step"] == 7
    for a, b in zip(eager, (ps.flat, opt.exp_avg, opt.exp_avg_sq, ps.shadow, ps.shadow_b)):
        assert torch.equal(a, b)
    assert not torch.equal(ps.flat, p0)


@pytest.mark.gpu
@pytest.mark.parametrize("resume_at", [3, 8])
def test_checkpoint_round_trip_continues_like_an_uninterrupted_run(golden_dir, resume_at):
    """Stop after `resume_at` steps, save model + optimizer state (reference RAdam layout), resume in a fresh model and
    optimizer: the continuation is bit-identical to an uninterrupted run. The same checkpoint loaded into the float64
    oracle continues to the same weights."""
    from vilbert_b200.optim import FusedRAdam
    total = 10

    def make():
        model, _ = _tiny_model(golden_dir)
        named = list(model.named_parameters())
        groups = AO.reference_param_groups(named, base_lr=1e-3)
        return model, named, groups, FusedRAdam(groups, lr=1e-3, model=model)

    def run(model, opt, base, t0, t1):
        for t in range(t0 + 1, t1 + 1):
            for g, b in zip(opt.param_groups, base):
                g["lr"] = b * (1.0 - 0.04 * t)
            gen = torch.Generator(device="cuda").manual_seed(100 + t)
            model.engine.ps.grad.copy_(torch.randn(model.engine.ps.numel, device="cuda", generator=gen) * 1e-2)
            opt.step()
        torch.cuda.synchronize()

    model_a, named_a, groups_a, opt_a = make()
    base = [g["lr"] for g in groups_a]
    run(model_a, opt_a, base, 0, total)
    model_b, _, _, opt_b = make()
    run(model_b, opt_b, base, 0, resume_at)
    buf = io.BytesIO()
    torch.save(dict(model=model_b.state_dict(), optimizer=opt_b.state_dict()), buf)
    buf.seek(0)
    ck = torch.load(buf)
    st = ck["optimizer"]["state"]
    assert len(st) == len(named_a) and all(set(s) == {"step", "exp_avg", "exp_avg_sq"} and s["step"] == resume_at for s in st.values())
    del model_b, opt_b
    model_c, named_c, _, opt_c = make()
    model_c.load_state_dict(ck["model"])
    opt_c.load_state_dict(ck["optimizer"])
    run(model_c, opt_c, base, resume_at, total)
    for (k, pa), (_, pc) in zip(named_a, named_c):
        assert torch.equal(pa.detach(), pc.detach()), k
    # the float64 oracle resumes from the same checkpoint (its own step counters restart at resume_at)
    ref = [torch.nn.Parameter(ck["model"][k].double()) for k, _ in named_a]
    ora = _oracle_for(groups_a, ref, 1e-3)
    ora.load_state_dict(ck["optimizer"])
    for g in ora.param_groups:
        g["betas"], g["eps"] = (0.9, 0.999), 1e-8
    flat = model_a.engine.ps.flat
    for t in range(resume_at + 1, total + 1):
        for g, b in zip(ora.param_groups, base):
            g["lr"] = _f32(b * (1.0 - 0.04 * t))
        gen = torch.Generator(device="cuda").manual_seed(100 + t)
        grad = torch.randn(model_a.engine.ps.numel, device="cuda", generator=gen) * 1e-2
        for r, (_, pa) in zip(ref, named_a):
            off = (pa.data_ptr() - flat.data_ptr()) // 4
            r.grad = grad[off:off + r.numel()].view(r.shape).double()
        ora.step()
    for r, (k, pa) in zip(ref, named_a):
        assert _rel(pa.detach(), r.detach(), 1e-6) < 2e-6, k


@pytest.mark.gpu
def test_training_loop_with_fused_radam(golden_dir):
    """Module surface: model(...) -> loss -> backward() -> FusedRAdam.step() lowers the loss of a fixed batch, and the next
    forward uses the updated weights without an explicit refresh."""
    import vilbert_b200
    from vilbert_b200.optim import FusedRAdam
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    cfgj = dict(cfgj, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, v_hidden_dropout_prob=0.0, v_attention_probs_dropout_prob=0.0)
    cfg = O.make_config(cfgj)
    inp = O.synth_inputs(cfg, 4, 11, 9, seed=1234, device="cuda")
    tgt = O.synth_vqa_target(4, 3129, device="cuda")
    args = (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1, dropout_prob=0.0)
    model.load_state_dict(O.synth_params(cfg, seed=0, device="cuda"), strict=True)
    model.train()
    opt = FusedRAdam(AO.reference_param_groups(model.named_parameters(), base_lr=1e-2), lr=1e-2, model=model)
    w0 = model.state_dict()["bert.encoder.layer.0.intermediate.dense.weight"].clone()
    losses = []
    for _ in range(7):
        loss = O.vqa_loss(model(*args)[0], tgt)
        loss.backward()
        opt.step(); model.zero_grad()
        losses.append(loss.item())
    assert losses[1] < losses[0] and losses[-1] < losses[0] * 0.97, losses
    assert (model.state_dict()["bert.encoder.layer.0.intermediate.dense.weight"] - w0).abs().max().item() > 0
    l_now = O.vqa_loss(model(*args)[0], tgt).item()
    model.engine.refresh_weights()
    l_fresh = O.vqa_loss(model(*args)[0], tgt).item()
    assert abs(l_fresh - l_now) < 1e-6 * abs(l_now) + 1e-7
