"""The arithmetic tests/test_optim_kernels_gpu.py relies on, pinned on the CPU: fp32 torch restatements of pytorch_transformers
1.0.0 AdamW and of the reference's RAdam (vilbert/optimization.py) with Python-scalar hyper-parameters meet the per-element
tolerances of tests/_optim_ref.py against the float64 oracles, the float64 block reference there is those oracles, the fp32
(1 - beta) constants are the reference's, and the schedule grid asserts every wrong reference somewhere."""
import math

import numpy as np
import pytest
import torch

import _optim_ref as R
import _radam_oracle as RO
from oracle import adamw_oracle as AO


# ---------------------------------------------------------------------------------------------------- fp32 restatements
def adamw_fp32(p, grad, exp_avg, exp_avg_sq, step, lr, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True,
               one_minus=None):
    """pytorch_transformers 1.0.0 AdamW.step on one fp32 tensor, line by line (the 1.0.0 `add_(1.0 - beta1, grad)` spelled with
    alpha=). one_minus=(o1, o2) replaces the Python `1.0 - beta` factors (to show what 1 - fp32(beta) would do)."""
    beta1, beta2 = betas
    o1, o2 = one_minus if one_minus is not None else (1.0 - beta1, 1.0 - beta2)
    exp_avg.mul_(beta1).add_(grad, alpha=o1)
    exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=o2)
    denom = exp_avg_sq.sqrt().add_(eps)
    step_size = lr
    if correct_bias:
        bias_correction1 = 1.0 - beta1 ** step
        bias_correction2 = 1.0 - beta2 ** step
        step_size = step_size * math.sqrt(bias_correction2) / bias_correction1
    p.addcdiv_(exp_avg, denom, value=-step_size)
    if weight_decay > 0.0:
        p.add_(p, alpha=-lr * weight_decay)


def radam_fp32(p, grad, exp_avg, exp_avg_sq, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, leader=None):
    """vilbert/optimization.py RAdam.step on one fp32 tensor, its fp32 data path, with the rectification of the leader group's
    (lr, betas) in Python floats."""
    beta1, beta2 = betas
    exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    exp_avg.mul_(beta1).add_(grad, alpha=1 - beta1)
    n_sma, step_size = RO.rectification(step, *(leader or (lr, beta1, beta2)))
    if weight_decay != 0:
        p.add_(p, alpha=-weight_decay * lr)
    if n_sma >= 5:
        denom = exp_avg_sq.sqrt().add_(eps)
        p.addcdiv_(exp_avg, denom, value=-step_size)
    else:
        p.add_(exp_avg, alpha=-step_size)


def _state(n=4096, seed=0):
    """The GPU test's per-element mix at a small size: ordinary, zero, sqrt(v) << eps and huge gradients (the 1e-20 class is left
    to the GPU test, where the flush to zero is part of what it checks), fresh and running moments, p0 = 0 on a quarter."""
    gen = torch.Generator().manual_seed(seed)
    cls = torch.randint(0, 7, (n,), generator=gen)
    sc = torch.tensor([1e-2] * 4 + [0.0, 1e-12, 1e15])[cls]
    st = torch.where(cls == 4, 1e-2, sc)
    fresh = torch.rand(n, generator=gen) < 1 / 3
    g = torch.randn(n, generator=gen) * sc
    m = torch.where(fresh, 0.0, 0.3 * torch.randn(n, generator=gen) * st)
    v = torch.where(fresh, 0.0, st * st * (0.1 + torch.rand(n, generator=gen)))
    p = torch.where(torch.rand(n, generator=gen) < 0.25, 0.0, 0.05 * torch.randn(n, generator=gen) + 1e-3)
    return p, g, m, v


def _hp(n, lr, wd, betas, eps, ss, rect=True):
    full = lambda x: torch.full((n,), float(x), dtype=torch.float64)     # noqa: E731
    return dict(lr=full(lr), wd=full(wd), b1=full(betas[0]), b2=full(betas[1]), eps=full(eps), ss=full(ss),
                rect=torch.full((n,), bool(rect)))


def _ratio(kind, fp32_out, state, hp, gs=1.0):
    p0, g, m0, v0 = (x.double() for x in state)
    pr, mr, vr, dmag, mmag, p1 = R.step(kind, p0, g, m0, v0, hp, gs)
    tols = R.tolerances(p0, pr, mmag, vr, dmag, p1)
    return {q: ((k.double() - r).abs() / t).max().item() for q, k, r, t in zip("pmv", fp32_out, (pr, mr, vr), (tols[2],) + tols[:2])}


# ---------------------------------------------------------------------------------------------------- the constants
@pytest.mark.parametrize("beta", [0.9, 0.999, 0.98])
def test_reference_ops_use_fp32_of_one_minus_beta(beta):
    """torch's fp32 ops round the Python scalar 1.0 - beta once: fp32(1 - beta), not 1 - fp32(beta)."""
    one = torch.ones(1)
    v = torch.zeros(1).addcmul_(one, one, value=1.0 - beta)
    m = torch.zeros(1).add_(one, alpha=1.0 - beta)
    assert v.item() == m.item() == R.f32(1.0 - beta)
    if beta != 0.9:
        assert R.f32(1.0 - beta) != float(np.float32(1.0) - np.float32(beta))


def test_group_row_carries_the_reference_constants():
    from vilbert_b200.optim import _GROUP_DT, group_row
    assert _GROUP_DT.itemsize == 32
    row = np.array([group_row(4e-5, (0.9, 0.999), 1e-6, 0.01, True), group_row(1e-4, (0.9, 0.98), 1e-8, 0.0)], dtype=_GROUP_DT)
    assert row["one_minus_beta2"][0] == np.float32(0.001) and row["one_minus_beta2"][0] != np.float32(1) - np.float32(0.999)
    assert row["one_minus_beta2"][1] == np.float32(1.0 - 0.98) and row["one_minus_beta1"].tolist() == [R.f32(1.0 - 0.9)] * 2
    assert row["correct_bias"].tolist() == [1, 0] and row["beta2"][0] == np.float32(0.999)
    # 1 - fp32(0.999) is 1.29e-5 low: the second moment every step of a default-betas run would be that much low
    assert abs((1.0 - R.f32(0.999)) / 0.001 - 1 + 1.287e-5) < 1e-8


# ---------------------------------------------------------------------------------------------------- the block reference
def _assert_same(ref, p0, oracle):
    """The two float64 restatements agree to a millionth of the fp32 tolerance (their operation order differs, and p0 - dp or
    b1 m0 + (1-b1) g may cancel, so relative to the terms rather than to the result)."""
    pr, mr, vr, dmag, mmag, p1 = ref
    tols = R.tolerances(p0, pr, mmag, vr, dmag, p1)
    for a, b, tol in zip((pr, mr, vr), oracle, (tols[2], tols[0], tols[1])):
        assert ((a - b).abs() <= 1e-6 * tol).all()


@pytest.mark.parametrize("t,correct_bias,wd", [(1, True, 0.0), (7, True, 0.01), (100, False, 0.1)])
def test_block_reference_is_the_adamw_oracle(t, correct_bias, wd):
    p0, g, m0, v0 = (x.double() for x in _state())
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    AO.adamw_step(p, g * 0.25, m, v, t, 3e-3, beta1=0.9, beta2=0.98, eps=1e-8, weight_decay=wd, correct_bias=correct_bias)
    ss = R.adamw_step_size(3e-3, (0.9, 0.98), t, correct_bias)
    _assert_same(R.step("adamw", p0, g, m0, v0, _hp(len(p0), 3e-3, wd, (0.9, 0.98), 1e-8, ss), 0.25), p0, (p, m, v))


@pytest.mark.parametrize("t", [1, 5, 6, 700])
def test_block_reference_is_the_radam_oracle_with_a_leader(t):
    p0, g, m0, v0 = (x.double() for x in _state())
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    leader = (R.LEADER["lr"], *R.LEADER["betas"])
    RO.radam_step(p, g, m, v, t, 4e-5, 0.9, 0.999, 1e-8, 0.1, leader=leader)
    rect, ss = R.radam_step_size(R.LEADER["lr"], R.LEADER["betas"], t)
    assert rect == (t >= 6)
    _assert_same(R.step("radam", p0, g, m0, v0, _hp(len(p0), 4e-5, 0.1, (0.9, 0.999), 1e-8, ss, rect), 1.0), p0, (p, m, v))


# ---------------------------------------------------------------------------------------------------- the tolerances
@pytest.mark.parametrize("betas", R.BETAS)
@pytest.mark.parametrize("t", [1, 10, 10 ** 4])
def test_fp32_adamw_meets_the_tolerances_and_one_minus_fp32_beta_does_not(betas, t):
    """A correct fp32 AdamW is within every per-element tolerance of the float64 reference; with 1 - fp32(beta) it misses the
    second moment by > 10 tolerances at beta2 = 0.999 (and is indistinguishable at 0.98, where the slip is 9.5e-7)."""
    state = _state(seed=t)
    hp = _hp(len(state[0]), 1e-2, 0.1, betas, 1e-6, R.adamw_step_size(1e-2, betas, t, True))
    outs = {}
    for slip in (None, "one_minus_fp32_beta"):
        p, g, m, v = (x.clone() for x in state)
        om = (1.0 - R.f32(betas[0]), 1.0 - R.f32(betas[1])) if slip else None
        adamw_fp32(p, g, m, v, t, 1e-2, betas, 1e-6, 0.1, True, one_minus=om)
        outs[slip] = _ratio("adamw", (p, m, v), state, hp)
    assert max(outs[None].values()) <= 1.0, outs[None]
    if betas[1] == 0.999:
        assert outs["one_minus_fp32_beta"]["v"] > R.MISS
    assert R.applicable("adamw", [dict(lr=1e-2, weight_decay=0.1, betas=betas, correct_bias=True)], 0, t, 1.0,
                        "one_minus_fp32_beta") == (betas[1] == 0.999)


@pytest.mark.parametrize("t", [1, 5, 6, 100])
def test_fp32_radam_meets_the_tolerances(t):
    state = _state(seed=100 + t)
    leader = (R.LEADER["lr"], *R.LEADER["betas"])
    rect, ss = R.radam_step_size(*leader[:1], R.LEADER["betas"], t)
    p, g, m, v = (x.clone() for x in state)
    radam_fp32(p, g, m, v, t, 1e-2, (0.9, 0.999), 1e-8, 0.1, leader=leader)
    r = _ratio("radam", (p, m, v), state, _hp(len(p), 1e-2, 0.1, (0.9, 0.999), 1e-8, ss, rect))
    assert max(r.values()) <= 1.0, r


def test_fp32_step_size_cancels_where_the_float64_one_does_not():
    """Why the kernel forms AdamW's bias correction in float64: in fp32, 1 - b2^t cancels (even with an exact pow): the step size
    alone is 4e-6 to 2e-5 off for t <= 100, several times the whole update tolerance."""
    for t in (1, 2, 5, 10, 100):
        exact = math.sqrt(1.0 - 0.999 ** t) / (1.0 - 0.9 ** t)
        b1, b2 = np.float32(0.9), np.float32(0.999)
        f = float(np.sqrt(np.float32(1) - b2 ** np.float32(t)) / (np.float32(1) - b1 ** np.float32(t)))
        assert abs(f / exact - 1) > 5 * R.REL["p"], t


# ---------------------------------------------------------------------------------------------------- the schedule grid
@pytest.mark.parametrize("kind", ["adamw", "radam"])
def test_schedule_grid_covers_every_value_and_asserts_every_slip(kind):
    cs = R.cases(kind)
    assert {c["t"] for c in cs} == set(R.T_VALUES) and {c["betas"] for c in cs} == set(R.BETAS)
    assert {c["eps"] for c in cs} == set(R.EPS) and {c["grad_scale"] for c in cs} == set(R.GRAD_SCALES)
    assert {(c["betas"], c["eps"]) for c in cs} == {(b, e) for b in R.BETAS for e in R.EPS}
    assert {c["copies"] for c in cs} == set(R.COPIES) and {c["zero_grad"] for c in cs} == {True, False}
    if kind == "adamw":
        assert {c["correct_bias"] for c in cs} == {True, False}
        assert {(c["t"], c["betas"]) for c in cs if c["correct_bias"]} == {(t, b) for t in R.T_VALUES for b in R.BETAS}
    names = [f"layer.{i}.weight" if i % 2 else f"layer.{i}.bias" for i in range(20)] + ["vil_prediction.weight"]
    slips = [s for s in R.SLIPS if kind == "radam" or s != "own_group_step"]
    hits = {s: [c["t"] for c in cs if R.applicable(kind, R.groups_for(names, kind, c), 0, c["t"], c["grad_scale"], s)] for s in slips}
    assert all(hits.values()), hits
    # what each slip cannot change is not asserted: t - 1 at t = 1, bias correction once 1 - b^t rounds to 1
    assert 1 not in hits["step_minus_1"] and 10 ** 5 not in hits["no_bias_correction"]
    assert 1 in hits["no_bias_correction"] and 6 in hits["step_minus_1"]
