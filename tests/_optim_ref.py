"""Per-element float64 references of the fused optimizer kernels (csrc/vb_optim.cu) on flat buffers, the fp32 error bounds the
kernels must meet against them, and the plausible wrong references those bounds must reject — TEST INFRASTRUCTURE, used by
tests/test_optim_kernels_gpu.py and pinned on the CPU by tests/test_optim_kernels_cpu.py.

The references restate pytorch_transformers 1.0.0 AdamW (oracle/adamw_oracle.py) and the reference's RAdam
(tests/_radam_oracle.py) for ONE step from an arbitrary state (p0, m0, v0) at step t, with the hyper-parameters as the Python
floats a user passes (beta2 = 0.999, not its fp32 neighbour): g' = grad_scale g (times the clip coefficient), then

    AdamW  m = b1 m0 + (1-b1) g';  v = b2 v0 + (1-b2) g'^2;  p = p0 - ss m / (sqrt(v) + eps);  p -= lr wd p
    RAdam  same m, v;  p = p0 - lr wd p0;  p -= ss m / (sqrt(v) + eps)  (N_sma >= 5)  or  p -= ss m  (otherwise)

with the step size ss of the group (AdamW) or of the leader group (RAdam) in float64.

Error bounds, per element, in units of the fp32 unit roundoff u = 2^-24 (the kernel rounds each operation to nearest; under
--use_fast_math sqrt and division are the approximate instructions, each within 2 ulp = 4u):
  m   two roundings (b1 m0, the sum; the product (1-b1) g' is the second term's) plus fp32 b1, fp32(1-b1) differing from the
      Python floats by <= 0.5u: 1.5u of |b1 m0| + |(1-b1) g'|, the terms' magnitude (the sum itself may cancel)  -> REL_M = 3u
  v   g'^2, (1-b2) g'^2, b2 v0, the sum (no cancellation: both terms >= 0), constants 0.8u: 2.8u of v        -> REL_V = 4u
  dp  m 1.5u; sqrt(v) 1.4u + 2u approximate; + eps 0.5u; division 4u; ss and ss q rounded 1u; the decay factor
      fl(1 - lr wd) and its product 1.5u: 11.9u of ss |m|_terms / (sqrt(v) + eps)                            -> REL_DP = 12u
  p   with p0 != 0 the kernel rounds two results where the reference is exact: the intermediate p1 (AdamW: p0 - dp before
      the decay; RAdam: p0 - lr wd p0) and the final p, 0.5 ulp each, and fl(1 - lr wd) is within 2^-25 of 1 - lr wd, at most
      0.5 ulp of p1: ULP_P = 1.5 ulp of the largest of |p0|, |p1|, |p| on top of the dp term. (Taking the ulp of p alone is not
      enough: where p1 lies in the binade above p, its rounding is a whole ulp of p.)
  A clip coefficient that is not a power of two rounds g' once more: +REL_CLIP = 2u on each bound.
  Below FLT_MIN the kernel flushes to zero (fast-math): every bound has an absolute floor of FLT_MIN. Such a v (g ~ 1e-20) has
  sqrt(v) < 1e-19, far below eps, so the flush does not reach p.
"""
import math

import numpy as np
import torch

import _radam_oracle as RO

U = 2.0 ** -24
FLT_MIN = float(np.finfo(np.float32).tiny)
REL = {"m": 3 * U, "v": 4 * U, "p": 12 * U}
REL_CLIP = 2 * U
ULP_P = 1.5
APPLICABLE = 20.0        # a slip is asserted where it moves some quantity by > 20 x its tolerance (an idealised effect)
MISS = 10.0              # ... and there it must miss the right reference by > 10 x the tolerance on the real data

SLIPS = ("decay_order", "no_bias_correction", "step_minus_1", "grad_scale_in_square", "own_group_step", "one_minus_fp32_beta")


def f32(x):
    return float(np.float32(x))


# ---------------------------------------------------------------------------------------------------- step sizes (float64)
def adamw_step_size(lr, betas, t, correct_bias):
    """pytorch_transformers 1.0.0: lr, or lr sqrt(1 - b2^t) / (1 - b1^t) in Python floats."""
    if not correct_bias:
        return lr
    return lr * math.sqrt(1.0 - betas[1] ** t) / (1.0 - betas[0] ** t)


def radam_step_size(lr, betas, t, bias_correction=True):
    """(rectified, step size) of RAdam step t from (lr, betas); bias_correction=False drops the 1 - b^t factors (a slip)."""
    n_sma, ss = RO.rectification(t, lr, betas[0], betas[1])
    if not bias_correction:
        b2t = betas[1] ** t
        ss = ss * (1.0 - betas[0] ** t) / (math.sqrt(1.0 - b2t) if n_sma >= 5 else 1.0)
    return n_sma >= 5, ss


def group_scalars(kind, groups, leader, t, slip=None):
    """Per group (step size, rectified) of one step, for the right reference (slip None) or a wrong one."""
    out = []
    for g in groups:
        if kind == "adamw":
            tt = t - 1 if slip == "step_minus_1" else t
            cb = g["correct_bias"] and slip != "no_bias_correction"
            out.append((adamw_step_size(g["lr"], g["betas"], tt, cb), True))
        else:
            src = g if slip == "own_group_step" else groups[leader]
            tt = t - 1 if slip == "step_minus_1" else t
            rect, ss = radam_step_size(src["lr"], src["betas"], tt, bias_correction=slip != "no_bias_correction")
            out.append((ss, rect))
    return out


def slip_effect(kind, groups, leader, t, grad_scale, slip):
    """Relative change a slip makes, per compared quantity, in idealised conditions the test data contain (fresh moments for v,
    p0 = 0 for p). A slip that changes nothing measurable at this step (bias correction at t = 1e5, step t-1 at t = 1) has
    effect 0 and is not asserted there."""
    if slip == "decay_order":
        return {"p": max(g["lr"] * g["weight_decay"] for g in groups)}
    if slip == "grad_scale_in_square":
        return {"v": abs(1.0 / grad_scale - 1.0)}
    if slip == "one_minus_fp32_beta":
        e = {}
        for g in groups:
            b1, b2 = g["betas"]
            e["m"] = max(e.get("m", 0.0), abs((1.0 - f32(b1)) / (1.0 - b1) - 1.0))
            e["v"] = max(e.get("v", 0.0), abs((1.0 - f32(b2)) / (1.0 - b2) - 1.0))
        return e
    if slip == "step_minus_1" and t < 2:
        return {}
    if kind == "adamw" and slip == "own_group_step":
        return {}
    right, wrong = group_scalars(kind, groups, leader, t), group_scalars(kind, groups, leader, t, slip)
    eff = 0.0
    for (s0, r0), (s1, r1) in zip(right, wrong):
        eff = max(eff, math.inf if r0 != r1 else abs(s1 / s0 - 1.0))
    return {"p": eff}


def applicable(kind, groups, leader, t, grad_scale, slip):
    return any(e > APPLICABLE * REL[q] for q, e in slip_effect(kind, groups, leader, t, grad_scale, slip).items())


# ---------------------------------------------------------------------------------------------------- element-wise step
def step(kind, p0, g, m0, v0, hp, grad_scale, slip=None):
    """One step of float64 tensors. hp: per-element float64 tensors lr, wd, b1, b2, eps, ss, rect (bool) for the right reference
    or the slip's. Returns (p, m, v, the update's magnitude |ss| |m|_terms / (sqrt(v) + eps) (without the division when
    unrectified), |m|_terms = |b1 m0| + |(1-b1) g'|, the intermediate p1 the kernel rounds before p)."""
    b1, b2 = hp["b1"], hp["b2"]
    if slip == "one_minus_fp32_beta":
        ob1, ob2 = 1.0 - b1.float().double(), 1.0 - b2.float().double()
    else:
        ob1, ob2 = 1.0 - b1, 1.0 - b2
    gg = g * grad_scale
    m = b1 * m0 + ob1 * gg
    v = b2 * v0 + ob2 * (gg * g if slip == "grad_scale_in_square" else gg * gg)
    den = v.sqrt() + hp["eps"]
    mag = (b1 * m0).abs() + (ob1 * gg).abs()
    lrwd = hp["lr"] * hp["wd"]
    if kind == "adamw":
        q, dmag = m / den, mag / den
        if slip == "decay_order":
            p1 = p0 - lrwd * p0
            p = p1 - hp["ss"] * q
        else:
            p1 = p0 - hp["ss"] * q
            p = p1 - lrwd * p1
    else:
        q = torch.where(hp["rect"], m / den, m)
        dmag = torch.where(hp["rect"], mag / den, mag)
        if slip == "decay_order":
            p1 = p0 - hp["ss"] * q
            p = p1 - lrwd * p1
        else:
            p1 = p0 - lrwd * p0
            p = p1 - hp["ss"] * q
    return p, m, v, hp["ss"].abs() * dmag, mag, p1


def ulp32(x):
    """Spacing of fp32 at |x| (float64 result)."""
    a = x.abs().float()
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


def tolerances(p0, p, m_mag, v, dmag, p1, clip=False):
    """Per-element absolute tolerances of (m, v, p) around the right reference."""
    extra = REL_CLIP if clip else 0.0
    tm = (REL["m"] + extra) * m_mag + FLT_MIN
    tv = (REL["v"] + extra) * v + FLT_MIN
    big = torch.maximum(torch.maximum(p0.abs(), p.abs()), p1.abs())
    tp = (REL["p"] + extra) * dmag + FLT_MIN + torch.where(p0 != 0, ULP_P * ulp32(big), 0.0)
    return tm, tv, tp


# ---------------------------------------------------------------------------------------------------- the schedules
T_VALUES = (1, 2, 5, 6, 10, 100, 700, 10 ** 4, 10 ** 5)
BETAS = ((0.9, 0.999), (0.9, 0.98))
EPS = (1e-6, 1e-8)
GRAD_SCALES = (1.0, 0.25, 2.0 ** -10)
# 16-bit copies a launch writes: (hi dtype or None, split-precision lo, always-bf16 copy)
COPIES = ((torch.float16, True, True), (torch.bfloat16, False, True), (torch.float16, False, False), (None, False, True),
          (torch.bfloat16, True, False))


def cases(kind):
    """Every t with both betas; eps, grad_scale, the copies written and zero_grad rotate; AdamW adds correct_bias off at four t."""
    out = []
    for i, (t, betas) in enumerate((t, b) for t in T_VALUES for b in BETAS):
        out.append(dict(t=t, betas=betas, eps=EPS[(i // 2) % 2], correct_bias=True,
                        grad_scale=GRAD_SCALES[i % 3], copies=COPIES[i % len(COPIES)], zero_grad=(i // 3) % 2 == 0))
    if kind == "adamw":
        for j, t in enumerate((1, 6, 700, 10 ** 5)):
            out.append(dict(t=t, betas=BETAS[j % 2], eps=EPS[(j + 1) % 2], correct_bias=False, grad_scale=GRAD_SCALES[(j + 1) % 3],
                            copies=COPIES[j % len(COPIES)], zero_grad=j % 2 == 1))
    return out


def case_id(c):
    return (f"t{c['t']}-b{c['betas'][1]}-eps{c['eps']:g}-{'cb' if c['correct_bias'] else 'nocb'}-gs{c['grad_scale']:g}"
            f"-{'zg' if c['zero_grad'] else 'keepg'}")


# the per-tensor hyper-parameters: the reference's grouping (train_tasks.py:401-421: lr 1e-4 for vil_* heads, no decay on bias /
# LayerNorm, 0.01 otherwise), a strong-decay group on every 7th tensor so that the order of decay and update is observable
# (lr wd = 1e-3), and for RAdam a leader group (the first tensor's) whose lr and betas differ from every other group's
BASE_LR = 4e-5
STRONG = dict(lr=1e-2, weight_decay=0.1)
LEADER = dict(lr=2e-3, betas=(0.8, 0.99))


def groups_for(names, kind, case):
    groups = []
    for i, name in enumerate(names):
        lr = 1e-4 if "vil_" in name else BASE_LR
        wd = 0.0 if any(k in name for k in ("bias", "LayerNorm.bias", "LayerNorm.weight")) else 0.01
        if i % 7 == 3:
            lr, wd = STRONG["lr"], STRONG["weight_decay"]
        g = dict(lr=lr, weight_decay=wd, betas=case["betas"], eps=case["eps"], correct_bias=case.get("correct_bias", False))
        if kind == "radam" and i == 0:
            g.update(lr=LEADER["lr"], betas=LEADER["betas"])
        groups.append(g)
    return groups
