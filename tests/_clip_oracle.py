"""Float64 restatement of gradient-norm clipping with non-finite step skipping, as `max_grad_norm=` of the fused optimizers
defines it — TEST INFRASTRUCTURE, used by tests/test_clip_cpu.py and tests/test_clip_gpu.py.

torch.nn.utils.clip_grad_norm_(params, max_norm) semantics, composed with the AdamW / RAdam restatements
(oracle/adamw_oracle.py, tests/_radam_oracle.py):

    norm = || grad_scale * g ||_2 over every trainable tensor (a tensor shared by two names counted once)
    skip = some element of g is NaN or +-inf          (the step then changes no weight, moment or step count)
    coef = min(1, max_norm * fp32(1 / (fp32(norm) + 1e-6)))   in fp32, as torch evaluates `max_norm / (norm + 1e-6)`
    the update uses grad_scale * g * coef

The norm itself is float64 here; the fused kernel sums squares in float64 too and rounds the norm to fp32 once.
"""
import math

import numpy as np
import torch


def global_norm(grads, grad_scale=1.0):
    """float64 L2 norm over a list of tensors (any dtype)."""
    s = sum(float(g.double().pow(2).sum()) for g in grads)
    return abs(grad_scale) * math.sqrt(s)


def clip_coefficient(norm, max_norm):
    """torch.nn.utils.clip_grad_norm_'s coefficient for an fp32 norm: clamp(reciprocal(norm + 1e-6) * max_norm, max=1)."""
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        r = np.float32(1.0) / (np.float32(norm) + np.float32(1e-6))
        c = r * np.float32(max_norm)
    return float(min(c, np.float32(1.0))) if not np.isnan(c) else 1.0


def clip_decision(grads, max_norm, grad_scale=1.0):
    """(norm as the fp32 value the device reports, coef, skip) for one step."""
    finite = all(bool(torch.isfinite(g).all()) for g in grads)
    if not finite:
        return float("nan"), 0.0, True
    with np.errstate(over="ignore"):
        norm = float(np.float32(global_norm(grads, grad_scale)))
    return norm, clip_coefficient(norm, max_norm), False


def clipped_grads(grads, max_norm, grad_scale=1.0):
    """The float64 gradients the update uses (grad_scale * g * coef), or None when the step is skipped."""
    _, coef, skip = clip_decision(grads, max_norm, grad_scale)
    if skip:
        return None
    return [g.double() * grad_scale * coef for g in grads]
