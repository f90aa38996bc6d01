"""CPU / float64-capable restatement of the reference's RAdam (vilbert/optimization.py:16-100, the optimizer of
`train_tasks.py --optim RAdam`, :427-428) — TEST INFRASTRUCTURE, used by tests/test_radam.py and tools/optim_probe.py.
tools/make_radam_golden.py pins it bit-exactly against the reference's own class (tests/golden/radam_reference_steps.pt).

Per tensor, at its step t (after the increment):

    exp_avg_sq = b2 exp_avg_sq + (1 - b2) g g          (own group's betas)
    exp_avg    = b1 exp_avg    + (1 - b1) g
    p         -= wd lr p                               (own group's lr / wd, only if wd != 0; FIRST, on the old p)
    p         -= step_size exp_avg / (sqrt(exp_avg_sq) + eps)   if N_sma >= 5
    p         -= step_size exp_avg                              otherwise

    N_sma_max = 2 / (1 - b2) - 1,  N_sma = N_sma_max - 2 t b2^t / (1 - b2^t)          (Python floats: float64)
    step_size = lr sqrt((1 - b2^t) (N_sma - 4) / (N_sma_max - 4) (N_sma - 2) / N_sma N_sma_max / (N_sma_max - 2)) / (1 - b1^t)
              = lr / (1 - b1^t)                                                        (N_sma < 5)

The reference keeps (t, N_sma, step_size) in ten slots indexed by t % 10 that all param groups share
(optimization.py:19, 59-86): the first tensor stepped at a given t computes them with ITS group's lr / b1 / b2 and every
later tensor at that t reuses them. `RAdamOracle` models that; `radam_step(..., leader=None)` is the naive per-group
version, which differs as soon as groups have different learning rates.
"""
import math

import torch


def rectification(step, lr, beta1, beta2):
    """(N_sma, step_size) of step `step` (1-based), in Python float64 and in the reference's order of operations."""
    beta2_t = beta2 ** step
    n_sma_max = 2 / (1 - beta2) - 1
    n_sma = n_sma_max - 2 * step * beta2_t / (1 - beta2_t)
    if n_sma >= 5:
        step_size = lr * math.sqrt((1 - beta2_t) * (n_sma - 4) / (n_sma_max - 4) * (n_sma - 2) / n_sma * n_sma_max / (n_sma_max - 2)) \
            / (1 - beta1 ** step)
    else:
        step_size = lr / (1 - beta1 ** step)
    return n_sma, step_size


def apply_update(p, grad, exp_avg, exp_avg_sq, n_sma, step_size, lr, beta1, beta2, eps, weight_decay):
    """The in-place element-wise part of one step, given the rectification scalars."""
    exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    exp_avg.mul_(beta1).add_(grad, alpha=1 - beta1)
    if weight_decay != 0:
        p.add_(p, alpha=-weight_decay * lr)
    if n_sma >= 5:
        p.addcdiv_(exp_avg, exp_avg_sq.sqrt().add_(eps), value=-step_size)
    else:
        p.add_(exp_avg, alpha=-step_size)


def radam_step(p, grad, exp_avg, exp_avg_sq, step, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, leader=None):
    """One in-place RAdam update of a single tensor at 1-based `step`. `leader` = (lr, beta1, beta2) of the group that supplies
    the rectification (the reference's leader group); None uses the tensor's own group."""
    n_sma, step_size = rectification(step, *(leader if leader is not None else (lr, beta1, beta2)))
    apply_update(p, grad, exp_avg, exp_avg_sq, n_sma, step_size, lr, beta1, beta2, eps, weight_decay)


class RAdamOracle(torch.optim.Optimizer):
    """Multi-tensor restatement with the reference's constructor, state layout ({step, exp_avg, exp_avg_sq} per parameter)
    and shared ten-slot step-size cache. Works in the dtype of the parameters it is given (float64 for the GPU tests)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._slots = [None] * 10

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st.update(step=0, exp_avg=torch.zeros_like(p), exp_avg_sq=torch.zeros_like(p))
                st["step"] += 1
                t = st["step"]
                slot = self._slots[t % 10]
                if slot is None or slot[0] != t:
                    slot = (t,) + rectification(t, group["lr"], beta1, beta2)
                    self._slots[t % 10] = slot
                apply_update(p, p.grad, st["exp_avg"], st["exp_avg_sq"], slot[1], slot[2], group["lr"], beta1, beta2, group["eps"],
                             group["weight_decay"])
        return loss
