"""Pins tests/_radam_oracle.py against the reference's own RAdam (vilbert/optimization.py:16-100) and writes
tests/golden/radam_reference_steps.pt, which tests/test_radam.py re-checks without the reference. Needs the reference
checkout (oracle/ref_loader.py; VILBERT_REFERENCE_ROOT overrides its location) and runs on the CPU:

    python tools/make_radam_golden.py

Six odd-sized fp32 tensors, one param group each with its own lr / weight decay (the reference's grouping has one group per
tensor, train_tasks.py:400-420); the largest lr sits in a group that is NOT first, one group has its own betas, and the lrs
change between steps like WarmupLinearSchedule. Twelve steps cover the unrectified steps 1-5 (N_sma < 5 at b2 = 0.999), the
switch at t = 6 and the wrap of the reference's ten-slot step-size cache at t = 10 / 11. The oracle must equal the reference
exactly; a per-group-lr restatement must NOT (the fixture exercises the shared-cache behaviour).
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_loader  # noqa: E402
import _radam_oracle as RO  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "radam_reference_steps.pt")
SHAPES = [(37, 5), (129,), (3, 7, 11), (1001,), (6,), (17, 3)]
HYPER = [  # lr, weight_decay, betas
    (1e-3, 0.01, (0.9, 0.999)),
    (3e-3, 0.0, (0.9, 0.999)),
    (2e-2, 0.01, (0.9, 0.999)),     # the largest lr, in a group that is not first
    (5e-4, 0.1, (0.8, 0.99)),
    (1e-3, 0.0, (0.9, 0.999)),
    (7e-4, 0.05, (0.9, 0.999)),
]
STEPS = 12


def lr_scale(t):
    """Warm-up over the first four steps, then linear decay (what WarmupLinearSchedule does to group["lr"])."""
    return t / 4 if t <= 4 else 1.0 - 0.05 * (t - 4)


def make_inputs():
    g = torch.Generator().manual_seed(20261015)
    params = [torch.randn(s, generator=g) * 0.5 for s in SHAPES]
    grads = [[torch.randn(s, generator=g) * 10 ** (-1 - i % 3) for i, s in enumerate(SHAPES)] for _ in range(STEPS)]
    return params, grads


def run(opt_cls, params, grads):
    ps = [torch.nn.Parameter(p.clone()) for p in params]
    opt = opt_cls([{"params": [p], "lr": lr, "weight_decay": wd, "betas": b} for p, (lr, wd, b) in zip(ps, HYPER)])
    traj = []
    for t in range(1, STEPS + 1):
        for grp, (lr, _, _) in zip(opt.param_groups, HYPER):
            grp["lr"] = lr * lr_scale(t)
        for p, gr in zip(ps, grads[t - 1]):
            p.grad = gr.clone()
        opt.step()
        traj.append([p.detach().clone() for p in ps])
    state = [(opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone(), int(opt.state[p]["step"])) for p in ps]
    return traj, state


def run_per_group(params, grads):
    ps = [p.clone() for p in params]
    mom = [(torch.zeros_like(p), torch.zeros_like(p)) for p in ps]
    traj = []
    for t in range(1, STEPS + 1):
        for p, (m, v), gr, (lr, wd, b) in zip(ps, mom, grads[t - 1], HYPER):
            RO.radam_step(p, gr, m, v, t, lr * lr_scale(t), b[0], b[1], 1e-8, wd)
        traj.append([p.clone() for p in ps])
    return traj


def main():
    ref_loader.load()
    from vilbert.optimization import RAdam
    params, grads = make_inputs()
    ref_traj, ref_state = run(RAdam, params, grads)
    ora_traj, ora_state = run(RO.RAdamOracle, params, grads)
    for t, (a, b) in enumerate(zip(ora_traj, ref_traj), 1):
        assert all(torch.equal(x, y) for x, y in zip(a, b)), f"oracle differs from the reference at step {t}"
    for (ma, va, sa), (mb, vb, sb) in zip(ora_state, ref_state):
        assert torch.equal(ma, mb) and torch.equal(va, vb) and sa == sb
    naive = run_per_group(params, grads)
    diff = max((x - y).abs().max().item() for x, y in zip(naive[-1], ref_traj[-1]))
    assert diff > 1e-4, f"a per-group-lr restatement matches the reference (max diff {diff:.2e}): the fixture misses the shared cache"
    torch.save(dict(shapes=SHAPES, hyper=HYPER, lr_scale=[lr_scale(t) for t in range(1, STEPS + 1)], params=params, grads=grads,
                    trajectory=ref_traj, exp_avg=[s[0] for s in ref_state], exp_avg_sq=[s[1] for s in ref_state],
                    reference="facebookresearch/vilbert-multi-task vilbert/optimization.py RAdam"), OUT)
    print(f"oracle == reference over {STEPS} steps; per-group-lr restatement differs by {diff:.3e}; wrote {OUT}")


if __name__ == "__main__":
    main()
