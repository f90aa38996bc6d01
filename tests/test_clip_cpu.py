"""Gradient-norm clipping and non-finite step skipping of the fused optimizers (`max_grad_norm=`), host side: argument checks,
the launches a step makes, and the float64 restatement (tests/_clip_oracle.py) against torch.nn.utils.clip_grad_norm_."""
import json
import math
import os
import sys

import pytest
import torch

import _clip_oracle as CO
from oracle import adamw_oracle as AO
from oracle import vilbert_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cpu_engine(golden_dir):
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    eng = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True)
    named = [(name, torch.nn.Parameter(eng.ps.p(name))) for name in eng.ps.entries]
    return eng, named


def _classes():
    from vilbert_b200.optim import FusedAdamW, FusedRAdam
    return FusedAdamW, FusedRAdam


# ---------------------------------------------------------------------------------------------------- the restatement
def test_oracle_coefficient_is_torch_clip_grad_norm_bit_for_bit():
    """The same fp32 norm gives torch's coefficient exactly: torch scales the gradients by it, so compare what it leaves."""
    gen = torch.Generator().manual_seed(0)
    for max_norm in (1.0, 0.37, 5.0, 1e-3, 123.456):
        for _ in range(50):
            g = torch.randn(97, generator=gen) * float(torch.rand(1, generator=gen)) * 3
            p = torch.nn.Parameter(torch.zeros(97)); p.grad = g.clone()
            total = torch.nn.utils.clip_grad_norm_([p], max_norm)
            coef = CO.clip_coefficient(float(total), max_norm)
            assert torch.equal(p.grad, g * torch.tensor(coef, dtype=torch.float32)), (max_norm, float(total))
    assert CO.clip_coefficient(1e-9, 1.0) == 1.0 and CO.clip_coefficient(3.0, float("inf")) == 1.0


def test_oracle_norm_and_skip_decision():
    gen = torch.Generator().manual_seed(1)
    gs = [torch.randn(n, generator=gen) for n in (5, 1000, 3)]
    ps = [torch.nn.Parameter(torch.zeros_like(g)) for g in gs]
    for p, g in zip(ps, gs):
        p.grad = g.clone()
    total = torch.nn.utils.clip_grad_norm_(ps, 1.0)
    norm, coef, skip = CO.clip_decision(gs, 1.0)
    assert not skip and abs(norm - float(total)) <= 1e-6 * float(total) and coef < 1
    assert CO.global_norm(gs, grad_scale=-0.5) == pytest.approx(0.5 * CO.global_norm(gs), rel=1e-15)
    for bad in (float("nan"), float("inf"), float("-inf")):
        g2 = [g.clone() for g in gs]
        g2[1][17] = bad
        assert CO.clip_decision(g2, 1.0)[2] and CO.clipped_grads(g2, 1.0) is None
    # finite fp32 extremes never overflow the float64 sum: no skip
    big = [torch.full((4096,), 3e38)]
    norm, _, skip = CO.clip_decision(big, 1.0)
    assert not skip and math.isinf(norm)        # the fp32 norm overflows, as torch's does; the step is still taken


def test_oracle_composes_with_the_adamw_restatement():
    """clip then AdamW == AdamW on the clipped float64 gradient (what the GPU tests compare the kernels against)."""
    g = torch.tensor([3.0, 4.0], dtype=torch.float64)
    p = torch.zeros(2, dtype=torch.float64); m = torch.zeros_like(p); v = torch.zeros_like(p)
    (cg,) = CO.clipped_grads([g], 1.0)
    assert torch.allclose(cg, g / (5.0 + 1e-6), rtol=1e-7)
    AO.adamw_step(p, cg, m, v, 1, lr=0.1, correct_bias=False)
    assert torch.allclose(m, 0.1 * cg)


# ---------------------------------------------------------------------------------------------------- argument checks
@pytest.mark.parametrize("bad", [0.0, -1.0, float("nan"), 0])
def test_max_grad_norm_must_be_positive(golden_dir, bad):
    eng, named = _cpu_engine(golden_dir)
    for cls in _classes():
        with pytest.raises(ValueError, match="max_grad_norm"):
            cls([p for _, p in named], engine=eng, max_grad_norm=bad)


def test_max_grad_norm_defaults_and_state(golden_dir):
    eng, named = _cpu_engine(golden_dir)
    for cls in _classes():
        opt = cls([p for _, p in named], engine=eng)
        assert opt.max_grad_norm is None and opt.grad_norm is None and opt.skipped_steps is None
        for value in (1, 2.5, float("inf")):
            opt = cls([p for _, p in named], engine=eng, max_grad_norm=value)
            assert opt.max_grad_norm == float(value)
            assert opt.grad_norm.dim() == 0 and opt.grad_norm.dtype == torch.float32
            assert opt.skipped_steps.dim() == 0 and opt.skipped_steps.dtype == torch.int32
            assert opt._norm_partials.numel() == opt.n_chunks


# ---------------------------------------------------------------------------------------------------- the launches
def test_none_keeps_the_single_step_launch(golden_dir):
    """max_grad_norm=None: op() is the plain step call with its argument layout, and the plan epilogue is that one op."""
    from vilbert_b200 import _lib as L
    FusedAdamW, FusedRAdam = _classes()
    eng, named = _cpu_engine(golden_dir)
    plan = eng.plan(4, 9, 11, grad_outputs=O.HEAD_NAMES, train=True)
    for cls, fn, n_args in ((FusedAdamW, L.lib().vb_adamw_step, 16), (FusedRAdam, L.lib().vb_radam_step, 18)):
        opt = cls([p for _, p in named], engine=eng)
        f, args = opt.op()
        assert f is fn and len(args) == n_args == len(fn.argtypes) - 1
        (f2, args2), = opt.ops()
        assert f2 is f and [str(a) for a in args2] == [str(a) for a in args]
        plan.enable_optimizer(opt)
        assert len(plan.epilogue) == 1 and plan.epilogue[0][0] is fn and plan.epilogue[0][2] == 0
        assert [str(a) for a in plan.epilogue[0][1]] == [str(a) for a in args]


def test_clipping_is_the_norm_launch_then_the_clipped_step(golden_dir):
    from vilbert_b200 import _lib as L
    FusedAdamW, FusedRAdam = _classes()
    eng, named = _cpu_engine(golden_dir)
    plan = eng.plan(4, 9, 11, grad_outputs=O.HEAD_NAMES, train=True)
    lib = L.lib()
    for cls, step_fn in ((FusedAdamW, lib.vb_adamw_step_clipped), (FusedRAdam, lib.vb_radam_step_clipped)):
        opt = cls([p for _, p in named], engine=eng, max_grad_norm=0.5)
        with pytest.raises(ValueError, match="ops"):
            opt.op()
        (nf, nargs), (sf, sargs) = opt.ops()
        assert nf is lib.vb_grad_norm and sf is step_fn
        assert len(nargs) == len(nf.argtypes) - 1 and len(sargs) == len(sf.argtypes) - 1
        g, cs, cc, n, gsc, mx, part, rec, step = nargs
        assert g == eng.ps.grad.data_ptr() and cs == opt._chunk_start.data_ptr() and cc == opt._chunk_count.data_ptr()
        assert n == opt.n_chunks and mx.value == 0.5 and gsc.value == 1.0
        assert part == opt._norm_partials.data_ptr() and rec == opt._clip_record.data_ptr()
        assert step == opt._step_dev.data_ptr()              # the norm advances the counter, unless it skips
        assert sargs[-1] == opt._clip_record.data_ptr()
        if cls is FusedRAdam:
            assert sargs[-4] == 0                            # advance_step: the norm did it
            # launch(advance_step=False): the norm leaves the counter alone
            assert opt.ops(advance_step=False)[0][1][-1] is None
        plan.enable_optimizer(opt)
        assert [op[0] for op in plan.epilogue] == [nf, sf] and all(op[2] == 0 for op in plan.epilogue)


def test_plan_listing_of_the_clipping_cases(golden_dir):
    """tools/plan_dump.py: the plain optimizer listing is what max_grad_norm=None gives, and the clipping listing is the norm
    launch followed by the clipped step over the same buffers."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import plan_dump as PD
    finally:
        sys.path.pop(0)
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    tiny = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    for cls in _classes():
        plain, none, clip = [], [], []
        PD.dump_optimizer_plan(plain, torch, O, Engine, BertConfig, tiny, "fp16", cls, "t")
        PD.dump_optimizer_plan(none, torch, O, Engine, BertConfig, tiny, "fp16", cls, "t", max_grad_norm=None)
        PD.dump_optimizer_plan(clip, torch, O, Engine, BertConfig, tiny, "fp16", cls, "t", max_grad_norm=1.0)
        assert plain == none
        assert [ln for ln in clip if not ln.startswith("epilogue")] == [ln for ln in plain if not ln.startswith("epilogue")]
        (step,) = [ln for ln in plain if ln.startswith("epilogue")]
        norm_ln, step_ln = [ln for ln in clip if ln.startswith("epilogue")]
        assert norm_ln.startswith("epilogue 0 s0 vb_grad_norm grad+0 opt._chunk_start+0 opt._chunk_count+0 ")
        assert norm_ln.endswith(" 1.0 1.0 opt._norm_partials+0 opt._clip_record+0 opt._step_dev+0")
        name = "vb_adamw_step" if cls.__name__ == "FusedAdamW" else "vb_radam_step"
        expect = step.replace(f"epilogue 0 s0 {name} ", f"epilogue 1 s0 {name}_clipped ")
        if name == "vb_radam_step":
            expect = expect.replace(" opt._step_dev+0 1 ", " opt._step_dev+0 0 ")      # advance_step moves to the norm
        assert step_ln == expect + " opt._clip_record+0"


def test_state_dict_reads_the_device_counter_for_adamw(golden_dir):
    """With clipping the host cannot know which steps were skipped: "step" comes from the device counter (reference layout)."""
    FusedAdamW, _ = _classes()
    eng, named = _cpu_engine(golden_dir)
    opt = FusedAdamW(AO.reference_param_groups(named, base_lr=1e-4), lr=1e-4, engine=eng, max_grad_norm=1.0)
    opt._step_dev.fill_(7)
    sd = opt.state_dict()
    assert all(s["step"] == 7 and set(s) == {"step", "exp_avg", "exp_avg_sq"} for s in sd["state"].values())
    opt2 = FusedAdamW(AO.reference_param_groups(named, base_lr=1e-4), lr=1e-4, engine=eng, max_grad_norm=1.0)
    opt2.load_state_dict(sd)
    assert int(opt2._step_dev.item()) == 7
