"""Deterministic plans on the GPU, with torch.use_deterministic_algorithms(True) set by this module's fixture: the same seeded work
gives bitwise identical losses, gradients and parameters eagerly, as a CUDA graph, with another plan run in between and in another
process, and stays within the default path's tolerances."""
import gc
import json
import os
import subprocess
import sys

import pytest
import torch

from _gpu_util import rel_l2
from oracle import vilbert_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import deterministic_probe as P  # noqa: E402

pytestmark = pytest.mark.gpu
FROZEN_TEXT = ("bert.embeddings.", "bert.encoder.layer.")


@pytest.fixture(autouse=True)
def release_engines():
    """Engines of earlier tests hold each other in reference cycles: collect them, an 80 GB card holds only a few config-2 engines."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True, scope="module")
def deterministic_algorithms():
    prev, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn_only)


def _equal(a, b):
    assert a.keys() == b.keys()
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, f"not bitwise equal: {diff}"


def _three_ways(eng, plan, other):
    """One step eagerly, one with `other` run in between, one as CUDA graphs: all bitwise equal."""
    r0 = P.step(eng, plan)
    other.run_forward()
    other.run_backward()
    r1 = P.step(eng, plan)
    plan.capture(separate=True)
    r2 = P.step(eng, plan)
    _equal(r0, r1)
    _equal(r0, r2)
    assert torch.isfinite(r0["grad"]).all()
    return r0


def _optimizer_steps(eng, plan, n=3, drop_step=11):
    """n training steps with a fresh FusedAdamW(max_grad_norm=1.0) from the current parameters at dropout step `drop_step` ->
    the parameters after them; the parameters, their 16-bit copy and the gradients are restored, so a second call starts from the
    same state."""
    p0 = eng.ps.flat.clone()
    eng.set_dropout_step(drop_step)
    eng.refresh_weights()
    eng.zero_grad(force=True)
    plan.enable_optimizer(P.optimizer(eng, max_grad_norm=1.0))
    for _ in range(n):
        plan.run_step()
    torch.cuda.synchronize()
    out = eng.ps.flat.clone()
    eng.ps.flat.copy_(p0)
    eng.refresh_weights()
    eng.zero_grad(force=True)
    return out


CASES = {
    "config2": dict(kind="vqa"),
    "pretraining_vt0": dict(kind="pretraining", Nv=37),
    "pretraining_vt2": dict(kind="pretraining", Nv=37, visual_target=2, v_target_size=2048),   # regresses the region features
    "fp32_split_precision": dict(kind="vqa", B=16, precision="fp32"),
    "bf16": dict(kind="vqa", B=16, precision="bf16"),
}


@pytest.mark.parametrize("name", list(CASES))
def test_reproducible_at_production_shapes(name):
    kw = CASES[name]
    eng, plan = P.build(deterministic=None, **kw)     # None: the flag of the fixture
    assert plan.det
    other = eng.plan(8, 20, 30, grad_outputs=plan.grad_outputs, loss=plan.loss_kind, train=True,
                     loss_in_forward=plan.loss_in_forward)
    P.load(other, kw["kind"], 5, dict(P.bench_config(), **{k: v for k, v in kw.items() if k in ("visual_target", "v_target_size")}))
    _three_ways(eng, plan, other)
    first = _optimizer_steps(eng, plan)
    eng.zero_grad(force=True)
    # a fresh engine from the same seed takes the same optimizer steps (the optimizer state starts from zero again)
    eng2, plan2 = P.build(deterministic=True, **kw)
    P.step(eng2, plan2)
    second = _optimizer_steps(eng2, plan2)
    assert torch.equal(first, second)


def test_frozen_text_stream_with_input_grads():
    from vilbert_b200.engine import INPUT_GRAD_NAMES, LOSS_HEADS
    eng, _ = P.build(kind="vqa", deterministic=True, B=64)
    frozen = frozenset(n for n in eng.ps.entries if n.startswith(FROZEN_TEXT))
    plan = eng.plan(64, 36, 100, grad_outputs=LOSS_HEADS["vqa"], loss="vqa", train=True, frozen=frozen,
                    input_grads=frozenset(INPUT_GRAD_NAMES))
    assert plan.det
    P.load(plan, "vqa", 3, P.bench_config())
    other = eng.plan(8, 20, 30, grad_outputs=LOSS_HEADS["vqa"], loss="vqa", train=True)
    P.load(other, "vqa", 5, P.bench_config())
    r = _three_ways(eng, plan, other)
    assert "input_grad.input_imgs" in r and "input_grad.image_loc" in r
    assert torch.equal(_optimizer_steps(eng, plan), _optimizer_steps(eng, plan))     # from the same parameters and a fresh optimizer


def test_packed_task_step():
    """A packed ForwardModelsTrain-style step (engine.pack_padding shapes: the valid rows only) is reproducible too."""
    from vilbert_b200.engine import LOSS_HEADS, pack_capacity
    eng, padded = P.build(kind="vqa", deterministic=True, B=64)
    rows_t = int(padded.in_amask.sum().item())
    rows_v = int(padded.in_imask.sum().item())
    plan = eng.plan(64, 36, 100, grad_outputs=LOSS_HEADS["vqa"], loss="vqa", train=True, outputs=LOSS_HEADS["vqa"],
                    packed=(rows_t, rows_v))
    assert plan.det
    P.load(plan, "vqa", 0, P.bench_config())
    r = _three_ways(eng, plan, padded)
    # the packed and the padded deterministic plans agree as the packed tests ask of the default path
    rp = P.step(eng, padded)
    _same_grads(eng, rp["grad"], r["grad"])
    assert torch.equal(_optimizer_steps(eng, plan), _optimizer_steps(eng, plan))


@pytest.mark.parametrize("kind", ["vqa", "pretraining"])
def test_deterministic_gradients_match_default(kind):
    kw = dict(kind=kind, B=32) if kind == "vqa" else dict(kind=kind, B=32, Nv=37)
    eng, det = P.build(deterministic=True, **kw)
    rd = P.step(eng, det)
    eng2, default = P.build(deterministic=False, **kw)
    assert not default.det
    r = P.step(eng2, default)
    _same_grads(eng, r["grad"], rd["grad"])
    for k in ("loss", "objective_out"):
        if k in r:
            assert torch.allclose(rd[k], r[k], rtol=1e-3, atol=1e-4), (k, rd[k], r[k])


def _same_grads(eng, g0, g1, bound=2e-3):
    """Every parameter's gradient within `bound` relative L2 (those above 1e-3 of the largest gradient entry)."""
    ps = eng.ps
    gmax = g0.abs().max().item()
    worst = max((rel_l2(g1[o:o + n], g0[o:o + n]), k) for k, (o, n) in ((k, ps.span(k)) for k in ps.entries)
                if g0[o:o + n].abs().max().item() > 1e-3 * gmax)
    assert worst[0] < bound, worst
    assert torch.isfinite(g1).all()


@pytest.mark.parametrize("B,Nv,Nt,seed,task,step,precision", [(4, 11, 9, 0, False, None, "fp16"), (3, 7, 12, 1, True, None, "fp16"),
                                                              (2, 37, 21, 2, False, None, "fp16"), (6, 33, 24, 4, True, None, "fp16"),
                                                              (4, 11, 9, 0, False, 3, "fp16"), (6, 33, 24, 4, False, 123456, "fp16"),
                                                              (6, 33, 24, 4, True, None, "fp32"), (6, 33, 24, 4, True, None, "bf16")])
def test_oracle_contract(golden_dir, B, Nv, Nt, seed, task, step, precision):
    """Deterministic plans meet the fp32-oracle contract of test_model_gpu.py at its sizes: every output and parameter gradient,
    eval and train mode (the oracle applies the kernels' dropout masks), the three precisions. The oracle's own torch ops run with
    warn_only=True; the engine still sees the flag on and builds deterministic plans."""
    from _gpu_util import model_case
    from test_model_gpu import _check
    cfgj = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], task_specific_tokens=task)
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        r = model_case(cfgj, B, Nv, Nt, seed=seed, train_step=step, precision=precision)
    finally:
        torch.use_deterministic_algorithms(True)
    assert r["plan"].det
    if precision == "fp16":
        _check(r)
    else:
        _check(r, precision, modes=("fp32",), grad_worst=5e-2 if precision == "bf16" else 2e-2,
               grad_median=2e-2 if precision == "bf16" else 1e-2)


def _module_step(model, cfg, seed=0):
    import torch.nn.functional as F
    inp = O.synth_inputs(cfg, 4, 11, 9, seed=seed, device="cuda")
    args = [inp[k] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")]
    model.zero_grad(set_to_none=False)
    out = model(*args, None, inp["task_ids"])
    tgt = O.synth_vqa_target(4, 3129, seed=seed, device="cuda")
    loss = F.binary_cross_entropy_with_logits(out[0], tgt) + 0.1 * out[2].float().pow(2).mean()
    loss.backward()
    torch.cuda.synchronize()
    return [loss.detach().clone()] + [o.detach().clone() for o in out if torch.is_tensor(o)] + \
        [p.grad.clone() for p in model.parameters() if p.grad is not None]


def test_module_surface(golden_dir):
    """VILBertForVLTasks forward + loss.backward() under the flag: the module surface builds deterministic plans, and five train-mode
    steps at one dropout step give bitwise identical losses, outputs and .grad (eager runs, then the captured passes)."""
    import vilbert_b200
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    cfg = O.make_config(cfgj)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.load_state_dict(O.synth_params(cfg, seed=3, device="cuda"), strict=False)
    model.train()
    eng = model.engine
    runs = []
    for _ in range(5):
        eng.set_dropout_step(7)
        runs.append(_module_step(model, cfg))
    assert all(p.det for p in eng.plans.values())
    for r in runs[1:]:
        assert len(r) == len(runs[0]) and all(torch.equal(a, b) for a, b in zip(runs[0], r))


def test_across_processes(tmp_path):
    here = P.hash_run()
    hashes = []
    for i in range(2):
        out = tmp_path / f"hash{i}.txt"
        subprocess.run([sys.executable, os.path.join(ROOT, "tools", "deterministic_probe.py"), "--hash", str(out)], check=True,
                       cwd=ROOT, timeout=900)
        hashes.append(out.read_text().strip())
    assert hashes[0] == hashes[1] == here
