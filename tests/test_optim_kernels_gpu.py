"""The fused optimizer entry points through the C ABI, update by update against float64, on the production parameter layout.

vb_adamw_step, vb_radam_step, vb_grad_norm, vb_adamw_step_clipped and vb_radam_step_clipped run over the chunk table of every
bert_base_6layer_6conect tensor (optim.build_chunks, 268M elements in ~8.5k chunks: more chunks than the 8 x SMs CTAs of the
grid, so CTAs stride to further chunks; ragged 3129- / 1533- / 1601-entry tails and 1-, 2-, 3-element head biases that only
reach the scalar path) with one group per tensor. The state is synthetic and per element mixes ordinary gradients, exact zeros,
gradients with sqrt(v) far below and far above eps, 1e-20 (g^2 underflows) and 1e15, fresh (zero) and running moments, and
p0 = 0 on a quarter of the elements so that the update itself is compared, relative to its own size. The tolerances and the
wrong references each case must reject are derived in tests/_optim_ref.py. The float64 reference runs over blocks of 4M
elements of the flat buffer, so beside the buffers themselves (~11 GB) it holds about 2 GB whatever the model.
"""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

import _clip_oracle as CO
import _optim_ref as R
from _gpu_util import launched

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")
BLOCK = 1 << 22
SENTINEL = 0x5A5A                     # 16-bit copy buffers start filled with this: a copy not asked for stays so
PAD = dict(p=7.0, g=1e3, m=0.5, v=0.25)   # padding between tensors: no chunk covers it, nothing may touch it
SLIPS = {"adamw": [s for s in R.SLIPS if s != "own_group_step"], "radam": list(R.SLIPS)}


def _lib():
    from vilbert_b200 import _lib as L
    return L


class Layout:
    pass


@pytest.fixture(scope="module")
def layout():
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    from vilbert_b200.optim import build_chunks
    eng = Engine(BertConfig.from_dict(json.load(open(CONFIG))), "cpu", _build_only=True)
    ps = eng.ps
    base = ps.flat.data_ptr()
    lay = Layout()
    lay.names = list(ps.entries)
    lay.ranges = [((ps.p(n).data_ptr() - base) // 4, ps.p(n).numel(), i) for i, n in enumerate(lay.names)]
    lay.numel = ps.numel
    del eng, ps
    st, cn, gr = build_chunks(lay.ranges)
    lay.chunks = (st, cn, gr)
    dev = torch.device("cuda")
    torch.cuda.reset_peak_memory_stats()
    lay.cs, lay.cc, lay.cg = (torch.from_numpy(x).to(dev) for x in (st, cn, gr))
    lay.n_chunks = len(st)
    N = lay.numel
    lay.gidx = torch.full((N,), -1, dtype=torch.int16, device=dev)
    for off, n, i in lay.ranges:
        lay.gidx[off:off + n] = i
    gen = torch.Generator(device=dev).manual_seed(0)
    # ordinary x4, exact zero, sqrt(v) << eps, g^2 underflowing, huge
    scales = torch.tensor([1e-2] * 4 + [0.0, 1e-12, 1e-20, 1e15], device=dev)
    lay.p0, lay.g0, lay.m0, lay.v0 = (torch.empty(N, device=dev) for _ in range(4))
    for s in range(0, N, BLOCK):
        e = min(N, s + BLOCK)
        n = e - s
        cls = torch.randint(0, 8, (n,), generator=gen, device=dev)
        sc = scales[cls]
        st_sc = torch.where(cls == 4, 1e-2, sc)            # zero gradients still carry running moments
        fresh = torch.rand(n, generator=gen, device=dev) < 1 / 3
        pad = lay.gidx[s:e] < 0
        lay.g0[s:e] = torch.randn(n, generator=gen, device=dev) * sc
        lay.m0[s:e] = torch.where(fresh, 0.0, 0.3 * torch.randn(n, generator=gen, device=dev) * st_sc)
        lay.v0[s:e] = torch.where(fresh, 0.0, st_sc * st_sc * (0.1 + torch.rand(n, generator=gen, device=dev)))
        lay.p0[s:e] = torch.where(torch.rand(n, generator=gen, device=dev) < 0.25, 0.0,
                                  0.05 * torch.randn(n, generator=gen, device=dev) + 1e-3)
        for k, x in (("p", lay.p0), ("g", lay.g0), ("m", lay.m0), ("v", lay.v0)):
            x[s:e][pad] = PAD[k]
    lay.p, lay.g, lay.m, lay.v = (torch.empty(N, device=dev) for _ in range(4))
    lay.p16, lay.lo, lay.b16 = (torch.empty(N, dtype=torch.int16, device=dev) for _ in range(3))
    lay.step = torch.zeros(1, dtype=torch.int32, device=dev)
    yield lay
    print(f"\ntest_optim_kernels_gpu: peak CUDA memory allocated {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB on "
          f"{torch.cuda.get_device_name()}")


def _reset(lay):
    for x, x0 in ((lay.p, lay.p0), (lay.g, lay.g0), (lay.m, lay.m0), (lay.v, lay.v0)):
        x.copy_(x0)
    for b in (lay.p16, lay.lo, lay.b16):
        b.fill_(SENTINEL)


def _group_table(groups):
    from vilbert_b200.optim import _GROUP_DT, group_row
    rows = np.array([group_row(g["lr"], g["betas"], g["eps"], g["weight_decay"], g["correct_bias"]) for g in groups], dtype=_GROUP_DT)
    return torch.from_numpy(rows.view(np.uint8).copy()).cuda()


def _copy_args(lay, copies):
    hi, lo, b = copies
    return (lay.p16 if hi is not None else None, lay.lo if (hi is not None and lo) else None, lay.b16 if b else None,
            1 if hi is torch.float16 else 0)


def _launch(kind, lay, groups, copies, grad_scale, zero_grad, leader=0, rec=None, advance_step=0, n_chunks=None):
    L = _lib()
    lib = L.lib()
    n_chunks = lay.n_chunks if n_chunks is None else n_chunks
    args = (lay.p, lay.g, lay.m, lay.v, *_copy_args(lay, copies), lay.cs, lay.cc, lay.cg, n_chunks, _group_table(groups))
    tail = (C.c_float(grad_scale), 1 if zero_grad else 0)
    if kind == "adamw":
        fn, a = (lib.vb_adamw_step, args + (lay.step,) + tail) if rec is None else (lib.vb_adamw_step_clipped, args + (lay.step,) + tail + (rec,))
    else:
        a = args + (leader, lay.step, advance_step) + tail
        fn, a = (lib.vb_radam_step, a) if rec is None else (lib.vb_radam_step_clipped, a + (rec,))
    L.call(fn, *a)
    torch.cuda.synchronize()


def _check(kind, lay, groups, t, grad_scale, copies, zero_grad, leader=0, clip=False, slips=()):
    """Compares the kernel's p, m, v, g and 16-bit copies with the float64 step from (p0, g0, m0, v0); returns the worst error
    over tolerance per quantity and, per slip, by how much its wrong reference misses the right one (in tolerances)."""
    dev = lay.p.device
    tab = lambda vals, dt=torch.float64: torch.tensor(vals, dtype=dt, device=dev)   # noqa: E731
    LR, WD, EPS = tab([g["lr"] for g in groups]), tab([g["weight_decay"] for g in groups]), tab([g["eps"] for g in groups])
    B1, B2 = tab([g["betas"][0] for g in groups]), tab([g["betas"][1] for g in groups])
    scal = {s: R.group_scalars(kind, groups, leader, t, s) for s in (None,) + tuple(slips)}
    SS = {s: tab([x[0] for x in v]) for s, v in scal.items()}
    RECT = {s: tab([x[1] for x in v], torch.bool) for s, v in scal.items()}
    worst = dict(m=0.0, v=0.0, p=0.0)
    miss = {s: 0.0 for s in slips}
    hi, want_lo, want_b = copies
    for s in range(0, lay.numel, BLOCK):
        e = min(lay.numel, s + BLOCK)
        gi = lay.gidx[s:e].long()
        valid = gi >= 0
        inv = ~valid
        gi.clamp_(min=0)
        hp = dict(lr=LR[gi], wd=WD[gi], b1=B1[gi], b2=B2[gi], eps=EPS[gi])
        p0, g0, m0, v0 = (x[s:e].double() for x in (lay.p0, lay.g0, lay.m0, lay.v0))
        pr, mr, vr, dmag, mmag, p1 = R.step(kind, p0, g0, m0, v0, dict(hp, ss=SS[None][gi], rect=RECT[None][gi]), grad_scale)
        tols = R.tolerances(p0, pr, mmag, vr, dmag, p1, clip)
        pk, mk, vk, gk = lay.p[s:e], lay.m[s:e], lay.v[s:e], lay.g[s:e]
        for name, k in (("p", pk), ("m", mk), ("v", vk)):
            assert torch.isfinite(k[valid]).all(), (name, s)
        for name, k, r, tol in (("m", mk, mr, tols[0]), ("v", vk, vr, tols[1]), ("p", pk, pr, tols[2])):
            worst[name] = max(worst[name], torch.where(valid, (k.double() - r).abs() / tol, 0.0).max().item())
        for k, k0 in ((pk, lay.p0), (mk, lay.m0), (vk, lay.v0), (gk, lay.g0)):
            assert torch.equal(k[inv], k0[s:e][inv]), "an element between tensors was written"
        if zero_grad:
            assert (gk[valid] == 0).all()
        else:
            assert torch.equal(gk, lay.g0[s:e])
        # the 16-bit copies: bitwise the casts of the kernel's own fp32 weights, on the float4 and the scalar-tail path alike
        sent = lambda b: (b[s:e] == SENTINEL).all().item()          # noqa: E731
        if hi is not None:
            h = pk.to(hi)
            assert torch.equal(lay.p16[s:e][valid], h.view(torch.int16)[valid]) and (lay.p16[s:e][inv] == SENTINEL).all()
            if want_lo:
                lo = (pk - h.float()).to(hi)
                assert torch.equal(lay.lo[s:e][valid], lo.view(torch.int16)[valid]) and (lay.lo[s:e][inv] == SENTINEL).all()
            else:
                assert sent(lay.lo)
        else:
            assert sent(lay.p16) and sent(lay.lo)
        if want_b:
            assert torch.equal(lay.b16[s:e][valid], pk.to(torch.bfloat16).view(torch.int16)[valid]) and (lay.b16[s:e][inv] == SENTINEL).all()
        else:
            assert sent(lay.b16)
        for slip in slips:
            pw, mw, vw, _, _, _ = R.step(kind, p0, g0, m0, v0, dict(hp, ss=SS[slip][gi], rect=RECT[slip][gi]), grad_scale, slip)
            for w, r, tol in ((mw, mr, tols[0]), (vw, vr, tols[1]), (pw, pr, tols[2])):
                miss[slip] = max(miss[slip], torch.where(valid, (w - r).abs() / tol, 0.0).max().item())
    return worst, miss


def _assert_case(kind, lay, case, clip=False, grad_scale=None):
    groups = R.groups_for(lay.names, kind, case)
    gs = case["grad_scale"] if grad_scale is None else grad_scale
    slips = [s for s in SLIPS[kind] if R.applicable(kind, groups, 0, case["t"], case["grad_scale"], s)]
    worst, miss = _check(kind, lay, groups, case["t"], gs, case["copies"], case["zero_grad"], clip=clip, slips=slips)
    assert all(w <= 1.0 for w in worst.values()), f"error / tolerance {worst}"
    missed = {s: x for s, x in miss.items() if not x > R.MISS}
    assert not missed, f"wrong references within {R.MISS} x the tolerance: {missed}"
    return worst, miss


# ---------------------------------------------------------------------------------------------------- the layout
def test_layout_is_the_production_chunk_table(layout):
    st, cn, gr = layout.chunks
    grid = 8 * torch.cuda.get_device_properties(0).multi_processor_count
    assert layout.n_chunks > grid                       # CTAs take further chunks by their grid stride
    # a tensor whose chunks are some CTAs' first chunks and other CTAs' second ones
    idx = np.arange(len(st))
    assert any((idx[gr == i] < grid).any() and (idx[gr == i] >= grid).any() for i in np.unique(gr))
    assert (cn % 4 != 0).any() and (cn < 4).any()        # ragged tails and biases that only the scalar path reaches
    assert len(layout.names) == len(layout.ranges) == int(gr.max()) + 1


# ---------------------------------------------------------------------------------------------------- the steps
@pytest.mark.parametrize("case", R.cases("adamw"), ids=R.case_id)
def test_adamw_step_matches_float64(layout, case):
    _reset(layout)
    layout.step.fill_(case["t"])
    groups = R.groups_for(layout.names, "adamw", case)
    _launch("adamw", layout, groups, case["copies"], case["grad_scale"], case["zero_grad"])
    assert layout.step.item() == case["t"]
    _assert_case("adamw", layout, case)


@pytest.mark.parametrize("case", R.cases("radam"), ids=R.case_id)
def test_radam_step_matches_float64(layout, case):
    """The leader group (the first tensor's) has its own lr and betas: its rectified step size drives every tensor."""
    _reset(layout)
    layout.step.fill_(case["t"] - 1)
    groups = R.groups_for(layout.names, "radam", case)
    _launch("radam", layout, groups, case["copies"], case["grad_scale"], case["zero_grad"], advance_step=1)
    assert layout.step.item() == case["t"]
    _assert_case("radam", layout, case)


def test_adamw_step_counter_zero_steps_like_one(layout):
    """A counter still at 0 with correct_bias would make 1 - b1^0 = 0 the divisor: the kernel clamps t to 1, as RAdam does."""
    case = dict(R.cases("adamw")[0])
    assert case["t"] == 1 and case["correct_bias"]
    groups = R.groups_for(layout.names, "adamw", case)
    n = int(layout.chunks[0][64])                       # the first 64 chunks (word embeddings) are enough for a scalar
    out = []
    for t in (0, 1):
        _reset(layout)
        layout.step.fill_(t)
        _launch("adamw", layout, groups, case["copies"], case["grad_scale"], case["zero_grad"], n_chunks=64)
        out.append([x[:n].clone() for x in (layout.p, layout.m, layout.v, layout.p16, layout.lo, layout.b16)])
    assert torch.isfinite(out[0][0]).all() and not torch.equal(out[0][0], layout.p0[:n])
    assert all(torch.equal(a, b) for a, b in zip(*out))


# ---------------------------------------------------------------------------------------------------- norm, clip and skip
@pytest.mark.parametrize("kind", ["adamw", "radam"])
def test_grad_norm_and_clipped_step_match_clip_then_step(layout, kind):
    """vb_grad_norm: the float64 norm of grad_scale g over the chunks (the 1e3 padding outside them excluded) rounded once,
    torch's clip coefficient from it, the counter advanced; the clipped step is the float64 step on grad_scale coef g."""
    L = _lib()
    case = dict(R.cases(kind)[4 if kind == "adamw" else 12], grad_scale=0.25, zero_grad=True)
    t = case["t"]
    _reset(layout)
    layout.step.fill_(t - 1)
    s2 = sum(float(layout.g0[s:e][layout.gidx[s:e] >= 0].double().square().sum())
             for s, e in ((s, min(layout.numel, s + BLOCK)) for s in range(0, layout.numel, BLOCK)))
    ref = 0.25 * math.sqrt(s2)
    max_norm = ref / 3
    partials = torch.zeros(layout.n_chunks, dtype=torch.float64, device="cuda")
    rec = torch.zeros(4, dtype=torch.int32, device="cuda")
    L.call(L.lib().vb_grad_norm, layout.g, layout.cs, layout.cc, layout.n_chunks, C.c_float(0.25), C.c_float(max_norm), partials,
           rec, layout.step)
    torch.cuda.synchronize()
    norm, coef = (float(x) for x in rec.view(torch.float32)[:2].tolist())
    assert abs(norm - ref) <= 2 * R.U * ref, (norm, ref)
    assert coef == CO.clip_coefficient(norm, float(np.float32(max_norm))) and 0.3 < coef < 0.34
    assert rec[2].item() == 0 and rec[3].item() == 0 and layout.step.item() == t
    groups = R.groups_for(layout.names, kind, case)
    _launch(kind, layout, groups, case["copies"], 0.25, True, rec=rec)
    _assert_case(kind, layout, case, clip=True, grad_scale=0.25 * coef)


@pytest.mark.parametrize("kind", ["adamw", "radam"])
def test_skip_record_leaves_the_state_and_zeroes_the_gradient(layout, kind):
    L = _lib()
    case = R.cases(kind)[5]
    _reset(layout)
    st, cn, _ = layout.chunks
    layout.g[int(st[-1]) + int(cn[-1]) - 1] = float("nan")      # the last element of the last chunk: a scalar-tail element
    layout.step.fill_(9)
    partials = torch.zeros(layout.n_chunks, dtype=torch.float64, device="cuda")
    rec = torch.zeros(4, dtype=torch.int32, device="cuda")
    L.call(L.lib().vb_grad_norm, layout.g, layout.cs, layout.cc, layout.n_chunks, C.c_float(1.0), C.c_float(1.0), partials, rec,
           layout.step)
    torch.cuda.synchronize()
    assert rec[2].item() == 1 and rec[3].item() == 1 and layout.step.item() == 9
    _launch(kind, layout, R.groups_for(layout.names, kind, case), R.COPIES[0], 1.0, True, rec=rec)
    assert layout.step.item() == 9
    for x, x0 in ((layout.p, layout.p0), (layout.m, layout.m0), (layout.v, layout.v0)):
        assert torch.equal(x, x0)
    assert all((b == SENTINEL).all() for b in (layout.p16, layout.lo, layout.b16))
    valid = layout.gidx >= 0
    assert (layout.g[valid] == 0).all() and torch.equal(layout.g[~valid], layout.g0[~valid])


# ---------------------------------------------------------------------------------------------------- refusals
def test_misaligned_buffers_are_refused_without_a_launch():
    """Each fp32 buffer 4 bytes off its 16-byte alignment, each 16-bit copy 2 bytes off its 8: every step entry point returns
    VB_ERR_INVALID, launches no kernel and leaves the step counter (RAdam's advance_step included) as it was."""
    L = _lib()
    lib = L.lib()
    n = 1024 + 3
    f = lambda: torch.zeros(n + 8, device="cuda")                        # noqa: E731
    h = lambda: torch.zeros(n + 8, dtype=torch.int16, device="cuda")     # noqa: E731
    bufs = dict(p=f(), g=f(), m=f(), v=f(), p16=h(), lo=h(), b16=h())
    cs = torch.zeros(1, dtype=torch.int64, device="cuda")
    cc = torch.full((1,), n, dtype=torch.int32, device="cuda")
    cg = torch.zeros(1, dtype=torch.int32, device="cuda")
    groups = _group_table([dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01, correct_bias=True)])
    step = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    rec = torch.zeros(4, dtype=torch.int32, device="cuda")
    partials = torch.zeros(1, dtype=torch.float64, device="cuda")

    def calls():
        out = []
        for bad in bufs:
            a = {k: (b[1:] if k == bad else b) for k, b in bufs.items()}
            head = (a["p"], a["g"], a["m"], a["v"], a["p16"], a["lo"], a["b16"], 1, cs, cc, cg, 1, groups)
            for fn, extra in ((lib.vb_adamw_step, (step, C.c_float(1.0), 1)),
                              (lib.vb_adamw_step_clipped, (step, C.c_float(1.0), 1, rec)),
                              (lib.vb_radam_step, (0, step, 1, C.c_float(1.0), 1)),
                              (lib.vb_radam_step_clipped, (0, step, 1, C.c_float(1.0), 1, rec))):
                out.append((fn.__name__, bad, fn(*L.launch_args(fn, *head, *extra), None)))
        fn = lib.vb_grad_norm
        out.append((fn.__name__, "g", fn(*L.launch_args(fn, bufs["g"][1:], cs, cc, 1, C.c_float(1.0), C.c_float(1.0), partials, rec,
                                                         step), None)))
        return out

    out, names = launched(calls)
    assert all(st == L.VB_ERR_INVALID for _, _, st in out), [o for o in out if o[2] != L.VB_ERR_INVALID]
    assert not [nm for nm in names if "vb::" in nm], sorted(set(names))
    assert step.item() == 5 and rec.abs().sum().item() == 0
