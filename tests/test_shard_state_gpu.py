"""Sharded optimizer state (shard_state=True) on the GPU.

Kernels: vb_adamw_step_sharded, vb_radam_step_sharded, vb_grad_norm_partial and vb_clip_finish on the bert_base_6layer_6conect
parameter layout, sliced over three ranks as ddp.shard_slices cuts the reducer's buckets (the middle rank: a non-zero state
offset, slices that start and end inside tensors and so cross group boundaries). The sharded steps over compact moments must
give bitwise what vb_adamw_step / vb_radam_step give over the flat ones (which tests/test_optim_kernels_gpu.py holds to float64),
and the AdamW update is also checked against float64 directly. The partial norm must add up to vb_grad_norm's sum, and
vb_clip_finish must write vb_grad_norm's record.

Training: tests/_shard_state_worker.py, launched like tests/test_retrieval_ddp_gpu.py (one GPU per rank over NCCL; both ranks on
one GPU over gloo), runs sharded and unsharded optimizers side by side; see its docstring for the cases."""
import ctypes as C
import json
import os
import signal
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")
WORKER = os.path.join(ROOT, "tests", "_shard_state_worker.py")


@pytest.fixture(scope="module")
def sharded_layout():
    from vilbert_b200.config import BertConfig
    from vilbert_b200.ddp import FlatGradAllReducer, shard_slices, trainable_ranges
    from vilbert_b200.engine import Engine
    from vilbert_b200.optim import build_chunks, shard_chunks, shard_state_layout
    eng = Engine(BertConfig.from_dict(json.load(open(CONFIG))), "cpu", _build_only=True)
    ps = eng.ps
    names = list(ps.entries)
    ranges = [(ps.span(n)[0], ps.span(n)[1], i % 7) for i, n in enumerate(names)]
    red = FlatGradAllReducer(ps.grad, n_buckets=8)
    red.set_ranges(trainable_ranges(ps, frozenset()))
    layout, total = shard_state_layout(shard_slices(red.table, 3), 1)
    per = shard_chunks(ranges, layout)
    st, ss, cn, gr = (np.concatenate([b[i] for b in per]) for i in range(4))
    full = build_chunks(ranges)
    numel = ps.numel
    del eng, ps, red
    return dict(numel=numel, layout=layout, total=total, sharded=(st, ss, cn, gr), full=full, n_groups=7)


def _groups(n, dev):
    from vilbert_b200.optim import _GROUP_DT, group_row
    g = np.zeros(n, _GROUP_DT)
    for i in range(n):
        g[i] = group_row(1e-3 * (1 + i), (0.9, 0.999 if i % 2 else 0.98), 1e-6, 0.01 * (i % 3), correct_bias=bool(i % 2))
    return torch.from_numpy(g.view(np.uint8).copy()).to(dev)


def _mask(st, cn, numel, dev):
    """The elements the chunk table (start, count) covers."""
    m = torch.zeros(numel, dtype=torch.bool, device=dev)
    for a, k in zip(st.tolist(), cn.tolist()):
        m[a:a + k] = True
    return m


def _state(numel, dev, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    p = torch.randn(numel, generator=gen, device=dev) * 0.02
    g = torch.randn(numel, generator=gen, device=dev) * 1e-2
    m = torch.randn(numel, generator=gen, device=dev) * 1e-3
    v = torch.rand(numel, generator=gen, device=dev) * 1e-4
    return p, g, m, v


@pytest.mark.parametrize("kind", ["adamw", "radam"])
@pytest.mark.parametrize("clip", [False, True])
def test_sharded_step_is_bitwise_the_flat_step(sharded_layout, kind, clip):
    from vilbert_b200 import _lib as L
    lib = L.lib()
    lay, dev = sharded_layout, torch.device("cuda")
    N = lay["numel"]
    p, g, m, v = _state(N, dev, 1)
    groups = _groups(lay["n_groups"], dev)
    st, ss, cn, gr = (torch.from_numpy(x).to(dev) for x in lay["sharded"])
    n_sh = len(lay["sharded"][0])
    assert lay["layout"][0][0] > 0 and lay["layout"][1][2] > 0      # the middle rank: slices start inside buckets, offsets > 0
    # compact moments of this rank's slices
    mc = torch.zeros(max(lay["total"], 4), device=dev)
    vc = torch.zeros_like(mc)
    for lo, hi, base in lay["layout"]:
        mc[base:base + hi - lo] = m[lo:hi]
        vc[base:base + hi - lo] = v[lo:hi]
    # the flat step over the same chunks (their flat offsets) on copies of the buffers
    pf, gf, mf, vf = p.clone(), g.clone(), m.clone(), v.clone()
    copies = [torch.full((N,), 0x5A5A, dtype=torch.int16, device=dev) for _ in range(4)]
    step = [torch.full((1,), 7, dtype=torch.int32, device=dev) for _ in range(2)]
    rec = [torch.zeros(4, dtype=torch.int32, device=dev) for _ in range(2)]
    if clip:                   # a record that clips: coefficient from a norm of 3
        for r in rec:
            r.view(torch.float32)[1] = 0.25
    recp = [r if clip else None for r in rec]
    if kind == "adamw":
        L.call(lib.vb_adamw_step_sharded, p, g, mc, vc, copies[0], None, copies[1], 0, st, ss, cn, gr, n_sh, groups, step[0],
               C.c_float(1.0), 1, recp[0], 0)
        fn = lib.vb_adamw_step_clipped if clip else lib.vb_adamw_step
        L.call(fn, pf, gf, mf, vf, copies[2], None, copies[3], 0, torch.from_numpy(lay["sharded"][0]).to(dev), cn, gr, n_sh, groups,
               step[1], C.c_float(1.0), 1, *([rec[1]] if clip else []))
    else:
        L.call(lib.vb_radam_step_sharded, p, g, mc, vc, copies[0], None, copies[1], 0, st, ss, cn, gr, n_sh, groups, 1, step[0], 1,
               C.c_float(1.0), 1, recp[0], 264)
        fn = lib.vb_radam_step_clipped if clip else lib.vb_radam_step
        L.call(fn, pf, gf, mf, vf, copies[2], None, copies[3], 0, torch.from_numpy(lay["sharded"][0]).to(dev), cn, gr, n_sh, groups,
               1, step[1], 1, C.c_float(1.0), 1, *([rec[1]] if clip else []))
    torch.cuda.synchronize()
    assert torch.equal(step[0], step[1])
    assert torch.equal(p, pf) and torch.equal(g, gf) and torch.equal(copies[0], copies[2]) and torch.equal(copies[1], copies[3])
    for lo, hi, base in lay["layout"]:
        assert torch.equal(mc[base:base + hi - lo], mf[lo:hi]) and torch.equal(vc[base:base + hi - lo], vf[lo:hi])
    if kind == "adamw" and not clip:
        # float64: the update of every element of the slices, from the group table's hyper-parameters
        from vilbert_b200.optim import _GROUP_DT
        gt = groups.cpu().numpy().view(_GROUP_DT)
        p0, g0, m0, v0 = _state(N, dev, 1)
        stt, cnt, grt = lay["sharded"][0], lay["sharded"][2], lay["sharded"][3]
        gmap = torch.full((N,), -1, dtype=torch.int64, device=dev)
        for a, k, q in zip(stt.tolist(), cnt.tolist(), grt.tolist()):
            gmap[a:a + k] = q
        elem = (gmap >= 0).nonzero().squeeze(1)
        grp = gmap[elem]
        col = lambda f: torch.from_numpy(np.asarray(gt[f], np.float64)).to(dev)[grp]
        lr, b1, b2, eps, wd, cb = (col(f) for f in ("lr", "beta1", "beta2", "eps", "weight_decay", "correct_bias"))
        ob1, ob2 = col("one_minus_beta1"), col("one_minus_beta2")
        t = 7.0                # AdamW reads the counter its caller advanced
        gg = g0[elem].double()
        mm = b1 * m0[elem].double() + ob1 * gg
        vv = b2 * v0[elem].double() + ob2 * gg * gg
        ss_ = torch.where(cb > 0, lr * torch.sqrt(1 - (1 - ob2) ** t) / (1 - (1 - ob1) ** t), lr)
        pp = (p0[elem].double() - ss_ * mm / (vv.sqrt() + eps)) * (1 - lr * wd)
        d_ref = pp - p0[elem].double()
        d_got = p[elem].double() - p0[elem].double()
        err = ((d_got - d_ref).abs() / d_ref.abs().clamp_min(1e-12)).median()
        # the fp32 weight rounds the update to half an ulp of |p| (twice: update, then decay); m, v and the step add a few ulps, of
        # m's terms rather than of m where they cancel
        m_err = 2.5e-7 * (b1 * m0[elem].double().abs() + ob1 * gg.abs())
        tol = 2e-6 * d_ref.abs() + 4e-7 * p0[elem].double().abs() + ss_ * m_err / (vv.sqrt() + eps)
        bad = ((d_got - d_ref).abs() > tol).sum()
        assert err < 1e-5 and int(bad) == 0, (float(err), int(bad))


def test_partial_norm_and_clip_finish_match_grad_norm(sharded_layout):
    from vilbert_b200 import _lib as L
    lib = L.lib()
    lay, dev = sharded_layout, torch.device("cuda")
    N = lay["numel"]
    _, g, _, _ = _state(N, dev, 2)
    st, cn, _ = (torch.from_numpy(x).to(dev) for x in lay["full"])
    n = len(lay["full"][0])
    partials = torch.zeros(n, dtype=torch.float64, device=dev)
    rec_a, rec_b = torch.zeros(4, dtype=torch.int32, device=dev), torch.zeros(4, dtype=torch.int32, device=dev)
    step_a, step_b = torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    L.call(lib.vb_grad_norm, g, st, cn, n, C.c_float(0.5), C.c_float(1.0), partials, rec_a, step_a)
    s = torch.zeros(1, dtype=torch.float64, device=dev)
    L.call(lib.vb_grad_norm_partial, g, st, cn, n, partials, s)
    L.call(lib.vb_clip_finish, s, C.c_float(0.5), C.c_float(1.0), rec_b, step_b)
    torch.cuda.synchronize()
    assert torch.equal(rec_a, rec_b) and int(step_b) == 1
    ref = float((g.double() ** 2)[_mask(lay["full"][0], lay["full"][1], N, dev)].sum())
    assert abs(float(s) - ref) <= 1e-12 * ref
    # this rank's slices: the partial sum over the sharded table is the float64 sum over the slices' trainable elements
    sst, _, scn, _ = lay["sharded"]
    sp = torch.zeros(len(sst), dtype=torch.float64, device=dev)
    L.call(lib.vb_grad_norm_partial, g, torch.from_numpy(sst).to(dev), torch.from_numpy(scn).to(dev), len(sst), sp, s)
    ref = float((g.double() ** 2)[_mask(sst, scn, N, dev)].sum())
    torch.cuda.synchronize()
    assert abs(float(s) - ref) <= 1e-12 * ref
    # a non-finite sum skips: counter unchanged, skipped counted, coefficient 0
    s.fill_(float("inf"))
    L.call(lib.vb_clip_finish, s, C.c_float(1.0), C.c_float(1.0), rec_b, step_b)
    torch.cuda.synchronize()
    assert int(step_b) == 1 and int(rec_b[2]) == 1 and int(rec_b[3]) == 1 and float(rec_b.view(torch.float32)[1]) == 0.0


# ------------------------------------------------------------------------------------------ two ranks
def _launch(tmp_path, backend, port):
    out = tmp_path / f"shard_state_{backend}.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), WORKER, str(out), backend]
    # own process group: on a timeout the launcher and both ranks are ended together, nothing is left running
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, start_new_session=True)
    try:
        _, err = proc.communicate(timeout=900)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        proc.communicate()
        pytest.fail(f"the 2-rank shard_state worker ({backend}) did not finish within 900 s")
    assert proc.returncode == 0, err[-4000:]
    return json.load(open(out))


def _check(ranks):
    from _shard_state_worker import CASES
    r0, r1 = ranks
    assert set(r0) == set(r1) == set(CASES)
    for name in CASES:
        for rank, res in enumerate(ranks):
            r = res[name]
            if name == "reload":
                assert all(r["step_equal"]) and r["state_equal"] and r["mid_equal"], (name, rank, r)
                continue
            assert all(r["ranks_equal"]), (name, rank, r)
            if r["det"] and r["exact"]:
                assert all(r["step_equal"]) and r["state_equal"], (name, rank, r)
            elif r["det"]:           # clipping: a norm summed in another order, the coefficient within an ulp
                assert r["rel"] <= 1e-6 and r["state_rel"] <= 1e-5, (name, rank, r)
            else:                    # default mode: each step from the unsharded run's state (_run_lockstep)
                assert r["rel"] <= 1e-6 and r["state_rel"] <= 1e-5, (name, rank, r)
            assert r["moments"] <= r["bound"], (name, rank, r)
            if "skip" in name:
                assert r["skipped"] == 1, (name, rank, r)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_over_nccl_match_the_unsharded_optimizer(tmp_path):
    _check(_launch(tmp_path, "nccl", 29571))


def test_two_ranks_on_one_gpu_over_gloo_match_the_unsharded_optimizer(tmp_path):
    _check(_launch(tmp_path, "gloo", 29573))
