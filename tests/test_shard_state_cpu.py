"""Sharded optimizer state (FusedAdamW / FusedRAdam shard_state=True) without a GPU: the bucket slices (ddp.shard_slices), the
compact state layout and its chunk tables, the reducer's reduce-scatter and all-gather over three gloo ranks on CPU tensors (padded buckets included), the
refusals, and the host-side state_dict assembly against the unsharded layout."""
import json
import os
import sys
import time
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cpu_engine():
    from vilbert_b200 import engine as E
    from vilbert_b200.config import BertConfig
    tiny = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"]
    return E.Engine(BertConfig.from_dict(tiny), "cpu", _build_only=True)


def _tables(ps):
    """Bucket tables of the reducer: whole buffer, and cut by a frozen text stream, at several bucket counts."""
    from vilbert_b200.ddp import FlatGradAllReducer, trainable_ranges
    frozen = frozenset(n for n in ps.entries if n.startswith(("bert.embeddings.", "bert.encoder.layer.")))
    out = []
    for n_buckets in (1, 3, 8):
        for fr in (frozenset(), frozen):
            red = FlatGradAllReducer(ps.grad, n_buckets=n_buckets)
            red.set_ranges(trainable_ranges(ps, fr))
            out.append((red.table, fr))
    return out


@pytest.mark.parametrize("world", [2, 3, 8])
def test_slices_cover_every_bucket_element_once_aligned(world):
    from vilbert_b200.ddp import shard_slices
    ps = _cpu_engine().ps
    for table, _ in _tables(ps) + [(((0, 8), (8, 24), (1024, 1024 + 4000)), None)]:
        slices = shard_slices(table, world)
        assert slices == shard_slices(tuple(table), world)        # a function of the table alone
        for (lo, hi), sl in zip(table, slices):
            assert len(sl) == world
            count = np.zeros(hi - lo, np.int64)
            for a, e in sl:
                assert lo <= a <= e <= hi and a % 4 == 0 and (e % 4 == 0 or e == hi)
                count[a - lo:e - lo] += 1
            assert (count == 1).all()
            per = sl[0][1] - sl[0][0]
            assert per % 4 == 0 and 0 <= per * world - (hi - lo) < 4 * world     # the bucket padded by less than 4 per rank


@pytest.mark.parametrize("world", [2, 3])
def test_state_layout_and_chunks_cover_each_trainable_element_once(world):
    from vilbert_b200.ddp import shard_slices
    from vilbert_b200.optim import shard_chunks, shard_state_layout
    ps = _cpu_engine().ps
    names = list(ps.entries)
    for table, frozen in _tables(ps):
        ranges = [(ps.span(n)[0], ps.span(n)[1], i % 5) for i, n in enumerate(names) if n not in frozen]
        slices = shard_slices(table, world)
        want = np.zeros(ps.numel, np.int64)
        for off, n, _ in ranges:
            want[off:off + n] = 1
        got = np.zeros(ps.numel, np.int64)
        for r in range(world):
            layout, total = shard_state_layout(slices, r)
            assert [(lo, hi) for lo, hi, _ in layout] == [sl[r] for sl in slices]
            assert total == sum(hi - lo for lo, hi, _ in layout) <= sum(-(-(hi - lo) // world) + 3 for lo, hi in table)
            at = 0
            for lo, hi, base in layout:                      # back to back, 4-aligned
                assert base == at and base % 4 == 0
                at += hi - lo
            state_seen = np.zeros(max(total, 1), np.int64)
            for (lo, hi, base), (st, ss, cn, gr) in zip(layout, shard_chunks(ranges, layout, chunk=4096)):
                for s, t, n, g in zip(st, ss, cn, gr):
                    assert lo <= s and s + n <= hi and s % 4 == 0 and t == s - lo + base and t % 4 == 0
                    assert g == next(gi for off, m, gi in ranges if off <= s < off + m)
                    got[s:s + n] += 1
                    state_seen[t:t + n] += 1
            assert state_seen.max(initial=0) <= 1
        assert np.array_equal(got, want)


def test_unshard_state_assembles_the_unsharded_state_dict():
    """The per-rank compact moments assembled on the host give the unsharded optimizer's state_dict: same keys, shapes, values."""
    from vilbert_b200.ddp import FlatGradAllReducer, shard_slices, trainable_ranges
    from vilbert_b200.optim import FusedAdamW, shard_state_layout, unshard_state
    eng = _cpu_engine()
    ps = eng.ps
    params = [torch.nn.Parameter(ps.p(n)) for n in ps.entries]
    model = types.SimpleNamespace(engine=eng, _ddp_sync=True, _step_in_backward=None)
    opt = FusedAdamW(params, lr=1e-3, model=model)
    g = torch.Generator().manual_seed(0)
    opt.exp_avg.copy_(torch.randn(ps.numel, generator=g))
    opt.exp_avg_sq.copy_(torch.rand(ps.numel, generator=g))
    want = opt.state_dict()
    red = FlatGradAllReducer(ps.grad, n_buckets=5)
    red.set_ranges(trainable_ranges(ps, frozenset()))
    slices = shard_slices(red.table, 2)
    layouts = [shard_state_layout(slices, r)[0] for r in range(2)]
    full = []
    for buf in (opt.exp_avg, opt.exp_avg_sq):
        compacts = []
        for layout in layouts:
            c = torch.zeros(sum(hi - lo for lo, hi, _ in layout))
            for lo, hi, base in layout:
                c[base:base + hi - lo] = buf[lo:hi]
            compacts.append(c)
        full.append(unshard_state(compacts, layouts, ps.numel))
    opt._expose(full)
    got = torch.optim.Optimizer.state_dict(opt)
    assert got["param_groups"] == want["param_groups"]
    assert set(got["state"]) == set(want["state"])
    for k, s in want["state"].items():
        assert set(got["state"][k]) == set(s)
        for name in ("exp_avg", "exp_avg_sq"):
            assert got["state"][k][name].shape == s[name].shape and torch.equal(got["state"][k][name], s[name])


def test_refusals():
    from vilbert_b200.ddp import DistributedDataParallel, FlatGradAllReducer
    from vilbert_b200.optim import FusedAdamW, FusedRAdam
    from oracle import vilbert_oracle as O
    eng = _cpu_engine()
    params = [torch.nn.Parameter(eng.ps.p(n)) for n in eng.ps.entries]
    model = types.SimpleNamespace(engine=eng, _ddp_sync=True, _step_in_backward=None)
    for cls in (FusedAdamW, FusedRAdam):
        with pytest.raises(ValueError, match="DistributedDataParallel"):
            cls(params, model=model, shard_state=True)
        ddp = object.__new__(DistributedDataParallel)         # a wrapper over a world of one
        ddp.module, ddp.reducer = model, FlatGradAllReducer(eng.ps.grad)
        assert ddp.reducer.world == 1
        with pytest.raises(ValueError, match="more than one rank"):
            cls(params, model=ddp, shard_state=True)
    plan = eng.plan(4, 9, 11, grad_outputs=O.HEAD_NAMES, train=True)
    with pytest.raises(ValueError, match="shard_state"):
        plan.enable_optimizer(types.SimpleNamespace(shard_state=True))


# ------------------------------------------------------------------------------------------ two gloo ranks
def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    from datetime import timedelta
    from vilbert_b200.ddp import FlatGradAllReducer, trainable_ranges
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=120))
    ps = _cpu_engine().ps
    res = {}
    frozen = frozenset(n for n in ps.entries if n.startswith("bert.embeddings."))
    from vilbert_b200.ddp import shard_slices
    for n_buckets in (3, 8):
        # small integers: the sum is exact in any order. Over 3 ranks most buckets do not split evenly and go through the padded
        # staging copy
        grads = [torch.randint(-64, 64, (ps.numel,), generator=torch.Generator().manual_seed(10 + r)).float() for r in range(world)]
        red = FlatGradAllReducer(ps.grad, n_buckets=n_buckets)
        red.set_ranges(trainable_ranges(ps, frozen))
        res[f"padded_{n_buckets}"] = any((sl[0][1] - sl[0][0]) * world != hi - lo for (lo, hi), sl in zip(red.table, red.slices))
        red.scatter = True
        ps.grad.copy_(grads[rank])
        red.allreduce()
        ok = True
        for sl in red.slices:
            a, e = sl[rank]
            ok &= bool(torch.equal(ps.grad[a:e], sum(g[a:e] for g in grads) / world))
        res[f"scatter_{n_buckets}"] = ok
        try:
            red.allreduce_range(*red.table[0])
            res[f"twice_{n_buckets}"] = "no error"
        except RuntimeError as ex:
            res[f"twice_{n_buckets}"] = str(ex)
        red.reset_exchange()
        # all-gather: every rank writes its slices, then every rank holds rank-specific values everywhere; -0.0 survives
        w = torch.full((ps.numel,), float("nan"))
        want = torch.randn(ps.numel, generator=torch.Generator().manual_seed(99))
        want[::7] = -0.0
        for (lo, hi), sl in zip(red.table, shard_slices(red.table, world)):
            a, e = sl[rank]
            w[a:e] = want[a:e]
        for lo, hi in red.table:
            red.all_gather_range(w, lo, hi, async_op=False)
        ok = all(torch.equal(w[lo:hi], want[lo:hi]) and torch.equal(torch.signbit(w[lo:hi]), torch.signbit(want[lo:hi]))
                 for lo, hi in red.table)
        res[f"gather_{n_buckets}"] = ok
        res[f"slices_{n_buckets}"] = red.slices
    gathered = [None] * world
    dist.all_gather_object(gathered, res)
    out[rank] = dict(res, same_slices=all(g[f"slices_{n}"] == res[f"slices_{n}"] for g in gathered for n in (3, 8)))
    dist.barrier()
    dist.destroy_process_group()


def test_three_gloo_ranks_reduce_scatter_and_all_gather():
    world = 3
    port = 35600 + (os.getpid() % 2000)
    mgr = mp.Manager()
    out = mgr.dict()
    ctx = mp.spawn(_worker, args=(world, port, out), nprocs=world, join=False)
    deadline = time.monotonic() + 300
    while not ctx.join(timeout=5):
        if time.monotonic() > deadline:
            for p in ctx.processes:
                p.kill()
            pytest.fail("the gloo ranks did not finish within 300 s")
    for rank in range(world):
        res = out[rank]
        for n in (3, 8):
            assert res[f"scatter_{n}"] and res[f"gather_{n}"] and res[f"padded_{n}"], (rank, n)
            assert "second synchronised backward" in res[f"twice_{n}"], res[f"twice_{n}"]
        assert res["same_slices"]
