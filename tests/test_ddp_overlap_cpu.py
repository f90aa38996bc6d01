"""The bucket schedule of the module surface's overlapped data parallelism (Plan.bucket_schedule, ddp.DistributedDataParallel(
delay_allreduce=False)) on plans built without a GPU: every training plan of tools/plan_dump.py's matrix, packed task and pre-training
plans at two capacities, frozen text streams, deterministic plans and the single-stream baseline. Every bucket of the reducer's table
is handed over once, in descending order, so all plans of one model issue the same collectives; no backward op after a bucket's
handover passes an address inside it; and two gloo ranks whose schedules cut the backward at different places average alike."""
import json
import os
import sys
from collections import defaultdict

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _modules():
    from oracle import vilbert_oracle as O
    from vilbert_b200 import engine as E
    from vilbert_b200.config import BertConfig
    import plan_dump
    return O, E, BertConfig, plan_dump


def _training_cases():
    """(name, config overrides, heads, B, plan kwargs, Nv, engine kwargs) of every plan with a backward."""
    O, E, _, P = _modules()
    tiny_base = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_basebert.json")))
    labels = tiny_base["num_labels"]
    every = P.cases(O, E, labels) + P.input_grad_cases(O, E, labels)
    for rows in ((24, 32), (32, 40)):            # two capacities of the packed steps
        for name, over, heads, B, kw, *extra in P.packed_cases(E) + P.packed_pretraining_cases(E):
            every.append((f"{name}_{rows[0]}_{rows[1]}", over, heads, B, dict(kw, packed=rows), *extra))
    every += [c for c in P.deterministic_cases(O, E, labels) if c[0] in ("det_heads_train", "det_packed_task_vqa", "det_pretraining")]
    out = []
    for name, over, heads, B, kw, *extra in every:
        if not (kw.get("grad_outputs") or kw.get("input_grads")):
            continue
        out.append((name, over, heads, B, kw, extra[0] if extra else P.NV, extra[1] if len(extra) > 1 else {}))
    return out


def _plans(n_buckets):
    """-> {(model, table): [(case name, plan)]}: the plans of one engine per (config overrides, heads), grouped by the reducer table
    of their frozen set."""
    O, E, BertConfig, P = _modules()
    from vilbert_b200.ddp import FlatGradAllReducer, trainable_ranges
    tiny = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"]
    tiny_base = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_basebert.json")))
    engines, groups = {}, defaultdict(list)
    for name, over, heads, B, kw, nv, engine_kw in _training_cases():
        model = (heads, json.dumps(over, sort_keys=True), json.dumps(engine_kw, sort_keys=True))
        if model not in engines:
            cfg = dict(tiny_base["config"] if heads.startswith("base") else tiny, **over)
            engines[model] = E.Engine(BertConfig.from_dict(cfg), "cpu", heads=heads, _build_only=True, **engine_kw)
        eng = engines[model]
        frozen = kw.get("frozen", frozenset())
        if frozen == "all" or isinstance(frozen, tuple):
            frozen = frozenset(n for n in eng.ps.entries if frozen == "all" or n.startswith(frozen))
        kw = dict(kw, frozen=frozen)
        try:
            plan = eng.plan(B, P.NT, nv, **kw)
        except (TypeError, ValueError):
            continue
        red = FlatGradAllReducer(eng.ps.grad, n_buckets=n_buckets)
        red.set_ranges(trainable_ranges(eng.ps, frozen))
        groups[(model, red.table)].append((name, plan))
    return groups


@pytest.fixture(scope="module", params=[8, 32], ids=["8_buckets", "32_buckets"])
def groups(request):
    return _plans(request.param)


def test_matrix_covers_every_kind(groups):
    names = {n for plans in groups.values() for n, _ in plans}
    for want in ("heads_train", "pretraining", "frozen_text_embeddings", "base_train", "det_heads_train", "packed_task_vqa_24_32",
                 "packed_task_vqa_32_40", "packed_pretraining_vt0_24_32", "packed_pretraining_vt0_32_40",
                 "packed_pretraining_frozen_text_24_32", "input_grads_heads_train"):
        assert want in names, want


def test_each_bucket_once_in_descending_order(groups):
    """The handover sequence is the table in descending order, for every plan: identical across the plans of one model."""
    for (_, table), plans in groups.items():
        want = tuple(reversed(table))
        for name, plan in plans:
            sched = plan.bucket_schedule(table)
            assert tuple(r for _, _, rs in sched for r in rs) == want, name
            # the pieces tile the backward list up to its last kernel, in order
            assert sched[0][0] == 0 and all(a[1] == b[0] for a, b in zip(sched, sched[1:])), name
            assert not any(op[0] is not None for op in plan.bwd[sched[-1][1]:]), name
            assert plan.bucket_schedule(table) is sched       # cached per table


def _extents(ps):
    """Flat (lo, hi) of every entry and fused projection: the ranges an op that passes an address inside them may write."""
    names = list(ps.entries) + list(ps.fused)
    return [(off, off + n) for off, n in (ps.span(nm) for nm in names)]


def test_no_op_after_a_cut_touches_its_bucket(groups):
    """Derived from the launches alone: each address an op passes that falls in the flat gradient buffer stands for the whole
    entry or fused projection containing it; no op after the piece a bucket is handed over at may reach into that bucket."""
    from vilbert_b200.engine import op_pointers
    for (_, table), plans in groups.items():
        for name, plan in plans:
            ps = plan.ps
            ext = _extents(ps)
            base, end = ps.grad.data_ptr(), ps.grad.data_ptr() + 4 * ps.numel
            reach = []      # per op: (lo, hi) ranges it may touch
            for fn, args, _ in plan.bwd:
                rs = []
                if fn is not None:
                    for p in op_pointers(fn, args):
                        if base <= p < end:
                            o = (p - base) // 4
                            inside = [(a, b) for a, b in ext if a <= o < b]
                            assert inside, (name, fn.__name__, o)
                            rs.append((min(a for a, _ in inside), max(b for _, b in inside)))
                reach.append(rs)
            cut_of = {r: hi for _, hi, rs in plan.bucket_schedule(table) for r in rs}
            for (lo, hi), cut in cut_of.items():
                for i in range(cut, len(plan.bwd)):
                    for a, b in reach[i]:
                        assert b <= lo or a >= hi, (name, (lo, hi), cut, i, plan.bwd[i][0].__name__)


def test_anomaly_plans_are_refused():
    O, E, BertConfig, P = _modules()
    tiny = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"]
    eng = E.Engine(BertConfig.from_dict(tiny), "cpu", _build_only=True)
    plan = eng.plan(4, P.NT, P.NV, grad_outputs=O.HEAD_NAMES, train=True, anomaly=True)
    with pytest.raises(ValueError, match="anomaly"):
        plan.bucket_schedule(((0, eng.ps.numel),))


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    from datetime import timedelta
    from oracle import vilbert_oracle as O
    from vilbert_b200.config import BertConfig
    from vilbert_b200.ddp import FlatGradAllReducer
    from vilbert_b200.engine import LOSS_HEADS, Engine
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=120))
    tiny = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"]
    eng = Engine(BertConfig.from_dict(tiny), "cpu", _build_only=True)
    # rank 0 runs the padded VQA step, rank 1 the packed one: the same table, cut at other places
    kw = dict(grad_outputs=LOSS_HEADS["vqa"], loss="vqa", train=True, score=True, loss_in_forward=True, outputs=LOSS_HEADS["vqa"])
    plan = eng.plan(4, 9, 11, **(kw if rank == 0 else dict(kw, packed=(24, 32))))
    red = FlatGradAllReducer(eng.ps.grad, n_buckets=8)
    sched = plan.bucket_schedule(red.table)
    vals = [torch.randn(eng.ps.numel, generator=torch.Generator().manual_seed(100 + r)) for r in range(world)]
    eng.ps.grad.zero_()
    for _, _, ranges in sched:
        for lo, hi in ranges:            # the piece finished these buckets: the backward's last write, then the handover
            eng.ps.grad[lo:hi] = vals[rank][lo:hi]
        for lo, hi in ranges:
            red.allreduce_range(lo, hi)
    expect = sum(vals) / world
    out[rank] = ([hi for _, hi, rs in sched if rs], bool(torch.allclose(eng.ps.grad, expect, atol=1e-6)))
    dist.barrier()
    dist.destroy_process_group()


def test_gloo_ranks_with_other_cuts_average_alike():
    world = 2
    port = 29500 + (os.getpid() % 2000) + 7
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    cuts0, ok0 = out[0]
    cuts1, ok1 = out[1]
    assert cuts0 != cuts1            # the two plans pause at other places of their backward
    assert ok0 and ok1
