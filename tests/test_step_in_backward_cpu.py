"""The step in the backward (FusedAdamW / FusedRAdam.step_in_backward) on plans built without a GPU, as tests/test_ddp_overlap_cpu.py
builds them: every training plan kind, padded, packed at two capacities, frozen text streams, deterministic, input-gradient,
dynamic_attention, in_batch_pairs, task-token, baseline and fused pre-training plans. Plan.step_schedule steps every bucket once, no
backward op after a bucket's step point passes an address inside its range of the gradient, the fp32 parameters or any 16-bit copy,
and under a data-parallel table the collectives keep bucket_schedule's sequence and cut points. The per-bucket chunk tables cover every
trainable element exactly once, and the context refuses what it cannot overlap and takes the post-backward path where it must."""
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))


@pytest.fixture(scope="module", params=["step_buckets", 32], ids=["step_buckets", "32_buckets"])
def groups(request):
    from test_ddp_overlap_cpu import _plans
    from vilbert_b200.optim import STEP_BUCKETS
    return _plans(STEP_BUCKETS if request.param == "step_buckets" else request.param)


def _extents(ps):
    names = list(ps.entries) + list(ps.fused)
    return [(off, off + n) for off, n in (ps.span(nm) for nm in names)]


def _reach(plan):
    """Per backward op: the (lo, hi) flat ranges of every entry or fused projection it passes an address inside, in the gradient,
    the fp32 parameters or a 16-bit copy (what it may read or write there)."""
    from vilbert_b200.engine import op_pointers
    ps = plan.ps
    ext = _extents(ps)
    bufs = [t for t in (ps.grad, ps.flat, ps.shadow, ps.shadow_lo, ps.shadow_b) if t is not None]
    spans = [(t.data_ptr(), t.data_ptr() + t.element_size() * ps.numel, t.element_size()) for t in bufs]
    out = []
    for fn, args, _ in plan.bwd:
        rs = []
        if fn is not None:
            for p in op_pointers(fn, args):
                for base, end, es in spans:
                    if base <= p < end:
                        o = (p - base) // es
                        inside = [(a, b) for a, b in ext if a <= o < b]
                        assert inside, (fn.__name__, o)
                        rs.append((min(a for a, _ in inside), max(b for _, b in inside)))
                        break
        out.append(rs)
    return out


def test_matrix_covers_every_kind(groups):
    names = {n for plans in groups.values() for n, _ in plans}
    for want in ("heads_train", "pretraining", "frozen_text_embeddings", "base_train", "det_heads_train", "packed_task_vqa_24_32",
                 "packed_pretraining_vt0_24_32", "input_grads_heads_train", "dynamic_attention", "in_batch_pairs", "task_tokens"):
        assert want in names, want


@pytest.mark.parametrize("allreduce", [False, True], ids=["single", "ddp"])
def test_no_op_after_a_step_point_touches_its_bucket(groups, allreduce):
    for (_, table), plans in groups.items():
        for name, plan in plans:
            sched = plan.step_schedule(table, allreduce)
            assert plan.step_schedule(table, allreduce) is sched           # cached
            assert sched[0][0] == 0 and all(a[1] == b[0] for a, b in zip(sched, sched[1:])), name
            assert not any(op[0] is not None for op in plan.bwd[sched[-1][1]:]), name
            steps = [k for *_, ks in sched for k in ks]
            assert sorted(steps) == list(range(len(table))), name          # every bucket once
            step_at = {k: hi for _, hi, _, ks in sched for k in ks}
            reach = _reach(plan)
            for k, cut in step_at.items():
                lo, hi = table[k]
                for i in range(cut, len(plan.bwd)):
                    for a, b in reach[i]:
                        assert b <= lo or a >= hi, (name, (lo, hi), cut, i, plan.bwd[i][0].__name__)
            if allreduce:
                # the collectives: bucket_schedule's sequence and cut points; a step no earlier than its bucket's collective
                comm = [(hi, rs) for _, hi, rs in plan.bucket_schedule(table) if rs]
                assert [(hi, rs) for _, hi, rs, _ in sched if rs] == comm, name
                handed = {r: hi for hi, rs in comm for r in rs}
                assert all(step_at[k] >= handed[table[k]] for k in step_at), name
            else:
                assert not any(rs for _, _, rs, _ in sched), name


def test_tied_decoder_bucket_is_stepped_last(groups):
    """The word embeddings are read by the tied decoder's dgrad at the start of the backward and written by the embedding
    scatter at its end: in a pre-training plan their bucket is stepped at the last step point."""
    seen = 0
    for (_, table), plans in groups.items():
        for name, plan in plans:
            if plan.loss_kind != "pretraining" or not plan.trainable("bert.embeddings.word_embeddings.weight"):
                continue
            off, n = plan.ps.span("bert.embeddings.word_embeddings.weight")
            for allreduce in (False, True):
                step_at = {k: hi for _, hi, _, ks in plan.step_schedule(table, allreduce) for k in ks}
                mine = [k for k, (lo, hi) in enumerate(table) if lo < off + n and off < hi]
                assert mine and all(step_at[k] == max(step_at.values()) for k in mine), name
            seen += 1
    assert seen


def test_anomaly_plans_are_refused():
    from oracle import vilbert_oracle as O
    from vilbert_b200 import engine as E
    from vilbert_b200.config import BertConfig
    tiny = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"]
    eng = E.Engine(BertConfig.from_dict(tiny), "cpu", _build_only=True)
    plan = eng.plan(4, 9, 11, grad_outputs=O.HEAD_NAMES, train=True, anomaly=True)
    with pytest.raises(ValueError, match="anomaly"):
        plan.step_schedule(((0, eng.ps.numel),), False)


# ------------------------------------------------------------------------------------------ chunk sub-tables
def _cpu_engine():
    from vilbert_b200 import engine as E
    from vilbert_b200.config import BertConfig
    tiny = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"]
    return E.Engine(BertConfig.from_dict(tiny), "cpu", _build_only=True)


def _covered(subs, numel):
    count = np.zeros(numel, np.int64)
    for st, cn, _ in subs:
        for s, n in zip(st, cn):
            count[s:s + n] += 1
    return count


@pytest.mark.parametrize("n_buckets", [1, 3, 8, 32])
def test_bucket_chunks_cover_each_trainable_element_once(n_buckets):
    from vilbert_b200.ddp import FlatGradAllReducer, trainable_ranges
    from vilbert_b200.optim import bucket_chunks, build_chunks
    eng = _cpu_engine()
    ps = eng.ps
    names = list(ps.entries)
    assert any(".q_dense1." in n for n in names) and any(".q_dense2." in n for n in names)
    for frozen in (frozenset(), frozenset(n for n in names if n.startswith(("bert.embeddings.", "bert.encoder.layer.")))):
        ranges = [(ps.span(n)[0], ps.span(n)[1], i % 5) for i, n in enumerate(names) if n not in frozen]
        red = FlatGradAllReducer(ps.grad, n_buckets=n_buckets)
        red.set_ranges(trainable_ranges(ps, frozen))
        subs = bucket_chunks(ranges, red.table, chunk=4096)
        want = np.zeros(ps.numel, np.int64)
        for off, n, _ in ranges:
            want[off:off + n] = 1
        assert np.array_equal(_covered(subs, ps.numel), want)
        assert np.array_equal(_covered([build_chunks(ranges, 4096)], ps.numel), want)
        for (lo, hi), (st, cn, gr) in zip(red.table, subs):
            assert all(lo <= s and s + n <= hi and s % 4 == 0 and 0 < n <= 4096 for s, n in zip(st, cn))
            for s, g in zip(st, gr):                 # each piece keeps its tensor's group
                assert g == next(gi for off, n, gi in ranges if off <= s < off + n)
    with pytest.raises(ValueError, match="outside every bucket"):
        bucket_chunks([(0, 64, 0), (1024, 64, 0)], ((0, 64),))


def _optimizer(cls, **kw):
    """An optimizer over the CPU engine's parameters with a stand-in for the model (the attributes step_in_backward reads)."""
    eng = _cpu_engine()
    params = [torch.nn.Parameter(eng.ps.p(n)) for n in eng.ps.entries]
    model = types.SimpleNamespace(engine=eng, _ddp_sync=True, _step_in_backward=None)
    return cls(params, lr=1e-3, model=model, **kw), params, model


def _classes():
    from vilbert_b200.optim import FusedAdamW, FusedRAdam
    return FusedAdamW, FusedRAdam


def test_frozen_parameter_leaves_the_sub_tables():
    from vilbert_b200.ddp import FlatGradAllReducer
    for cls in _classes():
        opt, params, _ = _optimizer(cls)
        red = FlatGradAllReducer(opt.engine.ps.grad, n_buckets=8)
        table = red.table
        from vilbert_b200.optim import bucket_chunks
        full = _covered(bucket_chunks(opt._trainable_ranges(), table), opt.engine.ps.numel)
        params[3].requires_grad_(False)
        assert opt._refresh_trainable()
        after = _covered(bucket_chunks(opt._trainable_ranges(), table), opt.engine.ps.numel)
        off = (params[3].data_ptr() - opt.engine.ps.flat.data_ptr()) // 4
        assert full[off:off + params[3].numel()].tolist() == [1] * params[3].numel()
        assert after[off:off + params[3].numel()].sum() == 0
        assert after.sum() == full.sum() - params[3].numel()


# ------------------------------------------------------------------------------------------ refusals and the post-backward path
@pytest.mark.parametrize("which", [0, 1], ids=["adamw", "radam"])
def test_refusals(which):
    cls = _classes()[which]
    opt, _, model = _optimizer(cls, max_grad_norm=1.0)
    with pytest.raises(ValueError, match="max_grad_norm"):
        with opt.step_in_backward():
            pass
    assert model._step_in_backward is None
    opt, _, model = _optimizer(cls)
    model._ddp_sync = False                         # inside model.no_sync()
    with pytest.raises(ValueError, match="no_sync"):
        with opt.step_in_backward():
            pass
    model._ddp_sync = True
    eng = opt.engine
    opt2 = cls([torch.nn.Parameter(eng.ps.p(n)) for n in eng.ps.entries], lr=1e-3, engine=eng)
    with pytest.raises(ValueError, match="model="):
        with opt2.step_in_backward():
            pass


@pytest.mark.parametrize("which", [0, 1], ids=["adamw", "radam"])
def test_no_plan_reached_steps_after_the_body_and_a_raising_body_steps_nothing(which):
    opt, _, model = _optimizer(_classes()[which])
    calls = []
    opt.step = lambda: calls.append("step")
    with opt.step_in_backward():
        assert model._step_in_backward is not None
    assert calls == ["step"] and model._step_in_backward is None
    with pytest.raises(RuntimeError, match="boom"):
        with opt.step_in_backward():
            raise RuntimeError("boom")
    assert calls == ["step"] and model._step_in_backward is None


def test_only_the_single_pending_plan_backward_takes_the_step():
    """_PlanCall._step_hook: the hook only for the model's only pending plan call, a plan without anomaly checks, and a gradient
    not all-reduced after the backward; every call leaves the pending set when its backward starts."""
    import weakref
    from vilbert_b200.modeling import _PlanCall

    def hook(plan, red):
        pass

    def call(model, anomaly=False):
        c = _PlanCall.__new__(_PlanCall)
        c.model, c.plan = model, types.SimpleNamespace(anomaly=anomaly)
        model._pending_calls.add(c)
        return c
    model = types.SimpleNamespace(_pending_calls=weakref.WeakSet(), _step_in_backward=hook)
    a = call(model)
    assert a._step_hook(None, False) is hook and not model._pending_calls           # single process
    a = call(model)
    assert a._step_hook(object(), True) is hook                                        # delay_allreduce=False
    a = call(model)
    assert a._step_hook(object(), False) is None                                       # delay_allreduce=True: after the all-reduce
    a = call(model, anomaly=True)
    assert a._step_hook(None, False) is None                                           # anomaly checks
    a, b = call(model), call(model)
    assert a._step_hook(None, False) is None                                           # two pending plan forwards
    assert b._step_hook(None, False) is hook                                           # ... the last one is alone again
    model._step_in_backward = None
    a = call(model)
    assert a._step_hook(None, False) is None                                           # outside the context
