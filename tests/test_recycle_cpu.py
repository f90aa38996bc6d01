"""Forward-only plans with their buffers placed by lifetime (Plan(recycle=True), Engine.recycle_forward_only), checked on CPU-built
plans of the tiny config across every forward-only case of the tools/plan_dump.py matrix and the three precisions: the same launches
as the plain plan with only the addresses of the plan's buffers changed, no two buffers sharing bytes unless every use of one
happens before every use of the other on the streams, and the buffers the host reads keeping bytes of their own."""
import json
import os
import subprocess
import sys

import pytest

from oracle import vilbert_oracle as O
from vilbert_b200 import engine as E
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import Engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import plan_dump as PD  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
TINY = json.load(open(os.path.join(GOLDEN, "tiny_b4.json")))["config"]
TINY_BASE = json.load(open(os.path.join(GOLDEN, "tiny_basebert.json")))


def _forward_only(kw):
    return not (kw.get("train") or kw.get("grad_outputs") or kw.get("input_grads"))


def _cases():
    nl = TINY_BASE["num_labels"]
    every = (PD.cases(O, E, nl) + PD.input_grad_cases(O, E, nl) + PD.packed_cases(E) + PD.packed_pretraining_cases(E) +
             PD.deterministic_cases(O, E, nl))
    return [c for c in every if _forward_only(c[4])]


CASES = _cases()


def _engine(over, heads, extra, precision):
    cfg = dict(TINY_BASE["config"] if heads.startswith("base") else TINY, **over)
    return Engine(BertConfig.from_dict(cfg), "cpu", heads=heads, _build_only=True, precision=precision,
                  **(extra[1] if len(extra) > 1 else {}))


def _pair(case, precision):
    """The plain and the recycled plan of one case, on one engine."""
    name, over, heads, B, kw, *extra = case
    eng = _engine(over, heads, extra, precision)
    nv = extra[0] if extra else PD.NV
    return eng.plan(B, PD.NT, nv, **kw), eng.plan(B, PD.NT, nv, recycle=True, **kw)


def _ops(plan):
    return [op for section in (plan.prefix, plan.fwd, plan.bwd) for op in section]


def _slots(fn, args):
    """(pointer slots, everything else) of one launch: the pointers in argument / struct-field order, and the launch with every
    pointer written as 'p' (null as '0')."""
    ptrs = []

    class Slots:
        def name(self, p):
            if p:
                ptrs.append(p)
                return "p"
            return "0"
    text = " ".join(PD.value(a, t, Slots()) for a, t in zip(args, fn.argtypes))
    return ptrs, text


def _happens_before(ops):
    """Ancestor bitsets of the kernel ops of `ops` (one run: the image prefix, forward and backward lists in order, every stream
    joined between them), computed by transitive closure over stream order and the barrier / join / event markers. -> list of
    (op index, ancestors) for the kernels, by position in `ops`."""
    n_streams = 4
    state = [0] * n_streams
    events, anc = {}, {}
    for i, (fn, args, sid) in enumerate(ops):
        if fn is None:
            if not args:
                state[0] = state[1] = state[0] | state[1]
            elif args[0] == "all":
                both = 0
                for s in state:
                    both |= s
                state = [both] * n_streams
            elif args[0] == "rec":
                events[args[1]] = state[sid]
            elif args[0] == "wait":
                state[sid] |= events[args[1]]
            continue
        anc[i] = state[sid]
        state[sid] |= 1 << i
    return anc


def _read_by_the_host(plan):
    """What the package's callers read from a plan after a run (modeling, tasks, retrieval, basebert), listed here apart from the
    engine's own rule: outputs, encoded layers, attention exports, the objective's scalars and results, the compacted masked-LM
    row count and the image states of an image prefix."""
    ts = list(plan.outputs.values())
    ts += [a.f32 for n in ("enc_t", "enc_v", "enc") for a in getattr(plan, n, [])]
    ts += [d[k] for d in plan.attn_t + plan.attn_v + [d for pair in plan.attn_c for d in pair] for k in ("attn", "q", "k")]
    ts += [getattr(plan, n) for n in ("objective_out", "results_out", "loss", "score", "preds")]
    ts += [(getattr(plan, "lm_c", None) or {}).get("count")] + list(getattr(plan, "image_states", ()))
    return [t for t in ts if t is not None]


def _sections_joined(plan):
    """The op lists of one plan as one list with a join of every stream between the sections (runs)."""
    join = (None, ("all",), 0)
    return list(plan.prefix) + [join] + list(plan.fwd) + [join] + list(plan.bwd)


@pytest.mark.parametrize("precision", E.PRECISIONS)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_recycled_plan_is_the_plain_plan_at_other_addresses(case, precision):
    """Op for op the same entry point, stream and non-pointer arguments; each pointer into a plan buffer moves by one offset per
    buffer, every other pointer (parameters, the dropout counter) stays where it is."""
    plain, rec = _pair(case, precision)
    a, b = _ops(plain), _ops(rec)
    assert len(a) == len(b) and plain.n_kernels_fwd == rec.n_kernels_fwd and rec.n_kernels_bwd == 0
    bufs = PD.allocations(plain)
    moved = {}
    for (fa, xa, sa), (fb, xb, sb) in zip(a, b):
        if fa is None or fb is None:
            assert (fa, xa, sa) == (fb, xb, sb)
            continue
        pa, ta = _slots(fa, xa)
        pb, tb = _slots(fb, xb)
        assert (fa.__name__, sa, ta) == (fb.__name__, sb, tb)
        for p, q in zip(pa, pb):
            owner = bufs.name(p).split("+")[0]
            if owner.startswith(("keep", "plan.")):
                assert moved.setdefault(owner, q - p) == q - p, f"{fa.__name__}: {owner} is not one block in the recycled plan"
            else:
                assert p == q, f"{fa.__name__}: an engine pointer ({owner}) moved"


@pytest.mark.parametrize("precision", E.PRECISIONS)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_shared_bytes_have_ordered_uses(case, precision):
    """An independent check of the recycled plan: every buffer of the plain plan has one byte range in the recycled plan; two
    ranges that overlap belong to buffers whose uses are all ordered one before the other by the streams' happens-before; what
    the host reads and the private buffers overlap no other buffer; what the image prefix leaves for the forwards (it runs once,
    they run many times) is private; held_bytes is below the plain plan's."""
    plain, rec = _pair(case, precision)
    a, b = _sections_joined(plain), _sections_joined(rec)
    anc = _happens_before(b)
    keep = [t for t in plain._keep if hasattr(t, "data_ptr") and t.numel()]
    spans = sorted((t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), k) for k, t in enumerate(keep))
    ranges, uses = {}, {}
    for i, ((fa, xa, _), (fb, xb, _)) in enumerate(zip(a, b)):
        if fa is None:
            continue
        for p, q in zip(_slots(fa, xa)[0], _slots(fb, xb)[0]):
            hit = [(lo, hi, k) for lo, hi, k in spans if lo <= p < hi]
            if not hit:
                continue
            lo, hi, k = hit[0]
            r = (q - (p - lo), q - (p - lo) + hi - lo)
            assert ranges.setdefault(k, r) == r
            uses.setdefault(k, set()).add(i)
    region = rec._region
    in_region = lambda r: region is not None and region.data_ptr() <= r[0] < region.data_ptr() + region.numel()
    outs = {t.data_ptr() for t in _read_by_the_host(rec)}
    pinned = {k for k, r in ranges.items() if not in_region(r) or any(r[0] <= p < r[1] for p in outs)}
    n_prefix = len(plain.prefix)
    for k, u in uses.items():
        if min(u) < n_prefix < max(u):
            assert not in_region(ranges[k]), f"the image prefix leaves {keep[k].shape} for the forwards in recycled bytes"
    ks = sorted(ranges)
    for x in ks:
        for y in ks:
            if x >= y or ranges[x][1] <= ranges[y][0] or ranges[y][1] <= ranges[x][0]:
                continue
            assert x not in pinned and y not in pinned, f"a private or host-read buffer shares bytes ({keep[x].shape}, {keep[y].shape})"
            ux = sum(1 << i for i in uses[x])
            uy = sum(1 << i for i in uses[y])
            x_first = all(anc[j] & ux == ux for j in uses[y])
            y_first = all(anc[j] & uy == uy for j in uses[x])
            assert x_first or y_first, f"buffers {keep[x].shape} and {keep[y].shape} share bytes with unordered uses"
    assert rec.held_bytes < plain.held_bytes


def test_lifetimes_follow_the_streams_not_the_list():
    """Two-stream plans: a buffer of the vision stream that ends in list order before a buffer of the text stream starts is
    still live while that one is (the streams run concurrently), so the clocks order the two only across a barrier."""
    class Fn:
        argtypes = [E.L.C.c_void_p, E.L.C.c_void_p]
        __name__ = "fake"
    fn = Fn()
    # x is written and read on stream 1; y is first used on stream 0 after x in list order, with no barrier in between
    ops = [(fn, (100, None), 1), (fn, (100, None), 1), (fn, (200, None), 0), (None, (), 0), (fn, (300, None), 0)]
    spans = [(100, 64), (200, 64), (300, 64)]
    off, extent = E.lifetime_layout((ops,), spans, set())
    assert off[0] != off[1], "x and y overlap in time: unordered across the two streams"
    assert off[2] == off[0] or off[2] == off[1], "z follows the barrier: it may take the bytes of either"
    assert extent == 2 * E.BUF_ALIGN
    # a buffer no op uses sits at offset 0 and the extent covers it, so its view in the plan's region is in bounds
    off, extent = E.lifetime_layout((ops,), spans + [(900, 10 * E.BUF_ALIGN)], set())
    assert off[3] == 0 and extent == 10 * E.BUF_ALIGN


def test_recording_build_writes_no_host_memory_under_deterministic_algorithms():
    """The recording build of a recycled plan takes host address ranges as large as the plain plan. Under
    torch.use_deterministic_algorithms(True) torch fills uninitialised memory, so the build must turn that off for them: building a
    recycled retrieval plan of bert_base_6layer_6conect whose plain plan holds several GB grows the peak RSS by far less."""
    script = r"""
import json, resource, sys, torch
sys.path.insert(0, sys.argv[1])
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import Engine
cfg = dict(json.load(open(sys.argv[2])), task_specific_tokens=True)
eng = Engine(BertConfig.from_dict(cfg), "cpu", _build_only=True)
eng.enable_activation_arena(2 << 30)
torch.use_deterministic_algorithms(True)
r0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
plan = eng.plan(64, 30, 101, outputs=("vil_logit",), fast_mode=True, image_prefix=True, recycle=True)
r1 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
print(json.dumps(dict(grown=(r1 - r0) * 1024, plain=sum(nb for nb, _ in plan._place[0]), fill=torch.utils.deterministic.fill_uninitialized_memory)))
"""
    cfg = os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")
    out = subprocess.run([sys.executable, "-c", script, ROOT, cfg], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert r["plain"] > 4e9 and r["fill"] is True
    assert r["grown"] < 1e9, r


@pytest.mark.parametrize("kw", [dict(train=True), dict(grad_outputs=("vil_prediction",)),
                                dict(grad_outputs=("vil_prediction",), input_grads=frozenset(E.INPUT_GRAD_NAMES))],
                         ids=["train", "grad_outputs", "input_grads"])
def test_recycle_refused_on_plans_with_a_backward(kw):
    eng = _engine({}, "vl", (), "fp16")
    with pytest.raises(ValueError, match="forward-only"):
        eng.plan(4, PD.NT, PD.NV, recycle=True, **kw)


def test_engine_switch_reaches_forward_only_plans_only():
    """engine.recycle_forward_only is the default of Engine.plan(recycle=None) for forward-only plans; plans with a backward build
    as before, and the flag is part of the plan key."""
    eng = _engine({}, "vl", (), "fp16")
    plain = eng.plan(4, PD.NT, PD.NV, outputs=("vil_logit",))
    eng.recycle_forward_only = True
    rec = eng.plan(4, PD.NT, PD.NV, outputs=("vil_logit",))
    train = eng.plan(4, PD.NT, PD.NV, grad_outputs=("vil_logit",), train=True)
    assert rec is not plain and rec.recycle and not plain.recycle and not train.recycle
    assert eng.plan(4, PD.NT, PD.NV, outputs=("vil_logit",), recycle=False) is plain


def test_recycled_plan_in_the_shared_arena():
    """With the shared activation arena the recycled region is the start of the arena and arena_bytes its extent."""
    eng = _engine({}, "vl", (), "fp16")
    eng.enable_activation_arena(PD.ARENA_BYTES)
    plain = eng.plan(4, PD.NT, PD.NV, outputs=("vil_prediction",), results="vqa")
    rec = eng.plan(4, PD.NT, PD.NV, outputs=("vil_prediction",), results="vqa", recycle=True)
    assert rec._region.data_ptr() == eng.arena.data_ptr()
    assert 0 < rec.arena_bytes < plain.arena_bytes
    assert rec.held_bytes - rec.arena_bytes == plain.held_bytes - plain.arena_bytes     # the same private buffers
