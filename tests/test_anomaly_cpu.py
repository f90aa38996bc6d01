"""Anomaly detection (torch.autograd.set_detect_anomaly(True) / Engine.plan(anomaly=True)), checked on CPU-built plans of the tiny
config across the tools/plan_dump.py case matrix: with the flag off (or check_nan=False) nothing changes; a checked plan is the
unchecked plan plus its vb_nan_check launches; every gradient a backward-role op writes is scanned after that op on its stream;
an entry point without an output-table entry fails at build; a checked plan refuses the in-plan optimizer and is cached apart."""
import json
import os
import re
import sys

import pytest
import torch

from oracle import vilbert_oracle as O
from vilbert_b200 import _lib as L
from vilbert_b200 import engine as E
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import Engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import plan_dump as PD  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
TINY = json.load(open(os.path.join(GOLDEN, "tiny_b4.json")))["config"]
TINY_BASE = json.load(open(os.path.join(GOLDEN, "tiny_basebert.json")))
LABELS = TINY_BASE["num_labels"]
EVERY = (PD.cases(O, E, LABELS) + PD.input_grad_cases(O, E, LABELS) + PD.packed_cases(E) + PD.packed_pretraining_cases(E) +
         PD.deterministic_cases(O, E, LABELS))
CHECKED = PD.anomaly_cases(O, E, LABELS)
ES = {L.VB_NAN_F32: 4, L.VB_NAN_F16: 2, L.VB_NAN_BF16: 2}


def _plan(name, over, heads, B, kw, *extra, precision="fp16", **plan_kw):
    nv = extra[0] if extra else PD.NV
    engine_kw = extra[1] if len(extra) > 1 else {}
    cfg = dict(TINY_BASE["config"] if heads.startswith("base") else TINY, **over)
    eng = Engine(BertConfig.from_dict(cfg), "cpu", heads=heads, _build_only=True, precision=precision, **engine_kw)
    frozen = kw.get("frozen")
    if frozen == "all" or isinstance(frozen, tuple):
        kw = dict(kw, frozen=frozenset(n for n in eng.ps.entries if frozen == "all" or n.startswith(frozen)))
    plan = eng.plan(B, PD.NT, nv, **dict(kw, **plan_kw))
    plan.enable_training_prologue()
    return plan


def _listing(plan, drop_checks=False):
    """plan_dump's listing of the plan without the op index, optionally without the vb_nan_check launches."""
    out = []
    PD.dump_plan(out, "", plan)
    lines = [re.sub(r"^(\w+) \d+ ", r"\1 ", ln) for ln in out[1:]]
    return [ln for ln in lines if not (drop_checks and " vb_nan_check " in ln)]


@pytest.mark.parametrize("case", EVERY, ids=[c[0] for c in EVERY])
def test_flag_off_or_check_nan_false_builds_the_unchecked_plan(case):
    name, over, heads, B, kw, *extra = case
    ref = _listing(_plan(*case))
    with torch.autograd.set_detect_anomaly(True, check_nan=False):
        off = _plan(*case)
    assert not off.anomaly and _listing(off) == ref


@pytest.mark.parametrize("case", CHECKED, ids=[c[0] for c in CHECKED])
def test_checked_plan_is_the_unchecked_plan_plus_its_checks(case):
    name, over, heads, B, kw, *extra = case
    checked = _plan(*case)
    assert checked.anomaly
    plain = _plan(name, over, heads, B, dict(kw, anomaly=False), *extra)
    assert _listing(checked, drop_checks=True) == _listing(plain)
    fn, args, sid = checked.fwd[0]
    assert fn.__name__ == "vb_nan_check" and args.reset == 1 and sid == 0       # the flag reset opens every forward


def _span(ptr, rows, cols, ld, dt):
    return ptr, ptr + ((rows - 1) * ld + cols) * ES[dt]


# every checked case in fp16, a few of them in the other two precisions
OTHER_PRECISIONS = ("anomaly_heads_train", "anomaly_base_train", "anomaly_packed_task_vqa", "anomaly_det_heads_train",
                    "anomaly_pretraining_fwd_vt2")
COVERAGE = [(c, "fp16") for c in CHECKED] + [(c, p) for c in CHECKED if c[0] in OTHER_PRECISIONS for p in ("fp32", "bf16")]


@pytest.mark.parametrize("case,precision", COVERAGE, ids=[f"{c[0]}-{p}" for c, p in COVERAGE])
def test_every_backward_gradient_is_checked_after_its_op(case, precision):
    plan = _plan(*case, precision=precision)
    regions = {}                 # (section, op) -> [(region span, id)]
    for (ptr, rows, cols, ld, dt, rid), rec in zip(sorted(plan.nan_regions, key=lambda r: r[5]), plan.nan_records):
        assert rid == rec.region
        regions.setdefault((rec.section, rec.op), []).append((_span(ptr, rows, cols, ld, dt), rid))
    # where each region is scanned: (section, index of the check launch, stream)
    scanned, table = {}, plan.nan_table.data_ptr()
    for section in ("fwd", "bwd"):
        for i, (fn, args, sid) in enumerate(getattr(plan, section)):
            if fn is not None and fn.__name__ == "vb_nan_check" and not args.reset:
                first = (args.regions - table) // E.C_SIZEOF_NAN_REGION
                for k in range(args.n_regions):
                    scanned[plan.nan_regions[first + k][5]] = (section, i, sid)
    assert sorted(scanned) == list(range(len(plan.nan_records)))
    assert [r.region for r in plan.nan_records] == sorted(scanned)       # ids follow op-list order (fwd objective first)
    # every kernel of the backward list declares its outputs, and each output lies in a region of its own op scanned later on its stream
    role_ops = [("bwd", i) for i, (fn, _, _) in enumerate(plan.bwd) if fn is not None and fn.__name__ != "vb_nan_check"]
    role_ops += sorted({(r.section, r.op) for r in plan.nan_records if r.section == "fwd"})
    for section, i in role_ops:
        fn, args, sid = getattr(plan, section)[i]
        for out, ptr, rows, cols, ld, dt in E.ANOMALY_OUTPUTS[fn.__name__](plan, args):
            if not ptr or rows <= 0 or cols <= 0:
                continue
            lo, hi = _span(ptr, rows, cols, ld, dt)
            hits = [rid for (a, b), rid in regions.get((section, i), ()) if a <= lo and hi <= b]
            assert hits, f"{section} {i} {fn.__name__}.{out} is not checked"
            s_sec, s_i, s_sid = scanned[hits[0]]
            assert s_sec == section and s_i > i and s_sid == sid, (fn.__name__, out, scanned[hits[0]], i, sid)
    # every gradient range the backward writes is inside a checked region of the flat buffer
    g0 = plan.ps.grad.data_ptr()
    spans = [s for rs in regions.values() for s, _ in rs]
    image_type = plan.ps.entries.get("bert.image_embeddings.token_type_embeddings.weight")
    for (off, n) in plan.grad_touch:      # a fused projection's range may be checked part by part (bias sums of Q, K and V)
        lo, hi = g0 + 4 * off, g0 + 4 * (off + n)
        if image_type is not None and off == image_type[0]:
            lo += 4 * image_type[1][1]          # the baseline's image tokens are all of type 1: the backward writes row 1 only
        for a, b in sorted(s for s in spans if s[0] < hi and s[1] > lo):
            if a <= lo:
                lo = max(lo, b)
        assert lo >= hi, f"gradient range {off}+{n} is not checked"
    # no region reaches past the buffer it starts in
    alloc = PD.allocations(plan)
    for (a, b) in spans:
        inside = [(base, base + nb) for _, base, nb in alloc.ranges if base <= a < base + nb]
        assert inside and all(b <= end for _, end in inside[:1]), f"region [{a:#x}, {b:#x}) leaves its buffer"


def test_a_backward_entry_point_without_an_output_entry_fails_at_build(monkeypatch):
    monkeypatch.delitem(E.ANOMALY_OUTPUTS, "vb_relu_bwd")
    case = next(c for c in CHECKED if c[0] == "anomaly_heads_train")
    with pytest.raises(L.VBError, match="vb_relu_bwd .*no entry in engine.ANOMALY_OUTPUTS"):
        _plan(*case)
    _plan(*case, anomaly=False)         # the unchecked plan does not consult the table


def test_refusal_and_cache_keys():
    from vilbert_b200.optim import FusedAdamW
    eng = Engine(BertConfig.from_dict(TINY), "cpu", _build_only=True)
    kw = dict(grad_outputs=O.HEAD_NAMES, train=True)
    plain = eng.plan(4, PD.NT, PD.NV, **kw)
    with torch.autograd.set_detect_anomaly(True):
        checked = eng.plan(4, PD.NT, PD.NV, **kw)
        assert eng.plan(4, PD.NT, PD.NV, **kw) is checked
        assert not eng.plan(4, PD.NT, PD.NV).anomaly            # nothing to check without a backward
    with torch.autograd.detect_anomaly():
        assert eng.plan(4, PD.NT, PD.NV, **kw) is checked
    with torch.autograd.detect_anomaly(check_nan=False):
        assert eng.plan(4, PD.NT, PD.NV, **kw) is plain
    assert checked is not plain and checked.anomaly and not plain.anomaly
    assert eng.plan(4, PD.NT, PD.NV, anomaly=True, **kw) is checked and eng.plan(4, PD.NT, PD.NV, **kw) is plain
    params = [torch.nn.Parameter(eng.ps.p(n)) for n in eng.ps.entries]
    opt = FusedAdamW(params, lr=1e-4, engine=eng)
    with pytest.raises(ValueError, match="anomaly"):
        checked.enable_optimizer(opt)
    plain.enable_optimizer(opt)
    with pytest.raises(ValueError, match="without anomaly checks"):
        plain.anomaly_report()


def test_records_name_the_module_and_the_output():
    case = next(c for c in CHECKED if c[0] == "anomaly_task_vqa")
    plan = _plan(*case)
    first = plan.nan_records[0]
    assert (first.section, first.module, first.entry, first.name) == ("fwd", "vqa", "vb_bce_logits_loss", "dlogits_f32")
    mods = {r.module for r in plan.nan_records}
    assert {"vil_prediction.logit_fc", "bert.encoder.c_layer.0.biOutput", "bert.embeddings", "bert.v_embeddings"} <= mods
    scale = [r for r in plan.nan_records if r.entry == "vb_scale_by_device"]
    assert scale and all(r.section == "bwd" and r.module == "vqa" for r in scale)
