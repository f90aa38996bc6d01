"""The plan cache (Engine.plan, keyed on PlanSpec), checked on CPU-built plans of the tiny config: a changed engine value the build
reads builds a new plan, equivalent spellings of one plan share it, and a refused option set leaves the cache as it was."""
import json
import os

import pytest

from vilbert_b200 import _lib as L
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import HEAD_NAMES, Engine

NT, NV = 9, 11


def _engine(golden_dir, heads="vl", **over):
    name = "tiny_basebert.json" if heads.startswith("base") else "tiny_b4.json"
    meta = json.load(open(os.path.join(golden_dir, name)))
    kw = dict(num_labels=meta["num_labels"]) if heads.startswith("base") else {}
    return Engine(BertConfig.from_dict(dict(meta["config"], **over)), "cpu", heads=heads, _build_only=True, **kw)


def _labels_rows(plan):
    return plan.loss_inputs["labels"].shape[0]


def _head_dropout(plan):
    return sorted({round(k.p, 4) for k in plan._keep if isinstance(k, L.Dropout)})


def _bwd_max_ctas(plan):
    return {k.max_ctas for k in plan._keep if isinstance(k, L.GemmArgs) and k.max_ctas}


# engine attribute, new value, the plan options, and what the plan's layout shows of the value
BUILD_VALUES = [
    ("loss_options", 2, dict(grad_outputs=("vil_logit",), loss="logit_ce", train=True), _labels_rows, 2, 4),
    ("head_dropout_prob", 0.25, dict(grad_outputs=HEAD_NAMES, train=True), _head_dropout, [0.1], [0.1, 0.25]),
    ("bwd_gemm_max_ctas", 100, dict(grad_outputs=HEAD_NAMES, train=True), _bwd_max_ctas, set(), {100}),
]


@pytest.mark.parametrize("attr,value,kw,layout,before,after", BUILD_VALUES, ids=[c[0] for c in BUILD_VALUES])
def test_a_changed_engine_value_builds_a_new_plan(golden_dir, attr, value, kw, layout, before, after):
    eng = _engine(golden_dir)
    old = eng.plan(8, NT, NV, **kw)
    assert layout(old) == before
    setattr(eng, attr, value)
    new = eng.plan(8, NT, NV, **kw)
    assert new is not old and layout(new) == after
    assert eng.plan(8, NT, NV, **kw) is new and eng.plan_builds[(8, NT, NV)] == 2


def test_equivalent_spellings_share_one_plan(golden_dir):
    eng = _engine(golden_dir)
    plan = eng.plan(4, NT, NV)
    assert eng.plan(4, NT, NV, heads="vl") is plan
    assert eng.plan(4, NT, NV, fast_mode=False) is plan
    assert eng.plan(4, NT, NV, choices=3, outputs=None, packed=None) is plan      # nothing reads choices without its objective
    vqa = eng.plan(4, NT, NV, grad_outputs=["vil_prediction"], vqa_loss=True)
    assert eng.plan(4, NT, NV, grad_outputs=("vil_prediction",), loss="vqa") is vqa
    ce = eng.plan(4, NT, NV, grad_outputs=("vil_logit",), loss="logit_ce")
    assert eng.plan(4, NT, NV, grad_outputs=("vil_logit",), loss="logit_ce", choices=eng.loss_options) is ce
    assert len(eng.plans) == 3 and eng.plan_builds[(4, NT, NV)] == 3


# (engine heads, config overrides, B, options, exception): one refused option set per place a check used to live
REFUSED = [
    ("base", {}, 4, dict(packed=(8, 8)), NotImplementedError),                                            # Engine.plan
    ("base", {}, 4, dict(loss="vqa", grad_outputs=("vil_prediction",)), ValueError),                      # BasePlan
    ("vl", {}, 4, dict(recycle=True, train=True), ValueError),                                            # Plan: recycle
    ("vl", {}, 4, dict(frozen={"no.such.entry"}), ValueError),                                            # Plan: frozen
    ("vl", {}, 4, dict(loss="nope"), ValueError),                                                         # Plan: loss
    ("vl", {}, 4, dict(loss="vlogit_mc", grad_outputs=("vision_logit",)), ValueError),                    # Plan: choices
    ("vl", dict(visualization=True), 4, dict(train=True), ValueError),                                    # _stream_modes
    ("vl", {}, 4, dict(fast_mode=True, train=True), ValueError),                                          # _stream_modes
    ("vl", {}, 4, dict(outputs=("vil_answer",)), ValueError),                                             # _check_outputs
    ("vl", {}, 4, dict(outputs=("vil_logit",), results="vqa"), ValueError),                               # _check_outputs
    ("vl", {}, 4, dict(loss="vqa", loss_in_forward=True, packed=(20, 30)), NotImplementedError),          # _check_packed
    ("vl", {}, 4, dict(outputs=("vil_logit",), packed=(4 * NT + 1, 24)), ValueError),                     # _check_packed
    ("vl", {}, 6, dict(grad_outputs=("vil_logit",), loss="logit_ce"), ValueError),                        # _head_layout
    ("vl", {}, 4, dict(loss="vqa"), ValueError),                                                          # _emit_loss
]


@pytest.mark.parametrize("heads,over,B,kw,exc", REFUSED)
def test_a_refused_call_leaves_the_cache_as_it_was(golden_dir, heads, over, B, kw, exc):
    eng = _engine(golden_dir, heads, **over)
    eng.max_plans = 1
    cached = eng.plan(B, NT, NV)
    builds = dict(eng.plan_builds)
    with pytest.raises(exc):
        eng.plan(B, NT, NV, **kw)
    assert len(eng.plans) == 1 and dict(eng.plan_builds) == builds
    assert eng.plan(B, NT, NV) is cached and dict(eng.plan_builds) == builds
