"""Deterministic plans (torch.use_deterministic_algorithms(True) / Engine.plan(deterministic=True)), checked on CPU-built plans of
the tiny config across the tools/plan_dump.py case matrix: no launch adds into a sum with float atomics whose order depends on
scheduling, every launch goes to one stream, the flag is part of the plan key, and the single-stream baseline follows torch's rule
(RuntimeError, or a warning and the default kernels with warn_only=True)."""
import json
import os
import sys
import warnings

import pytest
import torch

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
# entry points that add with float atomics; a deterministic plan launches their _det twins
ATOMIC_ENTRY_POINTS = set(E.DET_WORKSPACE) | {"vb_layernorm_bwd", "vb_add_layernorm_bwd", *E.DET_MISSING_BASELINE}


def _plan(name, over, heads, B, kw, *extra, precision="fp16"):
    nv = extra[0] if extra else PD.NV
    eng = Engine(BertConfig.from_dict(dict(TINY, **over)), "cpu", heads=heads, _build_only=True, precision=precision)
    frozen = kw.get("frozen")
    if frozen == "all" or isinstance(frozen, tuple):
        kw = dict(kw, frozen=frozenset(n for n in eng.ps.entries if frozen == "all" or n.startswith(frozen)))
    plan = eng.plan(B, PD.NT, nv, **kw)
    plan.enable_training_prologue()
    return plan


def _ops(plan):
    for section in ("prologue", "prefix", "fwd", "bwd", "epilogue"):
        for fn, args, sid in getattr(plan, section, ()):
            yield section, fn, args, sid


def _order_dependent(fn, args):
    """Why the launch (fn, args) would sum in a scheduling-dependent order, or None."""
    name = fn.__name__
    if name in ATOMIC_ENTRY_POINTS:
        return f"{name} adds with float atomics"
    if name == "vb_gemm_bf16":
        g = args[0]._obj
        if g.out_colsum:
            return "GEMM with out_colsum (atomic column sums in the epilogue)"
        if g.atomic_out == 1 and g.split_k != 1:
            return f"GEMM with atomic_out=1, split_k={g.split_k} (split-K atomics)"
    if name == "vb_attention_bwd":
        a = args[0]._obj
        if a.dbias_q or a.dbias_k or a.dbias_v:
            return "attention backward with a bias-sum pointer (atomic column sums)"
    return None


DET_CASES = PD.deterministic_cases(O, E, TINY_BASE["num_labels"])


@pytest.mark.parametrize("case", DET_CASES, ids=[c[0] for c in DET_CASES])
def test_deterministic_plan_has_no_order_dependent_sums(case):
    plan = _plan(*case)
    assert plan.det
    bad = [f"{sec} {fn.__name__}: {why}" for sec, fn, args, _ in _ops(plan) if fn is not None
           for why in [_order_dependent(fn, args)] if why]
    assert not bad, bad[:5]
    # one stream: no two launches add into the same gradient range concurrently (e.g. the tied decoder's weight gradient and the
    # word-embedding sums)
    assert {sid for *_, sid in _ops(plan)} <= {0}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_deterministic_training_plan_other_precisions(precision):
    plan = _plan("heads_train", {}, "vl", 4, dict(grad_outputs=O.HEAD_NAMES, train=True, deterministic=True), precision=precision)
    assert not [fn.__name__ for _, fn, args, _ in _ops(plan) if fn is not None and _order_dependent(fn, args)]


def test_default_plan_unchanged_and_keyed_apart():
    """The default plan still uses the atomic kernels (nothing changes without the flag); both plans sit in the cache side by side,
    and deterministic=None reads torch's flag at the call."""
    eng = Engine(BertConfig.from_dict(TINY), "cpu", _build_only=True)
    kw = dict(grad_outputs=O.HEAD_NAMES, train=True)
    default = eng.plan(4, PD.NT, PD.NV, **kw)
    assert not default.det
    assert any(_order_dependent(fn, args) for _, fn, args, _ in _ops(default) if fn is not None)
    det = eng.plan(4, PD.NT, PD.NV, deterministic=True, **kw)
    assert det is not default and det.det and det.det_ws_bytes > 0
    assert eng.plan(4, PD.NT, PD.NV, **kw) is default
    prev, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        assert eng.plan(4, PD.NT, PD.NV, **kw) is det
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn_only)
    assert eng.plan(4, PD.NT, PD.NV, **kw) is default


def _base_engine():
    return Engine(BertConfig.from_dict(TINY_BASE["config"]), "cpu", heads="base", _build_only=True, num_labels=TINY_BASE["num_labels"])


def test_baseline_refuses_deterministic_plans():
    eng = _base_engine()
    kw = dict(grad_outputs=E.BASE_HEAD_NAMES, train=True)
    with pytest.raises(RuntimeError, match="vb_concat_embed_ln_bwd"):
        eng.plan(3, PD.NT, PD.NV, deterministic=True, **kw)
    prev, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        with pytest.raises(RuntimeError, match="vb_embed_text_bwd_padded"):
            eng.plan(3, PD.NT, PD.NV, **kw)
        torch.use_deterministic_algorithms(True, warn_only=True)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            plan = eng.plan(3, PD.NT, PD.NV, **kw)
        assert any("vb_concat_embed_ln_bwd" in str(x.message) for x in w)
        assert not plan.det and "vb_concat_embed_ln_bwd" in {fn.__name__ for _, fn, _, _ in _ops(plan) if fn is not None}
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn_only)


def test_det_prototypes_take_the_default_arguments_plus_a_workspace():
    """The parameter names of each _det twin are its default entry point's plus a trailing ws: DET_WORKSPACE sizes the workspace
    and a twin's engine.ANOMALY_OUTPUTS entry, its default entry point's, reads its launch by those names."""
    args = E.L.ARGS
    for name, size in E.DET_WORKSPACE.items():
        assert args[name + "_det"]._fields == args[name]._fields + (() if size is None else ("ws",)), name
    assert args["vb_layernorm_bwd_det"]._fields == args["vb_add_layernorm_bwd"]._fields + ("ws",)
    assert {n for n in args if n.endswith("_det")} == {n + "_det" for n in E.DET_WORKSPACE} | {"vb_layernorm_bwd_det"}
