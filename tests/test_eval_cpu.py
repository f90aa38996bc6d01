"""EvaluatingModel without a GPU: the restatement in tests/_eval_oracle.py against what the reference's EvaluatingModel returned
(tests/golden/evaluating_model_reference.json, written by tools/make_eval_golden.py), the per-row rules of vb_task_results against
torch, and the structure of the forward-only plans that build only the head their task type reads (Plan(outputs=...))."""
import json
import math
import os

import pytest
import torch

import _eval_oracle as E
from oracle import vilbert_oracle as O

NT, NV = 9, 11
FIXTURE = "evaluating_model_reference.json"


def _engine(golden_dir, **over):
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    cfg = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over)
    return Engine(BertConfig.from_dict(cfg), "cpu", _build_only=True)


# ------------------------------------------------------------------------------------------ the reference's EvaluatingModel
def _case_batch(c):
    out = []
    for k in c["batch_order"]:
        spec = c["batch"][k]
        if "data" in spec:
            t = torch.tensor(spec["data"], dtype=torch.int64 if spec["dtype"] == "int64" else torch.float32)
        else:
            t = torch.zeros(spec["shape"], dtype=torch.int64 if k in ("question", "input_mask", "segment_ids", "image_mask") else torch.float32)
        out.append(t)
    return tuple(out)


def _case_model(c):
    heads = []
    for n in O.HEAD_NAMES:
        heads.append(torch.tensor(c["heads"][n]["data"], dtype=torch.float32) if n in c["heads"] else torch.zeros(c["model_batch"], 3))

    def model(question, *rest):
        assert question.size(0) == c["model_batch"]
        return tuple(heads) + (None,)
    return model


def _same(a, b, rel=0.0):
    """Equal values (NaN equals NaN); floats within `rel` relative."""
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k], rel) for k in a)
    if isinstance(a, list):
        return len(a) == len(b) and all(_same(x, y, rel) for x, y in zip(a, b))
    if isinstance(a, float) or isinstance(b, float):
        if math.isnan(a) or math.isnan(b):
            return math.isnan(a) and math.isnan(b)
        return type(a) is type(b) and abs(a - b) <= rel * abs(b)
    return type(a) is type(b) and a == b


def _fixture(golden_dir):
    return json.load(open(os.path.join(golden_dir, FIXTURE)))["cases"]


def test_fixture_covers_every_type_and_process(golden_dir):
    cases = _fixture(golden_dir)
    assert {c["task_cfg"]["type"] for c in cases} == set(E.EVAL_TYPES)
    assert {c["task_cfg"]["process"] for c in cases} == {"normal", "dialog", "expand", "retrieval", "nlvr"}
    binary = [c for c in cases if c["task_cfg"]["type"] == "VL-binary-classifier" and c["task_cfg"]["loss"] == "BCEWithLogitLoss"]
    assert {c["model_batch"] % 2 for c in binary} == {0, 1}


def test_oracle_reproduces_the_reference(golden_dir):
    """Indices, ids, answers and IoU values exactly; loss and probabilities to 1e-6 relative; errors of the same type after the
    same partial results (VisDial's one id per image, Foil's loss / score)."""
    for c in _fixture(golden_dir):
        task_cfg = {c["task_id"]: c["task_cfg"]}
        want = c["expect"]
        results = []
        if want["error"]:
            with pytest.raises({"IndexError": IndexError, "ValueError": ValueError}[want["error"]]):
                E.evaluating_step(task_cfg, c["task_id"], _case_batch(c), _case_model(c), c["label2ans"], results, [])
            assert _same(results, want["results"], 1e-6), c["name"]
            continue
        loss, score, bs, res, others = E.evaluating_step(task_cfg, c["task_id"], _case_batch(c), _case_model(c), c["label2ans"], results, [])
        assert res is results and others == [] and bs == want["batch_size"], c["name"]
        assert _same(loss, want["loss"], 1e-6) and score == want["score"], (c["name"], loss, want["loss"], score, want["score"])
        assert _same(results, want["results"], 1e-6), c["name"]


# ------------------------------------------------------------------------------------------ the rules of vb_task_results
def test_results_rules_match_torch():
    nan, inf = float("nan"), float("inf")
    rows = torch.tensor([[1.0, 3.0, 3.0, 2.0], [nan, 5.0, nan, 1.0], [-1e4, -1e4, -1e4, -1e4], [1.0, nan, 9.0, nan], [0.0, -0.0, 0.0, 0.0],
                         [-inf, -inf, -5.0, -5.0], [-inf, -inf, -inf, -inf], [inf, 1.0, 2.0, inf]])
    rows = torch.cat([rows, torch.randn(40, 4).round(), torch.randn(20, 4) * 8])
    pick, _ = E.task_results_rule(rows, "argmax")
    assert torch.equal(pick, torch.max(rows, 1)[1])
    _, probs = E.task_results_rule(rows, "softmax")
    # torch.softmax in float64, rounded: the CPU float32 softmax itself is up to ~2e-6 off (its vectorised exp); the GPU test
    # compares the kernel with the float32 torch.softmax of the device
    want = torch.softmax(rows.double(), 1).float()
    assert torch.equal(torch.isnan(probs), torch.isnan(want)) and torch.isnan(torch.softmax(rows, 1)).equal(torch.isnan(want))
    ok = ~torch.isnan(want)
    assert torch.allclose(probs[ok], want[ok], rtol=1e-6, atol=0)
    wide = torch.randn(16, 3129) * 3
    assert torch.allclose(E.task_results_rule(wide, "softmax")[1], torch.softmax(wide.double(), 1).float(), rtol=1e-6, atol=0)
    tgt = torch.rand(rows.shape)
    _, iou = E.task_results_rule(rows, "gather", tgt)
    assert torch.equal(iou, tgt.gather(1, torch.max(rows, 1)[1].view(-1, 1)).view(-1))


# ------------------------------------------------------------------------------------------ Plan(outputs=...)
HEAD_PARAMS = {"vil_prediction": ("vil_prediction.",), "vil_prediction_gqa": ("vil_prediction_gqa.",), "vil_logit": ("vil_logit.",),
               "vil_tri_prediction": ("vil_tri_prediction.",), "vision_logit": ("vision_logit.",), "linguisic_logit": ("linguisic_logit.",),
               "vision_prediction": ("cls.imagePredictions.",), "linguisic_prediction": ("cls.predictions.",)}
HEAD_PREFIXES = ("cls.", "vil_prediction.", "vil_prediction_gqa.", "vil_logit.", "vil_binary_prediction.", "vil_tri_prediction.",
                 "vision_logit.", "linguisic_logit.")

# (objective kind, plan options) of EvaluatingModel's plan per evaluation type
EVAL_PLANS = {
    "vqa": dict(outputs=("vil_prediction",), results="vqa"),
    "gqa": dict(outputs=("vil_prediction_gqa",), results="gqa"),
    "logit_ce": dict(loss="logit_ce", choices=2, score=True, loss_in_forward=True, outputs=("vil_logit",), results="logit_ce"),
    "vlogit_bce": dict(loss="vlogit_bce", score=True, loss_in_forward=True, outputs=("vision_logit",), results="vlogit_bce"),
    "vlogit_mc": dict(loss="vlogit_mc", choices=3, score=True, loss_in_forward=True, outputs=("vision_logit",), results="vlogit_mc"),
    "binary_bce": dict(loss="binary_bce", score=True, loss_in_forward=True, outputs=("vil_binary_prediction",)),
    "tri_bce": dict(loss="tri_bce", score=True, loss_in_forward=True, outputs=("vil_tri_prediction",)),
}


def _params_read(plan):
    """Names of the parameters the forward ops read (by their fp32 or 16-bit pointer, also inside GEMM argument structs)."""
    ps = plan.e.ps
    ptrs = {}
    for n in ps.entries:
        ptrs[ps.p(n).data_ptr()] = n
        ptrs[ps.w(n).hi.data_ptr()] = n
    seen = set()
    for fn, args, _ in plan.fwd:
        if fn is None:
            continue
        for a in args:
            vals = [a]
            if hasattr(a, "_obj"):
                vals = [getattr(a._obj, f) for f, _ in a._obj._fields_]
            seen.update(ptrs[v] for v in vals if isinstance(v, int) and v in ptrs)
    return seen


def _gemm_ns(plan):
    return [args[0]._obj.N for fn, args, _ in plan.fwd if fn is not None and fn.__name__ == "vb_gemm_bf16"]


def _plan_bytes(plan):
    return sum(t.numel() * t.element_size() for t in plan._keep if torch.is_tensor(t))


@pytest.mark.parametrize("kind", sorted(EVAL_PLANS))
@pytest.mark.parametrize("B", [4, 3])
def test_pruned_plan_builds_only_the_kept_head(golden_dir, kind, B):
    from vilbert_b200.engine import BERT_OUT_NAMES
    eng = _engine(golden_dir, task_specific_tokens=True)
    kw = EVAL_PLANS[kind]
    Nv = 110 if kind == "vlogit_mc" else NV
    if kind == "logit_ce":
        kw = dict(kw, choices=B)
    plan = eng.plan(B, NT, Nv, **kw)
    head = kw["outputs"][0]
    assert list(plan.outputs) == list(BERT_OUT_NAMES) + [head]
    assert plan.bwd == [] or all(fn is None for fn, _, _ in plan.bwd)
    c = eng.cfg
    assert not {c.vocab_size, c.v_target_size} & set(_gemm_ns(plan))          # no masked-LM decoder, no region decoder
    heads_read = {n for n in _params_read(plan) if n.startswith(HEAD_PREFIXES)}
    if head == "vil_binary_prediction":
        allowed = ("vil_binary_prediction.",) if B % 2 == 0 else ("cls.bi_seq_relationship.",)
    else:
        allowed = HEAD_PARAMS[head]
    assert heads_read and all(n.startswith(allowed) for n in heads_read), sorted(heads_read)
    full = eng.plan(B, NT, Nv, **{k: v for k, v in kw.items() if k not in ("outputs", "results")})
    lm_logits = B * (NT + 1) * c.vocab_size * 4
    assert _plan_bytes(plan) + lm_logits <= _plan_bytes(full)
    if kind in ("vqa", "gqa", "logit_ce", "vlogit_bce", "vlogit_mc"):
        assert [fn.__name__ for fn, _, _ in plan.fwd if fn is not None][-1] == "vb_task_results"


def test_all_heads_plan_is_the_default(golden_dir):
    """outputs=None builds the nine heads; naming all nine builds the same launches."""
    eng = _engine(golden_dir)
    full = eng.plan(4, NT, NV)
    named = eng.plan(4, NT, NV, outputs=O.HEAD_NAMES)
    assert named is not full
    assert [fn.__name__ for fn, _, _ in full.fwd if fn] == [fn.__name__ for fn, _, _ in named.fwd if fn]
    assert list(full.outputs) == list(named.outputs) and len(full.outputs) == 13


def test_outputs_are_part_of_the_plan_key(golden_dir):
    eng = _engine(golden_dir)
    a = eng.plan(4, NT, NV)
    b = eng.plan(4, NT, NV, outputs=("vil_logit",))
    c = eng.plan(4, NT, NV, outputs=("vision_logit",))
    assert len({id(a), id(b), id(c)}) == 3
    assert eng.plan(4, NT, NV, outputs=("vil_logit",)) is b and eng.plan(4, NT, NV) is a
    assert eng.plan(4, NT, NV, outputs=("vil_logit",), results=None) is b


def test_outputs_and_results_are_checked_at_build_time(golden_dir):
    eng = _engine(golden_dir)
    with pytest.raises(ValueError, match="unknown head"):
        eng.plan(4, NT, NV, outputs=("vil_prediction", "vil_answer"))
    with pytest.raises(ValueError, match="misses"):                       # the objective reads vil_logit
        eng.plan(4, NT, NV, loss="logit_ce", loss_in_forward=True, outputs=("vil_prediction",))
    with pytest.raises(ValueError, match="misses"):                       # a gradient output that is not built
        eng.plan(4, NT, NV, grad_outputs=("vision_logit", "vil_logit"), train=True, outputs=("vision_logit",))
    with pytest.raises(ValueError, match="misses"):                       # the results read the VQA head
        eng.plan(4, NT, NV, outputs=("vil_logit",), results="vqa")
    with pytest.raises(ValueError, match="results must be one of"):
        eng.plan(4, NT, NV, outputs=("vil_tri_prediction",), results="tri_bce")
    with pytest.raises(ValueError, match="reads the inputs"):
        eng.plan(4, NT, NV, outputs=("vision_logit",), results="vlogit_bce")
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    pre = Engine(BertConfig.from_dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]), "cpu", heads="pretraining",
                 _build_only=True)
    with pytest.raises(ValueError, match="heads='vl'"):
        pre.plan(4, NT, NV, outputs=("vil_logit",))
    # the BertModel outputs are always there and may take a gradient
    p = eng.plan(4, NT, NV, grad_outputs=("pooled_output_t", "vil_logit"), train=True, outputs=("vil_logit",))
    assert "pooled_output_t" in p.outputs


def test_results_buffer_packs_objective_argmax_and_values(golden_dir):
    """One private buffer holds (loss, score), the argmax and the values, so one device-to-host copy reads them."""
    eng = _engine(golden_dir)
    eng.enable_activation_arena(64 << 20)
    p = eng.plan(8, NT, NV, **dict(EVAL_PLANS["logit_ce"], choices=4))
    buf = p.results_out
    assert buf.dtype == torch.uint8 and buf.numel() == 8 + 8 * 2 + 4 * 2 * 4
    for t, off in ((p.objective_out, 0), (p.results_argmax, 8), (p.results_values, 24)):
        assert t.untyped_storage().data_ptr() == buf.untyped_storage().data_ptr() and t.data_ptr() - buf.data_ptr() == off
    assert p.loss.data_ptr() == buf.data_ptr() and p.score.data_ptr() == buf.data_ptr() + 4
    assert buf.untyped_storage().data_ptr() != eng.arena.untyped_storage().data_ptr()
    q = eng.plan(4, NT, NV, **EVAL_PLANS["vqa"])
    assert q.loss is None and q.score is None and q.results_values is None and q.results_out.numel() == 8 + 8 * 4


def test_evaluating_model_refuses_pairs_outside_the_table():
    from vilbert_b200.tasks import EvaluatingModel
    cfg = {"TASK14": {"type": "VL-tri-classifier", "loss": "CrossEntropyLoss", "process": "normal"},
           "TASK99": {"type": "VL-caption", "loss": "CrossEntropyLoss", "process": "normal"}}
    for task_id in cfg:
        with pytest.raises(NotImplementedError):
            EvaluatingModel(None, cfg, None, task_id, (torch.zeros(1),), None, None, None, [], [])
