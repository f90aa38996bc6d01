"""Canonical text listing of the launches the engine's plans make, for checking that a host-side refactor of engine.py /
optim.py launches exactly what it launched before. Needs the built libvilbert_b200.so, no GPU (plans are built with
_build_only=True on the CPU).

    python tools/plan_dump.py ROOT [--out FILE]

imports the package from the repository tree ROOT. For every plan of the case matrix below it lists each op of the prologue,
image prefix, forward, backward and epilogue: section, stream id, function name (MARK for a stream barrier / event marker) and every
argument. Structs passed by reference are expanded field by field, and every pointer (a c_void_p argument or struct field) is
written as `allocation+byte offset` against the plan's allocations, so two runs, or two trees that launch the same work,
produce byte-identical listings."""
import argparse
import ctypes as C
import json
import os
import sys

ARENA_BYTES = 64 << 20
NT, NV = 9, 11


def cases(O, E, base_labels):
    """(name, config overrides, engine heads, B, plan kwargs[, Nv[, Engine kwargs]]) of the case matrix. The overrides apply to
    tests/golden/tiny_b4.json, or for the single-stream baseline (heads "base*") to tests/golden/tiny_basebert.json, whose answer
    count is `base_labels`. A case the tree cannot build (an objective kind or a plan option it does not have) is skipped with a
    note on stderr, so listings of two trees compare case by case."""
    LOSS_HEADS = E.LOSS_HEADS
    train = dict(grad_outputs=O.HEAD_NAMES, train=True)
    base = dict(num_labels=base_labels)

    def obj(kind, **kw):
        return dict(grad_outputs=LOSS_HEADS.get(kind, ()), loss=kind, train=True, **kw)
    task = dict(score=True, loss_in_forward=True)
    return [
        ("heads_train", {}, "vl", 4, train),
        ("vqa_loss", {}, "vl", 4, dict(grad_outputs=("vil_prediction",), vqa_loss=True, train=True)),
        ("task_tokens", dict(task_specific_tokens=True), "vl", 4, train),
        ("dynamic_attention", dict(dynamic_attention=True), "vl", 4, train),
        ("fast_mode", dict(fast_mode=True), "vl", 4, {}),
        ("in_batch_pairs", dict(in_batch_pairs=True), "vl", 4, train),
        ("visualization", dict(visualization=True), "vl", 4, dict(grad_outputs=O.HEAD_NAMES)),
        ("fixed_t_layer", dict(fixed_t_layer=1), "vl", 4, train),
        ("pretraining", {}, "pretraining", 4, dict(grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining", train=True)),
        ("odd_b3", {}, "vl", 3, train),
        # the fine-tuning objectives, as emitted at the start of the backward
        ("loss_gqa", {}, "vl", 4, obj("gqa")),
        ("loss_vlogit_bce", {}, "vl", 4, obj("vlogit_bce")),
        ("loss_logit_ce", {}, "vl", 4, obj("logit_ce")),
        ("loss_binary_ce", {}, "vl", 4, obj("binary_ce")),
        ("loss_tri_ce", {}, "vl", 4, obj("tri_ce")),
        ("loss_vlogit_mc", {}, "vl", 4, obj("vlogit_mc", choices=4), 110),
        ("loss_binary_bce", {}, "vl", 4, obj("binary_bce")),
        ("loss_tri_bce", {}, "vl", 4, obj("tri_bce")),
        # ... and placed at the end of the forward with the batch score (vilbert_b200.tasks)
        ("task_vqa", {}, "vl", 4, obj("vqa", **task)),
        ("task_gqa_eval", {}, "vl", 4, dict(loss="gqa", **task)),
        ("task_logit_ce", {}, "vl", 4, obj("logit_ce", choices=2, **task)),
        ("task_vlogit_bce", {}, "vl", 4, obj("vlogit_bce", **task)),
        ("task_vlogit_mc", dict(task_specific_tokens=True), "vl", 4, obj("vlogit_mc", choices=6, **task), 110),
        ("task_binary_bce", {}, "vl", 4, obj("binary_bce", **task)),
        ("task_tri_bce", {}, "vl", 4, obj("tri_bce", **task)),
        ("task_binary_ce_nscore", {}, "vl", 4, obj("binary_ce", loss_in_forward=True)),
        # forward-only evaluation plans that build only the head their task type reads, with the per-row results
        # (vilbert_b200.tasks.EvaluatingModel)
        ("eval_vqa", {}, "vl", 4, dict(outputs=("vil_prediction",), results="vqa")),
        ("eval_gqa_odd", {}, "vl", 3, dict(outputs=("vil_prediction_gqa",), results="gqa")),
        ("eval_logit_ce", {}, "vl", 4, dict(loss="logit_ce", choices=2, outputs=("vil_logit",), results="logit_ce", **task)),
        ("eval_vlogit_bce", {}, "vl", 4, dict(loss="vlogit_bce", outputs=("vision_logit",), results="vlogit_bce", **task)),
        ("eval_vlogit_mc", dict(task_specific_tokens=True), "vl", 4,
         dict(loss="vlogit_mc", choices=6, outputs=("vision_logit",), results="vlogit_mc", **task), 110),
        ("eval_binary_bce", {}, "vl", 4, dict(loss="binary_bce", outputs=("vil_binary_prediction",), **task)),
        ("eval_binary_bce_odd", {}, "vl", 3, dict(loss="binary_bce", outputs=("vil_binary_prediction",), **task)),
        ("eval_tri_bce", {}, "vl", 4, dict(loss="tri_bce", outputs=("vil_tri_prediction",), **task)),
        # the pre-training objective for every config.visual_target: summed, and with three losses placed at the end of the forward
        # (train, and eval without gradients)
        *[case for vt, over in ((0, {}), (1, dict(visual_target=1, v_target_size=48)), (2, dict(visual_target=2, v_target_size=48)))
          for case in ([] if vt == 0 else [(f"pretraining_vt{vt}", over, "pretraining", 4, obj("pretraining"))]) +
          [(f"pretraining_fwd_vt{vt}", over, "pretraining", 4, obj("pretraining", loss_in_forward=True)),
           (f"pretraining_fwd_vt{vt}_eval", over, "pretraining", 4, dict(loss="pretraining", loss_in_forward=True))]],
        # caption-to-image retrieval (vilbert_b200.retrieval): fast-mode plans whose image embedding runs once per image chunk
        ("retrieval_prefix", {}, "vl", 4, dict(outputs=("vil_logit",), fast_mode=True, image_prefix=True)),
        ("retrieval_prefix_task_tokens", dict(task_specific_tokens=True), "vl", 4, dict(outputs=("vil_logit",), fast_mode=True, image_prefix=True)),
        ("retrieval_zero_shot", {}, "pretraining", 4, dict(outputs=("seq_relationship_score",), fast_mode=True, image_prefix=True)),
        # frozen parameters (requires_grad=False): the text embeddings; the image embedding and the image-side projections of the
        # first connection layer (partial co-attention backward)
        ("frozen_text_embeddings", {}, "vl", 4, dict(train, frozen=frozenset(
            f"bert.embeddings.{n}" for n in ("word_embeddings.weight", "position_embeddings.weight", "token_type_embeddings.weight",
                                             "LayerNorm.weight", "LayerNorm.bias")))),
        ("frozen_vision_input", {}, "vl", 4, dict(train, frozen=frozenset(
            [f"bert.v_embeddings.{n}" for n in ("image_embeddings.weight", "image_embeddings.bias", "image_location_embeddings.weight",
                                               "image_location_embeddings.bias", "LayerNorm.weight", "LayerNorm.bias")] +
            [f"bert.encoder.c_layer.0.biattention.{n}{i}.{w}" for n in ("query", "key", "value") for i in (1,) for w in ("weight", "bias")]))),
        # the single-stream baseline (vilbert_b200.basebert): training with all seven outputs, eval, its embeddings and first layer
        # frozen, and the bare BertModel with gradients into its outputs
        ("base_train", {}, "base", 3, dict(grad_outputs=E.BASE_HEAD_NAMES, train=True), NV, base),
        ("base_eval", {}, "base", 3, {}, NV, base),
        ("base_frozen_embeddings_layer0", {}, "base", 3, dict(grad_outputs=E.BASE_HEAD_NAMES, train=True, frozen=frozenset(
            [f"bert.embeddings.{n}" for n in ("word_embeddings.weight", "position_embeddings.weight", "token_type_embeddings.weight",
                                             "LayerNorm.weight", "LayerNorm.bias")] +
            [f"bert.image_embeddings.{n}" for n in ("image_embeddings.weight", "image_embeddings.bias", "token_type_embeddings.weight",
                                                   "image_location_embeddings.weight", "image_location_embeddings.bias",
                                                   "LayerNorm.weight", "LayerNorm.bias")] +
            [f"bert.encoder.layer.0.{n}.{w}" for n in ("attention.self.query", "attention.self.key", "attention.self.value",
                                                      "attention.output.dense", "attention.output.LayerNorm", "intermediate.dense",
                                                      "output.dense", "output.LayerNorm") for w in ("weight", "bias")])), NV, base),
        ("base_none_bert_outputs", {}, "base_none", 3, dict(grad_outputs=E.BASE_BERT_OUT_NAMES), NV, base),
    ]


def input_grad_cases(O, E, base_labels):
    """Cases of plans that also differentiate the region features and boxes (input_grads=), listed after the matrix above so that
    the listing of a tree without them is a prefix of this one. frozen="all" freezes every parameter entry (the saliency case)."""
    both = frozenset(E.INPUT_GRAD_NAMES)
    train = dict(grad_outputs=O.HEAD_NAMES, train=True, input_grads=both)
    base = dict(num_labels=base_labels)
    return [
        ("input_grads_heads_train", {}, "vl", 4, train),
        ("input_grads_all_frozen_eval", {}, "vl", 4, dict(grad_outputs=("vil_prediction",), input_grads=both, frozen="all")),
        ("input_grads_in_batch_pairs", dict(in_batch_pairs=True), "vl", 4, train),
        ("input_grads_base_train", {}, "base", 3, dict(grad_outputs=E.BASE_HEAD_NAMES, train=True, input_grads=both), NV, base),
        ("input_grads_pretraining", {}, "pretraining", 4, dict(grad_outputs=E.LOSS_HEADS["pretraining"], loss="pretraining", train=True,
                                                               loss_in_forward=True, input_grads=both)),
    ]


def packed_cases(E):
    """Packed task steps (packed=(rows_t, rows_v)) building heads of PACKED_HEADS only: a train-mode VQA step, a V-logit evaluation
    step with its results, a VL-logit step over two options and a train-mode V-logit step with the text stream frozen (frozen= as
    entry-name prefixes). Listed after every case above, so that the listing of a tree without them is a prefix of this one."""
    rows = (24, 32)

    def step(kind, **kw):
        return dict(grad_outputs=E.LOSS_HEADS[kind], loss=kind, train=True, score=True, loss_in_forward=True, outputs=E.LOSS_HEADS[kind],
                    packed=rows, **kw)
    return [
        ("packed_task_vqa", {}, "vl", 4, step("vqa")),
        ("packed_eval_vlogit_bce", {}, "vl", 4, dict(loss="vlogit_bce", score=True, loss_in_forward=True, outputs=("vision_logit",),
                                                     results="vlogit_bce", packed=rows)),
        ("packed_task_logit_ce", {}, "vl", 4, step("logit_ce", choices=2)),
        ("packed_task_vlogit_bce_frozen_text", {}, "vl", 4, step("vlogit_bce", frozen=("bert.embeddings.", "bert.encoder.layer."))),
    ]


def packed_pretraining_cases(E):
    """Packed pre-training steps: the fused objective with its three losses in the forward (BertForMultiModalPreTraining with
    engine.pack_padding) for every config.visual_target, in train mode and as a forward-only evaluation plan, and a train-mode step
    with the text stream frozen. Listed after every case above, so that the listing of a tree without them is a prefix of this one."""
    rows = (24, 32)
    train = dict(grad_outputs=E.LOSS_HEADS["pretraining"], train=True)

    def step(**kw):
        return dict(loss="pretraining", loss_in_forward=True, packed=rows, **kw)
    return [
        *[case for vt, over in ((0, {}), (1, dict(visual_target=1, v_target_size=48)), (2, dict(visual_target=2, v_target_size=48)))
          for case in ((f"packed_pretraining_vt{vt}", over, "pretraining", 4, step(**train)),
                       (f"packed_pretraining_vt{vt}_eval", over, "pretraining", 4, step()))],
        ("packed_pretraining_frozen_text", {}, "pretraining", 4, step(frozen=("bert.embeddings.", "bert.encoder.layer."), **train)),
    ]


def packed_retrieval_cases(E):
    """Packed retrieval plans (fast_mode and image_prefix with packed=(rows_t, rows_v), the score head alone): VILBertForVLTasks with
    and without task tokens, the zero-shot pre-training model, recycled and deterministic. Listed after every case above, so that
    the listing of a tree without them is a prefix of this one."""
    rows = (20, 24)
    kw = dict(outputs=("vil_logit",), fast_mode=True, image_prefix=True, packed=rows)
    return [
        ("packed_retrieval", {}, "vl", 4, kw),
        ("packed_retrieval_task_tokens", dict(task_specific_tokens=True), "vl", 4, kw),
        ("packed_retrieval_zero_shot", {}, "pretraining", 4, dict(kw, outputs=("seq_relationship_score",))),
        ("packed_retrieval_recycled", dict(task_specific_tokens=True), "vl", 4, dict(kw, recycle=True)),
        ("det_packed_retrieval_task_tokens", dict(task_specific_tokens=True), "vl", 4, dict(kw, deterministic=True)),
    ]


def deterministic_cases(O, E, base_labels):
    """The two-stream cases of every matrix above with deterministic=True (named det_...)."""
    every = (cases(O, E, base_labels) + input_grad_cases(O, E, base_labels) + packed_cases(E) + packed_pretraining_cases(E))
    return [(f"det_{name}", over, heads, B, dict(kw, deterministic=True), *extra)
            for name, over, heads, B, kw, *extra in every if not heads.startswith("base")]


def anomaly_cases(O, E, base_labels):
    """Every case above that has a backward (grad_outputs or input_grads) again with anomaly=True (named anomaly_...), the
    deterministic ones included: the plans torch.autograd.set_detect_anomaly(True) selects."""
    every = (cases(O, E, base_labels) + input_grad_cases(O, E, base_labels) + packed_cases(E) + packed_pretraining_cases(E) +
             deterministic_cases(O, E, base_labels))
    return [(f"anomaly_{name}", over, heads, B, dict(kw, anomaly=True), *extra)
            for name, over, heads, B, kw, *extra in every if kw.get("grad_outputs") or kw.get("input_grads")]


def dump_cases(out, case_list, prec, Engine, BertConfig, tiny, tiny_base):
    """Lists every plan of `case_list` in precision `prec`, without and with the shared activation arena. -> (plans, op records)"""
    n_plans = n_ops = 0
    for name, over, heads, B, kw, *extra in case_list:
        nv = extra[0] if extra else NV
        engine_kw = extra[1] if len(extra) > 1 else {}
        cfg = dict(tiny_base["config"] if heads.startswith("base") else tiny, **over)
        for arena in (False, True):
            eng = Engine(BertConfig.from_dict(cfg), "cpu", heads=heads, _build_only=True, precision=prec, **engine_kw)
            if arena:
                eng.enable_activation_arena(ARENA_BYTES)
            frozen = kw.get("frozen")
            if frozen == "all" or isinstance(frozen, tuple):     # every entry, or the entries under these name prefixes
                plan_kw = dict(kw, frozen=frozenset(n for n in eng.ps.entries if frozen == "all" or n.startswith(frozen)))
            else:
                plan_kw = kw
            try:
                plan = eng.plan(B, NT, nv, **plan_kw)
            except (TypeError, ValueError) as ex:
                print(f"plan_dump: {prec} {name} arena={int(arena)} skipped: {ex}", file=sys.stderr)
                continue
            plan.enable_training_prologue()
            n_ops += dump_plan(out, f"{prec} {name} arena={int(arena)}", plan)
            n_plans += 1
    return n_plans, n_ops


class Allocations:
    """Names pointers after the first allocation (in the order given) whose storage contains them."""

    def __init__(self, named):
        self.ranges = []
        for name, t in named:
            if t is None or not hasattr(t, "untyped_storage"):
                continue
            s = t.untyped_storage()
            if s.nbytes():
                self.ranges.append((name, s.data_ptr(), s.nbytes()))

    def name(self, p):
        if not p:
            return "0"
        for name, base, n in self.ranges:
            if base <= p < base + n:
                return f"{name}+{p - base}"
        raise ValueError(f"pointer {p:#x} lies in none of the plan's allocations")


def allocations(plan, opt=None):
    import torch
    e, ps = plan.e, plan.e.ps
    named = [("flat", ps.flat), ("grad", ps.grad), ("shadow", ps.shadow), ("shadow_b", ps.shadow_b), ("shadow_lo", ps.shadow_lo),
             ("drop_step", e.drop_step), ("arena", e.arena)]
    named += [(f"keep{i}", t) for i, t in enumerate(t for t in plan._keep if torch.is_tensor(t))]
    named += [(f"plan.{k}", v) for k, v in sorted(vars(plan).items()) if torch.is_tensor(v)]
    if opt is not None:
        named += [(f"opt.{k}", v) for k, v in sorted(vars(opt).items()) if torch.is_tensor(v)]
    return Allocations(named)


def value(v, ctype, alloc):
    if v is None:
        return "0"
    if hasattr(v, "_obj"):          # byref(struct), also where the argtype is a plain void*
        return struct(v._obj, alloc)
    if ctype is C.c_void_p:
        return alloc.name(v)
    if isinstance(ctype, type) and issubclass(ctype, C.Structure):
        return struct(v, alloc)
    if isinstance(v, C._SimpleCData):
        v = v.value
    return repr(float(v)) if isinstance(v, float) or ctype is C.c_float else str(int(v))


def struct(s, alloc):
    return "{" + ",".join(f"{f}={value(getattr(s, f), t, alloc)}" for f, t in s._fields_) + "}"


def dump_plan(out, title, plan, opt=None):
    alloc = allocations(plan, opt)
    n = 0
    out.append(f"== {title}")
    for section in ("prologue", "prefix", "fwd", "bwd", "epilogue"):
        for i, (fn, args, sid) in enumerate(getattr(plan, section, ())):     # prefix: image_prefix plans only
            if fn is None:
                rec = "MARK " + " ".join(str(a) for a in args)
            else:
                types = fn.argtypes[:len(args)]
                assert len(types) == len(args) == len(fn.argtypes) - 1, fn.__name__     # the trailing argument is the stream
                rec = fn.__name__ + " " + " ".join(value(a, t, alloc) for a, t in zip(args, types))
            out.append(f"{section} {i} s{sid} {rec.rstrip()}")
            n += 1
    return n


def dump_optimizer_plan(out, torch, O, Engine, BertConfig, tiny, prec, opt_cls, title, **opt_kw):
    """The training plan of the tiny config with the fused optimizer `opt_cls(**opt_kw)` in its epilogue."""
    eng = Engine(BertConfig.from_dict(tiny), "cpu", _build_only=True, precision=prec)
    plan = eng.plan(4, NT, NV, grad_outputs=O.HEAD_NAMES, train=True)
    params = [torch.nn.Parameter(eng.ps.p(nm)) for nm in eng.ps.entries]
    opt = opt_cls(params, lr=1e-4, engine=eng, **opt_kw)
    plan.enable_optimizer(opt)
    return dump_plan(out, title, plan, opt)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("root", help="repository tree to import the package from")
    ap.add_argument("--out", help="output file (default: stdout)")
    a = ap.parse_args()
    root = os.path.abspath(a.root)
    sys.path.insert(0, root)
    import torch
    from oracle import vilbert_oracle as O
    from vilbert_b200.config import BertConfig
    from vilbert_b200 import engine as E
    from vilbert_b200.engine import PRECISIONS, Engine
    from vilbert_b200.optim import FusedAdamW, FusedRAdam
    golden = os.path.join(root, "tests", "golden")
    tiny = json.load(open(os.path.join(golden, "tiny_b4.json")))["config"]
    tiny_base = json.load(open(os.path.join(golden, "tiny_basebert.json")))
    out, n_plans, n_ops = [], 0, 0
    for prec in PRECISIONS:
        p, o = dump_cases(out, cases(O, E, tiny_base["num_labels"]), prec, Engine, BertConfig, tiny, tiny_base)
        n_plans, n_ops = n_plans + p, n_ops + o
        for opt_cls in (FusedAdamW, FusedRAdam):
            n_ops += dump_optimizer_plan(out, torch, O, Engine, BertConfig, tiny, prec, opt_cls, f"{prec} {opt_cls.__name__}")
            n_plans += 1
    # gradient-norm clipping: listed after the matrix above, so that the listing of a tree without it is a prefix of this one
    for prec in PRECISIONS:
        for opt_cls in (FusedAdamW, FusedRAdam):
            n_ops += dump_optimizer_plan(out, torch, O, Engine, BertConfig, tiny, prec, opt_cls, f"{prec} {opt_cls.__name__} max_grad_norm=1.0",
                                         max_grad_norm=1.0)
            n_plans += 1
    # input gradients: listed last, so that the listing of a tree without them is a prefix of this one
    if hasattr(E, "INPUT_GRAD_NAMES"):
        for prec in PRECISIONS:
            p, o = dump_cases(out, input_grad_cases(O, E, tiny_base["num_labels"]), prec, Engine, BertConfig, tiny, tiny_base)
            n_plans, n_ops = n_plans + p, n_ops + o
    # packed task steps: listed last, so that the listing of a tree without them is a prefix of this one
    if hasattr(E, "PACKED_HEADS"):
        for prec in PRECISIONS:
            p, o = dump_cases(out, packed_cases(E), prec, Engine, BertConfig, tiny, tiny_base)
            n_plans, n_ops = n_plans + p, n_ops + o
    # packed pre-training steps: listed last, so that the listing of a tree without them is a prefix of this one
    if hasattr(E, "pretraining_pack_rows"):
        for prec in PRECISIONS:
            p, o = dump_cases(out, packed_pretraining_cases(E), prec, Engine, BertConfig, tiny, tiny_base)
            n_plans, n_ops = n_plans + p, n_ops + o
    # deterministic plans (torch.use_deterministic_algorithms(True)): every two-stream case above again with deterministic=True,
    # listed last, so that the listing of a tree without them is a prefix of this one (the baseline refuses them)
    if hasattr(E, "DET_WORKSPACE"):
        for prec in PRECISIONS:
            p, o = dump_cases(out, deterministic_cases(O, E, tiny_base["num_labels"]), prec, Engine, BertConfig, tiny, tiny_base)
            n_plans, n_ops = n_plans + p, n_ops + o
    # anomaly checks (torch.autograd.set_detect_anomaly(True)): listed last, so that the listing of a tree without them is a prefix
    # of this one
    if hasattr(E, "ANOMALY_OUTPUTS"):
        for prec in PRECISIONS:
            p, o = dump_cases(out, anomaly_cases(O, E, tiny_base["num_labels"]), prec, Engine, BertConfig, tiny, tiny_base)
            n_plans, n_ops = n_plans + p, n_ops + o
    # packed retrieval plans: listed last, so that the listing of a tree without them is a prefix of this one
    if hasattr(E, "RETRIEVAL_SCORE_HEADS"):
        for prec in PRECISIONS:
            p, o = dump_cases(out, packed_retrieval_cases(E), prec, Engine, BertConfig, tiny, tiny_base)
            n_plans, n_ops = n_plans + p, n_ops + o
    text = "\n".join(out) + "\n"
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)
    else:
        sys.stdout.write(text)
    print(f"plan_dump: {n_plans} plans, {n_ops} op records", file=sys.stderr)


if __name__ == "__main__":
    main()
