"""Writes tests/golden/tiny_input_grads.{json,pt}: the gradients of a scalar objective with respect to the region features and boxes
(input_imgs / image_loc, the reference's features / spatials) from the UNMODIFIED reference, after checking that the oracles
(oracle/vilbert_oracle.py, oracle/basebert_oracle.py) reproduce them (fp32, 1e-5 relative).

Cases (the tiny configs of oracle/make_golden.py and tools/make_basebert_golden.py, seeded parameters and inputs, ragged masks):
  eval              VILBertForVLTasks, eval mode, VQA loss + a small quadratic on every other head
  train             the same in train mode, every nn.Dropout replaced by the engine's stateless site mask (oracle.DropMasks)
  tasktok_odd_b3    task tokens, batch 3
  in_batch_pairs    BertModel's four outputs at batch b^2 under a fixed linear probe (each image's gradient sums its b copies)
  dynamic_attention the image attention gated by the pooled text states
  fixed_v_layer     fixed_v_layer=1 with the first image layer ahead of the first connection layer: the image stream is detached,
                    neither input gets a gradient (recorded as None)
  pretraining       BertForMultiModalPreTraining's three losses (visual_target 0), weighted 1 / 0.5 / 0.25
  baseline          BaseBertForVLTasks, eval mode, the fixed probe sum_o <out_o, R_o> of tests/golden/tiny_basebert.*

Tensors up to 512 elements (and every two-stream gradient) are kept in full; the baseline's 2048-wide feature gradient as
oracle.basebert_oracle.digest samples and norms.

Usage: python tools/make_input_grad_golden.py   (needs the reference checkout; see oracle/ref_loader.py)
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import basebert_oracle as BO  # noqa: E402
from oracle import basebert_ref_loader, ref_loader  # noqa: E402
from oracle import vilbert_oracle as O  # noqa: E402
from oracle.make_golden import TINY, _MaskDropout  # noqa: E402

TOL = 1e-5
BASE_TINY = dict(vocab_size=120, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128,
                 max_position_embeddings=40, type_vocab_size=2, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
BASE_LABELS = 7
TRAIN_STEP, HEAD_P = 5, 0.1
PRETRAIN_WEIGHTS = (1.0, 0.5, 0.25)
# name -> (config overrides, B, Nv, Nt, seed, train, objective)
VL_CASES = {
    "eval": ({}, 4, 11, 9, 0, False, "heads"),
    "train": ({}, 4, 11, 9, 0, True, "heads"),
    "tasktok_odd_b3": (dict(task_specific_tokens=True), 3, 7, 12, 1, False, "heads"),
    "in_batch_pairs": (dict(in_batch_pairs=True), 3, 11, 9, 0, False, "bert"),
    "dynamic_attention": (dict(dynamic_attention=True), 4, 11, 9, 0, False, "heads"),
    "fixed_v_layer": (dict(fixed_v_layer=1, v_biattention_id=[1, 2], t_biattention_id=[1, 2]), 4, 11, 9, 0, False, "heads"),
}


def rel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def heads_objective(heads, B):
    """VQA loss on vil_prediction + 0.1 * mean square of every other head (oracle/make_golden.py's total_loss)."""
    tgt = O.synth_vqa_target(B, 3129, device=heads[0].device)
    loss = O.vqa_loss(heads[0], tgt)
    for h in heads[1:]:
        loss = loss + 0.1 * h.float().clamp(-50, 50).pow(2).mean()
    return loss


def bert_objective(outs):
    """A fixed linear probe of the four BertModel outputs."""
    return sum((o * torch.linspace(0.5, 1.5, o.numel(), device=o.device).view_as(o)).sum() for o in outs)


def pretraining_targets(cfg, B, Nv, Nt):
    """Masked-LM labels, image labels, soft image targets and NSP labels of oracle/make_golden.py's pre-training case."""
    g = torch.Generator().manual_seed(5)
    lm = torch.full((B, Nt), -1, dtype=torch.long)
    sel = torch.rand(B, Nt, generator=g) < 0.15
    sel[:, 1] = True
    lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
    il = torch.full((B, Nv - 1), -1, dtype=torch.long)
    il[torch.rand(B, Nv - 1, generator=g) < 0.15] = 1
    il[:, 0] = 1
    it = torch.softmax(torch.randn(B, Nv - 1, cfg["v_target_size"], generator=g), -1)
    ns = torch.randint(0, 2, (B,), generator=g)
    return lm, il, it, ns


def _leaves(inp):
    return inp["input_imgs"].clone().requires_grad_(True), inp["image_loc"].clone().requires_grad_(True)


def _grads(feat, loc):
    return (None if feat.grad is None else feat.grad.clone()), (None if loc.grad is None else loc.grad.clone())


def _check(name, mine, theirs):
    for what, a, b in zip(("input_imgs", "image_loc"), mine, theirs):
        assert (a is None) == (b is None), (name, what, "gradient present in one of oracle / reference only")
        if b is not None:
            e = rel(a, b)
            assert e < TOL, (name, what, e)


def vl_case(ref, name):
    over, B, Nv, Nt, seed, train, objective = VL_CASES[name]
    cfgj = dict(TINY, **over)
    cfg = O.make_config(cfgj)
    model = ref.VILBertForVLTasks(ref.BertConfig.from_dict(dict(cfgj)), num_labels=1, default_gpu=False)
    P = O.synth_params(cfg, seed=seed)
    model.load_state_dict(P, strict=False)
    model.tie_weights()
    drop = None
    if train:
        model.train()
        drop = O.DropMasks(TRAIN_STEP, head_p=HEAD_P)
        for mname, mod in list(model.named_modules()):
            if isinstance(mod, torch.nn.Dropout):
                parent = model
                parts = mname.split(".")
                for q in parts[:-1]:
                    parent = getattr(parent, q)
                names = ["dropout.pooled", "dropout.seq_v", "dropout.seq_t"] if mname == "dropout" else [mname]
                setattr(parent, parts[-1], _MaskDropout(names, mod.p, drop))
    else:
        model.eval()
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=1234 + seed)

    def run(fn):
        feat, loc = _leaves(inp)
        args = (inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
        obj = fn(args)
        if obj.requires_grad:      # with the image stream detached the oracle's objective depends on nothing differentiable
            obj.backward()
        return _grads(feat, loc), float(obj.detach())

    if objective == "bert":
        theirs, obj = run(lambda a: bert_objective(model.bert(*a, inp["co_attention_mask"])[:4]))
        mine, _ = run(lambda a: bert_objective(O.bert_model(P, cfg, *a, drop=drop)))
    else:
        theirs, obj = run(lambda a: heads_objective(model(*a, inp["co_attention_mask"], inp["task_ids"])[:9], B))
        mine, _ = run(lambda a: heads_objective(O.vilbert_for_vl_tasks(P, cfg, *a, task_ids=inp["task_ids"], drop=drop)[1], B))
    _check(name, mine, theirs)
    meta = dict(kind="vl", config=cfgj, B=B, Nv=Nv, Nt=Nt, seed=seed, input_seed=1234 + seed, train_step=TRAIN_STEP if train else None,
                head_dropout_prob=HEAD_P, objective=objective, objective_value=obj)
    return meta, dict(zip(("input_imgs", "image_loc"), theirs))


def pretraining_case(ref):
    B, Nv, Nt = 4, 9, 8
    cfg = O.make_config(TINY)
    model = ref.BertForMultiModalPreTraining(ref.BertConfig.from_dict(dict(TINY)))
    P = O.synth_params(cfg, seed=3, with_task_heads=False)
    model.load_state_dict(P, strict=False)
    model.tie_weights()
    model.eval()
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=77)
    labels = pretraining_targets(cfg, B, Nv, Nt)

    def run(fn):
        feat, loc = _leaves(inp)
        losses = fn((inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"]) + labels)
        obj = sum(w * l.sum() for w, l in zip(PRETRAIN_WEIGHTS, losses))
        obj.backward()
        return _grads(feat, loc), float(obj.detach())

    theirs, obj = run(lambda a: model(*a))
    mine, _ = run(lambda a: O.pretraining_losses(P, cfg, *a))
    _check("pretraining", mine, theirs)
    meta = dict(kind="pretraining", config=TINY, B=B, Nv=Nv, Nt=Nt, seed=3, input_seed=77, loss_weights=PRETRAIN_WEIGHTS,
                objective_value=obj)
    return meta, dict(zip(("input_imgs", "image_loc"), theirs))


def baseline_case():
    base = basebert_ref_loader.load()
    B, Nt, Nv = 3, 9, 11
    cfg = O.make_config(BASE_TINY)
    torch.manual_seed(0)
    model = base.BaseBertForVLTasks(basebert_ref_loader.BertConfig(**cfg), num_labels=BASE_LABELS)
    P = BO.synth_params(cfg, BASE_LABELS, 0)
    sd = dict(P)
    sd["cls.predictions.decoder.weight"] = P["bert.embeddings.word_embeddings.weight"]
    model.load_state_dict(sd, strict=True)
    model.eval()
    inp = BO.synth_inputs(cfg, B, Nt, Nv, 1234)
    R = BO.probe_weights(B, Nt, Nv, BASE_LABELS, cfg["vocab_size"], 7)

    def run(fn):
        feat, loc = _leaves(inp)
        outs = fn((inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"]))
        obj = sum((outs[k] * R[k]).sum() for k in BO.OUT_NAMES)
        obj.backward()
        return _grads(feat, loc), float(obj.detach())

    theirs, obj = run(lambda a: dict(zip(BO.OUT_NAMES, model(*a))))
    mine, _ = run(lambda a: BO.base_bert_for_vl_tasks(P, cfg, *a))
    _check("baseline", mine, theirs)
    meta = dict(kind="baseline", config=BASE_TINY, num_labels=BASE_LABELS, B=B, Nv=Nv, Nt=Nt, seed=0, input_seed=1234, probe_seed=7,
                objective_value=obj)
    return meta, {"input_imgs": BO.digest(theirs[0], seed=0), "image_loc": theirs[1]}


def main():
    torch.set_num_threads(8)
    ref = ref_loader.load()
    meta, tensors = {}, {}
    for name in VL_CASES:
        meta[name], tensors[name] = vl_case(ref, name)
    meta["pretraining"], tensors["pretraining"] = pretraining_case(ref)
    meta["baseline"], tensors["baseline"] = baseline_case()
    for name, t in tensors.items():
        shapes = {k: (None if v is None else list(v["shape"]) if isinstance(v, dict) else list(v.shape)) for k, v in t.items()}
        meta[name]["grad_shapes"] = shapes
        print(f"{name:18s} oracle == reference (< {TOL:g}); gradients {shapes}")
    assert tensors["fixed_v_layer"]["input_imgs"] is None and tensors["fixed_v_layer"]["image_loc"] is None
    gdir = os.path.join(ROOT, "tests", "golden")
    with open(os.path.join(gdir, "tiny_input_grads.json"), "w") as f:
        json.dump(dict(cases=meta, tolerance=TOL), f, indent=1)
    torch.save(tensors, os.path.join(gdir, "tiny_input_grads.pt"))
    print("wrote tests/golden/tiny_input_grads.json / .pt")


if __name__ == "__main__":
    main()
