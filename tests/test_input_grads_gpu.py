"""Input gradients on the H100: `features.grad` / `spatials.grad` through every module surface, against the reference's fixtures
(fp32), the oracle in the engine's operand-rounding mode, and torch's autograd semantics; the vb_loc_proj_dx kernel against torch.

Bounds: the gradient bounds tests/test_model_gpu.py applies to the parameter gradients (worst rel-L2 2e-2, all-bf16 precision 5e-2
against the fp32 oracle), which include bert.v_embeddings.image_embeddings.weight, whose GEMM contracts the same bf16 d(embedding)
operand as the feature gradient. Run-to-run comparisons use 1e-5 max-rel, the bound of the split-K atomics' last-bit order effects
(tests/test_replay_gpu.py)."""
import ctypes as C
import json
import os
import sys

import pytest
import torch

from oracle import basebert_oracle as BO
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_input_grad_golden as MG  # noqa: E402

L2_BOUND = {"fp16": 2e-2, "fp32": 2e-2, "bf16": 5e-2}
NAMES = ("input_imgs", "image_loc")


def rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-30)).item()


def rel_l2(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


def _fixture(golden_dir):
    meta = json.load(open(os.path.join(golden_dir, "tiny_input_grads.json")))
    return meta["cases"], torch.load(os.path.join(golden_dir, "tiny_input_grads.pt"))


def _close(got, want, bound, what):
    if isinstance(want, dict):      # a digest of the baseline's 2048-wide feature gradient: sampled entries and norms
        samp, l2, _ = BO.digest_errors(got, want)
        assert samp < 3 * bound and l2 < bound, (what, samp, l2)
        return
    want = want.to(got.device)
    assert got.shape == want.shape and rel_l2(got, want) < bound, (what, rel_l2(got, want))


def _vl_model(meta, precision="fp16", cls=None):
    import vilbert_b200
    cfg = O.make_config(meta["config"])
    cls = cls or vilbert_b200.VILBertForVLTasks
    model = cls(vilbert_b200.BertConfig.from_dict(meta["config"]), precision=precision)
    model.load_state_dict(O.synth_params(cfg, seed=meta["seed"], device="cuda", with_task_heads=cls is vilbert_b200.VILBertForVLTasks),
                          strict=False)
    return model, cfg


def _inputs(cfg, meta, requires_grad=True):
    inp = O.synth_inputs(cfg, meta["B"], meta["Nv"], meta["Nt"], seed=meta["input_seed"], device="cuda")
    feat, loc = inp["input_imgs"].clone().requires_grad_(requires_grad), inp["image_loc"].clone().requires_grad_(requires_grad)
    return inp, feat, loc


def run_vl(meta, precision="fp16", train=None):
    """Module path of a two-stream fixture case: (features.grad, spatials.grad, model)."""
    model, cfg = _vl_model(meta, precision)
    inp, feat, loc = _inputs(cfg, meta)
    if meta["train_step"] is not None:
        model.train()
        model.engine.set_dropout_step(meta["train_step"] - 1)     # the forward bumps it to the fixture's step
    else:
        model.eval()
    args = (inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    if meta["objective"] == "bert":
        obj = MG.bert_objective(model.bert(*args)[:4])
    else:
        obj = MG.heads_objective(model(*args, inp["co_attention_mask"], inp["task_ids"])[:9], meta["B"])
    obj.backward()
    return feat.grad, loc.grad, model


def oracle_op(meta, cfg, precision):
    """The fp32 oracle under the engine's operand rounding (the `op` mode of tests/_gpu_util.model_case)."""
    P = O.synth_params(cfg, seed=meta["seed"], device="cuda")
    inp, feat, loc = _inputs(cfg, meta)
    drop = O.DropMasks(meta["train_step"], head_p=meta["head_dropout_prob"]) if meta["train_step"] is not None else None
    with (O.bf16_operand_mode() if precision == "bf16" else O.operand_mode()):
        heads = O.vilbert_for_vl_tasks(P, cfg, inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"],
                                       inp["image_attention_mask"], task_ids=inp["task_ids"], drop=drop)[1]
        MG.heads_objective(heads, meta["B"]).backward()
    return feat.grad, loc.grad


# ------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("M,H", [(1001, 1024), (333, 96), (257, 37), (6400, 1024)])
def test_loc_proj_dx_kernel(M, H):
    from vilbert_b200 import _lib as L
    lib = L.lib()
    dy = torch.randn(M, H, device="cuda")
    W = torch.randn(H, 5, device="cuda")
    outs = []
    for _ in range(2):
        dx = torch.full((M, 5), float("nan"), device="cuda")
        L.check(lib.vb_loc_proj_dx(dy.data_ptr(), W.data_ptr(), dx.data_ptr(), M, H, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        outs.append(dx)
    torch.cuda.synchronize()
    assert rel(outs[0], (dy.double() @ W.double()).float()) < 1e-5
    assert torch.equal(outs[0], outs[1])
    assert lib.vb_loc_proj_dx(dy.data_ptr(), W.data_ptr(), outs[0].data_ptr(), 0, H, None) != 0


# ------------------------------------------------------------------------------------------ tiny-shape parity
@pytest.mark.parametrize("precision", ["fp16", "fp32", "bf16"])
@pytest.mark.parametrize("case", ["eval", "train"])
def test_tiny_parity(golden_dir, precision, case):
    cases, tensors = _fixture(golden_dir)
    meta = cases[case]
    got = run_vl(meta, precision)[:2]
    bound = L2_BOUND[precision]
    for n, g in zip(NAMES, got):
        assert g is not None and g.dtype == torch.float32
        _close(g, tensors[case][n], bound, (case, precision, n, "fp32"))
    if precision != "fp32":
        for n, g, o in zip(NAMES, got, oracle_op(meta, O.make_config(meta["config"]), precision)):
            _close(g, o, bound, (case, precision, n, "op"))


@pytest.mark.parametrize("case", ["tasktok_odd_b3", "in_batch_pairs", "dynamic_attention", "fixed_v_layer"])
def test_other_configurations(golden_dir, case):
    cases, tensors = _fixture(golden_dir)
    got = run_vl(cases[case])[:2]
    for n, g in zip(NAMES, got):
        if tensors[case][n] is None:
            assert g is None, (case, n)
        else:
            _close(g, tensors[case][n], L2_BOUND["fp16"], (case, n))


def test_pretraining_fused_losses(golden_dir):
    import vilbert_b200
    cases, tensors = _fixture(golden_dir)
    meta = cases["pretraining"]
    cfg = O.make_config(meta["config"])
    model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(meta["config"]), fused_objective=True)
    model.load_state_dict(O.synth_params(cfg, seed=meta["seed"], device="cuda", with_task_heads=False), strict=False)
    model.eval()
    inp, feat, loc = _inputs(cfg, meta)
    labels = [t.cuda() for t in MG.pretraining_targets(cfg, meta["B"], meta["Nv"], meta["Nt"])]
    losses = model(inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"], *labels)
    sum(w * x.sum() for w, x in zip(meta["loss_weights"], losses)).backward()
    for n, g in zip(NAMES, (feat.grad, loc.grad)):
        _close(g, tensors["pretraining"][n], L2_BOUND["fp16"], n)


def test_baseline(golden_dir):
    from vilbert_b200 import BertConfig
    from vilbert_b200.basebert import BaseBertForVLTasks
    cases, tensors = _fixture(golden_dir)
    meta = cases["baseline"]
    cfg = O.make_config(meta["config"])
    model = BaseBertForVLTasks(BertConfig.from_dict(meta["config"]), meta["num_labels"])
    P = BO.synth_params(cfg, meta["num_labels"], meta["seed"], device="cuda")
    model.load_state_dict(dict(P, **{"cls.predictions.decoder.weight": P["bert.embeddings.word_embeddings.weight"]}))
    model.eval()
    inp = BO.synth_inputs(cfg, meta["B"], meta["Nt"], meta["Nv"], meta["input_seed"], device="cuda")
    R = BO.probe_weights(meta["B"], meta["Nt"], meta["Nv"], meta["num_labels"], cfg["vocab_size"], meta["probe_seed"], device="cuda")
    feat, loc = inp["input_imgs"].clone().requires_grad_(True), inp["image_loc"].clone().requires_grad_(True)
    out = model(inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    sum((o * R[k]).sum() for k, o in zip(BO.OUT_NAMES, out)).backward()
    for n, g in zip(NAMES, (feat.grad, loc.grad)):
        _close(g, tensors["baseline"][n], L2_BOUND["fp16"], n)


# ------------------------------------------------------------------------------------------ production shape, saliency setup
def test_saliency_everything_frozen_config2(golden_dir):
    """bert_base_6layer_6conect, B=64, 100 regions, 36 tokens, every parameter frozen, eval mode: gradients of the VQA loss into the
    features and boxes within the parameter-gradient bounds of the fp32 oracle; no Parameter gets a .grad and the flat gradient
    buffer stays zero."""
    import vilbert_b200
    cfgj = json.load(open(os.path.join(golden_dir, "base_6layer_6conect_b4.json")))["config"]
    cfg = O.make_config(cfgj)
    B, Nv, Nt = 64, 100, 36
    P = O.synth_params(cfg, seed=0, device="cuda")
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.load_state_dict(P, strict=False)
    model.eval()
    for p in model.parameters():
        p.requires_grad_(False)
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=1234, device="cuda")
    tgt = O.synth_vqa_target(B, 3129, device="cuda")
    feat, loc = inp["input_imgs"].clone().requires_grad_(True), inp["image_loc"].clone().requires_grad_(True)
    out = model(inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    assert out[0].requires_grad
    O.vqa_loss(out[0], tgt).backward()
    assert all(p.grad is None for p in model.parameters())
    assert model.engine.ps.grad.abs().max().item() == 0.0
    del model
    torch.cuda.empty_cache()
    f2, l2 = inp["input_imgs"].clone().requires_grad_(True), inp["image_loc"].clone().requires_grad_(True)
    heads = O.vilbert_for_vl_tasks(P, cfg, inp["input_txt"], f2, l2, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])[1]
    O.vqa_loss(heads[0], tgt).backward()
    for n, g, o in zip(NAMES, (feat.grad, loc.grad), (f2.grad, l2.grad)):
        _close(g, o, L2_BOUND["fp16"], n)
    # padded regions take no part in vil_prediction: their gradient is exactly zero, as in the reference
    pad = inp["image_attention_mask"] == 0
    assert pad.any() and feat.grad[pad].abs().max().item() == 0.0 and loc.grad[pad].abs().max().item() == 0.0


# ------------------------------------------------------------------------------------------ parameter gradients, reproducibility
def test_parameter_gradients_unchanged(golden_dir):
    cases, _ = _fixture(golden_dir)
    meta = cases["eval"]
    model, cfg = _vl_model(meta)
    model.eval()
    grads = []
    for want in (False, True):
        inp, feat, loc = _inputs(cfg, meta, requires_grad=want)
        model.zero_grad()
        MG.heads_objective(model(inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])[:9],
                           meta["B"]).backward()
        grads.append(model.engine.ps.grad.clone())
        assert (feat.grad is not None) == want
    assert rel(grads[1], grads[0]) < 1e-5


def test_graph_replays_and_recompute_reproduce_eager(golden_dir):
    """Eval: the first two calls run eagerly, later ones replay CUDA graphs. Train: a backward after another forward of a different
    batch recomputes its forward at its own dropout step. Both give the eager input gradients."""
    cases, _ = _fixture(golden_dir)
    meta = cases["eval"]
    model, cfg = _vl_model(meta)
    model.eval()
    runs = []
    for _ in range(4):
        inp, feat, loc = _inputs(cfg, meta)
        MG.heads_objective(model(inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])[:9],
                           meta["B"]).backward()
        runs.append((feat.grad, loc.grad))
    plan = model._last_plan
    assert plan.graph_fwd is not None and plan.graph_bwd is not None
    for f, l in runs[1:]:
        assert rel(f, runs[0][0]) < 1e-5 and rel(l, runs[0][1]) < 1e-5
    model.train()
    eng = model.engine

    def step_of(inp, feat, loc):
        return model(inp["input_txt"], feat, loc, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])[:9]
    eng.set_dropout_step(40)
    inp, feat, loc = _inputs(cfg, meta)
    MG.heads_objective(step_of(inp, feat, loc), meta["B"]).backward()
    eng.set_dropout_step(40)
    inp2, feat2, loc2 = _inputs(cfg, meta)
    heads = step_of(inp2, feat2, loc2)
    other = O.synth_inputs(cfg, meta["B"], meta["Nv"], meta["Nt"], seed=99, device="cuda")
    # another forward of the same plan in between: the backward recomputes its own forward at its own dropout step
    step_of(other, other["input_imgs"].requires_grad_(True), other["image_loc"].requires_grad_(True))
    MG.heads_objective(heads, meta["B"]).backward()
    assert rel(feat2.grad, feat.grad) < 1e-5 and rel(loc2.grad, loc.grad) < 1e-5


# ------------------------------------------------------------------------------------------ autograd semantics
def test_autograd_semantics(golden_dir):
    cases, _ = _fixture(golden_dir)
    meta = cases["eval"]
    model, cfg = _vl_model(meta)
    model.eval()
    inp, feat, loc = _inputs(cfg, meta)

    def objective(f, l):
        return MG.heads_objective(model(inp["input_txt"], f, l, inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])[:9],
                                  meta["B"])
    objective(feat, loc).backward()
    g1 = feat.grad.clone()
    objective(feat, loc).backward()                 # accumulates
    assert rel(feat.grad, 2 * g1) < 1e-5
    gf, gl = torch.autograd.grad(objective(feat, loc), (feat, loc))
    assert rel(gf, g1) < 1e-5 and gl.shape == loc.shape
    delta = torch.zeros_like(inp["input_imgs"], requires_grad=True)   # a perturbation in front of the model
    objective(inp["input_imgs"] + delta, inp["image_loc"]).backward()
    assert rel(delta.grad, g1) < 1e-5
    cpu = inp["input_imgs"].cpu().requires_grad_(True)
    objective(cpu, inp["image_loc"]).backward()
    assert cpu.grad.device.type == "cpu" and rel(cpu.grad, g1.cpu()) < 1e-5
    half = inp["input_imgs"].half().requires_grad_(True)
    objective(half, inp["image_loc"]).backward()
    assert half.grad.dtype == torch.float16 and rel_l2(half.grad, g1) < 1e-2
    g, = torch.autograd.grad(objective(feat, loc), feat, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()
