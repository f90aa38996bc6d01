"""Whole-path parity of the CUDA engine (through the C ABI) against the oracle and the reference's golden tensors.

Numerical contract (BASELINE.json north_star: outputs "within 1e-3 rel fp32 / 1e-2 bf16" of the reference), checked as
`max|a-b| / max|ref|` per tensor against the fp32 oracle (== the reference, bit-exact on CPU), on EVERY one of the 13 outputs
(sequence_output_t/v, pooled_output_t/v and the nine task-head outputs) with no per-head allowance:
  * default precision "fp16" (fp16 forward operands, bf16 gradient operands, fp32 accumulate): 1e-2;
  * precision "fp32" (split precision, fp16 hi+lo operands, 3 tensor-core passes): 1e-3.
Gradients are not part of the north_star contract; they are bounded against the fp32 oracle by rel-L2 per tensor (worst and
median over all parameter tensors), and against the oracle run under the engine's operand rounding ("op" mode).
"""
import json
import math
import os

import pytest
import torch

from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
OUT_TOL = {"fp16": 1e-2, "fp32": 1e-3, "bf16": 3e-2}


def _cfg(golden_dir, name):
    return json.load(open(os.path.join(golden_dir, name + ".json")))["config"]


def _check(r, precision="fp16", grad_worst=2e-2, grad_median=1e-2, modes=("fp32", "op")):
    tol = OUT_TOL[precision]
    for mode in modes:
        if "out_" + mode not in r:
            continue
        for n, e in r["out_" + mode].items():
            assert e < tol, (mode + "-oracle output", n, e)
    if "grad_fp32" in r:
        assert abs(r["loss"] - r["loss_fp32"]) < 1e-3 * abs(r["loss_fp32"])
        for mode in modes:
            if "grad_" + mode not in r:
                continue
            l2 = sorted((v[1], k) for k, v in r["grad_" + mode].items())
            assert l2[-1][0] < grad_worst, ("worst gradient rel-L2 vs " + mode + " oracle", l2[-3:])
            assert l2[len(l2) // 2][0] < grad_median, ("median gradient rel-L2 vs " + mode + " oracle", l2[len(l2) // 2])


@pytest.mark.parametrize("B,Nv,Nt,seed,task", [(4, 11, 9, 0, False), (3, 7, 12, 1, True), (2, 37, 21, 2, False), (6, 33, 24, 4, True)])
def test_tiny_config_outputs_and_gradients(golden_dir, B, Nv, Nt, seed, task):
    """Every output and every parameter gradient on the tiny config: odd batch (NSP branch of vil_binary_prediction),
    task tokens, ragged masks with a length-1 text row, odd extents."""
    from _gpu_util import model_case
    cfgj = dict(_cfg(golden_dir, "tiny_b4"), task_specific_tokens=task)
    r = model_case(cfgj, B, Nv, Nt, seed=seed)
    _check(r)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_tiny_config_other_precisions(golden_dir, precision):
    """The split-precision (fp32 parity) mode and the legacy all-bf16 mode on the tiny config, outputs and gradients."""
    from _gpu_util import model_case
    cfgj = dict(_cfg(golden_dir, "tiny_b4"), task_specific_tokens=True)
    r = model_case(cfgj, 6, 33, 24, seed=4, precision=precision)
    _check(r, precision, modes=("fp32",), grad_worst=5e-2 if precision == "bf16" else 2e-2, grad_median=2e-2 if precision == "bf16" else 1e-2)


@pytest.mark.parametrize("B,Nv,Nt,seed,task,step", [(4, 11, 9, 0, False, 3), (3, 7, 12, 1, True, 11), (6, 33, 24, 4, False, 123456)])
def test_train_mode_dropout_matches_oracle_masks(golden_dir, B, Nv, Nt, seed, task, step):
    """model.train(): every nn.Dropout of the reference (embeddings, attention probabilities incl. both co-attention
    directions, every dense-before-residual, pooled fusion, the two sequence dropouts of the logit heads) runs inside the
    CUDA kernels with a stateless counter-based mask; the oracle applies the SAME masks (oracle.DropMasks), so outputs
    and gradients are compared exactly like in eval mode. Odd B exercises the separate mask of BertPreTrainingHeads."""
    from _gpu_util import model_case
    cfgj = dict(_cfg(golden_dir, "tiny_b4"), task_specific_tokens=task)
    r = model_case(cfgj, B, Nv, Nt, seed=seed, train_step=step)
    _check(r)
    r_eval = model_case(cfgj, B, Nv, Nt, seed=seed)
    # sanity: train and eval outputs really differ (dropout is on)
    assert (r["plan"].outputs["sequence_output_t"] - r_eval["plan"].outputs["sequence_output_t"]).abs().max().item() > 1e-2


def test_train_mode_distinct_dropout_probabilities(golden_dir):
    """Five different probabilities (hidden 0.1, attention 0.15, v_hidden 0.2, v_attention 0.25, head 0.3): each fused dropout
    site must use the probability of ITS reference module. The site / probability / tensor-layout assignment of the oracle's
    DropMasks is itself pinned bit-exact against the reference with every nn.Dropout replaced by the same masks
    (tests/golden/tiny_train_mode_dropout.json, oracle/make_golden.py::check_train_mode_dropout_placement)."""
    from _gpu_util import model_case
    meta = json.load(open(os.path.join(golden_dir, "tiny_train_mode_dropout.json")))
    r = model_case(meta["config"], meta["B"], meta["Nv"], meta["Nt"], seed=0, train_step=meta["step"], head_dropout_prob=meta["head_p"])
    _check(r)
    r = model_case(dict(meta["config"], task_specific_tokens=True), 3, 7, 12, seed=1, train_step=7, head_dropout_prob=meta["head_p"])
    _check(r)


def test_dropout_statistics_and_step_counter(golden_dir):
    """Keep fraction ~ 1-p, masks change with the step counter, same counter -> bit-identical forward."""
    from _gpu_util import build_engine
    cfgj = _cfg(golden_dir, "tiny_b4")
    cfg = O.make_config(cfgj)
    eng = build_engine(cfgj, O.synth_params(cfg, seed=0, device="cuda"), "cuda")
    inp = O.synth_inputs(cfg, 8, 33, 24, seed=5, device="cuda")
    plan = eng.plan(8, 24, 33, train=True)
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    eng.drop_step.fill_(1); plan.run_forward(); torch.cuda.synchronize()
    a = plan.outputs["sequence_output_v"].clone()
    plan.run_forward(); torch.cuda.synchronize()
    assert torch.equal(a, plan.outputs["sequence_output_v"])
    eng.bump_dropout_step(); plan.run_forward(); torch.cuda.synchronize()
    assert int(eng.drop_step.item()) == 2 and not torch.equal(a, plan.outputs["sequence_output_v"])
    m = O.DropMasks(2).mask("bert.v_embeddings.dropout", cfg["hidden_dropout_prob"], (8 * 33, cfg["v_hidden_size"]), "cpu")
    assert abs((m > 0).float().mean().item() - 0.9) < 0.01


def test_tiny_against_reference_golden_tensors(golden_dir):
    """Directly against tensors saved from the UNMODIFIED reference (tests/golden/tiny_b4.pt)."""
    from _gpu_util import build_engine, rel
    meta = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))
    gold = torch.load(os.path.join(golden_dir, "tiny_b4.pt"))
    cfg = O.make_config(meta["config"])
    P = O.synth_params(cfg, seed=meta["seed"], device="cuda")
    eng = build_engine(meta["config"], P, "cuda")
    plan = eng.plan(meta["B"], meta["Nt"], meta["Nv"])
    i = gold["inputs"]
    plan.load_inputs(i["input_txt"], i["input_imgs"], i["image_loc"], i["token_type_ids"], i["attention_mask"], i["image_attention_mask"])
    plan.run_forward(); torch.cuda.synchronize()
    for k, v in {**gold["bert"], **gold["heads"]}.items():
        assert rel(plan.outputs[k].cpu().reshape(v.shape), v) < 1e-2, k


def test_peaked_attention_tiny(golden_dir):
    """query/key weights x8 (SURVEY.md §8c adversarial case i): a peaked softmax amplifies operand rounding of the scores
    (error ~ |S| * 2^-11); still inside the 1e-2 contract in the default precision and 1e-3 in split precision."""
    from _gpu_util import model_case
    _check(model_case(_cfg(golden_dir, "tiny_b4"), 2, 37, 21, seed=2, qk_scale=8.0))
    _check(model_case(_cfg(golden_dir, "tiny_b4"), 2, 37, 21, seed=2, qk_scale=8.0, precision="fp32", grads=False, oracle_modes=("fp32",)), "fp32", modes=("fp32",))


@pytest.mark.parametrize("task,Nt", [(False, 12), (True, 9)])
def test_fast_mode_text_broadcast(golden_dir, task, Nt):
    """config.fast_mode (BertEncoder FAST_MODE, vilbert.py:1042-1053; eval_retrieval.py): ONE caption (text batch 1) scored against
    a batch of images — the text stream runs at batch 1 up to the first connection layer and is broadcast from there. All 13
    outputs vs the oracle (pinned bit-exact against the reference for this path: tests/golden/tiny_fast_mode.json), through the
    engine and through the module surface; it is an inference path (train mode / gradients are refused)."""
    import vilbert_b200
    from _gpu_util import build_engine, rel
    cfgj = dict(_cfg(golden_dir, "tiny_b4"), fast_mode=True, task_specific_tokens=task)
    cfg = O.make_config(cfgj)
    B, Nv = 6, 33
    P = O.synth_params(cfg, seed=0, device="cuda")
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=4321, device="cuda", task_id=3 if task else None)
    txt = dict(input_txt=inp["input_txt"][:1], token_type_ids=inp["token_type_ids"][:1], attention_mask=inp["attention_mask"][:1],
               task_ids=inp["task_ids"][:1] if task else None)
    bert_o, heads_o = O.vilbert_for_vl_tasks(P, cfg, txt["input_txt"], inp["input_imgs"], inp["image_loc"], txt["token_type_ids"], txt["attention_mask"],
                                             inp["image_attention_mask"], None, txt["task_ids"])
    eng = build_engine(cfgj, P, "cuda")
    plan = eng.plan(B, Nt, Nv)
    plan.load_inputs(txt["input_txt"], inp["input_imgs"], inp["image_loc"], txt["token_type_ids"], txt["attention_mask"], inp["image_attention_mask"],
                     task_ids=txt["task_ids"])
    plan.run_forward(); torch.cuda.synchronize()
    for n, r in list(zip(O.BERT_OUT_NAMES, bert_o)) + list(zip(O.HEAD_NAMES, heads_o)):
        assert tuple(plan.outputs[n].shape) == tuple(r.shape) and rel(plan.outputs[n], r) < 1e-2, n
    with pytest.raises(ValueError):
        eng.plan(B, Nt, Nv, train=True)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1)
    model.load_state_dict(P, strict=True); model.eval()
    out = model(txt["input_txt"], inp["input_imgs"], inp["image_loc"], txt["token_type_ids"], txt["attention_mask"], inp["image_attention_mask"], None, txt["task_ids"])
    assert tuple(out[2].shape) == (B, 1) and rel(out[2], heads_o[2]) < 1e-2     # vil_logit: the retrieval score of each image


def test_roberta_config(golden_dir):
    """config.model == "roberta" (config/bert_base_6layer_6conect roberta variant): the reference's embeddings for it are the
    BERT ones (tests/golden/tiny_roberta.json pins this against the reference), so all outputs match the oracle; with task tokens
    the reference cannot run and the config is refused."""
    from _gpu_util import model_case
    _check(model_case(dict(_cfg(golden_dir, "tiny_b4"), model="roberta"), 4, 11, 9, seed=1234))
    import vilbert_b200
    with pytest.raises(NotImplementedError):
        vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(dict(_cfg(golden_dir, "tiny_b4"), model="roberta", task_specific_tokens=True)),
                                       num_labels=1)


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_dynamic_attention_gates(golden_dir, precision):
    """config.dynamic_attention (BertImageSelfAttention, vilbert.py:557-586; --dynamic_attention of train_tasks.py:357-358): the image
    self-attention's queries / keys gated by 1 + sigmoid(dyLinear(masked mean of the text states)). All 13 outputs and every
    parameter gradient (the dyLinear gates, and the text stream through the pooling) vs the oracle, which is pinned bit-exact
    against the reference for this path (tests/golden/tiny_dynamic_attention.json); ragged text masks, with and without task tokens."""
    from _gpu_util import model_case
    cfgj = dict(_cfg(golden_dir, "tiny_b4"), dynamic_attention=True)
    modes = ("fp32", "op") if precision == "fp16" else ("fp32",)
    r = model_case(cfgj, 4, 11, 9, seed=1234, precision=precision, oracle_modes=modes)
    _check(r, precision, modes=modes)
    gates = [k for k in r["grad_fp32"] if "dyLinear" in k]
    assert len(gates) == 8 and all(r["engine"].ps.g(k).abs().max().item() > 0 for k in gates)
    r = model_case(dict(cfgj, task_specific_tokens=True), 3, 7, 12, seed=1, precision=precision, oracle_modes=modes)
    _check(r, precision, modes=modes)


def test_dynamic_attention_base_shape(golden_dir):
    """dynamic_attention at the base 6-layer widths (Hv 1024 gated by Ht 768) and the VQA sequence lengths, small batch."""
    from _gpu_util import model_case
    cfgj = dict(_cfg(golden_dir, "base_6layer_6conect_b4"), dynamic_attention=True)
    # looser worst-case gradient bound: the query / key biases of the first text layers have an exact gradient close to zero at B=4
    _check(model_case(cfgj, 4, 100, 36, seed=0), grad_worst=5e-2, grad_median=1.5e-2)
    import vilbert_b200
    with pytest.raises(NotImplementedError):
        vilbert_b200.BertConfig.from_dict(dict(cfgj, fast_mode=True)).check_supported()


def test_in_batch_pairs_expansion(golden_dir):
    """config.in_batch_pairs (vilbert.py:1008-1040): at the first connection layer every (text i, image j) combination of the batch
    becomes a sample (batch b -> b^2). BertModel's four outputs and every parameter gradient (the backward sums each item's
    gradient over its b copies) vs the oracle, which is pinned bit-exact against the reference for this path
    (tests/golden/tiny_in_batch_pairs.json)."""
    from _gpu_util import build_engine, rel, rel_l2
    meta = json.load(open(os.path.join(golden_dir, "tiny_in_batch_pairs.json")))
    cfgj = meta["config"]
    cfg = O.make_config(cfgj)
    b, Nv, Nt = 4, 11, 9
    P = O.synth_params(cfg, seed=0, device="cuda")
    inp = O.synth_inputs(cfg, b, Nv, Nt, seed=555, device="cuda")
    eng = build_engine(cfgj, P, "cuda")
    plan = eng.plan(b, Nt, Nv, grad_outputs=O.BERT_OUT_NAMES, heads="none")
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    plan.run_forward(); torch.cuda.synchronize()
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
    Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
    ref = O.bert_model(Pg, cfg, inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    g = torch.Generator(device="cuda").manual_seed(3)
    ws = [torch.randn(r.shape, device="cuda", generator=g) * 0.1 for r in ref]
    for n, r in zip(O.BERT_OUT_NAMES, ref):
        assert tuple(plan.outputs[n].shape) == tuple(r.shape) and r.shape[0] == b * b and rel(plan.outputs[n], r) < 1e-2, n
    sum((r * w).sum() for r, w in zip(ref, ws)).backward()
    eng.zero_grad(force=True)
    for n, w in zip(O.BERT_OUT_NAMES, ws):
        plan.gout[n].copy_(w.reshape(plan.gout[n].shape))
    plan.run_backward(); torch.cuda.synchronize()
    gmax = max(v.grad.abs().max().item() for v in Pg.values() if v.grad is not None)
    l2 = sorted((rel_l2(eng.ps.g(k), Pg[k].grad), k) for k in eng.ps.entries if Pg[k].grad is not None and Pg[k].grad.abs().max().item() > 1e-3 * gmax)
    assert len(l2) > 40 and l2[-1][0] < 2e-2 and l2[len(l2) // 2][0] < 1e-2, l2[-3:]


def test_visualization_attention_export(golden_dir):
    """config.visualization + output_all_attention_masks=True: the attn_data dicts of every text / image / connection layer
    (probabilities, queries, keys; vilbert.py:451-458, 610-617, 813-821) through the module surface vs the oracle's attention hook
    (pinned against the reference: tests/golden/tiny_visualization.json). Without config.visualization the lists hold one None per
    layer, like the reference."""
    import vilbert_b200
    from _gpu_util import rel
    meta = json.load(open(os.path.join(golden_dir, "tiny_visualization.json")))
    cfgj = meta["config"]
    cfg = O.make_config(cfgj)
    P = O.synth_params(cfg, seed=0, device="cuda")
    inp = O.synth_inputs(cfg, 3, 11, 9, seed=777, device="cuda")
    args = (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1)
    model.load_state_dict(P, strict=True); model.eval()
    out = model(*args, None, None, False, True)
    at, av, ac = out[9]
    got = {}
    O.ATTN_HOOK = lambda name, p, q, k: got.__setitem__(name, (p, q, k))
    try:
        with torch.no_grad():
            O.vilbert_for_vl_tasks(P, cfg, *args)
    finally:
        O.ATTN_HOOK = None
    assert len(at) == cfg["num_hidden_layers"] and len(av) == cfg["v_num_hidden_layers"] and len(ac) == len(cfg["v_biattention_id"])
    for i, d in enumerate(at):
        p, q, k = got[f"bert.encoder.layer.{i}.attention.self.dropout"]
        assert d["attn"].shape == p.shape and rel(d["attn"], p) < 1e-2 and rel(d["queries"], q) < 1e-2 and rel(d["keys"], k) < 1e-2, ("text", i)
        assert (d["attn"].sum(-1) - 1).abs().max().item() < 1e-5
    for i, d in enumerate(av):
        p, q, k = got[f"bert.encoder.v_layer.{i}.attention.self.dropout"]
        assert rel(d["attn"], p) < 1e-2 and rel(d["queries"], q) < 1e-2 and rel(d["keys"], k) < 1e-2, ("image", i)
    for i, d in enumerate(ac):
        p1, q1, k1 = got[f"bert.encoder.c_layer.{i}.biattention.dropout1"]
        p2, q2, k2 = got[f"bert.encoder.c_layer.{i}.biattention.dropout2"]
        assert rel(d["attn1"], p1) < 1e-2 and rel(d["queries1"], q1) < 1e-2 and rel(d["keys1"], k1) < 1e-2, ("conn1", i)
        assert rel(d["attn2"], p2) < 1e-2 and rel(d["querues2"], q2) < 1e-2 and rel(d["keys2"], k2) < 1e-2, ("conn2", i)
    plain = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(dict(cfgj, visualization=False)), num_labels=1)
    plain.eval()
    m = plain(*args, None, None, False, True)[9]
    assert m == ([None] * cfg["num_hidden_layers"], [None] * cfg["v_num_hidden_layers"], [None] * len(cfg["v_biattention_id"]))
    assert plain(*args)[9] == ([], [], [])


def test_fixed_layers_stop_the_gradient(golden_dir):
    """config.fixed_t_layer (vilbert.py:968-1003: the first text layers run under torch.no_grad()): outputs unchanged, the frozen
    layers, the embeddings before them and nothing else lose their gradient (set of gradient-free tensors recorded from the
    reference: tests/golden/tiny_fixed_layers.json), every other gradient matches the oracle."""
    from _gpu_util import model_case
    meta = json.load(open(os.path.join(golden_dir, "tiny_fixed_layers.json")))
    r = model_case(meta["config"], meta["B"], meta["Nv"], meta["Nt"], names=("vil_prediction",))
    _check(r)
    eng = r["engine"]
    zero = sorted(k for k in eng.ps.entries if eng.ps.g(k).abs().max().item() == 0)
    assert zero == sorted(k for k in meta["frozen"] if k in eng.ps.entries), set(zero) ^ set(meta["frozen"])
    assert "bert.encoder.layer.0.output.dense.weight" in zero and "bert.encoder.layer.1.output.dense.weight" not in zero


def test_vqa_only_gradient_set_skips_dead_heads(golden_dir):
    from _gpu_util import model_case
    r = model_case(_cfg(golden_dir, "tiny_b4"), 4, 11, 9, names=("vil_prediction",))
    _check(r)
    eng = r["engine"]
    # heads that received no gradient keep exactly-zero parameter gradients; q_dense* never get one (vilbert.py:834,841)
    for k in eng.ps.entries:
        if k.startswith(("vil_prediction_gqa", "vil_logit", "vision_logit", "linguisic_logit", "cls.")) or "q_dense" in k:
            assert eng.ps.g(k).abs().max().item() == 0, k


def test_base_2layer_2conect_config1(golden_dir):
    """BASELINE.json configs[0] (B=2, 36 regions, 20 tokens) on the real 2-connection-layer config: all 13 outputs inside the
    contract in both precisions. With two samples the pooled path is ill-conditioned for GRADIENTS (vil_binary_prediction is ONE
    row of two logits; a single ReLU flip in a pooler moves whole gradient rows), so gradients are bounded against the oracle
    under the same operand rounding here and against fp32 in the full-size tests."""
    from _gpu_util import model_case
    r = model_case(_cfg(golden_dir, "base_2layer_2conect_cfg1"), 2, 36, 20)
    _check(r, modes=("op",), grad_worst=3e-2, grad_median=1.5e-2)
    for n, e in r["out_fp32"].items():
        assert e < 1e-2, ("fp32-oracle output", n, e)
    r = model_case(_cfg(golden_dir, "base_2layer_2conect_cfg1"), 2, 36, 20, precision="fp32", grads=False, oracle_modes=("fp32",))
    _check(r, "fp32", modes=("fp32",))


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_config2_full_size_parity(golden_dir, precision):
    """BASELINE.json configs[1] at its stated size: bert_base_6layer_6conect, B=64, 100 regions, 36 tokens — all 13 outputs and
    every parameter gradient vs the fp32 oracle (1e-2 default precision, 1e-3 split precision)."""
    from _gpu_util import model_case
    r = model_case(_cfg(golden_dir, "base_6layer_6conect_b4"), 64, 100, 36, precision=precision, oracle_modes=("fp32",))
    _check(r, precision, modes=("fp32",))


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_config3_cc_shape_full_size_parity(golden_dir, precision):
    """BASELINE.json configs[2] per-GPU share: B=64 (global 512 / 8), 36 + 1 regions, 36 tokens, outputs and gradients."""
    from _gpu_util import model_case
    r = model_case(_cfg(golden_dir, "base_6layer_6conect_b4"), 64, 37, 36, seed=3, precision=precision, oracle_modes=("fp32",))
    _check(r, precision, modes=("fp32",))


def test_config3_pretraining_objective_fused_losses(golden_dir):
    """The three-loss pre-training objective (vilbert.py:1578-1590) fused into the plan (masked-LM CE over 30522, masked-region
    KL over 1601, alignment CE; csrc/vb_loss.cu) at the CC shape: loss value and every parameter gradient vs the oracle."""
    from _gpu_util import build_engine, rel_l2
    from vilbert_b200.engine import LOSS_HEADS
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bench import synth_loss_inputs
    cfgj = _cfg(golden_dir, "base_6layer_6conect_b4")
    cfg = O.make_config(cfgj)
    B, Nv, Nt = 64, 37, 36
    P = O.synth_params(cfg, seed=0, device="cuda", with_task_heads=False)
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    eng = Engine(BertConfig.from_dict(cfgj), "cuda", heads="pretraining")
    for k in eng.ps.entries:
        eng.ps.p(k).copy_(P[k])
    eng.refresh_weights()
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=11, device="cuda")
    plan = eng.plan(B, Nt, Nv, grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining")
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    li = synth_loss_inputs(plan, "pretraining", 5, torch)
    for k, v in li.items():
        plan.loss_inputs[k].copy_(v.reshape(plan.loss_inputs[k].shape))
    eng.zero_grad(); plan.run_step(); torch.cuda.synchronize()
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
    Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
    lt, lv, ln = O.pretraining_losses(Pg, cfg, inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                                      inp["image_attention_mask"], li["masked_lm_labels"].view(B, Nt).cuda(), li["image_label"].cuda(),
                                      li["image_target"].cuda(), li["next_sentence_label"].cuda())
    ref = lt + lv + ln
    ref.backward()
    assert abs(plan.loss.item() - ref.item()) < 2e-3 * abs(ref.item()), (plan.loss.item(), ref.item())
    # tensors whose exact gradient is ~0 (key biases: softmax shift invariance) are excluded by a floor of 1e-3 of the largest gradient
    gmax = max(v.grad.abs().max().item() for v in Pg.values() if v.grad is not None)
    l2 = sorted((rel_l2(eng.ps.g(k), Pg[k].grad), k) for k in eng.ps.entries if Pg[k].grad is not None and Pg[k].grad.abs().max().item() > 1e-3 * gmax)
    assert len(l2) > 100 and l2[-1][0] < 5e-2 and l2[len(l2) // 2][0] < 1.5e-2, l2[-3:]


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_pretraining_objective_compacted_lm_head(golden_dir, precision):
    """The fused pre-training objective runs the tied 30522-way decoder on the labelled rows only (Plan.lm_head_compact):
    same loss and gradients as the full-logits plan; more labelled rows than the capacity poison the loss with NaN."""
    from _gpu_util import rel_l2
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine, LOSS_HEADS
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bench import synth_loss_inputs
    cfgj = _cfg(golden_dir, "tiny_b4")
    cfg = O.make_config(cfgj)
    B, Nv, Nt = 16, 11, 20
    P = O.synth_params(cfg, seed=0, device="cuda", with_task_heads=False)
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=3, device="cuda")
    res = {}
    for compact in (True, False):
        eng = Engine(BertConfig.from_dict(cfgj), "cuda", heads="pretraining", precision=precision)
        eng.lm_compact = compact
        for k in eng.ps.entries:
            eng.ps.p(k).copy_(P[k])
        eng.refresh_weights()
        plan = eng.plan(B, Nt, Nv, grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining")
        assert ("linguisic_prediction" in plan.outputs) == (not compact)
        plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
        li = synth_loss_inputs(plan, "pretraining", 5, torch)
        for k, v in li.items():
            plan.loss_inputs[k].copy_(v.reshape(plan.loss_inputs[k].shape))
        eng.zero_grad(); plan.run_step(); torch.cuda.synchronize()
        res[compact] = (plan.loss.item(), eng.ps.grad.clone())
        if compact:
            n, cap = plan.lm_rows()
            assert n == int((li["masked_lm_labels"] != -1).sum()) and n <= cap < B * Nt
            idx = plan.lm_c["idx"].cpu()
            assert idx[:n].tolist() == torch.nonzero(li["masked_lm_labels"] != -1).flatten().tolist() and (idx[n:] == -1).all()
            # every row labelled: 320 rows > capacity 80 -> the loss must not look valid
            plan.loss_inputs["masked_lm_labels"].fill_(7)
            eng.zero_grad(); plan.run_step(); torch.cuda.synchronize()
            assert plan.lm_rows()[0] == B * Nt and math.isnan(plan.loss.item())
    assert abs(res[True][0] - res[False][0]) < 1e-5 * abs(res[False][0]), (res[True][0], res[False][0])
    assert rel_l2(res[True][1], res[False][1]) < 1e-4


def test_shared_activation_arena(golden_dir):
    """Engine.enable_activation_arena (12-in-1 training keeps one plan per task shape but runs them one at a time): two plans of
    different shapes overlay their activations in one arena. Each still reproduces the all-private engine's loss and gradients,
    also after the other plan has run in between; a backward on clobbered activations is refused at the engine level and
    recomputed by the module surface."""
    import vilbert_b200
    from _gpu_util import build_engine, rel_l2
    from vilbert_b200._lib import VBError
    cfgj = _cfg(golden_dir, "tiny_b4")
    cfg = O.make_config(cfgj)
    P = O.synth_params(cfg, seed=0, device="cuda")
    shapes = [(4, 9, 11), (6, 24, 33)]
    inps = [O.synth_inputs(cfg, B, Nv, Nt, seed=10 + i, device="cuda") for i, (B, Nt, Nv) in enumerate(shapes)]
    tgts = [O.synth_vqa_target(B, 3129, seed=3 + i, device="cuda") for i, (B, _, _) in enumerate(shapes)]

    def engine(arena):
        eng = build_engine(cfgj, P, "cuda")
        if arena:
            eng.enable_activation_arena(64 << 20)
        plans = []
        for (B, Nt, Nv), inp, tgt in zip(shapes, inps, tgts):
            p = eng.plan(B, Nt, Nv, grad_outputs=("vil_prediction",), vqa_loss=True)
            p.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
            p.vqa_target.copy_(tgt)
            plans.append(p)
        return eng, plans

    def step(eng, p):
        eng.zero_grad(); p.run_step(); torch.cuda.synchronize()
        return p.loss.item(), eng.ps.grad.clone()

    e0, p0 = engine(False)
    ref = [step(e0, p) for p in p0]
    e1, p1 = engine(True)
    assert p1[0].mask_t.data_ptr() == p1[1].mask_t.data_ptr()
    for order in ((0, 1), (1, 0), (0, 0, 1, 1, 0)):
        for i in order:
            loss, g = step(e1, p1[i])
            assert abs(loss - ref[i][0]) <= 1e-5 * abs(ref[i][0]) and rel_l2(g, ref[i][1]) < 1e-4, (order, i)
    p1[0].run_forward(); p1[1].run_forward()
    with pytest.raises(VBError):
        p1[0].run_backward()
    torch.cuda.synchronize()
    # module surface: two forwards of different shapes, ONE backward of the summed loss -> the first forward is recomputed
    grads = []
    for arena in (False, True):
        model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1)
        model.load_state_dict(P, strict=True); model.eval()
        if arena:
            model.engine.enable_activation_arena(64 << 20)
        total = 0
        for inp, tgt in zip(inps, tgts):
            out = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
            total = total + torch.nn.functional.binary_cross_entropy_with_logits(out[0], tgt, reduction="mean") * tgt.size(1)
        model.zero_grad(); total.backward(); torch.cuda.synchronize()
        grads.append((total.item(), model.engine.ps.grad.clone()))
    assert abs(grads[0][0] - grads[1][0]) <= 1e-5 * abs(grads[0][0]) and rel_l2(grads[1][1], grads[0][1]) < 1e-4


def test_module_surface_autograd_and_state_dict(golden_dir):
    """Drop-in API: VILBertForVLTasks(config).forward(...) 10-tuple, loss.backward() through the autograd bridge,
    state_dict with the reference key names, load_state_dict round trip."""
    import vilbert_b200
    from _gpu_util import oracle_args, rel
    cfgj = _cfg(golden_dir, "tiny_b4")
    cfg = O.make_config(cfgj)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1, default_gpu=True)
    ref_names = set(O.param_shapes(cfg))
    assert set(model.state_dict().keys()) == ref_names
    P = O.synth_params(cfg, seed=0, device="cuda")
    missing, unexpected = model.load_state_dict(P, strict=True)
    assert not missing and not unexpected
    assert model.training           # a freshly constructed module is in train mode, like the reference's
    model.eval()                    # parity protocol: eval mode (from_pretrained also returns eval, vilbert/utils.py:1022)
    assert model.state_dict()["cls.predictions.decoder.weight"].data_ptr() == model.state_dict()["bert.embeddings.word_embeddings.weight"].data_ptr()
    inp = O.synth_inputs(cfg, 4, 11, 9, seed=1234, device="cuda")
    tgt = O.synth_vqa_target(4, 3129, device="cuda")
    out = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"],
                inp["co_attention_mask"], None)
    assert len(out) == 10 and out[9] == ([], [], [])
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
    Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
    _, heads_o = O.vilbert_for_vl_tasks(Pg, cfg, *oracle_args(inp))
    for n, a, b in zip(O.HEAD_NAMES, out[:9], heads_o):
        assert a.shape == b.shape and rel(a, b) < 1e-2, n
    for step in range(2):          # second iteration uses the gradient-set hint: single plan, no recompute
        model.zero_grad()
        out = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
        loss = O.vqa_loss(out[0], tgt) + 0.1 * out[2].pow(2).mean()
        loss.backward()
    lo = O.vqa_loss(heads_o[0], tgt) + 0.1 * heads_o[2].pow(2).mean()
    lo.backward()
    named = dict(model.named_parameters())
    for k in ("bert.encoder.layer.0.attention.self.query.weight", "bert.v_embeddings.image_embeddings.weight", "vil_prediction.logit_fc.3.weight",
              "bert.encoder.c_layer.1.biOutput.dense2.weight", "bert.embeddings.word_embeddings.weight", "vil_logit.weight"):
        assert rel(named[k].grad, Pg[k].grad) < 3e-2, k
    model.train()                   # dropout on: outputs change from call to call (new masks per forward)
    o1 = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])[0]
    o2 = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])[0]
    assert not torch.equal(o1, o2) and torch.isfinite(o1).all()
    model.eval()
    bert_out = model.bert(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    assert len(bert_out) == 5 and tuple(bert_out[0].shape) == (4, 9, cfg["hidden_size"])


def test_graph_replay_matches_eager_and_is_deterministic(golden_dir):
    """CUDA-graph capture of the whole step reproduces the eager plan; forward is run-to-run bit-identical."""
    from _gpu_util import build_engine
    cfgj = _cfg(golden_dir, "tiny_b4")
    cfg = O.make_config(cfgj)
    P = O.synth_params(cfg, seed=0, device="cuda")
    eng = build_engine(cfgj, P, "cuda")
    inp = O.synth_inputs(cfg, 4, 11, 9, seed=1234, device="cuda")
    plan = eng.plan(4, 9, 11, grad_outputs=("vil_prediction",), vqa_loss=True)
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    plan.vqa_target.copy_(O.synth_vqa_target(4, 3129, device="cuda"))
    eng.zero_grad(); plan.run_step(); torch.cuda.synchronize()
    out_e = plan.outputs["vil_prediction"].clone(); loss_e = plan.loss.clone(); g_e = eng.ps.grad.clone()
    plan.run_forward(); torch.cuda.synchronize()
    assert torch.equal(out_e, plan.outputs["vil_prediction"])
    plan.capture()
    eng.zero_grad(); plan.run_step(); torch.cuda.synchronize()
    assert torch.equal(out_e, plan.outputs["vil_prediction"])
    assert abs(loss_e.item() - plan.loss.item()) < 1e-6 * abs(loss_e.item())     # block-level atomics: last-bit order effects
    # split-K atomics make weight gradients order-dependent in the last bits only
    assert ((eng.ps.grad - g_e).abs().max() / g_e.abs().max()).item() < 1e-5


def test_full_size_config2_properties(golden_dir):
    """BASELINE.json configs[1] at full size (B=64, 100 regions, 36 tokens): size-independent properties —
    finite outputs, loss equals the BCE of the returned logits, gradient linearity in the loss scale, padded
    regions' vision_logit carries the -10000 mask, samples are independent of their batch neighbours."""
    from _gpu_util import build_engine
    cfgj = _cfg(golden_dir, "base_6layer_6conect_b4")
    cfg = O.make_config(cfgj)
    P = O.synth_params(cfg, seed=0, device="cuda")
    eng = build_engine(cfgj, P, "cuda")
    B, Nv, Nt = 64, 100, 36
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=7, device="cuda")
    tgt = O.synth_vqa_target(B, 3129, device="cuda")
    plan = eng.plan(B, Nt, Nv, grad_outputs=("vil_prediction",), vqa_loss=True)
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    plan.vqa_target.copy_(tgt)
    eng.zero_grad(); plan.run_step(); torch.cuda.synchronize()
    for n, t in plan.outputs.items():
        assert torch.isfinite(t).all(), n
    assert abs(plan.loss.item() - O.vqa_loss(plan.outputs["vil_prediction"], tgt).item()) < 1e-4 * plan.loss.item()
    pad = inp["image_attention_mask"] == 0
    assert (plan.outputs["vision_logit"].squeeze(-1)[pad] < -9000).all()
    g1 = eng.ps.grad.clone()
    assert torch.isfinite(g1).all() and g1.abs().max() > 0
    plan.run_step(); torch.cuda.synchronize()          # gradients accumulate: second identical step doubles them
    assert ((eng.ps.grad - 2 * g1).abs().max() / g1.abs().max()).item() < 1e-3
    # batch independence: the first 8 samples alone give the same sequence outputs
    first = plan.outputs["sequence_output_v"][:8].clone()
    p8 = eng.plan(8, Nt, Nv)
    p8.load_inputs(*(inp[k][:8] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")))
    p8.run_forward(); torch.cuda.synchronize()
    assert ((p8.outputs["sequence_output_v"] - first).abs().max() / first.abs().max()).item() < 1e-5


# the 8 distinct shapes of the 12 tasks (regions, tokens before the task token) at their per-GPU batch (vilbert_tasks.yml / 8)
TWELVE_IN_ONE = [(16, 101, 23), (16, 101, 26), (32, 200, 20), (64, 101, 30), (32, 101, 20), (16, 101, 40), (32, 101, 56), (8, 306, 256)]


@pytest.mark.parametrize("B,Nv,Nt", TWELVE_IN_ONE)
def test_config5_twelve_in_one_shapes(golden_dir, B, Nv, Nt):
    """BASELINE.json configs[4]: every shape of the 12-in-1 mix (tasks 1-2-4-7-8-9-10-11-12-13-15-17, task tokens on) at its
    per-GPU batch on bert_base_6layer_6conect, outputs AND gradients vs the fp32 oracle; the largest is TASK17 (306 regions x
    256 + 1 tokens)."""
    from _gpu_util import model_case
    cfgj = dict(_cfg(golden_dir, "base_6layer_6conect_b4"), task_specific_tokens=True)
    r = model_case(cfgj, B, Nv, Nt, seed=5, oracle_modes=("fp32",))
    _check(r, modes=("fp32",))


@pytest.mark.parametrize("B,Nv,Nt", [(8, 306, 256), (32, 200, 20)])
def test_config5_split_precision_forward(golden_dir, B, Nv, Nt):
    from _gpu_util import model_case
    cfgj = dict(_cfg(golden_dir, "base_6layer_6conect_b4"), task_specific_tokens=True)
    _check(model_case(cfgj, B, Nv, Nt, seed=5, precision="fp32", grads=False, oracle_modes=("fp32",)), "fp32", modes=("fp32",))


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_config4_bert_large_vcr_shape_full_size(precision):
    """BASELINE.json configs[3] per-GPU share: bert_large_6layer_6conect (24 text layers, 1024/4096, 16 heads), B=32 (global 256
    / 8), 100 regions, 60 tokens; all 13 outputs inside the contract, gradients of the VL-logit + VQA heads' paths bounded
    (36 sub-layers deep, hence the looser gradient bounds)."""
    from _gpu_util import model_case
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfgj = json.load(open(os.path.join(root, "vilbert-multi-task_b200", "configs", "bert_large_6layer_6conect.json")))
    r = model_case(cfgj, 32, 100, 60, seed=2, names=("vil_logit", "vil_prediction"), precision=precision, oracle_modes=("fp32",))
    _check(r, precision, modes=("fp32",), grad_worst=5e-2, grad_median=2e-2)


def test_pretraining_model_losses_and_gradients(golden_dir):
    """BertForMultiModalPreTraining (vilbert.py:1435-1597): masked-LM CE, masked-region KL and alignment CE through the
    module surface, eval mode, vs the oracle; backward through the autograd bridge."""
    import vilbert_b200
    from _gpu_util import rel
    cfgj = _cfg(golden_dir, "tiny_b4")
    cfg = O.make_config(cfgj)
    model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj))
    P = O.synth_params(cfg, seed=3, device="cuda", with_task_heads=False)
    model.load_state_dict(P, strict=True)
    model.eval()
    B, Nv, Nt = 4, 9, 8
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=77, device="cuda")
    g = torch.Generator().manual_seed(5)
    lm = torch.full((B, Nt), -1, dtype=torch.long)
    sel = torch.rand(B, Nt, generator=g) < 0.15; sel[:, 1] = True
    lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
    il = torch.full((B, Nv - 1), -1, dtype=torch.long); il[torch.rand(B, Nv - 1, generator=g) < 0.15] = 1; il[:, 0] = 1
    it = torch.softmax(torch.randn(B, Nv - 1, cfg["v_target_size"], generator=g), -1)
    ns = torch.randint(0, 2, (B,), generator=g)
    lm, il, it, ns = lm.cuda(), il.cuda(), it.cuda(), ns.cuda()
    args = (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"], lm, il, it, ns)
    losses = model(*args)
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
    Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
    ref = O.pretraining_losses(Pg, cfg, *args)
    gold = json.load(open(os.path.join(golden_dir, "tiny_pretraining_losses.json")))["losses"]     # from the reference itself
    for a, b, c in zip(losses, ref, gold):
        assert a.shape == (1,) and abs(a.item() - b.item()) < 5e-3 * abs(b.item()) and abs(a.item() - c) < 5e-3 * abs(c)
    model.zero_grad()
    sum(losses).sum().backward()
    sum(ref).backward()
    named = dict(model.named_parameters())
    for k in ("bert.encoder.layer.1.attention.self.value.weight", "cls.predictions.transform.dense.weight", "cls.imagePredictions.decoder.weight",
              "cls.bi_seq_relationship.weight", "bert.embeddings.word_embeddings.weight", "bert.encoder.c_layer.0.biattention.key1.weight"):
        assert rel(named[k].grad, Pg[k].grad) < 3e-2, k
    # without labels the reference returns the three score tensors + attention-mask tuple (:1591-1597)
    out = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    assert len(out) == 4 and tuple(out[0].shape) == (B, Nt, cfg["vocab_size"]) and tuple(out[1].shape) == (B, Nv, cfg["v_target_size"]) and tuple(out[2].shape) == (B, 2)


@pytest.mark.parametrize("visual_target", [1, 2])
def test_pretraining_other_visual_targets(golden_dir, visual_target):
    """config.visual_target 1 (feature regression, vilbert.py:1507-1513) and 2 (noise-contrastive, :1523-1575) through the module
    surface (v_target_size = feature size): the three losses vs the values recorded from the reference
    (tests/golden/tiny_visual_target_{1,2}.json; for 2 with the negatives the reference sampled, injected through `nce_sampler`) and
    the gradients vs the oracle; the module's own device-side sampler is checked for the exclusion rules."""
    import vilbert_b200
    from _gpu_util import rel_l2
    meta = json.load(open(os.path.join(golden_dir, f"tiny_visual_target_{visual_target}.json")))
    cfgj = meta["config"]
    cfg = O.make_config(cfgj)
    model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj))
    P = O.synth_params(cfg, seed=3, device="cuda", with_task_heads=False)
    model.load_state_dict(P, strict=True); model.eval()
    B, Nv, Nt = meta["B"], meta["Nv"], meta["Nt"]
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=77, device="cuda")
    g = torch.Generator().manual_seed(5)
    lm = torch.full((B, Nt), -1, dtype=torch.long); lm[:, 1] = torch.randint(0, cfg["vocab_size"], (B,), generator=g)
    il = torch.full((B, Nv - 1), -1, dtype=torch.long); il[:, 0] = 1; il[:, 3] = 1; il[2, 7] = 1
    it = torch.randn(B, Nv - 1, 48, generator=g)
    ns = torch.randint(0, 2, (B,), generator=g)
    lm, il, it, ns = lm.cuda(), il.cuda(), it.cuda(), ns.cuda()
    neg = torch.tensor(meta["neg_index"]).cuda() if visual_target == 2 else None
    if neg is not None:
        model.nce_sampler = lambda b, r, dev: neg.to(dev)
    a = (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"], lm, il, it, ns)
    losses = model(*a)
    assert all(x.shape == (1,) for x in losses)
    for x, y in zip(losses, meta["losses"]):
        assert abs(x.item() - y) < 5e-3 * abs(y), (x.item(), y)          # fp16-operand forward vs the reference's fp32 value
    model.zero_grad(); sum(losses).sum().backward()
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
    Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
    sum(O.pretraining_losses(Pg, cfg, *a, neg_index=neg)).backward()
    named = dict(model.named_parameters())
    gmax = max(v.grad.abs().max().item() for v in Pg.values() if v.grad is not None)
    l2 = sorted((rel_l2(named[k].grad, v.grad), k) for k, v in Pg.items() if k in named and v.grad is not None and v.grad.abs().max().item() > 1e-3 * gmax)
    assert len(l2) > 30 and l2[-1][0] < 5e-2 and l2[len(l2) // 2][0] < 2e-2, l2[-3:]
    if visual_target == 2:
        R = Nv - 1
        idx = model._nce_negatives(64, R, torch.device("cuda"))
        own = torch.arange(64, device="cuda").view(64, 1, 1)
        assert tuple(idx.shape) == (64, R, 20) and (idx[:, :, :14] // R != own).all() and (idx[:, :, 14:] // R == own).all()
        assert (idx[:, :, 14:] % R != torch.arange(R, device="cuda").view(1, R, 1)).all() and idx.min() >= 0 and idx.max() < 64 * R


def test_from_pretrained_local_file_with_legacy_names(tmp_path, golden_dir):
    """from_pretrained on a local checkpoint: gamma/beta -> weight/bias renaming, `module.` prefix stripping, base-model
    checkpoint into a model with heads, eval mode on return (vilbert/utils.py:945-958, 1022)."""
    import vilbert_b200
    cfgj = _cfg(golden_dir, "tiny_b4")
    cfg = O.make_config(cfgj)
    P = O.synth_params(cfg, seed=9)
    legacy = {}
    for k, v in P.items():
        k2 = "module." + k
        if "LayerNorm.weight" in k: k2 = k2.replace("LayerNorm.weight", "LayerNorm.gamma")
        if "LayerNorm.bias" in k: k2 = k2.replace("LayerNorm.bias", "LayerNorm.beta")
        legacy[k2] = v
    path = tmp_path / "pytorch_model.bin"
    torch.save(legacy, str(path))
    model = vilbert_b200.VILBertForVLTasks.from_pretrained(str(path), config=vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1, default_gpu=True)
    assert not model.training
    sd = model.state_dict()
    for k in ("bert.embeddings.LayerNorm.weight", "bert.encoder.c_layer.1.biOutput.LayerNorm2.bias", "vil_prediction.logit_fc.3.weight"):
        assert torch.equal(sd[k].cpu(), P[k]), k


def test_bert_model_surface_and_all_encoded_layers(golden_dir):
    """BertModel(config).forward 5-tuple (bare state_dict names, default masks) and output_all_encoded_layers=True: one entry
    per connection layer, pooled outputs taken from the last connection layer like the reference (vilbert.py:1388-1394)."""
    import vilbert_b200
    from _gpu_util import rel
    cfgj = _cfg(golden_dir, "tiny_b4")
    cfg = O.make_config(cfgj)
    model = vilbert_b200.BertModel(vilbert_b200.BertConfig.from_dict(cfgj))
    P = O.synth_params(cfg, seed=0, device="cuda")
    bare = {k[len("bert."):]: v for k, v in P.items() if k.startswith("bert.")}
    assert set(model.state_dict().keys()) == set(bare.keys())
    model.load_state_dict(bare)
    model.eval()
    inp = O.synth_inputs(cfg, 4, 11, 9, seed=1234, device="cuda", ragged=False)
    out = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"])                 # all masks defaulted (:1322-1329)
    ref = O.bert_model(P, cfg, inp["input_txt"], inp["input_imgs"], inp["image_loc"])
    assert len(out) == 5
    for a, b in zip(out[:4], ref):
        assert rel(a, b) < 1e-2
    all_t, all_v, pt, pv, _ = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], output_all_encoded_layers=True)
    r_t, r_v, r_pt, r_pv = O.bert_model(P, cfg, inp["input_txt"], inp["input_imgs"], inp["image_loc"], output_all_encoded_layers=True)
    assert len(all_t) == len(r_t) == len(cfg["t_biattention_id"])
    for a, b in zip(all_t + all_v, r_t + r_v):
        assert rel(a, b) < 1e-2
    assert rel(pt, r_pt) < 1e-2 and rel(pv, r_pv) < 1e-2
