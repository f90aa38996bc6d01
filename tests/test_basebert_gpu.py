"""Single-stream baseline (BaseBertForVLTasks) on the H100: the seven outputs and every parameter gradient against the fp32 oracle
(which tests/test_basebert_cpu.py pins to the reference) at the tiny golden shape and at full size across the 128-row attention
boundary, train mode, the new kernels against torch, graph-replay determinism, frozen parameters, the fused optimizer and loading."""
import gc
import json
import os

import pytest
import torch

from oracle import basebert_oracle as BO
from oracle.vilbert_oracle import DropMasks, make_config

pytestmark = pytest.mark.gpu
OUT_TOL = {"fp16": 1e-2, "fp32": 1e-3}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-20)).item()


def rel_l2(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-20)).item()


def _tiny(golden_dir):
    return json.load(open(os.path.join(golden_dir, "tiny_basebert.json")))


def _full_cfg():
    return json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))


def _model(cfgj, labels, P, precision="fp16"):
    # engines of earlier cases hold each other in reference cycles: collect them first, an 80 GB card does not hold several
    # full-size engines and oracles at once
    gc.collect()
    torch.cuda.empty_cache()
    from vilbert_b200.basebert import BaseBertForVLTasks
    from vilbert_b200.config import BertConfig
    m = BaseBertForVLTasks(BertConfig.from_dict(cfgj), labels, precision=precision)
    sd = dict(P)
    sd["cls.predictions.decoder.weight"] = P["bert.embeddings.word_embeddings.weight"]
    m.load_state_dict(sd)
    return m


def _engine_run(m, inp, R, train_step=None):
    """Outputs and parameter gradients of the seeded objective through the module surface (autograd bridge)."""
    m.train(train_step is not None)
    if train_step is not None:
        m.engine.set_dropout_step(train_step - 1)      # the train-mode forward bumps it to train_step
    m.zero_grad()
    outs = dict(zip(BO.OUT_NAMES, m(**inp)))
    sum((outs[k] * R[k]).sum() for k in BO.OUT_NAMES).backward()
    grads = {k: (None if p.grad is None else p.grad.clone()) for k, p in m._params.items()}
    return {k: v.detach() for k, v in outs.items()}, grads


def _oracle_run(P, cfg, inp, R, drop=None):
    Pl = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    out = BO.base_bert_for_vl_tasks(Pl, cfg, drop=drop, **inp)
    sum((out[k] * R[k]).sum() for k in BO.OUT_NAMES).backward()
    return {k: v.detach() for k, v in out.items()}, {k: v.grad for k, v in Pl.items()}


def _check(eo, eg, oo, og, precision, grad_worst=2e-2, grad_median=1e-2):
    for k in BO.OUT_NAMES:
        assert eo[k].shape == oo[k].shape, k
        assert rel(eo[k], oo[k]) < OUT_TOL[precision], (k, rel(eo[k], oo[k]))
    l2 = []
    for k, ref in og.items():
        if float(ref.abs().max()) == 0.0:
            assert float(eg[k].abs().max()) == 0.0, k
            continue
        if k.endswith(".attention.self.key.bias"):
            # exactly zero in exact arithmetic (softmax is invariant to a per-query shift): both sides are rounding noise, measured
            # against the query bias gradient of the same layer
            q = og[k.replace(".key.", ".query.")]
            l2.append(((eg[k].float() - ref.float()).norm().item() / (q.float().norm().item() + 1e-20), k))
            continue
        l2.append((rel_l2(eg[k], ref), k))
    l2.sort()
    assert l2[-1][0] < grad_worst, l2[-3:]
    assert l2[len(l2) // 2][0] < grad_median, l2[len(l2) // 2]
    for k in ("bert.embeddings.position_embeddings.weight", "bert.embeddings.token_type_embeddings.weight",
              "bert.image_embeddings.token_type_embeddings.weight"):
        assert float(eg[k][0].abs().max()) == 0.0, k         # padding_idx=0: row 0 takes exactly no gradient


def _case(cfgj, labels, B, Nt, Nv, precision, train_step=None, seeds=(0, 1234, 7), std=0.05):
    cfg = make_config(cfgj)
    P = BO.synth_params(cfg, labels, seeds[0], device="cuda", std=std)
    inp = BO.synth_inputs(cfg, B, Nt, Nv, seeds[1], device="cuda")
    R = BO.probe_weights(B, Nt, Nv, labels, cfg["vocab_size"], seeds[2], device="cuda")
    m = _model(cfgj, labels, P, precision)
    eo, eg = _engine_run(m, inp, R, train_step)
    drop = DropMasks(train_step, head_p=0.1) if train_step is not None else None
    oo, og = _oracle_run(P, cfg, inp, R, drop)
    return eo, eg, oo, og


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("train", [False, True])
def test_tiny_golden_shape(golden_dir, precision, train):
    meta = _tiny(golden_dir)
    r = _case(meta["config"], meta["num_labels"], meta["B"], meta["Nt"], meta["Nv"], precision,
              train_step=meta["train_step"] if train else None)
    _check(*r, precision)


def test_tiny_matches_recorded_reference(golden_dir):
    """The engine's outputs against the reference's recorded tensors themselves (split precision, eval mode)."""
    meta = _tiny(golden_dir)
    gold = torch.load(os.path.join(golden_dir, "tiny_basebert.pt"))["eval"]
    eo, eg, _, _ = _case(meta["config"], meta["num_labels"], meta["B"], meta["Nt"], meta["Nv"], "fp32")
    # the fixture keeps larger tensors as seeded samples plus norms: outputs to the split-precision tolerance; gradients (bf16
    # operands in the backward) by their L2 norm and sum to 2e-2, their samples to 5e-2 of the largest magnitude
    for k in BO.OUT_NAMES:
        assert max(BO.digest_errors(eo[k], gold["outputs"][k])) < OUT_TOL["fp32"], k
    for k, ref in gold["grads"].items():
        if k.endswith(".attention.self.key.bias"):
            continue            # exactly zero in exact arithmetic: rounding noise on both sides
        samp, l2, sm = BO.digest_errors(eg[k], ref)
        assert l2 < 2e-2 and sm < 2e-2 and samp < 5e-2, (k, samp, l2, sm)


@pytest.mark.parametrize("Nt", [36, 60])
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_full_size_past_128_rows(precision, Nt):
    """bert_base_6layer_6conect at B=64, 101 regions: a 137- / 161-row stream, past the single-pass fused attention backward."""
    r = _case(_full_cfg(), 3129, 64, Nt, 101, precision, seeds=(3, 11, 5), std=0.02)
    # the worst tensors are SimpleClassifier's and the pooler's: their weight gradients contract bf16 gradient operands over B = 64
    # rows, and weight_g = <dW, v> / ||v|| cancels over 1.2 M products, which amplifies that rounding (measured up to 5e-2)
    _check(*r, precision, grad_worst=8e-2)


def _lib():
    from vilbert_b200 import _lib as L
    return L, L.lib(), torch.cuda.current_stream().cuda_stream


def test_concat_embedding_layernorm_kernel():
    L, lib, st = _lib()
    torch.manual_seed(0)
    B, Nt, Nv, H = 5, 13, 21, 768
    xt, xv = torch.randn(B * Nt, H, device="cuda"), torch.randn(B * Nv, H, device="cuda") * 2 + 0.5
    trow = torch.randn(H, device="cuda")
    gt, bt, gv, bv = (torch.randn(H, device="cuda") * 0.2 + (1 if i % 2 == 0 else 0) for i in range(4))
    y = torch.empty(B * (Nt + Nv), H, device="cuda")
    y16, yb = torch.empty_like(y, dtype=torch.float16), torch.empty_like(y, dtype=torch.bfloat16)
    mean, rstd = torch.empty(B * (Nt + Nv), device="cuda"), torch.empty(B * (Nt + Nv), device="cuda")
    L.check(lib.vb_concat_embed_ln_fwd(xt.data_ptr(), xv.data_ptr(), trow.data_ptr(), gt.data_ptr(), bt.data_ptr(), gv.data_ptr(),
                                       bv.data_ptr(), y.data_ptr(), y16.data_ptr(), None, yb.data_ptr(), 1, mean.data_ptr(), rstd.data_ptr(),
                                       B, Nt, Nv, H, None, None, st))
    ref_in = [t.clone().requires_grad_(True) for t in (xt, xv, trow, gt, bt, gv, bv)]
    a, b, r, g1, b1, g2, b2 = ref_in

    def ln(x, w, bb):
        u = x.mean(-1, keepdim=True)
        return w * (x - u) / torch.sqrt((x - u).pow(2).mean(-1, keepdim=True) + 1e-12) + bb
    ref = torch.cat([ln(a, g1, b1).view(B, Nt, H), ln(b + r, g2, b2).view(B, Nv, H)], dim=1).view(-1, H)
    assert rel(y, ref) < 1e-5 and rel(y16, ref) < 1e-3 and rel(yb, ref) < 1e-2
    dy = torch.randn_like(y)
    ref.backward(dy)
    dxt, dxv, dxv16 = torch.empty_like(xt), torch.empty_like(xv), torch.empty_like(xv, dtype=torch.bfloat16)
    grads = [torch.zeros(H, device="cuda") for _ in range(6)]
    L.check(lib.vb_concat_embed_ln_bwd(dy.data_ptr(), xt.data_ptr(), xv.data_ptr(), trow.data_ptr(), gt.data_ptr(), gv.data_ptr(),
                                       mean.data_ptr(), rstd.data_ptr(), dxt.data_ptr(), dxv.data_ptr(), dxv16.data_ptr(),
                                       *[g.data_ptr() for g in grads], B, Nt, Nv, H, None, None, st))
    assert rel(dxt, a.grad) < 1e-4 and rel(dxv, b.grad) < 1e-4 and rel(dxv16, b.grad) < 1e-2
    for got, want in zip(grads, (g1.grad, b1.grad, g2.grad, b2.grad, b.grad.sum(0), r.grad)):
        assert rel(got, want) < 1e-4


def test_padded_text_embedding_backward_kernel():
    """Row 0 of the word, position and token-type tables receives exactly nothing; every other row the scatter-add."""
    L, lib, st = _lib()
    B, Nt, H, V = 4, 10, 64, 30
    ids = torch.randint(0, V, (B, Nt), device="cuda")
    ids[:, 3] = 0
    tt = torch.randint(0, 2, (B, Nt), device="cuda")
    d = torch.randn(B * Nt, H, device="cuda")
    dw, dp, dt = torch.zeros(V, H, device="cuda"), torch.zeros(Nt, H, device="cuda"), torch.zeros(2, H, device="cuda")
    L.check(lib.vb_embed_text_bwd_padded(d.data_ptr(), ids.data_ptr(), tt.data_ptr(), dw.data_ptr(), dp.data_ptr(), dt.data_ptr(), B, Nt, H, st))
    W = torch.zeros(V, H, device="cuda", requires_grad=True)
    Pm = torch.zeros(Nt, H, device="cuda", requires_grad=True)
    T = torch.zeros(2, H, device="cuda", requires_grad=True)
    pos = torch.arange(Nt, device="cuda").expand(B, Nt)
    F = torch.nn.functional
    out = F.embedding(ids, W, padding_idx=0) + F.embedding(pos, Pm, padding_idx=0) + F.embedding(tt, T, padding_idx=0)
    out.backward(d.view(B, Nt, H))
    for got, want in ((dw, W.grad), (dp, Pm.grad), (dt, T.grad)):
        assert float(got[0].abs().max()) == 0.0
        assert rel(got, want) < 1e-5


def test_weight_norm_kernel():
    L, lib, st = _lib()
    torch.manual_seed(1)
    v = torch.randn(1536, 768, device="cuda") * 0.03
    g = torch.tensor(3.7, device="cuda")
    w32, w16, wb = torch.empty_like(v), torch.empty_like(v, dtype=torch.float16), torch.empty_like(v, dtype=torch.bfloat16)
    scr = torch.empty(L.VB_WEIGHT_NORM_SCRATCH // 8, dtype=torch.float64, device="cuda")
    L.check(lib.vb_weight_norm_fwd(v.data_ptr(), g.data_ptr(), v.numel(), w32.data_ptr(), w16.data_ptr(), None, wb.data_ptr(), 1, scr.data_ptr(), st))
    vr, gr = v.clone().requires_grad_(True), g.clone().requires_grad_(True)
    ref = torch._weight_norm(vr, gr, -1) if hasattr(torch, "_weight_norm") else vr * (gr / vr.norm())
    assert rel(w32, ref) < 1e-5 and rel(w16, ref) < 1e-3
    dw = torch.randn_like(v)
    ref.backward(dw)
    outs = []
    for _ in range(2):
        dg, dv = torch.full((), 0.5, device="cuda"), torch.ones_like(v)
        L.check(lib.vb_weight_norm_bwd(dw.data_ptr(), v.data_ptr(), g.data_ptr(), v.numel(), dg.data_ptr(), dv.data_ptr(), scr.data_ptr(), st))
        outs.append((dg.clone(), dv.clone()))
        assert abs(float(dg) - 0.5 - float(gr.grad)) <= 1e-4 * abs(float(gr.grad)) + 1e-6
        assert rel(dv - 1.0, vr.grad) < 1e-4
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])     # fixed-order reductions


def test_tanh_pooler_kernels():
    L, lib, st = _lib()
    x = torch.randn(64, 768, device="cuda") * 2
    y, y16 = torch.empty_like(x), torch.empty_like(x, dtype=torch.float16)
    L.check(lib.vb_tanh_fwd(x.data_ptr(), y.data_ptr(), y16.data_ptr(), None, None, 1, x.numel(), st))
    assert rel(y, torch.tanh(x)) < 2e-5 and rel(y16, torch.tanh(x)) < 1e-3
    dy = torch.randn_like(x)
    dx, db = torch.empty_like(x, dtype=torch.bfloat16), torch.ones(768, device="cuda")
    L.check(lib.vb_tanh_bwd(dy.data_ptr(), y.data_ptr(), dx.data_ptr(), db.data_ptr(), 64, 768, st))
    want = dy * (1 - y * y)
    assert rel(dx, want) < 1e-2 and rel(db - 1.0, want.sum(0)) < 1e-5


def test_graph_replays_are_bit_identical(golden_dir):
    """Two replays of the captured train-mode step (same dropout step) give bit-identical outputs and weight-norm gradients."""
    from vilbert_b200.engine import BASE_HEAD_NAMES
    meta = _tiny(golden_dir)
    cfg = make_config(meta["config"])
    P = BO.synth_params(cfg, meta["num_labels"], 0, device="cuda")
    m = _model(meta["config"], meta["num_labels"], P)
    m.engine.refresh_weights()
    inp = BO.synth_inputs(cfg, 3, 9, 11, device="cuda")
    plan = m.engine.plan(3, 9, 11, grad_outputs=BASE_HEAD_NAMES, train=True)
    plan.load_inputs(**inp)
    for n in BASE_HEAD_NAMES:
        plan.gout[n].copy_(torch.randn(plan.gout[n].shape, device="cuda"))
    plan.capture(separate=True)
    res = []
    for _ in range(2):
        m.engine.zero_grad(force=True)
        plan.run_forward(); plan.run_backward()
        torch.cuda.synchronize()
        res.append(({n: plan.outputs[n].clone() for n in BASE_HEAD_NAMES}, m.engine.ps.grad.clone()))
    for n in BASE_HEAD_NAMES:
        assert torch.equal(res[0][0][n], res[1][0][n]), n
    ps = m.engine.ps
    for n in ps.entries:
        if n.startswith("vil_prediction."):
            assert torch.equal(ps._view(res[0][1], n), ps._view(res[1][1], n)), n
    assert rel_l2(res[1][1], res[0][1]) < 1e-6


def test_frozen_embeddings_and_first_layer(golden_dir):
    meta = _tiny(golden_dir)
    cfg = make_config(meta["config"])
    P = BO.synth_params(cfg, meta["num_labels"], 0, device="cuda")
    inp = BO.synth_inputs(cfg, 3, 9, 11, device="cuda")
    R = BO.probe_weights(3, 9, 11, meta["num_labels"], cfg["vocab_size"], 7, device="cuda")
    m = _model(meta["config"], meta["num_labels"], P)
    _, full = _engine_run(m, inp, R)
    frozen = [n for n in m._params if n.startswith(("bert.embeddings.", "bert.image_embeddings.", "bert.encoder.layer.0."))]
    frozen.remove("bert.embeddings.word_embeddings.weight")      # the tied decoder keeps the word table trainable
    for n in frozen:
        m._params[n].requires_grad_(False)
    m.engine.ps.grad.fill_(7.0)
    m.engine.grad_clean = False
    _, part = _engine_run(m, inp, R)
    ps = m.engine.ps
    for n in frozen:
        assert part[n] is None, n
        assert bool((ps.g(n) == 7.0).all()) or bool((ps.g(n) == 0.0).all()), n     # zero_grad may clear it; nothing else writes it
    for n, g in part.items():
        if g is not None:
            assert rel_l2(g, full[n]) < 1e-5, n


def test_fused_adamw_round_trip(golden_dir):
    """After a FusedAdamW step on g / v the next forward re-derives the weight-normed weights: it matches the oracle on the
    updated parameters."""
    from vilbert_b200.optim import FusedAdamW
    meta = _tiny(golden_dir)
    cfg = make_config(meta["config"])
    P = BO.synth_params(cfg, meta["num_labels"], 0, device="cuda")
    inp = BO.synth_inputs(cfg, 3, 9, 11, device="cuda")
    R = BO.probe_weights(3, 9, 11, meta["num_labels"], cfg["vocab_size"], 7, device="cuda")
    m = _model(meta["config"], meta["num_labels"], P, "fp32")
    opt = FusedAdamW(m.parameters(), lr=1e-2, model=m)
    _engine_run(m, inp, R)
    opt.step()
    P2 = {k: m._params[k].detach().clone() for k in P}
    assert float((P2["vil_prediction.main.0.weight_g"] - P["vil_prediction.main.0.weight_g"]).abs()) > 0
    m.eval()
    with torch.no_grad():
        eo = dict(zip(BO.OUT_NAMES, m(**inp)))
    oo = BO.base_bert_for_vl_tasks(P2, cfg, **inp)
    for k in BO.OUT_NAMES:
        assert rel(eo[k], oo[k]) < OUT_TOL["fp32"], k


def test_loading_reference_and_text_only_checkpoints(golden_dir, tmp_path):
    from vilbert_b200.basebert import BaseBertForVLTasks
    from vilbert_b200.config import BertConfig
    meta = _tiny(golden_dir)
    cfg = make_config(meta["config"])
    P = BO.synth_params(cfg, meta["num_labels"], 0)
    sd = {k: v for k, v in P.items()}
    sd["cls.predictions.decoder.weight"] = P["bert.embeddings.word_embeddings.weight"]
    assert sorted(sd) == sorted(k for k, _ in meta["state_dict"])
    torch.save(sd, tmp_path / "reference.bin")
    config = BertConfig.from_dict(meta["config"])
    m = BaseBertForVLTasks.from_pretrained(str(tmp_path / "reference.bin"), config=config, num_labels=meta["num_labels"], default_gpu=True)
    assert m.loading_info == {"missing_keys": [], "unexpected_keys": []}
    for k, v in P.items():
        assert torch.equal(m._params[k].detach().cpu(), v), k
    text = {k[len("bert."):].replace("LayerNorm.weight", "LayerNorm.gamma"): v for k, v in sd.items()
            if k.startswith(("bert.embeddings.", "bert.encoder.", "bert.pooler."))}
    torch.save(text, tmp_path / "text.bin")
    m2 = BaseBertForVLTasks.from_pretrained(str(tmp_path / "text.bin"), config=config, num_labels=meta["num_labels"])
    missing = m2.loading_info["missing_keys"]
    assert any(k.startswith("bert.image_embeddings.") for k in missing)
    assert "vil_prediction.main.0.weight_g" in missing and "cls.imagePredictions.decoder.weight" in missing
    assert not any(k.startswith(("bert.embeddings.", "bert.encoder.")) for k in missing)
    assert m2.loading_info["unexpected_keys"] == []


def test_bert_submodule_and_output_modes(golden_dir):
    meta = _tiny(golden_dir)
    cfg = make_config(meta["config"])
    P = BO.synth_params(cfg, meta["num_labels"], 0, device="cuda")
    inp = BO.synth_inputs(cfg, 3, 9, 11, device="cuda")
    m = _model(meta["config"], meta["num_labels"], P, "fp32")
    m.eval()
    with torch.no_grad():
        seq, pooled = m.bert(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                             inp["image_attention_mask"], output_all_encoded_layers=False)
        layers, pooled2 = m.bert(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                                 inp["image_attention_mask"])
    ref_seq, ref_pooled = BO.bert_model(P, cfg, **inp)
    ref_layers, _ = BO.bert_model(P, cfg, all_layers=True, **inp)
    assert seq.shape == (3, 20, cfg["hidden_size"]) and rel(seq, ref_seq) < 1e-3 and rel(pooled, ref_pooled) < 1e-3
    assert len(layers) == cfg["num_hidden_layers"] and all(rel(a, b) < 1e-3 for a, b in zip(layers, ref_layers))
    with pytest.raises(NotImplementedError):
        m(**inp, output_all_encoded_layers=True)
    with pytest.raises(TypeError):
        m(inp["input_txt"], inp["input_imgs"], inp["image_loc"])
