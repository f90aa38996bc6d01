"""The fused pre-training objective on the GPU: the masked-MSE and NCE region kernels through the C ABI against the float64 closed
forms, and BertForMultiModalPreTraining(fused_objective=True) against the reference's recorded losses, the oracle and the module's
own torch objective, with per-loss gradient scaling, graph replay and the capacity limit (recomputation: test_replay_gpu.py)."""
import ctypes as C
import json
import math
import os

import pytest
import torch

import _pretraining_oracle as PO
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
S = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
HEADS = ("linguisic_prediction", "vision_prediction", "seq_relationship_score")


# ------------------------------------------------------------------------------------------ kernels
def _launch(kind, s, t, lab, neg, loss, row_loss, d, acc=0):
    from vilbert_b200 import _lib as L
    B, Nv, D = s.shape
    if kind == "mse":
        st = L.lib().vb_mse_masked_loss(s.data_ptr(), t.data_ptr(), lab.data_ptr(), B, Nv, D, 1.0, row_loss.data_ptr(), loss.data_ptr(), acc,
                                        None if d is None else d.data_ptr(), S())
    else:
        st = L.lib().vb_nce_region_loss(s.data_ptr(), t.data_ptr(), lab.data_ptr(), neg.data_ptr(), B, Nv, D, neg.shape[2], 1.0,
                                        row_loss.data_ptr(), loss.data_ptr(), acc, None if d is None else d.data_ptr(), S())
    L.check(st)


@pytest.mark.parametrize("kind,n", [("mse", 0), ("nce", 127), ("nce", 254)])
@pytest.mark.parametrize("mask", ["none", "one", "15pct", "all"])
def test_region_kernels_against_closed_form(kind, n, mask):
    B, Nv, D = 4, 12, 2048
    R = Nv - 1
    s = torch.randn(B, Nv, D, device="cuda") * 0.05
    t = torch.randn(B, R, D, device="cuda") * 0.05
    lab = torch.full((B, R), -1, dtype=torch.int64, device="cuda")
    if mask == "one":
        lab[2, 5] = 1
    elif mask == "15pct":
        lab[torch.rand(B, R, device="cuda") < 0.15] = 1
        lab[0, 0] = 1
        lab[1, 1] = 0
    elif mask == "all":
        lab[:] = 1
    neg = torch.randint(0, B * R, (B, R, max(n, 1)), device="cuda")
    if n:
        neg[:, :, 1] = neg[:, :, 0]                                     # duplicates
        neg[:, :, 2] = torch.arange(B * R, device="cuda").view(B, R)    # the positive's own row as a negative
    loss, row_loss = torch.full((1,), 3.0, device="cuda"), torch.empty(B * Nv, device="cuda")
    d = torch.full((B, Nv, D), float("nan"), device="cuda")
    _launch(kind, s, t, lab, neg, loss, row_loss, d)
    sd, td, ld, nd = s.cpu().double(), t.cpu().double(), lab.cpu(), neg.cpu()
    ref_loss, ref_d = PO.mse_closed_form(sd, td, ld) if kind == "mse" else PO.nce_closed_form(sd, td, ld, nd)
    got = loss.item()
    if mask == "none":
        assert (got == 0.0) if kind == "mse" else math.isnan(got)
        assert d.abs().max().item() == 0
    else:
        assert abs(got - ref_loss.item()) <= 1e-4 * abs(ref_loss.item()), (got, ref_loss.item())
        scale = ref_d.abs().max().item()
        assert torch.allclose(d.cpu().double(), ref_d, rtol=1e-4, atol=1e-4 * scale)
    assert d[:, 0].abs().max().item() == 0
    # no atomics: a second launch (and an accumulating one) is bitwise reproducible
    again, loss2 = torch.empty_like(d), loss.clone()
    _launch(kind, s, t, lab, neg, loss2, row_loss, again)
    assert torch.equal(again, d) and (torch.equal(loss2, loss) or mask == "none")
    _launch(kind, s, t, lab, neg, loss2, row_loss, None, acc=1)
    if mask != "none":
        assert loss2.item() == pytest.approx(2 * got, rel=1e-6)


def test_nce_out_of_range_index_reads_nothing():
    """Index B * R points just past the target view, into memory of the larger buffer it was carved from: without the guard the
    kernel would return a wrong finite loss; with it the loss is NaN."""
    B, Nv, D, n = 3, 8, 2048, 127
    R = Nv - 1
    big = torch.randn(B * R + 4, D, device="cuda") * 0.05
    t = big[:B * R].view(B, R, D)
    s = torch.randn(B, Nv, D, device="cuda") * 0.05
    lab = torch.full((B, R), -1, dtype=torch.int64, device="cuda")
    lab[1, 3] = 1; lab[2, 0] = 1
    neg = torch.randint(0, B * R, (B, R, n), device="cuda")
    neg[1, 3, 5] = B * R
    loss, row_loss, d = torch.zeros(1, device="cuda"), torch.empty(B * Nv, device="cuda"), torch.empty(B, Nv, D, device="cuda")
    _launch("nce", s, t, lab, neg, loss, row_loss, d)
    assert math.isnan(loss.item()) and torch.isfinite(d).all()
    neg[1, 3, 5] = -1
    _launch("nce", s, t, lab, neg, loss, row_loss, d)
    assert math.isnan(loss.item())


# ------------------------------------------------------------------------------------------ module surface helpers
def _cfgj(golden_dir, name):
    meta = json.load(open(os.path.join(golden_dir, f"{name}.json")))
    return meta, meta["config"]


def _model(cfgj, fused=True, precision=None, seed=3):
    import vilbert_b200
    cfg = O.make_config(cfgj)
    model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj), precision=precision, fused_objective=fused)
    P = O.synth_params(cfg, seed=seed, device="cuda", with_task_heads=False)
    model.load_state_dict(P, strict=True)
    return model, cfg, P


def _labels(cfg, B, Nv, Nt, vt, seed=5, frac=0.15):
    g = torch.Generator().manual_seed(seed)
    lm = torch.full((B, Nt), -1, dtype=torch.long)
    sel = torch.rand(B, Nt, generator=g) < frac; sel[:, 1] = True
    lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
    il = torch.full((B, Nv - 1), -1, dtype=torch.long); il[torch.rand(B, Nv - 1, generator=g) < frac] = 1; il[:, 0] = 1
    C_ = cfg["v_target_size"]
    it = torch.softmax(torch.randn(B, Nv - 1, C_, generator=g), -1) if vt == 0 else torch.randn(B, Nv - 1, C_, generator=g) * 0.1
    ns = torch.randint(0, 2, (B,), generator=g)
    return [x.cuda() for x in (lm, il, it, ns)]


def _args(cfg, B, Nv, Nt, vt, seed=77, **kw):
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=seed, device="cuda")
    return (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"],
            *_labels(cfg, B, Nv, Nt, vt, **kw))


def _oracle(P, cfg, args, neg=None, weights=(1.0, 1.0, 1.0)):
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
    Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
    losses = O.pretraining_losses(Pg, cfg, *args, neg_index=neg)
    sum(w * x for w, x in zip(weights, losses)).backward()
    return losses, Pg


def _grads_vs_oracle(model, Pg, worst=5e-2, median=2e-2, min_tensors=30):
    from _gpu_util import rel_l2
    named = dict(model.named_parameters())
    gmax = max(v.grad.abs().max().item() for v in Pg.values() if v.grad is not None)
    l2 = sorted((rel_l2(named[k].grad, v.grad), k) for k, v in Pg.items()
                if k in named and v.grad is not None and v.grad.abs().max().item() > 1e-3 * gmax)
    assert len(l2) > min_tensors and l2[-1][0] < worst and l2[len(l2) // 2][0] < median, l2[-3:]


# ------------------------------------------------------------------------------------------ against the reference
@pytest.mark.parametrize("vt", [0, 1, 2])
def test_fused_losses_against_the_reference(golden_dir, vt):
    """The three losses vs the values recorded from the reference itself (tiny_pretraining_losses.json, tiny_visual_target_{1,2}.json
    with the reference's negatives through nce_sampler), and every parameter gradient of their sum vs the oracle."""
    meta, cfgj = _cfgj(golden_dir, "tiny_pretraining_losses" if vt == 0 else f"tiny_visual_target_{vt}")
    if vt == 0:
        cfgj = _cfgj(golden_dir, "tiny_b4")[1]
    model, cfg, P = _model(cfgj)
    model.eval()
    B, Nv, Nt = meta["B"], meta["Nv"], meta["Nt"]
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=77, device="cuda")
    g = torch.Generator().manual_seed(5)
    if vt == 0:       # the inputs tiny_pretraining_losses.json was recorded with
        lm = torch.full((B, Nt), -1, dtype=torch.long)
        sel = torch.rand(B, Nt, generator=g) < 0.15; sel[:, 1] = True
        lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
        il = torch.full((B, Nv - 1), -1, dtype=torch.long); il[torch.rand(B, Nv - 1, generator=g) < 0.15] = 1; il[:, 0] = 1
        it = torch.softmax(torch.randn(B, Nv - 1, cfg["v_target_size"], generator=g), -1)
    else:             # ... and tiny_visual_target_{1,2}.json
        lm = torch.full((B, Nt), -1, dtype=torch.long); lm[:, 1] = torch.randint(0, cfg["vocab_size"], (B,), generator=g)
        il = torch.full((B, Nv - 1), -1, dtype=torch.long); il[:, 0] = 1; il[:, 3] = 1; il[2, 7] = 1
        it = torch.randn(B, Nv - 1, 48, generator=g)
    ns = torch.randint(0, 2, (B,), generator=g)
    a = (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"],
         lm.cuda(), il.cuda(), it.cuda(), ns.cuda())
    neg = torch.tensor(meta["neg_index"]).cuda() if vt == 2 else None
    if neg is not None:
        model.nce_sampler = lambda b, r, dev: neg.to(dev)
    model.zero_grad()
    losses = model(*a)
    assert len(losses) == 3 and all(x.shape == (1,) and x.is_cuda and x.requires_grad for x in losses)
    for x, y in zip(losses, meta["losses"]):
        assert abs(x.item() - y) < 5e-3 * abs(y), (x.item(), y)
    assert model._last_plan.loss_in_forward and model._last_plan.cfg.visual_target == vt
    sum(losses).sum().backward()
    _, Pg = _oracle(P, cfg, a, neg)
    _grads_vs_oracle(model, Pg)


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_fused_matches_the_module_objective(golden_dir, precision):
    """Same weights, inputs and dropout step, train mode: the fused objective against the module's torch objective."""
    cfgj = _cfgj(golden_dir, "tiny_b4")[1]
    model, cfg, _ = _model(cfgj, precision=precision)
    model.train()
    a = _args(cfg, 8, 11, 12, 0)
    res = {}
    for fused in (False, True):
        model.fused_objective = fused
        model.engine.set_dropout_step(11)
        model.zero_grad()
        losses = model(*a)
        (losses[0] + losses[1] + losses[2]).sum().backward()
        res[fused] = (torch.cat(losses).detach(), model.engine.ps.grad.clone())
    (l0, g0), (l1, g1) = res[False], res[True]
    assert torch.allclose(l1, l0, rtol=1e-4, atol=0), (l1, l0)
    assert ((g1 - g0).norm() / g0.norm()).item() < 1e-3


@pytest.mark.parametrize("vt", [0, 2])
def test_config3_shape_against_the_oracle(golden_dir, vt):
    """base-6-6 at the per-GPU pre-training shape (B=64, 36 + 1 regions, 36 tokens); visual_target 2 with num_negative 255."""
    cfgj = dict(_cfgj(golden_dir, "base_6layer_6conect_b4")[1], visual_target=vt)
    if vt == 2:
        cfgj.update(num_negative=255, v_target_size=cfgj["v_feature_size"])
    B, Nv, Nt = 64, 37, 36
    model, cfg, P = _model(cfgj, seed=0)
    model.eval()
    # the inputs and labels of test_config3_pretraining_objective_fused_losses (bench.synth_loss_inputs with seed 5)
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=11, device="cuda")
    g = torch.Generator().manual_seed(5)
    lm = torch.full((B * Nt,), -1, dtype=torch.long)
    sel = torch.rand(B * Nt, generator=g) < 0.15
    lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
    il = torch.full((B, Nv - 1), -1, dtype=torch.long)
    il[torch.rand(B, Nv - 1, generator=g) < 0.15] = 1
    il[:, 0] = 1
    it = torch.softmax(torch.randn(B, Nv - 1, cfg["v_target_size"], generator=g), -1).cuda()
    ns = torch.randint(0, 2, (B,), generator=g)
    if vt == 2:
        it = inp["input_imgs"][:, 1:].clone()            # the region features (train_concap.py's image_target)
    a = (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"],
         lm.view(B, Nt).cuda(), il.cuda(), it, ns.cuda())
    neg = None
    if vt == 2:
        neg = O.nce_negative_indices(B, Nv - 1, 255).cuda()
        model.nce_sampler = lambda b, r, dev: neg.to(dev)
    model.zero_grad()
    losses = model(*a)
    sum(losses).sum().backward()
    ref, Pg = _oracle(P, cfg, a, neg)
    for x, y in zip(losses, ref):
        assert abs(x.item() - y.item()) < 2e-3 * abs(y.item()), (x.item(), y.item())
    _grads_vs_oracle(model, Pg, worst=5e-2, median=1.5e-2, min_tensors=100)
    del Pg


# ------------------------------------------------------------------------------------------ per-loss scaling
def test_per_loss_scaling(golden_dir):
    cfgj = _cfgj(golden_dir, "tiny_b4")[1]
    model, cfg, P = _model(cfgj)
    model.eval()
    a = _args(cfg, 4, 9, 8, 0)
    # masked_loss_t + masked_loss_v * img_weight + next_sentence_loss * 0 (--objective 2)
    model.zero_grad()
    lt, lv, ln = model(*a)
    (lt + 0.7 * lv + 0 * ln).sum().backward(retain_graph=True)
    first = model.engine.ps.grad.clone()
    _, Pg = _oracle(P, cfg, a, weights=(1.0, 0.7, 0.0))
    _grads_vs_oracle(model, Pg)
    # a second backward of the same forward gives the same gradient
    model.zero_grad()
    (lt + 0.7 * lv + 0 * ln).sum().backward()
    assert ((model.engine.ps.grad - first).abs().max() / first.abs().max()).item() < 1e-5
    # the masked-LM loss alone: the other two heads receive nothing
    model.zero_grad()
    lt, lv, ln = model(*a)
    lt.sum().backward()
    _, Pg = _oracle(P, cfg, a, weights=(1.0, 0.0, 0.0))
    _grads_vs_oracle(model, Pg, min_tensors=10)
    for k in ("cls.imagePredictions.decoder.weight", "cls.bi_seq_relationship.weight"):
        assert model.engine.ps.g(k).abs().max().item() == 0, k


def test_backward_does_not_synchronise(golden_dir):
    cfgj = _cfgj(golden_dir, "tiny_b4")[1]
    model, cfg, _ = _model(cfgj)
    model.train()
    a = _args(cfg, 4, 9, 8, 0)
    for _ in range(3):        # eager runs, then both passes captured into graphs
        model.zero_grad()
        lt, lv, ln = model(*a)
        (lt + lv + ln).sum().backward()
    assert model._last_plan.graph_fwd is not None and model._last_plan.graph_bwd is not None
    lt, lv, ln = model(*a)
    total = ((lt + 0.5 * lv + ln) / 4).sum()
    torch.cuda.set_sync_debug_mode("error")
    try:
        total.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ edges
def test_eval_under_no_grad_uses_a_forward_only_plan(golden_dir):
    cfgj = _cfgj(golden_dir, "tiny_b4")[1]
    model, cfg, _ = _model(cfgj)
    model.eval()
    a = _args(cfg, 4, 9, 8, 0)
    with_grad = torch.cat(model(*a)).detach()
    with torch.no_grad():
        losses = model(*a)
    plan = model._last_plan
    assert plan.loss_in_forward and not plan.grad_outputs and not any(fn is not None for fn, _, _ in plan.bwd)
    assert not any(x.requires_grad for x in losses)
    assert torch.allclose(torch.cat(losses), with_grad, rtol=1e-6, atol=0)


def test_graph_replay_matches_eager(golden_dir):
    cfgj = _cfgj(golden_dir, "tiny_visual_target_2")[1]
    model, cfg, _ = _model(cfgj)
    model.train()
    a = _args(cfg, 4, 9, 8, 2)
    neg = O.nce_negative_indices(4, 8, cfg["num_negative"]).cuda()
    model.nce_sampler = lambda b, r, dev: neg.to(dev)
    res = []
    for _ in range(4):
        model.engine.set_dropout_step(21)
        model.zero_grad()
        losses = model(*a)
        sum(losses).sum().backward()
        res.append((torch.cat(losses).detach(), model.engine.ps.grad.clone()))
    plan = model._last_plan
    assert plan.graph_fwd is not None and plan.graph_bwd is not None
    (l0, g0), (l3, g3) = res[0], res[3]
    assert torch.equal(l0, l3) or torch.allclose(l0, l3, rtol=1e-6, atol=0)
    assert ((g3 - g0).abs().max() / g0.abs().max()).item() < 1e-5


def test_labels_beyond_the_capacity_give_a_nan_masked_lm_loss(golden_dir):
    cfgj = _cfgj(golden_dir, "tiny_b4")[1]
    model, cfg, _ = _model(cfgj)
    model.eval()
    B, Nv, Nt = 16, 9, 20                       # 320 token rows, capacity 80
    a = list(_args(cfg, B, Nv, Nt, 0))
    a[6] = torch.randint(0, cfg["vocab_size"], (B, Nt), device="cuda")     # every token labelled
    for grad in (True, False):
        with torch.set_grad_enabled(grad):
            lt, lv, ln = model(*a)
        assert math.isnan(lt.item()) and math.isfinite(lv.item()) and math.isfinite(ln.item())


def test_summed_plan_dispatches_the_nce_objective(golden_dir):
    """visual_target == 2 with the summed Plan(loss="pretraining"): the NCE region loss, not a KL over the regression head."""
    from _gpu_util import rel_l2
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine, LOSS_HEADS
    meta, cfgj = _cfgj(golden_dir, "tiny_visual_target_2")
    cfg = O.make_config(cfgj)
    B, Nv, Nt = 8, 9, 10
    P = O.synth_params(cfg, seed=3, device="cuda", with_task_heads=False)
    eng = Engine(BertConfig.from_dict(cfgj), "cuda", heads="pretraining")
    for k in eng.ps.entries:
        eng.ps.p(k).copy_(P[k])
    eng.refresh_weights()
    a = _args(cfg, B, Nv, Nt, 2)
    neg = O.nce_negative_indices(B, Nv - 1, cfg["num_negative"]).cuda()
    plan = eng.plan(B, Nt, Nv, grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining")
    assert "vb_nce_region_loss" in [fn.__name__ for fn, _, _ in plan.bwd if fn is not None]
    plan.load_inputs(*a[:6])
    for k, v in zip(("masked_lm_labels", "image_label", "image_target", "next_sentence_label", "neg_index"), (*a[6:], neg)):
        plan.loss_inputs[k].copy_(v.reshape(plan.loss_inputs[k].shape))
    eng.zero_grad(); plan.run_step(); torch.cuda.synchronize()
    ref, Pg = _oracle(P, cfg, a, neg)
    assert abs(plan.loss.item() - sum(ref).item()) < 5e-3 * abs(sum(ref).item()), (plan.loss.item(), [x.item() for x in ref])
    gmax = max(v.grad.abs().max().item() for v in Pg.values() if v.grad is not None)
    l2 = sorted((rel_l2(eng.ps.g(k), Pg[k].grad), k) for k in eng.ps.entries if Pg[k].grad is not None and Pg[k].grad.abs().max().item() > 1e-3 * gmax)
    assert len(l2) > 30 and l2[-1][0] < 5e-2 and l2[len(l2) // 2][0] < 2e-2, l2[-3:]
