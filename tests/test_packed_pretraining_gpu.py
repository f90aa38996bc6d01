"""Packed pre-training steps (engine.pack_padding with BertForMultiModalPreTraining(fused_objective=True)) on the GPU: the same batch
through the padded and the packed plan gives the same three losses and parameter gradients (up to fp32 summation order) for every
visual_target, in train and eval mode, without gradients, in split precision and with a frozen text stream; at the per-GPU
pre-training shape against the fp32 oracle; batches that cannot be packed run padded and are counted; the device-side pack summary
agrees with the host decision; neither pass synchronises the host where it must not; and a captured packed plan replays to the eager
result."""
import json
import os

import pytest
import torch

from _gpu_util import rel_l2
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu

# five distinct dropout probabilities (the four of the config and cls.dropout's 0.1), so a site that drew another site's mask or
# probability would show
DROPOUT = dict(hidden_dropout_prob=0.12, attention_probs_dropout_prob=0.15, v_hidden_dropout_prob=0.2, v_attention_probs_dropout_prob=0.25)


def _cfgj(golden_dir, vt, **over):
    name = "tiny_b4" if vt == 0 else f"tiny_visual_target_{vt}"
    return dict(json.load(open(os.path.join(golden_dir, f"{name}.json")))["config"], **over)


def _model(cfgj, precision=None, seed=3):
    import vilbert_b200
    model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj), precision=precision, fused_objective=True)
    P = O.synth_params(O.make_config(cfgj), seed=seed, device="cuda", with_task_heads=False)
    model.load_state_dict(P, strict=True)
    return model, P


def _prefix(lens, n):
    return (torch.arange(n) < lens.unsqueeze(1)).long()


def _batch(cfgj, B, Nv, Nt, lt, lv, seed=5, frac=0.15):
    """Inputs with prefix-valid masks of lengths lt / lv (host tensors) and labels on valid tokens and regions only: region 1 of
    every sample and token 1 of every sample with two or more tokens are labelled. The masks and labels stay on the host."""
    cfg = O.make_config(cfgj)
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=seed + 1, device="cuda")
    g = torch.Generator().manual_seed(seed)
    mt, mv = _prefix(lt, Nt), _prefix(lv, Nv)
    lm = torch.full((B, Nt), -1, dtype=torch.long)
    sel = (torch.rand(B, Nt, generator=g) < frac) & mt.bool()
    sel[:, 1] |= lt > 1
    lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
    il = torch.full((B, Nv - 1), -1, dtype=torch.long)
    il[(torch.rand(B, Nv - 1, generator=g) < frac) & mv[:, 1:].bool()] = 1
    il[:, 0] = 1
    C_ = cfg["v_target_size"]
    vt = cfgj.get("visual_target", 0)
    it = torch.softmax(torch.randn(B, Nv - 1, C_, generator=g), -1) if vt == 0 else torch.randn(B, Nv - 1, C_, generator=g) * 0.1
    feats = inp["input_imgs"] * mv.cuda().unsqueeze(-1)
    ns = torch.randint(0, 2, (B,), generator=g)
    return [inp["input_txt"], feats, inp["image_loc"], inp["token_type_ids"], mt, mv, lm, il, it.cuda(), ns.cuda()]


def _negatives(model, B, Nv, n_neg, seed=9):
    g = torch.Generator().manual_seed(seed)
    neg = torch.randint(0, B * (Nv - 1), (B, Nv - 1, n_neg), generator=g).cuda()
    model.nce_sampler = lambda b, r, dev: neg.to(dev)


def _step(model, args, pack, step=7, backward=True):
    eng = model.engine
    eng.pack_padding = pack
    eng.set_dropout_step(step)          # the forward bumps it: both arms draw the masks of step + 1
    model.zero_grad()
    losses = model(*args)
    if backward:
        (losses[0] + losses[1] + losses[2]).sum().backward()
    assert (model._last_plan.packed is not None) == pack
    return torch.cat(losses).detach(), eng.ps.grad.clone()


def _same_grads(model, g0, g1, bound=2e-3):
    ps = model.engine.ps
    gmax = g0.abs().max().item()
    worst = max((rel_l2(g1[o:o + n], g0[o:o + n]), k) for k, (o, n) in ((k, ps.span(k)) for k in ps.entries)
                if g0[o:o + n].abs().max().item() > 1e-3 * gmax)
    assert worst[0] < bound, worst
    assert torch.isfinite(g1).all()


# (visual_target, train mode, precision, frozen text stream)
CASES = [(0, True, None, False), (1, True, None, False), (2, True, None, False), (0, False, None, False), (1, False, None, False),
         (2, False, None, False), (0, True, "fp32", False), (2, True, None, True)]


@pytest.mark.parametrize("vt,train,precision,freeze", CASES)
def test_packed_step_matches_padded(golden_dir, vt, train, precision, freeze):
    """Packed vs padded at the same dropout step: the three losses to 1e-5 relative, every parameter gradient to 2e-3 relative L2,
    and the losses of a forward-only (torch.no_grad()) call to 1e-5; a frozen text stream takes no gradient."""
    cfgj = _cfgj(golden_dir, vt, **(DROPOUT if train else {}))
    model, _ = _model(cfgj, precision)
    model.train(train)
    B, Nv, Nt = 6, 11, 9
    args = _batch(cfgj, B, Nv, Nt, torch.tensor([9, 1, 4, 7, 2, 9]), torch.tensor([11, 3, 6, 2, 9, 10]))
    if vt == 2:
        _negatives(model, B, Nv, cfgj["num_negative"])
    frozen = []
    if freeze:
        frozen = [n for n in model._params if n.startswith(("bert.embeddings.", "bert.encoder.layer."))]
        for n in frozen:
            model._params[n].requires_grad_(False)
    l0, g0 = _step(model, args, False)
    l1, g1 = _step(model, args, True)
    assert not model.engine.pack_fallbacks
    assert torch.isfinite(l0).all() and torch.allclose(l1, l0, rtol=1e-5, atol=0), (l0, l1)
    _same_grads(model, g0, g1)
    for n in frozen:
        o, k = model.engine.ps.span(n)
        assert g1[o:o + k].abs().max().item() == 0.0, n
    with torch.no_grad():
        n0, _ = _step(model, args, False, backward=False)
        n1, _ = _step(model, args, True, backward=False)
    assert not model._last_plan.grad_outputs
    assert torch.allclose(n1, n0, rtol=1e-5, atol=0) and torch.allclose(n0, l0, rtol=1e-5, atol=0), (n0, n1, l0)


def _concap_lengths(B, seed):
    """The default length distribution of tools/packed_pretrain_probe.py: captions of U{6..24} tokens, 1 + U{10..36} regions."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(6, 25, (B,), generator=g), 1 + torch.randint(10, 37, (B,), generator=g)


@pytest.mark.parametrize("vt", [0, 2])
def test_production_shape_against_the_oracle(golden_dir, vt):
    """base-6-6 at the per-GPU pre-training shape (B=64, 36 + 1 regions, 36 tokens) with ragged prefix masks: the packed losses
    against the fp32 oracle within the tolerance of test_config3_shape_against_the_oracle, and the gradients against the padded
    step to 2e-3 relative L2."""
    cfgj = dict(json.load(open(os.path.join(golden_dir, "base_6layer_6conect_b4.json")))["config"], visual_target=vt)
    if vt == 2:
        cfgj.update(num_negative=255, v_target_size=cfgj["v_feature_size"])
    B, Nv, Nt = 64, 37, 36
    model, P = _model(cfgj, seed=0)
    model.eval()
    args = _batch(cfgj, B, Nv, Nt, *_concap_lengths(B, 11))
    neg = None
    if vt == 2:
        args[8] = args[1][:, 1:].clone()                 # the region features (train_concap.py's image_target)
        neg = O.nce_negative_indices(B, Nv - 1, 255).cuda()
        model.nce_sampler = lambda b, r, dev: neg.to(dev)
    l0, g0 = _step(model, args, False)
    l1, g1 = _step(model, args, True)
    assert not model.engine.pack_fallbacks
    rows_t, rows_v = model._last_plan.packed
    assert rows_t < B * Nt and rows_v < B * Nv
    _same_grads(model, g0, g1)
    with torch.no_grad():
        ref = O.pretraining_losses(P, O.make_config(cfgj), *[a.cuda() for a in args], neg_index=neg)
    for x, y in zip(l1.tolist(), ref):
        assert abs(x - y.item()) < 2e-3 * abs(y.item()), (x, y.item())


def test_unpackable_batches_run_padded(golden_dir):
    """A non-prefix mask ("mask"), a labelled token on a masked position and a labelled region on a masked region ("label") run the
    plan the same call runs with pack_padding off, are counted once each, and give its losses and gradients; the same holds when
    the masks and labels are on the device. The plan's own run-to-run spread bounds the comparison: its loss and weight-gradient
    kernels add across CTAs with atomics, so two runs of one plan on one batch need not agree to the last bit."""
    cfgj = _cfgj(golden_dir, 1)
    model, _ = _model(cfgj)
    model.eval()
    B, Nv, Nt = 4, 11, 9
    base = _batch(cfgj, B, Nv, Nt, torch.tensor([9, 3, 5, 2]), torch.tensor([11, 4, 8, 6]))
    cases = []
    a = list(base); a[4] = a[4].clone(); a[4][1, 0] = 0; cases.append(("mask", a))
    a = list(base); a[6] = a[6].clone(); a[6][3, 7] = 4; cases.append(("label", a))
    a = list(base); a[7] = a[7].clone(); a[7][1, 6] = 1; cases.append(("label", a))
    a = list(cases[1][1]); a[4:8] = [t.cuda() for t in a[4:8]]; cases.append(("label", a))
    for reason, a in cases:
        l0, g0 = _step(model, a, False)
        padded = model._last_plan
        before = model.engine.pack_fallbacks[reason]
        model.engine.pack_padding = True
        model.zero_grad()
        losses = model(*a)
        sum(losses).sum().backward()
        assert model._last_plan is padded and model.engine.pack_fallbacks[reason] == before + 1, reason
        assert torch.allclose(torch.cat(losses).detach(), l0, rtol=1e-6, atol=0), (reason, losses, l0)
        g1 = model.engine.ps.grad
        assert ((g1 - g0).abs().max() / g0.abs().max()).item() < 1e-5, reason
    assert sum(model.engine.pack_fallbacks.values()) == len(cases)


def test_device_summary_equals_the_host_decision():
    """vb_pack_summary on device tensors decides as the host does on the same tensors, on random batches that include every
    fallback case and absent masks; its counts are the masks' lengths and the labelled tokens."""
    from vilbert_b200.engine import pack_summary, pretraining_pack_rows, pretraining_pack_rows_from_summary
    g = torch.Generator().manual_seed(0)
    seen = set()
    for i in range(60):
        B, Nt, Nv = int(torch.randint(1, 80, (1,), generator=g)), int(torch.randint(1, 40, (1,), generator=g)), int(torch.randint(2, 40, (1,), generator=g))
        mt = _prefix(torch.randint(1, Nt + 1, (B,), generator=g), Nt)
        mv = _prefix(torch.randint(1, Nv + 1, (B,), generator=g), Nv)
        lm = torch.where((torch.rand(B, Nt, generator=g) < 0.2) & mt.bool(), torch.randint(0, 100, (B, Nt), generator=g), -1)
        il = torch.where((torch.rand(B, Nv - 1, generator=g) < 0.2) & mv[:, 1:].bool(), 1, -1)
        k = i % 6
        b = int(torch.randint(0, B, (1,), generator=g))
        if k == 1:
            mt[b] = torch.randint(0, 2, (Nt,), generator=g)       # not prefix-valid unless it happens to be
        elif k == 2:
            mv[b] = 0
        elif k == 3:
            mt[b, -1] = 0; lm[b, -1] = 3
        elif k == 4:
            mv[b, -1] = 0; il[b, -1] = 1
        host = [None if (k == 5 and j < 2) else t for j, t in enumerate((mt, mv, lm, il))]
        want = pretraining_pack_rows(*host, B, Nt, Nv)
        s = pack_summary(*[None if t is None else t.cuda() for t in host], B, Nt, Nv)
        assert pretraining_pack_rows_from_summary(s, B, Nt, Nv) == want, (i, k)
        assert s[:B].tolist() == (mt.ne(0).sum(1).tolist() if host[0] is not None else [Nt] * B)
        assert s[B:2 * B].tolist() == (mv.ne(0).sum(1).tolist() if host[1] is not None else [Nv] * B)
        assert int(s[2 * B + 4]) == int(lm.ne(-1).sum())
        seen.add(want if isinstance(want, str) else "pack")
    assert seen == {"mask", "label", "pack"}


def _warm(model, args, n=3):
    for _ in range(n):      # eager runs, then both passes captured into graphs
        model.zero_grad()
        lt, lv, ln = model(*args)
        (lt + lv + ln).sum().backward()
    assert model._last_plan.packed is not None
    assert model._last_plan.graph_fwd is not None and model._last_plan.graph_bwd is not None


def test_no_synchronisation(golden_dir):
    """With host masks and labels neither the forward nor the backward synchronises; with device masks the forward reads the pack
    summary once, and the backward does not synchronise."""
    cfgj = _cfgj(golden_dir, 0)
    model, _ = _model(cfgj)
    model.train()
    model.engine.pack_padding = True
    args = _batch(cfgj, 4, 9, 8, torch.tensor([8, 2, 5, 3]), torch.tensor([9, 4, 2, 7]))
    args[4:8] = [t.pin_memory() for t in args[4:8]]
    _warm(model, args)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lt, lv, ln = model(*args)
        ((lt + 0.5 * lv + ln) / 4).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    dev = list(args); dev[4:8] = [t.cuda() for t in args[4:8]]
    _warm(model, dev)
    lt, lv, ln = model(*dev)
    total = ((lt + 0.5 * lv + ln) / 4).sum()
    torch.cuda.set_sync_debug_mode("error")
    try:
        total.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert not model.engine.pack_fallbacks


def test_graph_replay_matches_eager(golden_dir):
    """A packed train-mode step replayed from its captured graphs gives the eager step's losses and gradients."""
    cfgj = _cfgj(golden_dir, 2, **DROPOUT)
    model, _ = _model(cfgj)
    model.train()
    B, Nv, Nt = 4, 9, 8
    args = _batch(cfgj, B, Nv, Nt, torch.tensor([8, 2, 5, 3]), torch.tensor([9, 4, 2, 7]))
    _negatives(model, B, Nv, cfgj["num_negative"])
    res = [_step(model, args, True, step=21) for _ in range(4)]
    plan = model._last_plan
    assert plan.packed is not None and plan.graph_fwd is not None and plan.graph_bwd is not None
    (l0, g0), (l3, g3) = res[0], res[3]
    assert torch.allclose(l0, l3, rtol=1e-6, atol=0), (l0, l3)
    assert ((g3 - g0).abs().max() / g0.abs().max()).item() < 1e-5
