"""Frozen parameters on the GPU: the partial attention backward and the NULL parameter-gradient outputs of the row kernels are
bitwise the full kernels' outputs and write nothing else; plans with frozen parameters keep the forward bit-identical and the
trainable gradients; the module surface leaves frozen parameters' .grad None and their values untouched by optimizers."""
import ctypes as C
import json
import math
import os

import pytest
import torch

from _gpu_util import build_engine, oracle_args
from oracle import vilbert_oracle as O
from test_freeze_cpu import patterns
from vilbert_b200 import _lib as L

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def S():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ kernels
def _attn_args(B, H, Nq, Nk, D, p_drop, bias, seed):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(seed)
    Hd = H * D
    q = torch.randn(B * Nq, 3 * Hd, device=dev, generator=g).half()
    k = torch.randn(B * Nk, 3 * Hd, device=dev, generator=g).half()
    mask = ((torch.rand(B, Nk, device=dev, generator=g) < 0.2).float() * -10000.0).contiguous()
    mask[:, 0] = 0.0
    O_ = torch.zeros(B * Nq, Hd, device=dev, dtype=torch.float16)
    Ob = torch.zeros(B * Nq, Hd, device=dev, dtype=BF)
    lse = torch.zeros(B, H, Nq, device=dev)
    dO = torch.randn(B * Nq, Hd, device=dev, generator=g).to(BF)
    step = torch.full((1,), 5, dtype=torch.int32, device=dev)
    a = L.AttnArgs()
    a.B, a.H, a.Nq, a.Nk, a.D = B, H, Nq, Nk, D
    a.Q, a.ldq, a.K, a.ldk, a.V, a.ldv = q.data_ptr(), 3 * Hd, k[:, Hd:].data_ptr(), 3 * Hd, k[:, 2 * Hd:].data_ptr(), 3 * Hd
    a.mask, a.scale = mask.data_ptr(), 1.0 / math.sqrt(D)
    a.O, a.ldo, a.lse, a.O_b16, a.qkv_fp16 = O_.data_ptr(), Hd, lse.data_ptr(), Ob.data_ptr(), 1
    a.dO, a.lddo = dO.data_ptr(), Hd
    if p_drop:
        a.dropout.step, a.dropout.site, a.dropout.p = step.data_ptr(), 1234, p_drop
    L.check(L.lib().vb_attention_fwd(C.byref(a), S()), "vb_attention_fwd")
    return a, (q, k, mask, O_, Ob, lse, dO, step)


def _attn_bwd(a, B, H, Nq, Nk, D, want_q, want_kv, bias):
    """Runs the backward into sentinel-filled outputs; returns (dq, dk, dv, dbq, dbk, dbv)."""
    dev = torch.device("cuda")
    Hd = H * D
    sent = torch.tensor(-7.25, dtype=BF)
    dq = torch.full((B * Nq, Hd), sent.item(), device=dev, dtype=BF)
    dk = torch.full((B * Nk, Hd), sent.item(), device=dev, dtype=BF)
    dv = torch.full((B * Nk, Hd), sent.item(), device=dev, dtype=BF)
    db = [torch.full((Hd,), 0.5, device=dev) for _ in range(3)]
    delta = torch.zeros(B, H, Nq, device=dev)
    a.dQ, a.lddq = (dq.data_ptr() if want_q else None), Hd
    a.dK, a.lddk = (dk.data_ptr() if want_kv else None), Hd
    a.dV, a.lddv = (dv.data_ptr() if want_kv else None), Hd
    a.delta = delta.data_ptr()
    a.dbias_q, a.dbias_k, a.dbias_v = (db[0].data_ptr(), db[1].data_ptr(), db[2].data_ptr()) if bias else (None, None, None)
    L.check(L.lib().vb_attention_bwd(C.byref(a), S()), "vb_attention_bwd")
    torch.cuda.synchronize()
    return dq, dk, dv, *db


@pytest.mark.parametrize("D", [32, 64, 128])
@pytest.mark.parametrize("Nq,Nk", [(37, 101), (101, 36), (150, 101), (36, 200)])     # fused; fused; two kernels; two kernels
@pytest.mark.parametrize("p_drop,bias", [(0.0, False), (0.1, True)])
def test_partial_attention_backward_is_bitwise_the_full_one(D, Nq, Nk, p_drop, bias):
    B, H = 3, 2
    a, keep = _attn_args(B, H, Nq, Nk, D, p_drop, bias, seed=D + Nq)
    full = _attn_bwd(a, B, H, Nq, Nk, D, True, True, bias)
    q_only = _attn_bwd(a, B, H, Nq, Nk, D, True, False, bias)
    kv_only = _attn_bwd(a, B, H, Nq, Nk, D, False, True, bias)
    sentinel = torch.tensor(-7.25, dtype=BF).item()
    assert torch.equal(q_only[0], full[0]) and torch.equal(kv_only[1], full[1]) and torch.equal(kv_only[2], full[2])
    assert (q_only[1] == sentinel).all() and (q_only[2] == sentinel).all() and (kv_only[0] == sentinel).all()
    if bias:
        # the bias sums accumulate across CTAs with atomics: the order of additions is free, so the comparison allows the float
        # rounding of reordering
        torch.testing.assert_close(q_only[3], full[3], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(kv_only[4], full[4], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(kv_only[5], full[5], rtol=1e-4, atol=1e-5)
        assert (q_only[4] == 0.5).all() and (q_only[5] == 0.5).all() and (kv_only[3] == 0.5).all()   # a bias sum follows its gradient
    del keep


def test_partial_attention_backward_rejects_invalid_sets():
    B, H, Nq, Nk, D = 2, 2, 16, 16, 32
    a, keep = _attn_args(B, H, Nq, Nk, D, 0.0, False, seed=1)
    dk = torch.zeros(B * Nk, H * D, device="cuda", dtype=BF)
    delta = torch.zeros(B, H, Nq, device="cuda")
    a.delta = delta.data_ptr()
    a.dQ = a.dK = a.dV = None
    assert L.lib().vb_attention_bwd(C.byref(a), S()) == L.VB_ERR_INVALID
    a.dK, a.lddk = dk.data_ptr(), H * D                       # dK without dV
    assert L.lib().vb_attention_bwd(C.byref(a), S()) == L.VB_ERR_INVALID
    a.dK, a.dV, a.lddv = None, dk.data_ptr(), H * D           # dV without dK
    assert L.lib().vb_attention_bwd(C.byref(a), S()) == L.VB_ERR_INVALID
    torch.cuda.synchronize()
    del keep


def test_embedding_box_small_linear_gate_and_fuse_backward_null_outputs():
    lib, dev = L.lib(), torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(3)
    # text embedding scatter with task tokens: each table NULL in turn
    B, Nt, H, V = 4, 9, 64, 50
    ids = torch.randint(0, V, (B, Nt), device=dev, generator=g); tt = torch.randint(0, 2, (B, Nt), device=dev, generator=g)
    task = torch.randint(0, 20, (B,), device=dev, generator=g)
    d = torch.randn(B * (Nt + 1), H, device=dev, generator=g)

    def emb(which):
        outs = [torch.full(s, 0.125, device=dev) for s in ((V, H), (Nt + 1, H), (2, H), (20, H))]
        ptr = [o.data_ptr() if w else None for o, w in zip(outs, which)]
        L.check(lib.vb_embed_text_bwd(d.data_ptr(), ids.data_ptr(), tt.data_ptr(), task.data_ptr(), *ptr, B, Nt, H, S()))
        torch.cuda.synchronize()
        return outs
    full = emb((1, 1, 1, 1))
    for i in range(4):
        part = emb(tuple(int(j != i) for j in range(4)))
        assert (part[i] == 0.125).all()
        for j in range(4):
            if j != i:     # atomics: the order of additions is free, so the comparison allows the float rounding of reordering
                torch.testing.assert_close(part[j], full[j], rtol=1e-5, atol=1e-5)
    # box projection
    M, Hv = 300, 96
    dy, loc = torch.randn(M, Hv, device=dev, generator=g), torch.rand(M, 5, device=dev, generator=g)

    def box(w, b):
        dW, db = torch.full((Hv, 5), 0.5, device=dev), torch.full((Hv,), 0.5, device=dev)
        L.check(lib.vb_loc_proj_bwd(dy.data_ptr(), loc.data_ptr(), dW.data_ptr() if w else None, db.data_ptr() if b else None, M, Hv, S()))
        torch.cuda.synchronize()
        return dW, db
    fW, fb = box(1, 1)
    pW, pb = box(0, 1)
    assert (pW == 0.5).all(); torch.testing.assert_close(pb, fb, rtol=1e-5, atol=1e-5)
    pW, pb = box(1, 0)
    assert (pb == 0.5).all(); torch.testing.assert_close(pW, fW, rtol=1e-5, atol=1e-5)
    # small linear: dx is written without atomics and stays bitwise; dW / db NULL
    Ms, K, N = 37, 128, 3
    x, W, dys = torch.randn(Ms, K, device=dev, generator=g), torch.randn(N, K, device=dev, generator=g), torch.randn(Ms, N, device=dev, generator=g)

    def small(dx_on, w, b):
        dx, dW, db = torch.full((Ms, K), 0.5, device=dev), torch.full((N, K), 0.5, device=dev), torch.full((N,), 0.5, device=dev)
        L.check(lib.vb_small_linear_bwd(dys.data_ptr(), x.data_ptr(), K, W.data_ptr(), dx.data_ptr() if dx_on else None, K, 0,
                                        dW.data_ptr() if w else None, db.data_ptr() if b else None, Ms, K, N, None, S()))
        torch.cuda.synchronize()
        return dx, dW, db
    f = small(1, 1, 1)
    p = small(1, 0, 0)
    assert torch.equal(p[0], f[0]) and (p[1] == 0.5).all() and (p[2] == 0.5).all()
    p = small(0, 1, 0)
    assert (p[0] == 0.5).all() and (p[2] == 0.5).all(); torch.testing.assert_close(p[1], f[1], rtol=1e-5, atol=1e-5)
    # gate backward: the in-place scaling of dq / dk is bitwise; dz / dz16 NULL each
    Bg, Ng, cols = 4, 11, 64
    qk = torch.randn(Bg * Ng, 96, device=dev, generator=g).half()
    z = torch.randn(Bg, cols, device=dev, generator=g)
    dqk0 = torch.randn(Bg * Ng, 96, device=dev, generator=g).to(BF)

    def gate(a32, a16):
        dqk = dqk0.clone()
        dz, dz16 = torch.full((Bg, cols), 0.5, device=dev), torch.full((Bg, cols), 0.5, device=dev, dtype=BF)
        L.check(lib.vb_gate_scale_bwd(dqk.data_ptr(), 96, qk.data_ptr(), None, 96, z.data_ptr(), dz.data_ptr() if a32 else None,
                                      dz16.data_ptr() if a16 else None, Bg, Ng, cols, 1, S()))
        torch.cuda.synchronize()
        return dqk, dz, dz16
    f = gate(1, 1)
    for a32, a16 in ((0, 1), (1, 0), (0, 0)):
        p = gate(a32, a16)
        assert torch.equal(p[0], f[0])
        assert torch.equal(p[1], f[1]) if a32 else (p[1] == 0.5).all()
        assert torch.equal(p[2], f[2]) if a16 else (p[2] == 0.5).all()
    # fused pooled product: one side NULL
    n = 4 * 64
    dd, pa, pb_ = (torch.randn(n, device=dev, generator=g) for _ in range(3))

    def fuse(a_on, b_on):
        da, db = torch.full((n,), 0.5, device=dev), torch.full((n,), 0.5, device=dev)
        L.check(lib.vb_fuse_pooled_bwd(dd.data_ptr(), pa.data_ptr(), pb_.data_ptr(), da.data_ptr() if a_on else None,
                                       db.data_ptr() if b_on else None, n, 1, None, S()))
        torch.cuda.synchronize()
        return da, db
    f = fuse(1, 1)
    p = fuse(1, 0)
    assert torch.equal(p[0], f[0]) and (p[1] == 0.5).all()


# ------------------------------------------------------------------------------------------------ engine plans
CONFIGS = {"tiny": "tiny_b4.json", "base_2layer_2conect": "base_2layer_2conect_cfg1.json"}


def _engine_case(golden_dir, cfg_name):
    cfgj = json.load(open(os.path.join(golden_dir, CONFIGS[cfg_name])))["config"]
    cfg = O.make_config(cfgj)
    P = O.synth_params(cfg, seed=5, device="cuda")
    eng = build_engine(cfgj, P, torch.device("cuda"))
    return cfgj, cfg, P, eng


def _run(eng, plan, inp, gout, train):
    if train:
        eng.drop_step.fill_(9)
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                     inp["image_attention_mask"], inp["task_ids"])
    plan.run_forward()
    outs = {n: plan.outputs[n].clone() for n in O.HEAD_NAMES}
    eng.zero_grad(force=True)
    for n in O.HEAD_NAMES:
        plan.gout[n].copy_(gout[n].reshape(plan.gout[n].shape))
    plan.run_backward()
    torch.cuda.synchronize()
    return outs, eng.ps.grad.clone()


@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("pattern", ["text_below_first_connection", "vision_stream", "heads_only"])
@pytest.mark.parametrize("cfg_name", list(CONFIGS))
def test_frozen_plan_forward_bitwise_and_trainable_gradients_kept(golden_dir, cfg_name, pattern, train):
    cfgj, cfg, P, eng = _engine_case(golden_dir, cfg_name)
    frozen = patterns(eng.cfg, list(eng.ps.entries))[pattern]
    B, Nv, Nt = 4, 11, 9
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=77, device="cuda")
    kw = dict(grad_outputs=O.HEAD_NAMES, train=train)
    full, frz = eng.plan(B, Nt, Nv, **kw), eng.plan(B, Nt, Nv, frozen=frozen, **kw)
    g = torch.Generator(device="cuda").manual_seed(11)
    gout = {n: torch.randn(full.outputs[n].shape, device="cuda", generator=g) * 1e-2 for n in O.HEAD_NAMES}
    o1, g1 = _run(eng, full, inp, gout, train)
    _, g2 = _run(eng, full, inp, gout, train)
    o3, g3 = _run(eng, frz, inp, gout, train)
    for n in O.HEAD_NAMES:
        assert torch.equal(o1[n], o3[n]), n
    ps = eng.ps
    gmax = g1.abs().max().item()
    for name, (off, _) in ps.entries.items():
        n = ps.g(name).numel()
        a, b, c = g1[off:off + n], g2[off:off + n], g3[off:off + n]
        if name in frozen:
            assert (c == 0).all(), f"frozen {name} has a gradient"
            continue
        spread = (a - b).abs().max().item()          # run-to-run spread of the all-trainable plan (atomic accumulation order)
        assert (c - a).abs().max().item() <= 2 * spread + 1e-6 * gmax, name
    # against the oracle with the same flags (autograd's gradient of every trainable parameter), as closely as the all-trainable
    # plan matches it: tensors whose exact gradient is ~0 (key biases: softmax shift invariance) carry the same relative error in both
    drop = O.DropMasks(9, head_p=eng.head_dropout_prob) if train else None
    Pg = {k: v.clone().requires_grad_(k not in frozen) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
    Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
    with O.operand_mode():
        _, heads = O.vilbert_for_vl_tasks(Pg, cfg, *oracle_args(inp), drop=drop)
        sum((h.float() * gout[n].reshape(h.shape)).sum() for n, h in zip(O.HEAD_NAMES, heads)).backward()
    ref_max = max(v.grad.abs().max().item() for v in Pg.values() if v.grad is not None)
    errs = []
    for name, (off, _) in ps.entries.items():
        r = Pg[name].grad
        if name in frozen:
            assert r is None
            continue
        if r is None:
            continue
        den = max(r.norm().item(), 1e-3 * ref_max * math.sqrt(r.numel()) * 0.1)
        e_frz = ((g3[off:off + r.numel()].view(r.shape) - r).norm() / den).item()
        e_full = ((g1[off:off + r.numel()].view(r.shape) - r).norm() / den).item()
        assert e_frz <= 1.05 * e_full + 1e-3, (name, e_frz, e_full)
        errs.append(e_frz)
    errs.sort()
    assert errs[len(errs) // 2] < 1.5e-2, errs[len(errs) // 2]


# ------------------------------------------------------------------------------------------------ module surface
def _model(golden_dir, cls_name="VILBertForVLTasks", **over):
    import vilbert_b200
    cfgj = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over)
    cfg = O.make_config(cfgj)
    model = getattr(vilbert_b200, cls_name)(vilbert_b200.BertConfig.from_dict(cfgj), **({"fused_objective": True} if "Pre" in cls_name else {}))
    model.load_state_dict(O.synth_params(cfg, seed=3, device="cuda", with_task_heads="Pre" not in cls_name), strict=False)
    return cfgj, cfg, model


def _vl_loss(model, cfg, seed=0):
    import torch.nn.functional as F
    inp = O.synth_inputs(cfg, 4, 11, 9, seed=seed, device="cuda")
    args = [inp[k] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")]
    out = model(*args, None, inp["task_ids"])
    tgt = O.synth_vqa_target(4, 3129, seed=seed, device="cuda")
    return F.binary_cross_entropy_with_logits(out[0], tgt) + 0.1 * out[2].float().pow(2).mean() + 0.1 * out[6].float().pow(2).mean()


@pytest.mark.parametrize("train", [False, True])
def test_module_frozen_grads_are_none_and_optimizers_skip_them(golden_dir, train):
    from vilbert_b200.optim import FusedAdamW
    _, cfg, model = _model(golden_dir)
    model.train(train)
    frozen = patterns(model.engine.cfg, list(model._params))["text_below_first_connection"]
    for n in frozen:
        model._params[n].requires_grad_(False)
    before = {n: model._params[n].detach().clone() for n in frozen}
    model.zero_grad()
    assert all(model._params[n].grad is None for n in frozen)
    _vl_loss(model, cfg).backward()
    ps = model.engine.ps
    for n in frozen:
        assert model._params[n].grad is None
        assert (ps.g(n) == 0).all()
    assert all(p.grad is not None for n, p in model._params.items() if n not in frozen)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-2)
    opt.step()
    for n in frozen:
        assert torch.equal(model._params[n].detach(), before[n]), n
    # FusedAdamW built while everything was trainable: a parameter frozen afterwards is left alone from the next step on
    _, cfg, model = _model(golden_dir)
    model.train(train)
    fused = FusedAdamW(model.parameters(), lr=1e-2, model=model)
    name = "bert.encoder.c_layer.0.biattention.query1.weight"
    model._params[name].requires_grad_(False)
    keep = model._params[name].detach().clone()
    other = model._params["bert.encoder.c_layer.0.biattention.key1.weight"].detach().clone()
    _vl_loss(model, cfg).backward()
    fused.step()
    torch.cuda.synchronize()
    assert torch.equal(model._params[name].detach(), keep)
    assert not torch.equal(model._params["bert.encoder.c_layer.0.biattention.key1.weight"].detach(), other)


def test_module_everything_frozen_backward_raises(golden_dir):
    _, cfg, model = _model(golden_dir)
    for p in model.parameters():
        p.requires_grad_(False)
    loss = _vl_loss(model, cfg)
    assert not loss.requires_grad
    with pytest.raises(RuntimeError, match="does not require grad"):
        loss.backward()


def test_task_step_with_frozen_encoder(golden_dir):
    import _task_oracle as T
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    cfgj, cfg, model = _model(golden_dir, task_specific_tokens=True, max_position_embeddings=300)
    model.train()

    def step():
        batch = T.make_batch(cfgj, "TASK1", 4, 11, 9, seed=5)
        model.zero_grad()
        model.engine.set_dropout_step(3)       # the same dropout masks in every call
        loss, _ = ForwardModelsTrain(None, T.TASK_CFG, torch.device("cuda"), "TASK1", {"TASK1": 0}, {}, {"TASK1": [batch]}, model,
                                     LoadLosses(None, T.TASK_CFG, ["1"]))
        return loss
    loss_full = step()
    loss_full.backward()
    g_full = model.engine.ps.grad.clone()
    frozen = [n for n in model._params if n.startswith("bert.")]
    for n in frozen:
        model._params[n].requires_grad_(False)
    loss = step()
    # the loss kernel sums its rows with atomics: equal up to the rounding of the summation order
    torch.testing.assert_close(loss, loss_full, rtol=1e-6, atol=0)
    loss.backward()
    ps = model.engine.ps
    for n in frozen:
        assert model._params[n].grad is None and (ps.g(n) == 0).all()
    for n in ("vil_prediction.logit_fc.3.weight", "vil_prediction.logit_fc.0.weight"):
        torch.testing.assert_close(ps.g(n), g_full[ps.entries[n][0]:ps.entries[n][0] + ps.g(n).numel()].view(ps.g(n).shape),
                                   rtol=1e-3, atol=1e-6)
    for p in model.parameters():
        p.requires_grad_(False)
    loss = step()
    with pytest.raises(RuntimeError):
        loss.backward()


def test_fused_pretraining_with_frozen_text_embeddings(golden_dir):
    from test_replay_gpu import _pretraining_labels
    cfgj, cfg, model = _model(golden_dir, "BertForMultiModalPreTraining", visual_target=2, v_target_size=48, num_negative=20)
    neg = O.nce_negative_indices(4, 8, cfg["num_negative"])      # the same negatives in every call
    model.nce_sampler = lambda b, r, dev: neg.to(dev)
    model.train()
    inp = O.synth_inputs(cfg, 4, 9, 8, seed=2, device="cuda")
    args = [inp[k] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")]
    labels = _pretraining_labels(cfg, 4, 9, 8, 2)

    def losses():
        model.engine.set_dropout_step(4)
        model.zero_grad()
        return model(*args, *labels)
    full = losses()
    sum(full).sum().backward()
    g_full = model.engine.ps.grad.clone()
    frozen = [n for n in model._params if n.startswith("bert.embeddings.")]
    for n in frozen:
        model._params[n].requires_grad_(False)
    part = losses()
    for a, b in zip(part, full):     # summed with atomics: equal up to the rounding of the summation order
        torch.testing.assert_close(a, b, rtol=1e-6, atol=0)
    sum(part).sum().backward()
    ps = model.engine.ps
    for n in frozen:
        assert model._params[n].grad is None and (ps.g(n) == 0).all()
    n = "bert.encoder.layer.0.attention.self.query.weight"
    ref = g_full[ps.entries[n][0]:ps.entries[n][0] + ps.g(n).numel()].view(ps.g(n).shape)
    torch.testing.assert_close(ps.g(n), ref, rtol=1e-3, atol=1e-3 * ref.abs().max().item())
