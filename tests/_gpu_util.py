"""Shared GPU check helpers (used by the -m gpu tests and by the tools/ probe drivers).
Every check runs the CUDA path through the C ABI (ctypes) and compares with torch fp32 / the oracle."""
import ctypes as C
import gc
import math

import torch
import torch.nn.functional as F

from oracle import vilbert_oracle as O
from vilbert_b200 import _lib as L

BF = torch.bfloat16


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-20)).item()


def rel_l2(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-20)).item()


def launched(fn, *expect, tries=10, pad_cycles=2_000_000):
    """Runs fn() under torch.profiler (CUDA activity); returns (its result, the names of the recorded events). Kernel names are
    demangled, e.g. "void vb::ln_fwd_kernel<4, false>(float const*, ...)". The profiler now and then delivers a capture without its
    device records (only the runtime calls such as cudaLaunchKernelExC), most often for a capture that holds a single short launch
    late in a long-running process. So fn's launches are bracketed on the stream by two GPU busy-waits of `pad_cycles` clock cycles
    each (about 1 ms), which the capture records too. With expect
    (regular expressions), a capture in which one of them matches no name is taken again, up to `tries` captures, and then asserted:
    the launches are deterministic, so a kernel that is really not launched is missing from every capture. fn must be repeatable."""
    import re
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(pad_cycles)
            r = fn()
            torch.cuda._sleep(pad_cycles)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        if all(any(re.search(pat, n) for n in names) for pat in expect):
            break
    assert_launched(names, *expect)
    return r, names


def assert_launched(names, *patterns):
    """Every regular expression in patterns matches the name of a launched kernel (a boundary case stays on its variant)."""
    import re
    for pat in patterns:
        assert any(re.search(pat, n) for n in names), (pat, sorted(set(names)))


# ------------------------------------------------------------------------------------------ GEMM
def gemm_case(M, N, K, a_mn=False, b_mn=False, bias=False, res=False, act=0, out_bf16=False, atomic=False, split_k=1, block_n=0,
              alpha=1.0, check=True, iters=0, seed=0, both_outputs=False, a_fp16=False, b_fp16=False, out_fp16=False,
              split=False):
    """Returns (max relative error vs fp32 matmul of the 16-bit operands, ms per launch or None). a_fp16 / b_fp16 / out_fp16
    pick fp16 instead of bf16 per operand (mixed formats = the dgrad / wgrad configuration). split=True stores A and B as
    hi + lo (split precision, three passes) and compares with the float64 product of the fp32 operands."""
    dev = torch.device("cuda")
    g_ = torch.Generator(device=dev).manual_seed(seed)
    lib = L.lib()
    dA, dB, dO = (torch.float16 if a_fp16 else BF), (torch.float16 if b_fp16 else BF), (torch.float16 if out_fp16 else BF)
    A32 = torch.randn(M, K, device=dev, generator=g_) * 0.5
    B32 = torch.randn(N, K, device=dev, generator=g_) * 0.5
    A, B = A32.to(dA), B32.to(dB)
    pad8 = lambda x: (x + 7) // 8 * 8
    def store(X, rows, cols, mn, dt):
        if mn:
            st = torch.zeros(cols, pad8(rows), device=dev, dtype=dt); st[:, :rows] = X.t(); return st, pad8(rows)
        st = torch.zeros(rows, pad8(cols), device=dev, dtype=dt); st[:, :cols] = X; return st, pad8(cols)
    A_st, lda = store(A, M, K, a_mn, dA)
    B_st, ldb = store(B, N, K, b_mn, dB)
    if split:
        Al_st, _ = store((A32 - A.float()).to(dA), M, K, a_mn, dA)
        Bl_st, _ = store((B32 - B.float()).to(dB), N, K, b_mn, dB)
    bias_t = torch.randn(N, device=dev, generator=g_) if bias else None
    res_t = torch.randn(M, N, device=dev, generator=g_) if res else None
    aux_t = torch.randn(M, N, device=dev, generator=g_).to(BF) if act == L.VB_ACT_DGELU else None
    out32 = torch.full((M, N), 0.0 if atomic else float("nan"), device=dev)
    out16 = torch.empty(M, N, device=dev, dtype=dO) if out_bf16 else None
    outlo = torch.empty(M, N, device=dev, dtype=dO) if (out_bf16 and split) else None
    outb = torch.empty(M, N, device=dev, dtype=BF) if (out_bf16 and out_fp16 and not atomic) else None   # bf16 copy for the backward
    pre16 = torch.empty(M, N, device=dev, dtype=BF) if (act == L.VB_ACT_GELU and out_bf16 and N % 8 == 0) else None
    g = L.GemmArgs()
    g.M, g.N, g.K = M, N, K
    g.A, g.lda, g.a_mn_major = A_st.data_ptr(), lda, int(a_mn)
    g.B, g.ldb, g.b_mn_major = B_st.data_ptr(), ldb, int(b_mn)
    g.alpha = alpha
    g.bias = bias_t.data_ptr() if bias else None
    g.residual, g.ld_res = (res_t.data_ptr(), N) if res else (None, 0)
    g.aux, g.ld_aux = (aux_t.data_ptr(), N) if aux_t is not None else (None, 0)
    g.act = act
    # like the engine: a bf16-output GEMM has no fp32 output unless both are requested explicitly
    want_f32 = (not out_bf16) or atomic or both_outputs
    g.out_f32, g.ld_out_f32 = (out32.data_ptr(), N) if want_f32 else (None, 0)
    g.out_bf16, g.ld_out_bf16 = (out16.data_ptr(), N) if out_bf16 and not atomic else (None, 0)
    g.out_pre, g.ld_out_pre = (pre16.data_ptr(), N) if pre16 is not None else (None, 0)
    g.atomic_out, g.split_k, g.block_n, g.max_ctas = int(atomic), split_k, block_n, 0
    g.a_fp16, g.b_fp16, g.out_fp16 = int(a_fp16), int(b_fp16), int(out_fp16)
    if split:
        g.A_lo, g.B_lo = Al_st.data_ptr(), Bl_st.data_ptr()
        if outlo is not None and not atomic: g.out_lo = outlo.data_ptr()
    if outb is not None: g.out_b16 = outb.data_ptr()
    L.check(lib.vb_gemm_bf16(C.byref(g), stream()), "vb_gemm_bf16")
    torch.cuda.synchronize()
    err = None
    if check:
        ref = alpha * ((A32.double() @ B32.double().t()).float() if split else (A.float() @ B.float().t()))
        if bias: ref = ref + bias_t
        if act == L.VB_ACT_GELU:
            x_ = ref.clone(); ref = O.gelu(ref)
            pre_ref = 0.5 * (1 + torch.erf(x_ / 2 ** 0.5)) + x_ * torch.exp(-0.5 * x_ * x_) / math.sqrt(2 * math.pi)   # saved gelu'(pre)
        elif act == L.VB_ACT_RELU:
            ref = ref.clamp_min(0)
        elif act == L.VB_ACT_DGELU:
            ref = ref * aux_t.float()            # aux = saved gelu'(pre)
        if res: ref = ref + res_t
        scale = ref.abs().max().item() + 1e-9
        err = ((out32 - ref).abs().max() / scale).item() if want_f32 else 0.0
        if out16 is not None and not atomic:
            if outlo is not None:   # hi + lo reconstructs the fp32 epilogue value
                err = max(err, (((out16.float() + outlo.float()) - ref).abs().max() / scale).item())
            else:
                err = max(err, ((out16.float() - ref).abs().max() / scale).item() - (5e-4 if out_fp16 else 4e-3))   # output rounding
        if outb is not None:
            err = max(err, ((outb.float() - ref).abs().max() / scale).item() - 4e-3)
        if pre16 is not None:
            err = max(err, ((pre16.float() - pre_ref).abs().max() / (pre_ref.abs().max() + 1e-9)).item() - 4e-3)
        if err != err: err = float("inf")
    ms = None
    if iters:
        if atomic: out32.zero_()
        for _ in range(3): lib.vb_gemm_bf16(C.byref(g), stream())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        torch.cuda._sleep(int(4e6))          # hold the GPU so that the launches below are queued ahead (kernel time, not launch rate)
        e0.record()
        for _ in range(iters): lib.vb_gemm_bf16(C.byref(g), stream())
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
    return err, ms


# ------------------------------------------------------------------------------------------ attention
def attn_case(B, H, Nq, Nk, D, cross, peaked=1.0, iters=0, seed=0, fp16=False, split=False):
    """Returns (dict of relative errors of O, dQ, dK, dV, lse vs fp32 torch on the same 16-bit inputs, timing str).
    fp16: Q/K/V/O are fp16 (gradients stay bf16). split: Q/K/V given as hi + lo, O checked as hi + lo against the
    fp32 inputs (forward only carries the low parts)."""
    dev = torch.device("cuda"); lib = L.lib()
    g_ = torch.Generator(device=dev).manual_seed(seed)
    Hd = H * D
    DT = torch.float16 if fp16 else BF
    if cross:
        q32 = torch.randn(B * Nq, 3 * Hd, device=dev, generator=g_) * peaked
        k32 = torch.randn(B * Nk, 3 * Hd, device=dev, generator=g_) * peaked
        qsrc, ksrc = q32.to(DT), k32.to(DT)
    else:
        q32 = k32 = torch.randn(B * Nq, 3 * Hd, device=dev, generator=g_) * peaked
        qsrc = ksrc = q32.to(DT)
    q, k, v = qsrc[:, :Hd], ksrc[:, Hd:2 * Hd], ksrc[:, 2 * Hd:]
    if split:
        qlo_src, klo_src = (q32 - qsrc.float()).to(DT), (k32 - ksrc.float()).to(DT)
    lens = torch.randint(1, Nk + 1, (B,), device=dev, generator=g_); lens[0] = Nk
    if B > 1: lens[1] = 1                                                 # a row with a single valid key
    mask = ((torch.arange(Nk, device=dev)[None] >= lens[:, None]).float() * -10000.0).contiguous()
    Ot = torch.zeros(B * Nq, Hd, device=dev, dtype=DT); lse = torch.zeros(B, H, Nq, device=dev)
    Olo = torch.zeros(B * Nq, Hd, device=dev, dtype=DT) if split else None
    Ob = torch.zeros(B * Nq, Hd, device=dev, dtype=BF) if fp16 else None
    dO = torch.randn(B * Nq, Hd, device=dev, generator=g_).to(BF)
    dqb = torch.zeros(B * Nq, 3 * Hd, device=dev, dtype=BF); dkb = torch.zeros(B * Nk, 3 * Hd, device=dev, dtype=BF)
    delta = torch.zeros(B, H, Nq, device=dev)
    a = L.AttnArgs()
    a.B, a.H, a.Nq, a.Nk, a.D = B, H, Nq, Nk, D
    a.Q, a.ldq, a.K, a.ldk, a.V, a.ldv = q.data_ptr(), 3 * Hd, k.data_ptr(), 3 * Hd, v.data_ptr(), 3 * Hd
    a.mask, a.scale = mask.data_ptr(), 1.0 / math.sqrt(D)
    a.O, a.ldo, a.lse = Ot.data_ptr(), Hd, lse.data_ptr()
    a.dO, a.lddo = dO.data_ptr(), Hd
    a.dQ, a.lddq = dqb[:, :Hd].data_ptr(), 3 * Hd
    a.dK, a.lddk = dkb[:, Hd:2 * Hd].data_ptr(), 3 * Hd
    a.dV, a.lddv = dkb[:, 2 * Hd:].data_ptr(), 3 * Hd
    a.delta = delta.data_ptr()
    a.qkv_fp16 = int(fp16)
    if split:
        a.Q_lo, a.K_lo, a.V_lo = qlo_src[:, :Hd].data_ptr(), klo_src[:, Hd:2 * Hd].data_ptr(), klo_src[:, 2 * Hd:].data_ptr()
        a.O_lo = Olo.data_ptr()
    if Ob is not None:
        a.O_b16 = Ob.data_ptr()
    L.check(lib.vb_attention_fwd(C.byref(a), stream()), "vb_attention_fwd")
    L.check(lib.vb_attention_bwd(C.byref(a), stream()), "vb_attention_bwd")
    torch.cuda.synchronize()
    def ref(qq, kk, vv):
        qf = qq.float().view(B, Nq, H, D).permute(0, 2, 1, 3).detach().requires_grad_(True)
        kf = kk.float().view(B, Nk, H, D).permute(0, 2, 1, 3).detach().requires_grad_(True)
        vf = vv.float().view(B, Nk, H, D).permute(0, 2, 1, 3).detach().requires_grad_(True)
        s = qf @ kf.transpose(-1, -2) / math.sqrt(D) + mask[:, None, None, :]
        p = torch.softmax(s, -1)
        o = (p @ vf).permute(0, 2, 1, 3).reshape(B * Nq, Hd)
        o.backward(dO.float())
        return qf, kf, vf, s, o.detach()
    qf, kf, vf, s, o = ref(q, k, v)
    if fp16:
        # the backward kernels contract in bf16 (dO / dS are bf16 operands): their Q / K / V panels are the fp16 values rounded to
        # bf16, so the gradient reference is the attention of those rounded inputs; the forward reference keeps the fp16 values
        qf, kf, vf, _, _ = ref(q.to(BF), k.to(BF), v.to(BF))
    if split:
        # forward against the fp32 (hi + lo) inputs; the backward of split precision contracts the hi parts only
        qs = q32[:, :Hd].view(B, Nq, H, D).permute(0, 2, 1, 3); ks = k32[:, Hd:2 * Hd].view(B, Nk, H, D).permute(0, 2, 1, 3)
        vs = k32[:, 2 * Hd:].view(B, Nk, H, D).permute(0, 2, 1, 3)
        s32 = qs.double() @ ks.double().transpose(-1, -2) / math.sqrt(D) + mask[:, None, None, :].double()
        o32 = (torch.softmax(s32, -1) @ vs.double()).permute(0, 2, 1, 3).reshape(B * Nq, Hd).float()
        o_split = rel(Ot.float() + Olo.float(), o32)
    # dQ and dK are products of dS = P o (dP - delta), which is 0 in exact arithmetic when every row has one key (Nk = 1): their
    # error is measured against a floor of 1e-3 of the dV scale, so rounding residue of size ~1e-6 is not divided by ~0
    gfloor = 1e-3 * vf.grad.abs().max().item()
    relg = lambda a, b: ((a.float() - b.float()).abs().max() / max(b.float().abs().max().item(), gfloor, 1e-20)).item()
    errs = dict(O=rel(Ot, o), dQ=relg(dqb[:, :Hd].view(B, Nq, H, D).permute(0, 2, 1, 3), qf.grad),
                dK=relg(dkb[:, Hd:2 * Hd].view(B, Nk, H, D).permute(0, 2, 1, 3), kf.grad),
                dV=rel(dkb[:, 2 * Hd:].view(B, Nk, H, D).permute(0, 2, 1, 3), vf.grad),
                lse=rel(lse * math.log(2.0), torch.logsumexp(s, -1)))
    if split:
        errs["O_split"] = o_split
    if Ob is not None:
        errs["O_b16"] = max(rel(Ob, o) - 4e-3, 0.0)
    timing = ""
    if iters:
        for fn, nm in ((lib.vb_attention_fwd, "fwd"), (lib.vb_attention_bwd, "bwd")):
            e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
            for _ in range(3): fn(C.byref(a), stream())
            e0.record()
            for _ in range(iters): fn(C.byref(a), stream())
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / iters
            fl = 4.0 * B * H * Nq * Nk * D * (1 if nm == "fwd" else 2.5)
            timing += f" {nm} {ms*1e3:.1f}us {fl/ms/1e9:.1f}TF"
    return errs, timing


# ------------------------------------------------------------------------------------------ full model
def build_engine(cfgj, P, device, precision="fp16"):
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    eng = Engine(BertConfig.from_dict(cfgj), device, precision=precision)
    for k in eng.ps.entries:
        eng.ps.p(k).copy_(P[k])
    eng.refresh_weights()
    return eng


def oracle_args(inp):
    return (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
            inp["image_attention_mask"], inp["co_attention_mask"], inp["task_ids"])


def probe_loss(heads, names, tgt):
    """VQA loss on vil_prediction + a small quadratic on every other requested head (touches every grad path)."""
    l = 0
    for n, h in zip(O.HEAD_NAMES, heads):
        if n in names:
            l = l + (O.vqa_loss(h, tgt) if n == "vil_prediction" else 0.1 * h.float().clamp(-50, 50).pow(2).mean())
    return l


def model_case(cfgj, B, Nv, Nt, seed=0, qk_scale=1.0, names=None, grads=True, device="cuda", train_step=None, precision="fp16",
               oracle_modes=("fp32", "op"), head_dropout_prob=None):
    """Engine vs the oracle in fp32 and in the engine's operand-rounding mode ("op": fp16 forward / bf16 gradient operands for
    precision "fp16" and "fp32", all-bf16 for "bf16"). Returns dict(out_fp32, out_op, grad_fp32, grad_op, ...)
    where each is {tensor name: error}; gradient errors are (max-rel with floor, rel-L2).
    train_step=k runs the engine in TRAIN mode (every nn.Dropout of the reference active, dropout step counter = k) against
    the oracle with the same stateless masks (oracle.DropMasks(k))."""
    # engines and plans of earlier cases hold each other in reference cycles: collect them before building a new one, an 80 GB
    # card does not hold several full-size engines at once
    gc.collect()
    torch.cuda.empty_cache()
    dev = torch.device(device)
    cfg = O.make_config(cfgj)
    names = O.HEAD_NAMES if names is None else names
    P = O.synth_params(cfg, seed=seed, device=dev, qk_scale=qk_scale)
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=1234 + seed, device=dev)
    eng = build_engine(cfgj, P, dev, precision)
    if head_dropout_prob is not None:
        eng.head_dropout_prob = head_dropout_prob     # VILBertForVLTasks(dropout_prob=...)
    drop = None
    if train_step is not None:
        eng.drop_step.fill_(int(train_step))
        drop = O.DropMasks(train_step, head_p=eng.head_dropout_prob)
    plan = eng.plan(B, Nt, Nv, grad_outputs=names if grads else (), train=train_step is not None)
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                     inp["image_attention_mask"], inp["task_ids"])
    plan.run_forward()
    torch.cuda.synchronize()
    tgt = O.synth_vqa_target(B, 3129, device=dev)
    result = dict(plan=plan, engine=eng)
    mine_heads = [plan.outputs[n].detach().clone().requires_grad_(True) for n in O.HEAD_NAMES]
    if grads:
        lm = probe_loss(mine_heads, names, tgt); lm.backward()
        eng.zero_grad()
        for n, t in zip(O.HEAD_NAMES, mine_heads):
            if n in names:
                plan.gout[n].copy_(t.grad.reshape(plan.gout[n].shape))
        plan.run_backward()
        torch.cuda.synchronize()
        result["loss"] = lm.item()
    for mode in oracle_modes:
        Pg = {k: v.clone().requires_grad_(True) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
        Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
        if mode == "op":
            with (O.bf16_operand_mode() if precision == "bf16" else O.operand_mode()):
                bert_o, heads_o = O.vilbert_for_vl_tasks(Pg, cfg, *oracle_args(inp), drop=drop)
                if grads:
                    lo = probe_loss(heads_o, names, tgt); lo.backward()
        else:
            bert_o, heads_o = O.vilbert_for_vl_tasks(Pg, cfg, *oracle_args(inp), drop=drop)
            if grads:
                lo = probe_loss(heads_o, names, tgt); lo.backward()
        oe = {}
        for n, r in list(zip(O.BERT_OUT_NAMES, bert_o)) + list(zip(O.HEAD_NAMES, heads_o)):
            oe[n] = rel(plan.outputs[n].reshape(r.shape), r)
        result["out_" + mode] = oe
        if grads:
            result["loss_" + mode] = lo.item()
            gmax = max(v.grad.abs().max().item() for v in Pg.values() if v.grad is not None)
            ge = {}
            for k in eng.ps.entries:
                rg, mg = Pg[k].grad, eng.ps.g(k)
                if rg is None:
                    ge[k] = (0.0 if mg.abs().max().item() == 0 else float("inf"), 0.0)
                    continue
                # gradients that are ~0 in exact arithmetic (key biases: softmax shift invariance) are compared
                # against a floor of 1e-3 of the largest gradient in the model
                floor = 1e-3 * gmax
                ge[k] = (((mg - rg).abs().max() / max(rg.abs().max().item(), floor)).item(),
                         ((mg - rg).norm() / max(rg.norm().item(), floor * math.sqrt(rg.numel()) * 0.1)).item())
            result["grad_" + mode] = ge
    return result
