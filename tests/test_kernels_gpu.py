"""Attention forward/backward and the row-wise kernels through the C ABI vs plain torch fp32 (same inputs)."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from vilbert_b200 import _lib as L

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", [
    (2, 4, 9, 9, 16, False), (3, 3, 11, 11, 32, False), (2, 2, 12, 7, 32, True), (2, 2, 7, 12, 32, True),
    (4, 12, 36, 36, 64, False), (4, 8, 100, 100, 128, False), (4, 8, 36, 100, 128, True), (4, 8, 100, 36, 128, True),
    (2, 8, 306, 306, 128, False), (2, 8, 257, 306, 128, True), (2, 12, 257, 257, 64, False), (3, 8, 65, 129, 128, True)])
def test_attention_fwd_bwd(B, H, Nq, Nk, D, cross):
    """Self- and cross-attention incl. the largest 12-in-1 shapes (306 regions x 257 tokens), ragged key masks with a
    single valid key, odd extents. bf16 inputs, fp32 reference: 2e-2 tolerance (P and dS are bf16 MMA operands)."""
    from _gpu_util import attn_case
    errs, _ = attn_case(B, H, Nq, Nk, D, cross)
    assert errs["lse"] < 1e-5
    assert max(errs.values()) < 2e-2, errs


# The backward's dispatch edges (vb_attention_bwd): the fused single-pass kernel runs for Nq, Nk <= 128 and D >= 32, and is at its
# largest (~205 KiB of shared memory) at Nq = Nk = 128, D = 128; one query or one key more, or D = 16, takes the dQ + dK / dV
# pair, which holds whole panels up to Nq = Nk = 320 at D = 128. Each shape asserts the variant it reaches.
_FUSED = r"attn_bwd_fused_kernel<{D}, true, true>"
_TWO = (r"attn_bwd_dq_kernel<{D}, true>", r"attn_bwd_dkv_kernel<{D}>")
BWD_EDGES = {(Nq, Nk, D): ((_FUSED,) if Nq <= 128 and Nk <= 128 else _TWO)
             for D in (32, 64, 128) for Nq, Nk in [(128, 128), (128, 129), (129, 128), (1, 128), (128, 1), (1, 1), (320, 320),
                                                   (320, 36), (36, 320)]}
BWD_EDGES[(128, 128, 16)] = _TWO


@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", [
    (3, 3, 11, 11, 32, False), (4, 12, 36, 36, 64, False), (4, 8, 100, 100, 128, False), (4, 8, 36, 100, 128, True),
    (4, 8, 100, 36, 128, True), (2, 8, 257, 306, 128, True), (2, 2, 7, 12, 16, True)]
    + [(2, 2, Nq, Nk, D, Nq != Nk) for (Nq, Nk, D) in BWD_EDGES])
def test_attention_fp16_operands(B, H, Nq, Nk, D, cross):
    """The engine's default arithmetic: Q/K/V/O fp16 (forward operands), dO/dQ/dK/dV bf16. The forward is checked at fp16
    accuracy; the backward converts its Q/K/V panels to bf16 (dS and dO are bf16 MMA operands); whole-model gradient parity is
    bounded in tests/test_model_gpu.py."""
    from _gpu_util import attn_case, launched
    run = lambda: attn_case(B, H, Nq, Nk, D, cross, fp16=True)
    errs, _ = launched(run, *(p.format(D=D) for p in BWD_EDGES[(Nq, Nk, D)]))[0] if (Nq, Nk, D) in BWD_EDGES else run()
    assert errs["lse"] < 1e-5 and errs["O"] < 2e-3 and errs["O_b16"] < 1e-3, errs
    # gradients vs the attention of the bf16-rounded inputs (what the backward kernels contract); the saved row log-sum-exp comes
    # from the fp16 forward, so the recomputed probabilities differ from the reference's by the bf16 rounding of the scores
    assert max(errs.values()) < 3e-2, errs


@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", [
    (3, 3, 11, 11, 32, False), (4, 12, 36, 36, 64, False), (4, 8, 100, 100, 128, False), (4, 8, 36, 100, 128, True),
    (2, 8, 257, 306, 128, True)])
def test_attention_split_precision_forward(B, H, Nq, Nk, D, cross):
    """fp32 parity mode: Q/K/V as fp16 hi + lo, three MMA passes for QK^T and for PV (P split in registers), O written as
    hi + lo. Checked against a float64 attention of the fp32 inputs: 2e-5 (north_star fp32 tolerance is 1e-3)."""
    from _gpu_util import attn_case
    errs, _ = attn_case(B, H, Nq, Nk, D, cross, fp16=True, split=True)
    assert errs["O_split"] < 2e-5, errs


def test_attention_peaked_softmax():
    from _gpu_util import attn_case
    for args in [(4, 8, 100, 100, 128, False), (4, 12, 36, 36, 64, False)]:
        errs, _ = attn_case(*args, peaked=5.0)
        assert max(errs.values()) < 2e-2, errs


def S():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-20)).item()


@pytest.mark.parametrize("M,H", [(37, 64), (50, 96), (2304, 768), (6400, 1024), (33, 2048), (128, 128)])
def test_layernorm_fwd_bwd(M, H):
    lib, dev = L.lib(), "cuda"
    x = torch.randn(M, H, device=dev) * 2 + 0.5; g = torch.randn(H, device=dev); b = torch.randn(H, device=dev)
    y32 = torch.empty(M, H, device=dev); y16 = torch.empty(M, H, device=dev, dtype=BF); mean = torch.empty(M, device=dev); rstd = torch.empty(M, device=dev)
    L.check(lib.vb_layernorm_fwd(x.data_ptr(), H, g.data_ptr(), b.data_ptr(), 1e-12, y32.data_ptr(), y16.data_ptr(), H, mean.data_ptr(), rstd.data_ptr(), M, H, None, 0, None, None, S()))
    # fp16 operand copy as hi + lo (split precision): hi + lo reconstructs the fp32 output to ~2^-22
    yh = torch.empty(M, H, device=dev, dtype=torch.float16); yl = torch.empty(M, H, device=dev, dtype=torch.float16)
    yb = torch.empty(M, H, device=dev, dtype=BF)
    L.check(lib.vb_layernorm_fwd(x.data_ptr(), H, g.data_ptr(), b.data_ptr(), 1e-12, None, yh.data_ptr(), H, None, None, M, H, None, 1, yl.data_ptr(), yb.data_ptr(), S()))
    xr = x.clone().requires_grad_(True); gr = g.clone().requires_grad_(True); br = b.clone().requires_grad_(True)
    yr = F.layer_norm(xr, (H,), gr, br, 1e-12)
    dy = torch.randn(M, H, device=dev); yr.backward(dy)
    dx32 = torch.empty(M, H, device=dev); dx16 = torch.empty(M, H, device=dev, dtype=BF); dg = torch.zeros(H, device=dev); db = torch.zeros(H, device=dev)
    L.check(lib.vb_layernorm_bwd(dy.data_ptr(), H, x.data_ptr(), H, g.data_ptr(), mean.data_ptr(), rstd.data_ptr(), dx32.data_ptr(), dx16.data_ptr(), H, None, 0,
                                 dg.data_ptr(), db.data_ptr(), None, M, H, None, None, S()))
    torch.cuda.synchronize()
    assert rel(y32, yr) < 1e-5 and rel(y16, yr) < 5e-3
    assert torch.equal(yh, y32.to(torch.float16)) and rel(yh.float() + yl.float(), y32) < 2e-6 and torch.equal(yb, y16)
    assert rel(dx32, xr.grad) < 1e-5 and rel(dx16, xr.grad) < 5e-3 and rel(dg, gr.grad) < 1e-5 and rel(db, br.grad) < 1e-5


def test_layernorm_bwd_fused_gelu_grad():
    lib, dev = L.lib(), "cuda"
    M, H = 64, 2048
    x = torch.randn(M, H, device=dev); g = torch.randn(H, device=dev); b = torch.randn(H, device=dev); pre = torch.randn(M, H, device=dev).to(BF)
    mean = x.mean(-1); rstd = 1 / torch.sqrt(x.var(-1, unbiased=False) + 1e-12); dy = torch.randn(M, H, device=dev)
    xr = x.clone().requires_grad_(True); F.layer_norm(xr, (H,), g, b, 1e-12).backward(dy)
    gp = pre.float()          # the buffer holds gelu'(pre-activation) as saved by the forward GEMM epilogue
    dx16 = torch.empty(M, H, device=dev, dtype=BF); dg = torch.zeros(H, device=dev); db = torch.zeros(H, device=dev)
    L.check(lib.vb_layernorm_bwd(dy.data_ptr(), H, x.data_ptr(), H, g.data_ptr(), mean.data_ptr(), rstd.data_ptr(), None, dx16.data_ptr(), H, pre.data_ptr(), H,
                                 dg.data_ptr(), db.data_ptr(), None, M, H, None, None, S()))
    torch.cuda.synchronize()
    assert rel(dx16, xr.grad * gp) < 5e-3


@pytest.mark.parametrize("has_task", [False, True])
def test_text_embedding_gather_and_scatter(has_task):
    lib, dev = L.lib(), "cuda"
    B, Nt, H, V = 5, 9, 64, 50
    ids = torch.randint(0, V, (B, Nt), device=dev); ids[0, 3] = 0; tt = torch.randint(0, 2, (B, Nt), device=dev); task = torch.randint(0, 20, (B,), device=dev)
    word = torch.randn(V, H, device=dev); pos = torch.randn(40, H, device=dev); typ = torch.randn(2, H, device=dev); tk = torch.randn(20, H, device=dev)
    out = torch.empty(B, Nt + int(has_task), H, device=dev)
    L.check(lib.vb_embed_text_fwd(ids.data_ptr(), tt.data_ptr(), task.data_ptr() if has_task else None, word.data_ptr(), pos.data_ptr(), typ.data_ptr(),
                                  tk.data_ptr() if has_task else None, out.data_ptr(), B, Nt, H, S()))
    wr, pr, tr, kr = (t.clone().requires_grad_(True) for t in (word, pos, typ, tk))
    e = F.embedding(ids, wr, padding_idx=0) + F.embedding(torch.arange(Nt, device=dev)[None].expand(B, Nt), pr) + F.embedding(tt, tr)
    if has_task:
        e = torch.cat([e[:, :1], F.embedding(task[:, None], kr), e[:, 1:]], 1)
    d = torch.randn_like(e); e.backward(d)
    dw, dp, dt, dk = (torch.zeros_like(t) for t in (word, pos, typ, tk))
    L.check(lib.vb_embed_text_bwd(d.contiguous().data_ptr(), ids.data_ptr(), tt.data_ptr(), task.data_ptr() if has_task else None, dw.data_ptr(), dp.data_ptr(),
                                  dt.data_ptr(), dk.data_ptr() if has_task else None, B, Nt, H, S()))
    torch.cuda.synchronize()
    assert torch.equal(out, e.detach())                       # pure gather + adds in the same order: bit-exact
    assert rel(dw, wr.grad) < 1e-5 and rel(dp, pr.grad) < 1e-5 and rel(dt, tr.grad) < 1e-5
    assert dw[0].abs().max().item() == 0                      # padding_idx row gets no gradient
    if has_task:
        assert rel(dk, kr.grad) < 1e-5


def test_misc_rowops():
    lib, dev = L.lib(), "cuda"
    # casts
    x = torch.randn(1000003, device=dev); y = torch.empty(1000003, device=dev, dtype=BF)
    L.check(lib.vb_cast_f32_to_bf16(x.data_ptr(), y.data_ptr(), x.numel(), 0, None, None, S())); torch.cuda.synchronize()
    assert torch.equal(y, x.to(BF))
    yh = torch.empty(1000003, device=dev, dtype=torch.float16); yl = torch.empty_like(yh)
    yb = torch.empty(1000003, device=dev, dtype=BF)
    L.check(lib.vb_cast_f32_to_bf16(x.data_ptr(), yh.data_ptr(), x.numel(), 1, yl.data_ptr(), yb.data_ptr(), S())); torch.cuda.synchronize()
    assert torch.equal(yh, x.to(torch.float16)) and torch.equal(yl, (x - yh.float()).to(torch.float16)) and torch.equal(yb, x.to(BF))
    x = torch.randn(77, 3129, device=dev); y = torch.zeros(77, 3136, device=dev, dtype=BF)
    L.check(lib.vb_cast2d_f32_to_bf16(x.data_ptr(), 3129, y.data_ptr(), 3136, 77, 3129, 0.5, S())); torch.cuda.synchronize()
    assert torch.equal(y[:, :3129], (x * 0.5).to(BF)) and y[:, 3129:].abs().max().item() == 0
    # image location projection
    M, H = 333, 96
    loc = torch.rand(M, 5, device=dev); W = torch.randn(H, 5, device=dev); b = torch.randn(H, device=dev); out = torch.empty(M, H, device=dev)
    L.check(lib.vb_loc_proj_fwd(loc.data_ptr(), W.data_ptr(), b.data_ptr(), out.data_ptr(), M, H, S()))
    dy = torch.randn(M, H, device=dev); dW = torch.zeros(H, 5, device=dev); db = torch.zeros(H, device=dev)
    L.check(lib.vb_loc_proj_bwd(dy.data_ptr(), loc.data_ptr(), dW.data_ptr(), db.data_ptr(), M, H, S())); torch.cuda.synchronize()
    assert rel(out, loc @ W.t() + b) < 1e-5 and rel(dW, dy.t() @ loc) < 1e-5 and rel(db, dy.sum(0)) < 1e-5
    # column sums
    for dt_ in (torch.float32, BF):
        X = torch.randn(2304, 776, device=dev).to(dt_); o = torch.zeros(770, device=dev)
        L.check(lib.vb_colsum(X.data_ptr(), int(dt_ == BF), 776, o.data_ptr(), 2304, 770, S())); torch.cuda.synchronize()
        assert rel(o, X.float().sum(0)[:770]) < 1e-5
    # tiny-N linears
    for (M, K, N) in [(64, 1024, 1), (64, 1024, 3), (32, 2048, 2), (6400, 1024, 1)]:
        x = torch.randn(M, K, device=dev); W = torch.randn(N, K, device=dev); b = torch.randn(N, device=dev); add = torch.randn(M, device=dev)
        y = torch.empty(M, N, device=dev)
        L.check(lib.vb_small_linear_fwd(x.data_ptr(), K, W.data_ptr(), b.data_ptr(), add.data_ptr(), y.data_ptr(), M, K, N, None, S()))
        dy = torch.randn(M, N, device=dev); dx = torch.ones(M, K, device=dev); dW = torch.zeros(N, K, device=dev); db = torch.zeros(N, device=dev)
        L.check(lib.vb_small_linear_bwd(dy.data_ptr(), x.data_ptr(), K, W.data_ptr(), dx.data_ptr(), K, 1, dW.data_ptr(), db.data_ptr(), M, K, N, None, S()))
        torch.cuda.synchronize()
        assert rel(y, x @ W.t() + b + add[:, None]) < 1e-5 and rel(dx, 1 + dy @ W) < 1e-5 and rel(dW, dy.t() @ x) < 1e-5
        # the bias gradient is a sum of M signed values (N = 1: a single number that may cancel to ~0): bound the error by the summands
        assert (db - dy.sum(0)).abs().max().item() <= 1e-6 * dy.abs().sum().item()
    # pooled fusion, relu backward
    a = torch.randn(64, 1024, device=dev); b = torch.randn(64, 1024, device=dev); o32 = torch.empty_like(a); o16 = torch.empty(64, 1024, device=dev, dtype=BF)
    L.check(lib.vb_fuse_pooled_fwd(a.data_ptr(), b.data_ptr(), o32.data_ptr(), o16.data_ptr(), a.numel(), 1, None, 0, None, None, S()))
    d = torch.randn_like(a); da = torch.ones_like(a); db = torch.ones_like(a)
    L.check(lib.vb_fuse_pooled_bwd(d.data_ptr(), a.data_ptr(), b.data_ptr(), da.data_ptr(), db.data_ptr(), a.numel(), 1, None, S())); torch.cuda.synchronize()
    assert torch.equal(o32, a * b) and rel(da, 1 + d * b) < 1e-6 and rel(db, 1 + d * a) < 1e-6
    # VQA BCE objective (task_utils.py:325-327)
    z = torch.randn(64, 3129, device=dev) * 3; t = (torch.rand(64, 3129, device=dev) < 0.001).float() * 0.6
    loss = torch.zeros(1, device=dev); dz = torch.empty_like(z); dz16 = torch.zeros(64, 3136, device=dev, dtype=BF)
    L.check(lib.vb_bce_logits_loss(z.data_ptr(), t.data_ptr(), loss.data_ptr(), dz.data_ptr(), dz16.data_ptr(), 3136, 64, 3129, 1.0, S())); torch.cuda.synchronize()
    zr = z.clone().requires_grad_(True); lr = F.binary_cross_entropy_with_logits(zr, t, reduction="mean") * 3129; lr.backward()
    assert abs(loss.item() - lr.item()) < 1e-5 * lr.item() and rel(dz, zr.grad) < 1e-5
    # additive masks (vilbert.py:1341-1362) incl. the task-token extension
    m = (torch.rand(7, 13, device=dev) < 0.6).long(); o0 = torch.empty(7, 13, device=dev); o1 = torch.empty(7, 14, device=dev)
    L.check(lib.vb_mask_to_additive(m.data_ptr(), o0.data_ptr(), 7, 13, 0, S())); L.check(lib.vb_mask_to_additive(m.data_ptr(), o1.data_ptr(), 7, 13, 1, S()))
    torch.cuda.synchronize()
    ref0 = (1.0 - m.float()) * -10000.0
    assert torch.equal(o0, ref0) and torch.equal(o1[:, 1:], ref0) and o1[:, 0].abs().max().item() == 0


def test_batch_expansion_and_prefetcher():
    """Input-pipeline edge (task_utils.py:186-310): device-side `expand` / `dialog` replication (vb_repeat_rows), the view-only
    `retrieval` / `nlvr` reshapes, and the pinned double-buffered host -> device prefetcher."""
    from vilbert_b200.data import PinnedBatchPrefetcher, expand_batch
    dev = "cuda"
    B, R, Nv, Nt = 3, 4, 7, 5
    feats = torch.randn(B, Nv, 2048, device=dev); sp = torch.rand(B, Nv, 5, device=dev); im = (torch.rand(B, Nv, device=dev) < 0.7).long()
    q = torch.randint(0, 100, (B, R, Nt), device=dev); am = torch.ones_like(q); seg = torch.zeros_like(q)
    co = torch.zeros(B, R, Nv, Nt, device=dev)
    f2, s2, m2, q2, a2, g2, c2, bs, no = expand_batch("expand", feats, sp, im, q, am, seg, co)
    # the reference's own expressions (task_utils.py:248-274)
    assert torch.equal(f2, feats.unsqueeze(1).expand(B, R, Nv, 2048).contiguous().view(-1, Nv, 2048))
    assert torch.equal(s2, sp.unsqueeze(1).expand(B, R, Nv, 5).contiguous().view(-1, Nv, 5))      # 140-byte items: falls back to views
    assert torch.equal(m2, im.unsqueeze(1).expand(B, R, Nv).contiguous().view(-1, Nv))
    assert torch.equal(q2, q.view(-1, Nt)) and c2.shape == (B * R, Nv, Nt) and (bs, no) == (B, R)
    f3, s3, m3, q3, a3, g3, _, bs3, _ = expand_batch("nlvr", torch.randn(B, 2 * Nv, 2048, device=dev), torch.rand(B, 2 * Nv, 5, device=dev),
                                                   torch.ones(B, 2 * Nv, device=dev).long(), q[:, 0], am[:, 0], seg[:, 0])
    assert f3.shape == (2 * B, Nv, 2048) and torch.equal(q3[0], q3[1]) and torch.equal(q3[0], q[0, 0])
    batches = [(torch.randn(4, 3), torch.arange(4) + i) for i in range(5)]
    n = 0
    for g, bt in zip(PinnedBatchPrefetcher(batches), batches):      # a yielded batch is valid until `depth` more are requested: consume it now
        assert g[0].is_cuda and torch.equal(g[1].cpu(), bt[1]) and torch.equal(g[0].cpu(), bt[0])
        n += 1
    assert n == 5
