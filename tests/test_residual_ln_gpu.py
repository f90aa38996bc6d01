"""vb_add_layernorm_fwd / _bwd give the same bits as the GEMM-epilogue residual they replace: GEMM(+bias, dropout, +residual) ->
vb_layernorm_fwd against GEMM(+bias) -> vb_add_layernorm_fwd, and dgrad GEMM(+residual) -> vb_layernorm_bwd against dgrad GEMM ->
vb_add_layernorm_bwd, at the residual-stream shapes of config 2, fp16 and split-precision operands, dropout on and off."""
import ctypes as C

import pytest
import torch

from vilbert_b200 import _lib as L

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gemm(A, B, M, N, K, out, bias=None, res=None, drop=None, fp16=True, A_lo=None, B_lo=None, b_mn=0):
    g = L.GemmArgs()
    g.M, g.N, g.K = M, N, K
    g.A, g.lda = A.data_ptr(), K
    g.B, g.ldb, g.b_mn_major = B.data_ptr(), (N if b_mn else K), b_mn
    g.alpha = 1.0
    g.bias = bias.data_ptr() if bias is not None else None
    g.residual, g.ld_res = (res.data_ptr(), N) if res is not None else (None, 0)
    g.out_f32, g.ld_out_f32 = out.data_ptr(), N
    g.a_fp16 = g.b_fp16 = g.out_fp16 = int(fp16)
    if A_lo is not None:
        g.A_lo, g.B_lo = A_lo.data_ptr(), B_lo.data_ptr()
    if drop is not None:
        g.dropout = drop
    L.check(L.lib().vb_gemm_bf16(C.byref(g), _st()), "vb_gemm_bf16")


@pytest.mark.parametrize("M,H", [(2304, 768), (6400, 1024)])
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("split", [False, True])
def test_add_layernorm_matches_gemm_residual(M, H, dropout, split):
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(M + H + 2 * dropout + split)
    lib = L.lib()
    K = H
    A32, W32 = torch.randn(M, K, device=dev, generator=gen), torch.randn(H, K, device=dev, generator=gen) * 0.05
    A, W = A32.half(), W32.half()
    A_lo, W_lo = ((A32 - A.float()).half(), (W32 - W.float()).half()) if split else (None, None)
    bias, r = torch.randn(H, device=dev, generator=gen), torch.randn(M, H, device=dev, generator=gen)
    gm, bt = torch.randn(H, device=dev, generator=gen), torch.randn(H, device=dev, generator=gen)
    step = torch.full((1,), 3, dtype=torch.int32, device=dev)
    drop = None
    if dropout:
        drop = L.Dropout(); drop.step, drop.site, drop.p = step.data_ptr(), 12345, 0.1

    def outs():
        return dict(y32=torch.empty(M, H, device=dev), hi=torch.empty(M, H, device=dev, dtype=F16),
                    lo=torch.empty(M, H, device=dev, dtype=F16) if split else None, b16=torch.empty(M, H, device=dev, dtype=BF),
                    mean=torch.empty(M, device=dev), rstd=torch.empty(M, device=dev))
    p = lambda t: t.data_ptr() if t is not None else None

    # forward: old pair, then the new one
    x_old, o_old = torch.empty(M, H, device=dev), outs()
    _gemm(A, W, M, H, K, x_old, bias=bias, res=r, drop=drop, A_lo=A_lo, B_lo=W_lo)
    L.check(lib.vb_layernorm_fwd(x_old.data_ptr(), H, gm.data_ptr(), bt.data_ptr(), 1e-12, o_old["y32"].data_ptr(), o_old["hi"].data_ptr(), H,
                                 o_old["mean"].data_ptr(), o_old["rstd"].data_ptr(), M, H, None, 1, p(o_old["lo"]), o_old["b16"].data_ptr(), _st()))
    d, o_new = torch.empty(M, H, device=dev), outs()
    _gemm(A, W, M, H, K, d, bias=bias, A_lo=A_lo, B_lo=W_lo)
    L.check(lib.vb_add_layernorm_fwd(d.data_ptr(), r.data_ptr(), H, C.byref(drop) if drop else None, d.data_ptr(), gm.data_ptr(), bt.data_ptr(),
                                     1e-12, o_new["y32"].data_ptr(), o_new["hi"].data_ptr(), H, o_new["mean"].data_ptr(), o_new["rstd"].data_ptr(),
                                     M, H, 1, p(o_new["lo"]), o_new["b16"].data_ptr(), _st()))
    torch.cuda.synchronize()
    assert torch.equal(d, x_old)                        # the sum written back for the backward
    for k in o_old:
        if o_old[k] is not None:
            assert torch.equal(o_old[k], o_new[k]), k

    # backward: the dgrad GEMM adding the residual-path gradient e, against the LayerNorm backward adding it
    dy16 = torch.randn(M, 3 * H, device=dev, generator=gen).to(BF)
    Wq = (torch.randn(3 * H, H, device=dev, generator=gen) * 0.05).to(BF)
    e = torch.randn(M, H, device=dev, generator=gen)
    g_old, g_new = torch.empty(M, H, device=dev), torch.empty(M, H, device=dev)
    _gemm(dy16, Wq, M, H, 3 * H, g_old, res=e, fp16=False, b_mn=1)
    _gemm(dy16, Wq, M, H, 3 * H, g_new, fp16=False, b_mn=1)

    def bwd(fn, *first):
        dx32, dx16 = torch.empty(M, H, device=dev), torch.empty(M, H, device=dev, dtype=BF)
        dg, db, dbias = torch.zeros(H, device=dev), torch.zeros(H, device=dev), torch.zeros(H, device=dev)
        L.check(fn(*first, H, d.data_ptr(), H, gm.data_ptr(), o_new["mean"].data_ptr(), o_new["rstd"].data_ptr(), dx32.data_ptr(),
                   dx16.data_ptr(), H, None, 0, dg.data_ptr(), db.data_ptr(), dbias.data_ptr(), M, H, None,
                   C.byref(drop) if drop else None, _st()))
        torch.cuda.synchronize()
        return dx32, dx16, dg, db, dbias
    old = bwd(lib.vb_layernorm_bwd, g_old.data_ptr())
    new = bwd(lib.vb_add_layernorm_bwd, g_new.data_ptr(), e.data_ptr())
    assert torch.equal(old[0], new[0]) and torch.equal(old[1], new[1])
    for a, b in zip(old[2:], new[2:]):       # column sums: one atomic per CTA, in no fixed order
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-3)
