"""wgmma GEMM (vb_gemm_bf16) through the C ABI. Every case runs through the float64 checker of tests/_gpu_util.py (gemm_case):
per-element bounds, correctly rounded 16-bit outputs, guard bands, the tile width's kernel asserted, wrong references. The value
returned and compared with TOL is the largest error past the correctly rounded result, relative to max|ref|."""
import pytest

from vilbert_b200 import _lib as L

pytestmark = pytest.mark.gpu
TOL = 2e-3


@pytest.mark.parametrize("M,N,K,bn", [(128, 128, 64, 128), (128, 256, 64, 256), (384, 512, 256, 0), (2304, 768, 768, 0),
                                       (2304, 2304, 768, 0), (6400, 1024, 1024, 128), (6400, 3072, 1024, 256), (100, 72, 40, 0),
                                       (333, 1601, 1024, 0), (130, 30522, 768, 0), (64, 1024, 768, 0), (1, 8, 8, 0)])
def test_forward_layout_plain(M, N, K, bn):
    """nn.Linear forward layout (both operands K-major), incl. ragged edges and the 30522/1601-wide heads."""
    from _gpu_util import gemm_case
    err, _ = gemm_case(M, N, K, block_n=bn)
    assert err < TOL


@pytest.mark.parametrize("kw", [dict(bias=True), dict(bias=True, act=L.VB_ACT_GELU, out_bf16=True), dict(bias=True, res=True),
                                dict(act=L.VB_ACT_DGELU, out_bf16=True), dict(bias=True, act=L.VB_ACT_RELU, out_bf16=True),
                                dict(atomic=True, split_k=3), dict(atomic=True, split_k=0), dict(alpha=0.125, res=True),
                                dict(bias=True, out_bf16=True), dict(bias=True, out_bf16=True, both_outputs=True),
                                dict(bias=True, act=L.VB_ACT_GELU, out_bf16=True, both_outputs=True)])
@pytest.mark.parametrize("shape", [(2304, 768, 768), (300, 200, 136), (256, 1601, 128)])
def test_fused_epilogues(kw, shape):
    """bias / erf-GELU (+ saved pre-activation) / ReLU / GELU' / fp32 residual / split-K atomics."""
    from _gpu_util import gemm_case
    err, _ = gemm_case(*shape, **kw)
    assert err < TOL


@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K,bn", [(128, 128, 64, 128), (256, 256, 128, 256), (768, 768, 2304, 0), (1000, 520, 200, 0), (3072, 768, 6400, 0)])
def test_mn_major_operands(a_mn, b_mn, M, N, K, bn):
    """dgrad (B MN-major) and wgrad (A and B MN-major) operand layouts, read in place through TMA."""
    from _gpu_util import gemm_case
    err, _ = gemm_case(M, N, K, a_mn=a_mn, b_mn=b_mn, block_n=bn)
    assert err < TOL


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("kw,shape", [
    (dict(bias=True, res=True), (2304, 768, 768)),                       # even number of row blocks
    (dict(bias=True, out_bf16=True), (6400, 3072, 1024)),                # several tiles per CTA
    (dict(bias=True, res=True), (333, 1601, 1024)),                      # odd number of row blocks (3); ragged N
    (dict(bias=True, act=L.VB_ACT_GELU, out_bf16=True), (1000, 520, 200)),
    (dict(b_mn=True, res=True), (2304, 768, 3072)),                      # dgrad form: B read MN-major
    (dict(a_mn=True, b_mn=True, atomic=True, split_k=0), (1024, 1024, 6400)),   # wgrad form with split-K
    (dict(a_mn=True, b_mn=True, atomic=True, split_k=3), (768, 520, 2304)),
])
def test_forced_tile_widths(kw, shape, bn):
    """block_n fixed by the caller: both tile widths on even and odd row-block counts, the dgrad and wgrad operand forms and
    split-K."""
    from _gpu_util import gemm_case
    err, _ = gemm_case(*shape, block_n=bn, **kw)
    assert err < 2e-3, err


@pytest.mark.parametrize("kw,shape", [
    (dict(bias=True, res=True), (2304, 768, 768)),
    (dict(bias=True, out_bf16=True, out_fp16=True), (6400, 3072, 1024)),
    (dict(bias=True, act=L.VB_ACT_GELU, out_bf16=True, out_fp16=True), (300, 200, 136)),
    (dict(b_mn=True, res=True), (2304, 768, 3072)),
    (dict(a_mn=True, b_mn=True, atomic=True, split_k=0), (1024, 1024, 6400)),
    (dict(b_mn=True, out_bf16=True), (333, 1601, 1024)),
    (dict(bias=True, out_bf16=True, out_fp16=True, block_n=256), (1000, 520, 200)),
])
def test_fp16_operands(kw, shape):
    """fp16 x fp16 (the forward operand format of the default precision), fp16 16-bit outputs, every operand major."""
    from _gpu_util import gemm_case
    err, _ = gemm_case(*shape, a_fp16=True, b_fp16=True, **kw)
    assert err < TOL, err


def test_mixed_operand_formats_are_rejected():
    """wgmma takes one 16-bit operand type for both A and B: the library refuses fp16 x bf16 instead of launching it."""
    import ctypes as C
    import torch
    lib = L.lib()
    x = torch.zeros(128, 64, device="cuda", dtype=torch.float16); w = torch.zeros(128, 64, device="cuda", dtype=torch.bfloat16)
    o = torch.zeros(128, 128, device="cuda")
    g = L.GemmArgs()
    g.M, g.N, g.K, g.A, g.lda, g.B, g.ldb = 128, 128, 64, x.data_ptr(), 64, w.data_ptr(), 64
    g.out_f32, g.ld_out_f32, g.alpha, g.split_k, g.a_fp16, g.b_fp16 = o.data_ptr(), 128, 1.0, 1, 1, 0
    assert lib.vb_gemm_bf16(C.byref(g), None) == 2 and b"same 16-bit format" in lib.vb_last_error()


@pytest.mark.parametrize("kw,shape", [
    (dict(bias=True, res=True), (2304, 768, 768)),
    (dict(bias=True, out_bf16=True), (6400, 3072, 1024)),
    (dict(bias=True, out_bf16=True, block_n=128), (1000, 520, 200)),
    (dict(bias=True, act=L.VB_ACT_GELU, out_bf16=True), (300, 200, 136)),
    (dict(bias=True, act=L.VB_ACT_RELU, out_bf16=True, both_outputs=True), (64, 1024, 768)),
    (dict(bias=True), (130, 30522, 768)),
    (dict(bias=True, res=True), (6400, 1024, 4096)),
])
def test_split_precision(kw, shape):
    """fp32 parity mode: operands as fp16 hi + lo, three passes (hi.hi + lo.hi + hi.lo) into one register accumulator; the
    16-bit output is written as hi + lo too. Compared with the float64 product of the fp32 operands: 5e-5 of max|ref|
    (single-pass fp16 operands give ~5e-4, bf16 ~4e-3)."""
    from _gpu_util import gemm_case
    err, _ = gemm_case(*shape, a_fp16=True, b_fp16=True, out_fp16=True, split=True, **kw)
    assert err < 5e-5, err


def test_invalid_arguments_are_rejected():
    import ctypes as C
    import torch
    lib = L.lib()
    g = L.GemmArgs()
    x = torch.zeros(64, 64, device="cuda", dtype=torch.bfloat16)
    o = torch.zeros(64, 64, device="cuda")
    g.M, g.N, g.K = 64, 64, 60
    g.A, g.lda, g.B, g.ldb = x.data_ptr(), 60, x.data_ptr(), 64      # lda not a multiple of 8
    g.out_f32, g.ld_out_f32, g.alpha, g.split_k = o.data_ptr(), 64, 1.0, 1
    assert lib.vb_gemm_bf16(C.byref(g), None) == 1
    assert b"ld % 8" in lib.vb_last_error()
    g.lda, g.out_f32 = 64, None
    assert lib.vb_gemm_bf16(C.byref(g), None) == 1                      # no output
    with pytest.raises(L.VBError):
        L.check(lib.vb_gemm_bf16(C.byref(g), None), "vb_gemm_bf16")
