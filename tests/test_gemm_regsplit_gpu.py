"""GEMM tile widths and production signatures: the 128- and 256-wide tiles accumulate every output element over k in the same
order (one m64n256k16 per k step is the two m64n128k16 halves side by side), so their outputs are bitwise identical; every
GEMM signature of the config-2 training step matches a float64 reference; and the build log shows no GEMM kernel spilling."""
import ctypes as C
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from vilbert_b200 import _lib as L  # noqa: E402

PTXAS_LOG = os.path.join(ROOT, "vilbert-multi-task_b200", "csrc", "vb_gemm.ptxas.log")
TOL = 2e-3   # tests/test_gemm_gpu.py: max error relative to the largest reference value
RND16 = {torch.bfloat16: 4e-3, torch.float16: 5e-4}   # output rounding allowance of a 16-bit result


def test_gemm_kernels_do_not_spill():
    if not os.path.exists(PTXAS_LOG):
        pytest.skip("no vb_gemm.ptxas.log (written by build.sh)")
    text = open(PTXAS_LOG).read()
    entries = re.findall(r"Compiling entry function '(\w*gemm_wgmma_kernel\w*)'[^\n]*\n[^\n]*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(entries) == 26, f"found {len(entries)} gemm_wgmma_kernel entries in {PTXAS_LOG}"
    spilling = [(n, int(s), int(l)) for n, s, l in entries if int(s) or int(l)]
    assert not spilling, spilling
    assert "setmaxnreg' ignored" not in text


# ------------------------------------------------------------------------------------------ float64 reference
def _hash32(x):
    x = x & 0xFFFFFFFF
    x = x ^ (x >> 16); x = (x * 0x7FEB352D) & 0xFFFFFFFF
    x = x ^ (x >> 15); x = (x * 0x846CA68B) & 0xFFFFFFFF
    return x ^ (x >> 16)


def _keep_scale(M, N, site, ctr, p):
    seed = _hash32(torch.tensor(site + ctr * 0x9E3779B9, dtype=torch.int64))
    idx = (torch.arange(M, device="cuda", dtype=torch.int64)[:, None] * N + torch.arange(N, device="cuda", dtype=torch.int64)[None]) & 0xFFFFFFFF
    p32 = float(torch.tensor(p, dtype=torch.float32))   # the kernel's threshold and scale come from the float p
    keep = _hash32(idx ^ seed) >= int(p32 * 4294967296.0)
    return keep.double() * float(1.0 / (1.0 - torch.tensor(p32, dtype=torch.float32)))


def reference(ln):
    """float64 epilogue value (before the residual), the column sums, the value after the residual and gelu'(pre)."""
    s, v = ln.s, ln.views
    M, N, K = s["M"], s["N"], s["K"]
    op = lambda X, mn, rows: (X[:K, :rows].t() if mn else X[:rows, :K]).double()
    A = op(v["A"], s["a_mn_major"], M) + (op(v["A_lo"], s["a_mn_major"], M) if "A_lo" in v else 0)
    B = op(v["B"], s["b_mn_major"], N) + (op(v["B_lo"], s["b_mn_major"], N) if "B_lo" in v else 0)
    x = s["alpha"] * (A @ B.t())
    if "bias" in v:
        x = x + v["bias"][0, :N].double()
    pre = None
    if s["act"] == L.VB_ACT_GELU:
        pre = 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5
        x = x * 0.5 * (1 + torch.erf(x / 2 ** 0.5))
    elif s["act"] == L.VB_ACT_RELU:
        x = x.clamp_min(0)
    elif s["act"] == L.VB_ACT_DGELU:
        x = x * v["aux"][:M, :N].double()
    if s["dropout"]:
        x = x * _keep_scale(M, N, s["dropout"][0], int(ln.ctr.item()), s["dropout"][1])
    colsum = x.sum(0)
    y = x + v["residual"][:M, :N].double() if "residual" in v else x
    return y, colsum, pre


def rel(a, ref):
    return ((a.double() - ref).abs().max() / (ref.abs().max() + 1e-9)).item()


def check_against_reference(ln):
    s, v = ln.s, ln.views
    M, N = s["M"], s["N"]
    y, colsum, pre = reference(ln)
    errs = {}
    if "out_f32" in v:
        out = v["out_f32"]
        if s["atomic_out"] == L.VB_GEMM_PARTIALS:
            out = out.view(-1, M, out.shape[1]).sum(0)
        errs["out_f32"] = rel(out[:M, :N], y)
    for f in ("out_bf16", "out_b16"):
        if f in v:
            hi = v[f][:M, :N].double() + (v["out_lo"][:M, :N].double() if (f == "out_bf16" and "out_lo" in v) else 0)
            errs[f] = rel(hi, y) - (0 if (f == "out_bf16" and "out_lo" in v) else RND16[v[f].dtype])
    if "out_pre" in v:
        errs["out_pre"] = rel(v["out_pre"][:M, :N], pre) - RND16[torch.bfloat16]
    if "out_colsum" in v:
        errs["out_colsum"] = rel(v["out_colsum"][0, :N], colsum)
    assert errs and max(errs.values()) < TOL, (s, errs)


# ------------------------------------------------------------------------------------------ the config-2 step's signatures
def _config2_signatures():
    from gemm_sig_probe import plan_gemm_signatures, short, describe
    return [pytest.param(k, id=short(describe(k)).replace(" ", "_")) for k in plan_gemm_signatures(2)]


@pytest.mark.gpu
@pytest.mark.parametrize("sig", _config2_signatures())
def test_config2_signature_against_float64(sig):
    from gemm_sig_probe import Launch
    ln = Launch(sig, seed=3)
    ln(C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    check_against_reference(ln)


# ------------------------------------------------------------------------------------------ 128- vs 256-wide tiles
def _sig(M, N, K, a_mn=False, b_mn=False, act=0, bias=False, res=False, aux=False, f32=False, b16=False, pre=False, colsum=False,
         atomic=0, split_k=0, out_fp16=False, a_fp16=False, out_lo=False, out_b16=False, drop=None):
    """A signature in gemm_sig_probe's format for a dense problem of the given flags."""
    from gemm_sig_probe import SCALAR_FIELDS
    p8 = lambda x: (x + 7) // 8 * 8
    s = dict(M=M, N=N, K=K, lda=p8(M) if a_mn else p8(K), a_mn_major=int(a_mn), ldb=p8(N) if b_mn else p8(K), b_mn_major=int(b_mn),
             alpha=0.75, ld_res=N if res else 0, ld_aux=N if aux else 0, act=act, ld_out_f32=N if f32 else 0, ld_out_bf16=N if b16 else 0,
             ld_out_pre=N if pre else 0, atomic_out=atomic, split_k=split_k, block_n=0, max_ctas=0, a_fp16=int(a_fp16),
             b_fp16=int(a_fp16), out_fp16=int(out_fp16))
    ptrs = [f for f, on in (("A", 1), ("B", 1), ("bias", bias), ("residual", res), ("aux", aux), ("out_f32", f32), ("out_bf16", b16),
                            ("out_pre", pre), ("out_colsum", colsum), ("out_lo", out_lo), ("out_b16", out_b16)) if on]
    return tuple(s[f] for f in SCALAR_FIELDS) + (tuple((f, 0) for f in ptrs), drop)


EPILOGUES = {
    "f32_bias_drop_res": dict(bias=True, res=True, f32=True, drop=(7, 0.1)),
    "bf16_out16_0": dict(bias=True, b16=True),
    "bf16_out16_1": dict(bias=True, b16=True, out_fp16=True, a_fp16=True),
    "bf16_out16_2": dict(bias=True, b16=True, out_fp16=True, out_b16=True, a_fp16=True),
    "bf16_out16_3": dict(bias=True, b16=True, out_fp16=True, out_lo=True, out_b16=True, a_fp16=True),
    "gelu": dict(act=L.VB_ACT_GELU, bias=True, b16=True, pre=True, out_fp16=True, out_b16=True, a_fp16=True),
    "dgelu_colsum": dict(act=L.VB_ACT_DGELU, aux=True, b16=True, colsum=True),
    "atomic_split_k": dict(atomic=1, f32=True, split_k=2),
    "partials": dict(atomic=L.VB_GEMM_PARTIALS, f32=True),
}
REORDERED = ("atomic_split_k", "partials")   # float atomics / slice sums: compared with the float64 reference instead


def _run(sig, block_n):
    from gemm_sig_probe import Launch, resolved_tiles, SCALAR_FIELDS
    s = dict(zip(SCALAR_FIELDS, sig[:len(SCALAR_FIELDS)]), block_n=block_n)
    if s["atomic_out"] == L.VB_GEMM_PARTIALS:
        from gemm_sig_probe import describe
        s["split_k"] = resolved_tiles(dict(describe(sig), block_n=block_n))[1]
    sig = tuple(s[f] for f in SCALAR_FIELDS) + sig[len(SCALAR_FIELDS):]
    ln = Launch(sig, seed=5)
    ln(C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return ln


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(300, 200, 136), (6400, 1601, 1024)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("majors", [(False, False), (False, True), (True, True)], ids=["AB", "AB^T", "A^TB^T"])
@pytest.mark.parametrize("epi", sorted(EPILOGUES))
def test_tile_widths_give_the_same_bits(epi, majors, shape):
    M, N, K = shape
    sig = _sig(M, N, K, a_mn=majors[0], b_mn=majors[1], **EPILOGUES[epi])
    n128, n256 = _run(sig, 128), _run(sig, 256)
    if epi in REORDERED:
        check_against_reference(n128)
        check_against_reference(n256)
        return
    for f, v in n128.views.items():
        if f in ("A", "B", "bias", "residual", "aux"):
            continue
        if f == "out_colsum":   # float atomics across row blocks
            check_against_reference(n256)
            continue
        assert torch.equal(v, n256.views[f]), (epi, f)
    check_against_reference(n256)
