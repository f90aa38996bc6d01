"""GEMM tile widths and production signatures: the 128- and 256-wide tiles accumulate every output element over k in the same
order (one m64n256k16 per k step is the two m64n128k16 halves side by side), so their outputs are bitwise identical; every GEMM
form of the bench configs' plans (training steps; config 2's evaluation, capped-backward and deterministic plans) passes the float64
checker of tests/_gpu_util.py; and the build log shows no GEMM kernel spilling."""
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from vilbert_b200 import _lib as L  # noqa: E402
from _gpu_util import GEMM_OUTPUTS, GemmCase, _bits  # noqa: E402

PTXAS_LOG = os.path.join(ROOT, "vilbert-multi-task_b200", "csrc", "vb_gemm.ptxas.log")


def test_gemm_kernels_do_not_spill():
    if not os.path.exists(PTXAS_LOG):
        pytest.skip("no vb_gemm.ptxas.log (written by build.sh)")
    text = open(PTXAS_LOG).read()
    entries = re.findall(r"Compiling entry function '(\w*gemm_wgmma_kernel\w*)'[^\n]*\n[^\n]*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(entries) == 26, f"found {len(entries)} gemm_wgmma_kernel entries in {PTXAS_LOG}"
    spilling = [(n, int(s), int(l)) for n, s, l in entries if int(s) or int(l)]
    assert not spilling, spilling
    assert "setmaxnreg' ignored" not in text


# ------------------------------------------------------------------------------------------ the plans' signatures
class SigCase(GemmCase):
    """A signature in gemm_sig_probe's format on guarded device buffers (tests/_gpu_util.GemmCase): the plan's row pitches and
    base addresses modulo 256, random 16-bit operands (split precision: the low parts of fp32 values), random fp32 bias / residual,
    bf16 aux; every output filled with a NaN sentinel around and inside its range (atomic outputs and column sums start from
    random values)."""

    def __init__(self, sig, seed=0):
        from gemm_sig_probe import SCALAR_FIELDS, describe
        s = describe(sig)
        ld = {f: s[k] for f, k in (("A", "lda"), ("B", "ldb"), ("residual", "ld_res"), ("aux", "ld_aux"), ("out_f32", "ld_out_f32"),
                                   ("out_bf16", "ld_out_bf16"), ("out_pre", "ld_out_pre")) if f in s["set"]}
        st = set(s["set"])
        super().__init__(s["M"], s["N"], s["K"], outs=[f for f in GEMM_OUTPUTS if f in st], a_mn=bool(s["a_mn_major"]),
                         b_mn=bool(s["b_mn_major"]), fp16=bool(s["a_fp16"]), out_fp16=bool(s["out_fp16"]), alpha=s["alpha"],
                         bias="bias" in st, act=s["act"], res="residual" in st, drop=s["dropout"], a_lo="A_lo" in st,
                         b_lo="B_lo" in st, atomic=s["atomic_out"], split_k=s["split_k"], block_n=s["block_n"],
                         max_ctas=s["max_ctas"], ld=ld, align=dict(sig[len(SCALAR_FIELDS)]), seed=seed)
        self.s = s


def check_against_reference(ln):
    """(Re)runs the launch under the profiler (the kernel of the tile width vb_gemm_plan resolves) and holds it to the float64
    checker of tests/_gpu_util.py: per-element bounds, correctly rounded 16-bit outputs, guard bands, wrong references."""
    from _gpu_util import gemm_verdict
    from gemm_sig_probe import short
    gemm_verdict(ln, short(ln.s), expect=rf"gemm_wgmma_kernel<{ln.bn}, ")


def _config2_signatures():
    from gemm_sig_probe import plan_gemm_signatures, short, describe
    return [pytest.param(k, id=short(describe(k)).replace(" ", "_")) for k in plan_gemm_signatures(2)]


@pytest.mark.gpu
@pytest.mark.parametrize("sig", _config2_signatures())
def test_config2_signature_against_float64(sig):
    check_against_reference(SigCase(sig, seed=3))


def _other_plan_signatures():
    """One signature per GEMM form of every bench config's training step, config 2's forward-only evaluation plan, its backward
    capped at SMs - 16 CTAs and its deterministic step, without the forms of config 2's training step (the test above)."""
    from gemm_sig_probe import plan_gemm_signatures, plan_signature_union, short, describe
    seen = set(plan_gemm_signatures(2))
    out = []
    for k, src in plan_signature_union().items():
        if k not in seen:
            tag = "+".join(f"{c}{kind}" for c, kind in src[:2]) + ("+" if len(src) > 2 else "")
            out.append(pytest.param(k, id=f"{tag}:{short(describe(k))}".replace(" ", "_")))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("sig", _other_plan_signatures())
def test_plan_signature_against_float64(sig):
    check_against_reference(SigCase(sig, seed=3))


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
    from gemm_sig_probe import resolved_tiles, SCALAR_FIELDS
    s = dict(zip(SCALAR_FIELDS, sig[:len(SCALAR_FIELDS)]), block_n=block_n)
    if s["atomic_out"] == L.VB_GEMM_PARTIALS:
        from gemm_sig_probe import describe
        s["split_k"] = resolved_tiles(dict(describe(sig), block_n=block_n))[1]
    sig = tuple(s[f] for f in SCALAR_FIELDS) + sig[len(SCALAR_FIELDS):]
    ln = SigCase(sig, seed=5)
    ln.run()
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
    for f in n128.outs:
        if f == "out_colsum":   # float atomics across row blocks
            continue
        assert torch.equal(_bits(n128.raw[f])[n128.inside[f]], _bits(n256.raw[f])[n256.inside[f]]), (epi, f)
    check_against_reference(n128)
    check_against_reference(n256)
