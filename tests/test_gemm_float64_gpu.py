"""vb_gemm_bf16 cases no other GEMM test reaches, each held to the float64 checker of tests/_gpu_util.py (GemmCase, gemm_verdict):
per-element bounds against float64, correctly rounded 16-bit outputs, NaN-filled guard bands around every output, the kernel
instantiation asserted through the profiler, and wrong references that must miss by more than 10x the bound.

- every one of the 26 gemm_wgmma_kernel<BN, EPI, OUT16> instantiations (KERNELS), at a shape whose epilogue chunks are all full
  (the unrolled fast path) and at a ragged one (the generic chunk routines inside the same kernel), with the engine's operand majors;
- each vector-access condition of the epilogue made false once (the scalar / generic fallbacks);
- the persistent scheduler under a CTA cap (max_ctas) at work-item counts around the SM count, split-K forced and automatic, and
  deterministic partials (VB_GEMM_PARTIALS) with the split count vb_gemm_plan resolves under the cap;
- the residual read in place from out_f32;
- split precision with A_lo only, B_lo only and both, and split-K whose splits straddle a pass boundary (each partial slice checked
  against the k-blocks of its own split)."""
import ctypes as C
import zlib

import pytest
import torch

from _gpu_util import EPI, GemmCase, gemm_kernel_name, gemm_verdict
from vilbert_b200 import _lib as L

GELU, DGELU, RELU = L.VB_ACT_GELU, L.VB_ACT_DGELU, L.VB_ACT_RELU
PARTIALS = L.VB_GEMM_PARTIALS
FULL, RAGGED = (256, 512, 192), (200, 328, 136)      # every 16 x 32 chunk inside / M % 16 = 8, N % 32 = 8, K % 64 = 8

# (EPI, OUT16) -> the arguments that reach gemm_wgmma_kernel<BN, EPI, OUT16>, in the engine's form of that epilogue
KERNELS = {
    ("F32", 0): dict(outs=("out_f32",), fp16=True, bias=True, res=True, drop=(7, 0.1)),          # out-proj: LN(dropout(dense) + res)
    ("BF16", 0): dict(outs=("out_bf16",), b_mn=True),                                              # plain dgrad, bf16 gradient operand
    ("BF16", 1): dict(outs=("out_bf16",), fp16=True, out_fp16=True, bias=True),                    # QKV of a forward-only plan
    ("BF16", 2): dict(outs=("out_bf16", "out_b16"), fp16=True, out_fp16=True, bias=True),          # QKV + the backward's bf16 copy
    ("BF16", 3): dict(outs=("out_bf16", "out_lo", "out_b16"), fp16=True, out_fp16=True, bias=True, a_lo=True, b_lo=True),
    ("GELU", 0): dict(outs=("out_bf16", "out_pre"), bias=True, act=GELU),                           # bf16 precision FFN1
    ("GELU", 1): dict(outs=("out_bf16", "out_pre"), fp16=True, out_fp16=True, bias=True, act=GELU),  # forward-only FFN1
    ("GELU", 2): dict(outs=("out_bf16", "out_pre", "out_b16"), fp16=True, out_fp16=True, bias=True, act=GELU),
    ("GELU", 3): dict(outs=("out_bf16", "out_lo", "out_b16", "out_pre"), fp16=True, out_fp16=True, bias=True, act=GELU,
                      a_lo=True, b_lo=True),
    ("DGELU", 0): dict(outs=("out_bf16", "out_colsum"), act=DGELU, b_mn=True),                     # FFN1 dgrad + bias gradient
    ("ATOMIC", 0): dict(outs=("out_f32",), a_mn=True, b_mn=True, atomic=1, split_k=0),              # split-K wgrad
    ("GENERIC", 0): dict(outs=("out_f32", "out_bf16"), fp16=True, out_fp16=True, bias=True),        # fp32 + 16-bit outputs
    ("PARTIAL", 0): dict(outs=("out_f32",), a_mn=True, b_mn=True, atomic=PARTIALS, split_k=0),      # deterministic wgrad
}
INSTANTIATIONS = [(bn, epi, o16) for bn in (128, 256) for (epi, o16) in KERNELS]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(label, bn, epi, out16, shape, **kw):
    case = GemmCase(*shape, block_n=bn, seed=zlib.crc32(label.encode()) & 0xFFFF, **kw)
    assert case.bn == bn
    gemm_verdict(case, label, expect=gemm_kernel_name(bn, epi, out16))
    return case


def test_instantiation_table_is_complete():
    """26 distinct kernels: 13 epilogue variants per tile width, as test_gemm_kernels_do_not_spill counts in the build log."""
    assert len(set(INSTANTIATIONS)) == len(INSTANTIATIONS) == 26
    assert {e for e, _ in KERNELS} == set(EPI)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [FULL, RAGGED], ids=["full", "ragged"])
@pytest.mark.parametrize("bn,epi,out16", INSTANTIATIONS, ids=[f"{b}-{e}-{o}" for b, e, o in INSTANTIATIONS])
def test_every_instantiation(bn, epi, out16, shape):
    _run(f"<{bn},{epi},{out16}> {'x'.join(map(str, shape))}", bn, epi, out16, shape, **KERNELS[(epi, out16)])


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 256])
def test_pooler_chunk(bn):
    """ReLU(acc + bias) -> fp32 + 16-bit copy: the F32 kernel's out-of-line pooler chunk."""
    _run(f"pooler bn{bn}", bn, "F32", 0, FULL, outs=("out_f32", "out_bf16"), fp16=True, out_fp16=True, bias=True, act=RELU)


N_ = FULL[1]
ALIGNMENT = {
    "ld_out_f32 % 4 != 0": (("F32", 0), dict(ld={"out_f32": N_ + 1})),
    "ld_res % 4 != 0": (("F32", 0), dict(ld={"residual": N_ + 3})),
    "ld_aux % 4 != 0": (("DGELU", 0), dict(ld={"aux": N_ + 1})),
    "ld_out_pre % 4 != 0": (("GELU", 1), dict(ld={"out_pre": N_ + 1})),
    "out_bf16 4-byte aligned": (("BF16", 0), dict(align={"out_bf16": 4})),
}


@pytest.mark.gpu
@pytest.mark.parametrize("what", sorted(ALIGNMENT))
def test_alignment_fallbacks(what):
    (epi, out16), over = ALIGNMENT[what]
    _run(what, 128, epi, out16, FULL, **dict(KERNELS[(epi, out16)], **over))


# ------------------------------------------------------------------------------------------ scheduler
CAPS = ["1", "7", "SMs-16", "0"]
WORK = ["SMs-1", "SMs", "SMs+1", "2SMs+1"]


def _value(expr, sms):
    return int(eval(expr.replace("2SMs", "2*SMs"), {"SMs": sms}))


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("work", WORK)
@pytest.mark.parametrize("cap", CAPS)
def test_capped_grid_tiles(cap, work, bn):
    """W = work tiles (128 x bn), one k split, on a grid of min(W, cap) persistent CTAs."""
    sms = _sms()
    w = _value(work, sms)
    b = max(d for d in range(1, 9) if w % d == 0)          # tile columns; the rest are row blocks
    shape = (128 * (w // b), bn * b, 64)
    _run(f"cap {cap} work {w} bn{bn}", bn, "F32", 0, shape, outs=("out_f32",), fp16=True, bias=True, max_ctas=_value(cap, sms))


@pytest.mark.gpu
@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("form", ["forced3", "auto", "partials"])
def test_capped_grid_split_k(cap, form):
    """Split-K weight gradients under a cap: forced split_k = 3, the automatic choice, and deterministic partials with the split
    count vb_gemm_plan resolves under that cap (the slices past it must stay untouched)."""
    sms = _sms()
    mc = _value(cap, sms)
    kw = dict(outs=("out_f32",), a_mn=True, b_mn=True, max_ctas=mc)
    if form == "forced3":
        shape, kw = (1000, 520, 640), dict(kw, atomic=1, split_k=3)
        epi = "ATOMIC"
    else:
        shape, kw = (768, 768, 6400), dict(kw, atomic=1 if form == "auto" else PARTIALS, split_k=0)
        epi = "ATOMIC" if form == "auto" else "PARTIAL"
    case = GemmCase(*shape, block_n=128, seed=5, **kw)
    if form == "forced3":
        assert case.split == 3
    if form == "partials":
        free = GemmCase(*shape, block_n=128, seed=5, **dict(kw, max_ctas=0))
        print(f"\n[gemm] partials split under cap {mc}: {case.split} (uncapped {free.split})")
        case.g.split_k = 0                    # partials need the split count as resolved: 0 (automatic) is refused
        assert L.lib().vb_gemm_bf16(C.byref(case.g), None) == L.VB_ERR_INVALID
        case.g.split_k = case.split
    gemm_verdict(case, f"split-K {form} cap {mc}", expect=gemm_kernel_name(128, epi, 0))


# ------------------------------------------------------------------------------------------ residual in place, split precision
@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("shape", [FULL, RAGGED], ids=["full", "ragged"])
def test_residual_in_place(shape, bn):
    """residual == out_f32 (dgrad into the residual stream): each element is read before it is overwritten."""
    _run(f"in-place residual bn{bn} {'x'.join(map(str, shape))}", bn, "F32", 0, shape, outs=("out_f32",), fp16=True,
         bias=True, res_inplace=True)


@pytest.mark.gpu
@pytest.mark.parametrize("lo", ["A", "B", "AB"])
def test_split_precision_passes(lo):
    """pass_sel of every combination: hi.hi + lo.hi (A_lo), hi.hi + hi.lo (B_lo), all three; fp32 + hi / lo outputs."""
    _run(f"split precision {lo}_lo", 128, "GENERIC", 0, (200, 328, 192), outs=("out_f32", "out_bf16", "out_lo"), fp16=True,
         out_fp16=True, bias=True, a_lo="A" in lo, b_lo="B" in lo)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["partials", "atomic"])
def test_split_precision_split_k_straddles_passes(form):
    """K = 192 (3 k-blocks) x 3 passes = 9 virtual k-blocks in 2 splits of 5 + 4: the first ends inside pass 1, the second
    begins there. Partials are checked slice by slice against the k-blocks of their own split."""
    kw = dict(outs=("out_f32",), a_mn=True, b_mn=True, fp16=True, a_lo=True, b_lo=True)
    if form == "partials":
        _run("split precision partials straddling", 128, "PARTIAL", 0, (300, 200, 192), atomic=PARTIALS, split_k=2, **kw)
    else:
        _run("split precision atomic straddling", 128, "ATOMIC", 0, (300, 200, 192), atomic=1, split_k=2, **kw)
