"""The float64 GEMM checker (tests/_gpu_util.GemmCase) discriminates, without a GPU: an emulated kernel (fp32 accumulation of
16-wide k groups in the kernel's pass order, an fp32 epilogue, round-to-nearest 16-bit outputs) written into the checker's guarded
CPU buffers passes it, and each planted defect fails it."""
import pytest
import torch

from _gpu_util import BF, GEMM_TOLS, GemmCase, _bits, _sentinel, keep_scale, rz16, ulp_up
from vilbert_b200 import _lib as L

F16 = torch.float16


def emulate(case, drop_lo_kblock=False):
    """Writes what a correct kernel writes into case's output regions (drop_lo_kblock: the last k-block of low-part pass 1 skipped)."""
    M, N = case.M, case.N
    ps = case.passes()
    rk = -(-case.K // 64)
    blocks = [b for i, b in enumerate(case.kblocks()) if not (drop_lo_kblock and i == 2 * rk - 1)]
    acc = torch.zeros(M, N, dtype=torch.float32)
    for p, k0, k1 in blocks:
        A, B = ps[p]
        for k in range(k0, k1, 16):
            acc = (acc.double() + A[:, k:min(k + 16, k1)] @ B[:, k:min(k + 16, k1)].t()).float()
    v = acc.double() * case.alpha
    if "bias" in case.fields:
        v = v + case.region["bias"].double()
    v = v.float()                                                    # fmaf(acc, alpha, bias)
    pre = None
    if case.act == L.VB_ACT_GELU:
        x = v.double()
        cdf = 0.5 * (1 + torch.erf(x / 2 ** 0.5))
        pre = (cdf + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5).float()
        v = (x * cdf).float()
    elif case.act == L.VB_ACT_DGELU:
        v = v * case.region["aux"].float()
    if case.drop is not None:
        v = v * keep_scale(M, N, case.drop[0], 1, case.drop[1], "cpu").float()
    if "out_colsum" in case.outs:
        case.region["out_colsum"] += v.sum(0, keepdim=True)
    if "residual" in case.fields:
        v = v + case.res0[:M, :N]
    if "out_f32" in case.outs:
        case.region["out_f32"].copy_(v)
    if "out_bf16" in case.outs:
        hi = v.to(case.dt["out_bf16"])
        case.region["out_bf16"].copy_(hi)
        if "out_lo" in case.outs:
            case.region["out_lo"].copy_((v - hi.float()).to(case.dt["out_lo"]))
    if "out_b16" in case.outs:
        case.region["out_b16"].copy_(v.to(BF))
    if "out_pre" in case.outs:
        case.region["out_pre"].copy_(pre.to(BF))


def failed(e):
    return [k for k, tol in GEMM_TOLS.items() if k in e and not e[k] <= tol]


CASES = {
    "f32 bias residual": dict(outs=("out_f32",), bias=True, res=True, fp16=True),
    "bf16 out": dict(outs=("out_bf16",)),
    "fp16 out + bf16 copy": dict(outs=("out_bf16", "out_b16"), fp16=True, out_fp16=True, bias=True),
    "gelu": dict(outs=("out_bf16", "out_pre", "out_b16"), act=L.VB_ACT_GELU, bias=True, fp16=True, out_fp16=True),
    "dgelu colsum": dict(outs=("out_bf16", "out_colsum"), act=L.VB_ACT_DGELU),
    "split precision": dict(outs=("out_f32", "out_bf16", "out_lo"), a_lo=True, b_lo=True, fp16=True, out_fp16=True, bias=True),
    "dropout in-place residual": dict(outs=("out_f32",), bias=True, res_inplace=True, drop=(7, 0.1), fp16=True),
}


def _case(kw, M=45, N=40, K=256):
    return GemmCase(M, N, K, device="cpu", seed=11, **kw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_kernel_passes(name):
    c = _case(CASES[name])
    emulate(c)
    e = c.errors()
    assert not failed(e), (name, e)
    if "exact" in e:      # most 16-bit elements are held bitwise, not merely within a window (GELU's absolute erf error widens
        assert e["exact"] > 0.5, e   # the window of its small negative outputs)


def _defect(name, plant):
    c = _case(CASES[name])
    emulate(c, drop_lo_kblock=(plant == "drop_lo_kblock"))
    M, N = c.M, c.N
    f = c.outs[0] if plant != "lo_ulp" else "out_lo"
    if plant == "rz":
        y = c.reference()["y"]
        c.region["out_bf16"].copy_(rz16(y, c.dt["out_bf16"]))
    elif plant == "stray_pad":
        c.view[f][3, N] = 1.0                      # one element into the row pitch's padding
    elif plant == "stray_row":
        c.view[f][M, 5] = 1.0                      # one element of the row past M
    elif plant == "unwritten":
        _bits(c.region[f])[M // 2, N // 3] = _sentinel(c.dt.get(f, torch.float32)).item()
    elif plant == "lost_chunk":
        m0 = (M - 1) // 16 * 16
        _bits(c.region[f])[m0:M] = _sentinel(c.dt.get(f, torch.float32)).item()
    elif plant == "lo_ulp":
        c.region["out_lo"].copy_(ulp_up(c.region["out_lo"]))
    return failed(c.errors())


@pytest.mark.parametrize("name,plant,expect", [
    ("bf16 out", "rz", "out_bf16"),
    ("fp16 out + bf16 copy", "rz", "out_bf16"),
    ("split precision", "drop_lo_kblock", "out_f32"),
    ("bf16 out", "stray_pad", "guard"),
    ("f32 bias residual", "stray_row", "guard"),
    ("gelu", "stray_pad", "guard"),
    ("bf16 out", "unwritten", "unwritten"),
    ("f32 bias residual", "unwritten", "unwritten"),
    ("dgelu colsum", "lost_chunk", "out_bf16"),
    ("dropout in-place residual", "lost_chunk", "out_f32"),
    ("split precision", "lo_ulp", "out_lo"),
])
def test_planted_defect_fails(name, plant, expect):
    assert expect in _defect(name, plant)


def test_wrong_references_miss():
    """The wrong references a GPU case asserts against miss the emulated kernel by more than 10x the bound."""
    from _gpu_util import gemm_wrongs, REF_OF
    for name in ("f32 bias residual", "split precision", "gelu", "dropout in-place residual"):
        c = _case(CASES[name])
        emulate(c)
        ref = c.reference()
        for lab, wr in gemm_wrongs(c).items():
            e = c.errors(wr)
            ks = [k for k in ("out_f32", "out_bf16", "out_lo", "out_b16", "out_pre") if k in e and not torch.equal(wr[REF_OF[k]], ref[REF_OF[k]])]
            assert ks and all(e[k] > 10 for k in ks), (name, lab, {k: e[k] for k in ks})
