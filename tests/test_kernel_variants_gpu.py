"""The kernel variants that the host code picks from the problem shape, each at the edges of its range, against float64 references;
the entry points that no other test calls directly; and the launches the library refuses.

Every LayerNorm case runs under torch.profiler and asserts the templates it is meant to reach, so that a case stays a boundary case
when a threshold moves (the attention backward's edges do the same in tests/test_kernels_gpu.py). Where a plausible slip would go unnoticed by the other cases (a row mean over the full lanes of a partly
filled float4 chunk, a softmax that forgets the keys of earlier chunks) a case also recomputes its reference with that slip and
asserts that it misses by more than 10x the tolerance."""
import ctypes as C
import math
import re
import zlib

import pytest
import torch

from _gpu_util import launched
from vilbert_b200 import _lib as L

pytestmark = pytest.mark.gpu
BF, F16, F64 = torch.bfloat16, torch.float16, torch.float64
DEV = "cuda"
NAN = float("nan")


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def _p(t):
    return None if t is None else t.data_ptr()


def relmax(a, ref):
    a, ref = a.to(F64), ref.to(F64)
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()


def colsum_err(got, base, terms):
    """max over columns of |got - base - sum_m terms[m, col]| / (|base| + sum_m |terms[m, col]|)  (terms [M, cols]): the sum is
    added into a non-zero buffer, whose value its roundings are relative to (at M = 1 a single term may be much smaller)."""
    terms = terms.to(F64).reshape(terms.shape[0], -1)
    base = base.to(F64).flatten()
    s, a = terms.sum(0), terms.abs().sum(0) + base.abs()
    return ((got.to(F64).flatten() - base - s).abs() / a.clamp_min(1e-300)).max().item()


def verdict(case, errs, tols, wrongs=None):
    """errs / tols: {output: value}; wrongs: {label: {output: error of that wrong reference}}, each more than 10x its tolerance."""
    wrongs = wrongs or {}
    w = "  ".join(f"{lab}:" + ",".join(f"{k}={v:.2e}" for k, v in we.items()) for lab, we in wrongs.items())
    print(f"\n[kernel-variants] {case} | err/tol " + ",".join(f"{k}={v:.2e}/{tols[k]:.0e}" for k, v in errs.items())
          + (f" | wrong {w}" if w else ""))
    for k, v in errs.items():
        assert v <= tols[k], (case, k, v, tols[k])
    for lab, we in wrongs.items():
        for k, v in we.items():
            assert v > 10 * tols[k], (case, lab, k, v, tols[k])


def _refused(status, code, pattern):
    assert status == code, (status, code)
    msg = L.lib().vb_last_error().decode()
    assert re.search(pattern, msg), msg


def _no_kernel(names, pattern):
    assert not any(re.search(pattern, n) for n in names), sorted(set(names))


# ============================================================================================ LayerNorm
# ln_fwd_kernel<NV4, ADD>: NV4 = ceil(H / 128) rounded up to {1, 2, 4, 6, 8, 16} (one warp per row, NV4 float4 chunks per lane);
# ln_bwd_kernel<NV> / ln_bwd_det_kernel<NV>: NV = ceil(H / 256) rounded up to {1, 2, 3, 4, 8} (a 64-lane team per row). The widths
# take the lower and upper end of every template, and widths that leave the last float4 chunk of some lanes empty.
LN_VARIANTS = {   # H: (forward NV4, backward NV)
    4: (1, 1), 128: (1, 1), 132: (2, 1), 256: (2, 1), 260: (4, 2), 384: (4, 2), 512: (4, 2), 516: (6, 3), 772: (8, 4),
    1020: (8, 4), 1028: (16, 8), 1536: (16, 8), 2044: (16, 8)}
LN_TOL = dict(x=0.0, y=1e-5, mean=1e-5, rstd=1e-5, hilo=2e-6, dx32=1e-5, dx16=0.0, dgamma=2e-5, dbeta=2e-5, dbias=2e-5, det=0.0)


def _ln64(x):
    x = x.to(F64)
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + 1e-12)
    return (x - mean) * rstd, mean.squeeze(-1), rstd.squeeze(-1)


# M = 9001 rows at H = 260 is past row_grid's cap (SMs x 8 CTAs x 8 rows, 8448 on 132 SMs): the grid-stride row loop goes round
@pytest.mark.parametrize("M,H", [(M, H) for H in LN_VARIANTS for M in (1, 3, 5, 333)] + [(9001, 260)])
def test_layernorm_variants(M, H):
    """vb_layernorm_fwd (fp32 + bf16, then fp16 hi + lo + bf16 copy), vb_add_layernorm_fwd, vb_layernorm_bwd, vb_add_layernorm_bwd
    (dy + dy2, gelu_pre, dbias) and vb_layernorm_bwd_det against float64. 16-bit outputs are bitwise the cast of the kernel's own
    fp32 value; accumulated column sums start from non-zero buffers and are bounded per column by 2e-5 * (|base| + sum_m |term|)."""
    nv4, nv = LN_VARIANTS[H]
    gen = _gen("ln", M, H)
    lib = L.lib()
    x = torch.randn(M, H, device=DEV, generator=gen) * 2 + 3.0
    r = torch.randn(M, H, device=DEV, generator=gen)
    gm, bt = torch.randn(H, device=DEV, generator=gen), torch.randn(H, device=DEV, generator=gen)
    dy, dy2 = torch.randn(M, H, device=DEV, generator=gen), torch.randn(M, H, device=DEV, generator=gen)
    pre = torch.rand(M, H, device=DEV, generator=gen).to(BF) * 1.2      # a saved gelu'(pre-activation)
    base = {k: torch.randn(H, device=DEV, generator=gen) for k in ("dgamma", "dbeta", "dbias")}
    o = {}

    def run():
        full = lambda dt=torch.float32: torch.full((M, H), NAN, device=DEV, dtype=dt)
        o["y32"], o["y16"], o["mean"], o["rstd"] = full(), full(BF), torch.full((M,), NAN, device=DEV), torch.full((M,), NAN, device=DEV)
        L.check(lib.vb_layernorm_fwd(x.data_ptr(), H, gm.data_ptr(), bt.data_ptr(), 1e-12, o["y32"].data_ptr(), o["y16"].data_ptr(), H,
                                     o["mean"].data_ptr(), o["rstd"].data_ptr(), M, H, None, 0, None, None, _st()))
        o["hi"], o["lo"], o["yb"] = full(F16), full(F16), full(BF)
        L.check(lib.vb_layernorm_fwd(x.data_ptr(), H, gm.data_ptr(), bt.data_ptr(), 1e-12, None, o["hi"].data_ptr(), H, None, None, M, H,
                                     None, 1, o["lo"].data_ptr(), o["yb"].data_ptr(), _st()))
        # residual LayerNorm: x = d + r written over d
        o["xa"] = x - r
        o["a32"], o["ahi"], o["alo"], o["ab"] = full(), full(F16), full(F16), full(BF)
        o["amean"], o["arstd"] = torch.full((M,), NAN, device=DEV), torch.full((M,), NAN, device=DEV)
        L.check(lib.vb_add_layernorm_fwd(o["xa"].data_ptr(), r.data_ptr(), H, None, o["xa"].data_ptr(), gm.data_ptr(), bt.data_ptr(), 1e-12,
                                         o["a32"].data_ptr(), o["ahi"].data_ptr(), H, o["amean"].data_ptr(), o["arstd"].data_ptr(), M, H, 1,
                                         o["alo"].data_ptr(), o["ab"].data_ptr(), _st()))
        # backward: plain (dx32, dx16, dgamma, dbeta)
        o["dx32"], o["dx16"] = full(), full(BF)
        o["acc"] = {k: v.clone() for k, v in base.items()}
        L.check(lib.vb_layernorm_bwd(dy.data_ptr(), H, x.data_ptr(), H, gm.data_ptr(), o["mean"].data_ptr(), o["rstd"].data_ptr(),
                                     o["dx32"].data_ptr(), o["dx16"].data_ptr(), H, None, 0, o["acc"]["dgamma"].data_ptr(),
                                     o["acc"]["dbeta"].data_ptr(), None, M, H, None, None, _st()))
        # dy + dy2 with the GELU derivative and the bias gradient
        o["ex32"], o["ex16"] = full(), full(BF)
        o["eacc"] = {k: v.clone() for k, v in base.items()}
        L.check(lib.vb_add_layernorm_bwd(dy.data_ptr(), dy2.data_ptr(), H, x.data_ptr(), H, gm.data_ptr(), o["mean"].data_ptr(),
                                         o["rstd"].data_ptr(), o["ex32"].data_ptr(), o["ex16"].data_ptr(), H, pre.data_ptr(), H,
                                         o["eacc"]["dgamma"].data_ptr(), o["eacc"]["dbeta"].data_ptr(), o["eacc"]["dbias"].data_ptr(),
                                         M, H, None, None, _st()))
        # deterministic plans: the same sums through per-CTA slices
        o["tx32"], o["tx16"] = full(), full(BF)
        o["tacc"] = {k: v.clone() for k, v in base.items()}
        grid = min((M + 3) // 4, L.VB_DET_LN_SLICES)
        ws = torch.full((3 * grid * H,), NAN, device=DEV)
        L.check(lib.vb_layernorm_bwd_det(dy.data_ptr(), dy2.data_ptr(), H, x.data_ptr(), H, gm.data_ptr(), o["mean"].data_ptr(),
                                         o["rstd"].data_ptr(), o["tx32"].data_ptr(), o["tx16"].data_ptr(), H, pre.data_ptr(), H,
                                         o["tacc"]["dgamma"].data_ptr(), o["tacc"]["dbeta"].data_ptr(), o["tacc"]["dbias"].data_ptr(),
                                         M, H, None, None, ws.data_ptr(), _st()))

    launched(run, rf"ln_fwd_kernel<{nv4}, false>", rf"ln_fwd_kernel<{nv4}, true>", rf"ln_bwd_kernel<{nv}>", rf"ln_bwd_det_kernel<{nv}>")

    xh, mu, rs = _ln64(x)
    y = xh * gm.to(F64) + bt.to(F64)
    xs = (x - r) + r                                                    # the kernel's one fp32 add
    xha, mua, rsa = _ln64(xs)
    ya = xha * gm.to(F64) + bt.to(F64)
    gamma64 = gm.to(F64)

    def dx_of(g, xhat, rstd):
        gg = g * gamma64
        return rstd[:, None] * (gg - gg.mean(-1, keepdim=True) - xhat * (gg * xhat).mean(-1, keepdim=True))

    dx = dx_of(dy.to(F64), xh, rs)
    g2 = (dy + dy2).to(F64)                                             # dy + dy2 is one fp32 add in the kernel
    dx2 = dx_of(g2, xh, rs)
    dxp = dx2 * pre.to(F64)
    e = o
    errs = dict(y=max(relmax(e["y32"], y), relmax(e["a32"], ya)), mean=max(relmax(e["mean"], mu), relmax(e["amean"], mua)),
                rstd=max(relmax(e["rstd"], rs), relmax(e["arstd"], rsa)),
                x=(e["xa"] != xs).double().mean().item(),
                hilo=max(relmax(e["hi"].float() + e["lo"].float(), e["y32"]), relmax(e["ahi"].float() + e["alo"].float(), e["a32"])),
                # 16-bit copies: fraction of elements that are not the cast of the kernel's fp32 value
                dx16=max((e["y16"] != e["y32"].to(BF)).double().mean().item(), (e["hi"] != e["y32"].to(F16)).double().mean().item(),
                         (e["yb"] != e["y32"].to(BF)).double().mean().item(), (e["ahi"] != e["a32"].to(F16)).double().mean().item(),
                         (e["ab"] != e["a32"].to(BF)).double().mean().item(), (e["dx16"] != e["dx32"].to(BF)).double().mean().item(),
                         (e["ex16"] != (e["ex32"] * pre.float()).to(BF)).double().mean().item()),
                dx32=max(relmax(e["dx32"], dx), relmax(e["ex32"], dx2)),
                dgamma=max(colsum_err(e["acc"]["dgamma"], base["dgamma"], dy.to(F64) * xh),
                           colsum_err(e["eacc"]["dgamma"], base["dgamma"], g2 * xh), colsum_err(e["tacc"]["dgamma"], base["dgamma"], g2 * xh)),
                dbeta=max(colsum_err(e["acc"]["dbeta"], base["dbeta"], dy), colsum_err(e["eacc"]["dbeta"], base["dbeta"], g2),
                          colsum_err(e["tacc"]["dbeta"], base["dbeta"], g2)),
                dbias=max(colsum_err(e["eacc"]["dbias"], base["dbias"], dxp), colsum_err(e["tacc"]["dbias"], base["dbias"], dxp)),
                # the deterministic kernel's rows are the default kernel's: bitwise
                det=max((e["tx32"] != e["ex32"]).double().mean().item(), (e["tx16"] != e["ex16"]).double().mean().item()))
    assert torch.equal(base["dbias"], e["acc"]["dbias"])                # dbias NULL in the plain backward: untouched
    wrongs = {}
    if (H // 4) % (32 * nv4):
        # sensitivity: the row mean taken over every lane's full chunks (H rounded up to 128 * NV4 columns, the missing ones 0)
        xw = x.to(F64)
        mean_w = xw.sum(-1) / (128 * nv4)
        rstd_w = 1.0 / torch.sqrt(((xw - mean_w[:, None]) ** 2).mean(-1) + 1e-12)
        yw = (xw - mean_w[:, None]) * rstd_w[:, None] * gamma64 + bt.to(F64)
        wrongs["full-lane mean"] = dict(y=relmax(e["y32"], yw))
    verdict(f"layernorm {M}x{H} fwd<{nv4}> bwd<{nv}>", errs, LN_TOL, wrongs)


# ============================================================================================ attention, streamed forward
# Split precision at D = 128 keeps Q plus hi and lo panels of K and V for every padded key: (D + 8) * 2 bytes * 2 parts = 544 bytes
# per key and panel. With 64 query rows (34816 B) and the mask (4 B per key), 2 * 192 keys need 243 KiB > 227 KiB, so from a
# padded key count of 192 (Nk >= 129) the forward streams the keys in chunks of 128 (kchunk) through the same panels:
# Nk = 129 -> chunks 128 + 1 key, 192 -> 128 + 64, 256 -> 128 + 128, 320 -> 128 + 128 + 64.
@pytest.mark.parametrize("Nq", [1, 37, 100])
@pytest.mark.parametrize("Nk", [129, 192, 256, 320])
def test_attention_split_streamed_forward(Nq, Nk):
    """Cross-attention in split precision (Q / K / V as fp16 hi + lo, O as hi + lo) on the streamed path, against the float64
    attention of the fp32 inputs. Masks: sample 0 all keys valid, sample 1 a single valid key, sample 2 valid keys in the first chunk
    only (every later chunk masked), sample 3 every key masked. A fully masked row is the softmax of the unmasked scores over all
    Nk keys, and the padding keys past Nk stay excluded. Its scores sit near -10000 * log2(e) in the kernel's fp32 log2 domain,
    where one rounding of s * scale + mask is 2^-11: its rows are bounded by ln(2) 2^-10 sum_j p_j |v_j| beyond the 2e-5 bound."""
    B, H, D = 4, 2, 128
    gen = _gen("streamed", Nq, Nk)
    lib = L.lib()
    Hd = H * D
    q32 = torch.randn(B * Nq, Hd, device=DEV, generator=gen)
    k32 = torch.randn(B * Nk, 2 * Hd, device=DEV, generator=gen)
    qh, kh = q32.half(), k32.half()
    ql, kl = (q32 - qh.float()).half(), (k32 - kh.float()).half()
    lens = torch.tensor([Nk, 1, min(100, Nk - 1), 0], device=DEV)
    mask = ((torch.arange(Nk, device=DEV)[None] >= lens[:, None]).float() * -10000.0).contiguous()
    O, Ol = torch.full((B * Nq, Hd), NAN, device=DEV, dtype=F16), torch.full((B * Nq, Hd), NAN, device=DEV, dtype=F16)
    lse = torch.full((B, H, Nq), NAN, device=DEV)
    a = L.AttnArgs()
    a.B, a.H, a.Nq, a.Nk, a.D = B, H, Nq, Nk, D
    a.Q, a.ldq, a.K, a.ldk, a.V, a.ldv = qh.data_ptr(), Hd, kh.data_ptr(), 2 * Hd, kh[:, Hd:].data_ptr(), 2 * Hd
    a.Q_lo, a.K_lo, a.V_lo = ql.data_ptr(), kl.data_ptr(), kl[:, Hd:].data_ptr()
    a.mask, a.scale, a.O, a.O_lo, a.ldo, a.lse, a.qkv_fp16 = mask.data_ptr(), 1.0 / math.sqrt(D), O.data_ptr(), Ol.data_ptr(), Hd, lse.data_ptr(), 1
    # no profiler check here: the streamed and the resident forward are the same template (attn_fwd_kernel<128, true, true>) with a
    # runtime kchunk, so the kernel name cannot tell them apart; the arithmetic above puts every case on the streamed side
    L.check(lib.vb_attention_fwd(C.byref(a), _st()), "vb_attention_fwd")

    q = q32.to(F64).view(B, Nq, H, D).permute(0, 2, 1, 3)
    k = k32[:, :Hd].to(F64).view(B, Nk, H, D).permute(0, 2, 1, 3)
    v = k32[:, Hd:].to(F64).view(B, Nk, H, D).permute(0, 2, 1, 3)
    s = q @ k.transpose(-1, -2) / math.sqrt(D) + mask.to(F64)[:, None, None, :]
    p = torch.softmax(s, -1)
    ref = p @ v                                                          # [B, H, Nq, D]
    got = (O.float() + Ol.float()).to(F64).view(B, Nq, H, D).permute(0, 2, 1, 3)
    scale = ref.abs().max().item()
    live = slice(0, 3)
    bound = 2e-5 * scale + math.log(2) * 2 ** -10 * (p @ v.abs())[3]   # the fully masked sample's rows

    def masked_ratio(r):
        return ((got[3] - r[3]).abs() / bound).max().item()

    errs = dict(O=((got[live] - ref[live]).abs().max() / scale).item(), O_masked=masked_ratio(ref),
                lse=relmax((lse * math.log(2.0))[live], torch.logsumexp(s, -1)[live]))
    wrongs = {}
    if Nk >= 256:
        # sensitivity: the fully masked row's softmax over the first chunk only (the later chunks' keys forgotten); at Nk = 129 / 192 the
        # first chunk holds most of the keys and the slip moves O by less than 10x the masked-row bound
        p1 = torch.softmax(s[..., :128], -1)
        wrongs["first chunk only"] = dict(O_masked=masked_ratio(torch.cat([ref[:3], (p1 @ v[..., :128, :])[3:]])))
    if Nk % 64:
        # sensitivity: the padding keys past Nk (zero-filled panel rows) treated as masked (-10000) rather than absent, which only
        # the fully masked row can tell: its softmax would also spread over the zero scores of the padding
        pad = (Nk + 63) // 64 * 64 - Nk
        sp = torch.cat([s, torch.full(s.shape[:-1] + (pad,), -10000.0, dtype=F64, device=DEV)], -1)
        wrongs["padding as masked"] = dict(O_masked=masked_ratio(torch.cat([ref[:3], (torch.softmax(sp, -1)[..., :Nk] @ v)[3:]])))
    verdict(f"attn split streamed Nq={Nq} Nk={Nk}", errs, dict(O=2e-5, O_masked=1.0, lse=1e-5), wrongs)


# ============================================================================================ attention, backward partial at the fused ceiling
def test_attention_partial_backward_fused_ceiling():
    """Nq = Nk = 128, D = 128 (the fused kernel's largest shared-memory footprint, where test_attention_fp16_operands pins
    attn_bwd_fused_kernel<128, true, true>): dQ only and dK / dV only write bitwise what the full backward writes, and nothing else."""
    from _gpu_util import attn_case
    B, H, Nq, Nk, D = 2, 4, 128, 128, 128
    gen = _gen("partial", B, H)
    lib = L.lib()
    Hd = H * D
    qkv = torch.randn(B * Nq, 3 * Hd, device=DEV, generator=gen).half()
    mask = torch.zeros(B, Nk, device=DEV); mask[1, 77:] = -10000.0
    O, Ob = torch.empty(B * Nq, Hd, device=DEV, dtype=F16), torch.empty(B * Nq, Hd, device=DEV, dtype=BF)
    lse, delta = torch.empty(B, H, Nq, device=DEV), torch.empty(B, H, Nq, device=DEV)
    dO = torch.randn(B * Nq, Hd, device=DEV, generator=gen).to(BF)
    a = L.AttnArgs()
    a.B, a.H, a.Nq, a.Nk, a.D = B, H, Nq, Nk, D
    a.Q, a.ldq, a.K, a.ldk, a.V, a.ldv = qkv.data_ptr(), 3 * Hd, qkv[:, Hd:].data_ptr(), 3 * Hd, qkv[:, 2 * Hd:].data_ptr(), 3 * Hd
    a.mask, a.scale, a.O, a.ldo, a.lse, a.O_b16, a.qkv_fp16 = mask.data_ptr(), 1.0 / math.sqrt(D), O.data_ptr(), Hd, lse.data_ptr(), Ob.data_ptr(), 1
    a.dO, a.lddo, a.delta = dO.data_ptr(), Hd, delta.data_ptr()
    L.check(lib.vb_attention_fwd(C.byref(a), _st()))

    def bwd(dq, dkv):
        g = torch.full((B * Nq, 3 * Hd), NAN, device=DEV, dtype=BF)
        a.dQ, a.lddq = (g.data_ptr(), 3 * Hd) if dq else (None, 0)
        a.dK, a.dV, a.lddk, a.lddv = (g[:, Hd:].data_ptr(), g[:, 2 * Hd:].data_ptr(), 3 * Hd, 3 * Hd) if dkv else (None, None, 0, 0)
        L.check(lib.vb_attention_bwd(C.byref(a), _st()))
        torch.cuda.synchronize()
        return g

    full, only_q, only_kv = bwd(True, True), bwd(True, False), bwd(False, True)
    assert not full.isnan().any()
    assert torch.equal(only_q[:, :Hd], full[:, :Hd]) and only_q[:, Hd:].isnan().all()
    assert torch.equal(only_kv[:, Hd:], full[:, Hd:]) and only_kv[:, :Hd].isnan().all()
    # and the full backward at this shape is right (fp16 operands, the tolerances of test_attention_fp16_operands)
    errs, _ = attn_case(B, H, Nq, Nk, D, False, fp16=True)
    assert errs["lse"] < 1e-5 and errs["O"] < 2e-3 and max(errs.values()) < 3e-2, errs


# ============================================================================================ entry points at the engine's shapes
# B = 64 samples, 36 text tokens + the task token, 101 regions, Ht = 768, Hv = 1024
EB, ENT, ENV, EHT, EHV = 64, 37, 101, 768, 1024


def _prefix_mask(B, N, gen):
    lens = torch.randint(1, N + 1, (B,), device=DEV, generator=gen)
    lens[0], lens[1] = 1, N
    m = (torch.arange(N, device=DEV)[None] < lens[:, None])
    return m, ((1.0 - m.float()) * -10000.0).contiguous()


def test_masked_mean_fwd_bwd():
    """vb_masked_mean_fwd / _bwd (dynamic_attention's text pool) with prefix masks of random length (including 1 and all tokens):
    pool against the float64 masked mean, its operand copies bitwise the casts of pool, dx with accumulate 0 (from NaN) and 1."""
    gen = _gen("masked_mean")
    lib = L.lib()
    x = torch.randn(EB, ENT, EHT, device=DEV, generator=gen)
    m, add = _prefix_mask(EB, ENT, gen)
    w = m.to(F64)
    ref = (w[:, :, None] * x.to(F64)).sum(1) / w.sum(1, keepdim=True)
    bnd = (w[:, :, None] * x.to(F64).abs()).sum(1) / w.sum(1, keepdim=True)     # mean of |x|: the scale of the rounding
    for fp16 in (1, 0):
        pool = torch.full((EB, EHT), NAN, device=DEV)
        p16, plo = (torch.full((EB, EHT), NAN, device=DEV, dtype=F16 if fp16 else BF) for _ in range(2))
        pb = torch.full((EB, EHT), NAN, device=DEV, dtype=BF)                # the always-bf16 copy
        L.check(lib.vb_masked_mean_fwd(x.data_ptr(), add.data_ptr(), pool.data_ptr(), p16.data_ptr(), plo.data_ptr() if fp16 else None,
                                       pb.data_ptr() if fp16 else None, fp16, EB, ENT, EHT, _st()))
        torch.cuda.synchronize()
        assert ((pool.to(F64) - ref).abs() <= 3e-6 * bnd + 1e-30).all(), ((pool.to(F64) - ref).abs() / bnd).max()
        if fp16:
            assert torch.equal(p16, pool.half()) and torch.equal(plo, (pool - p16.float()).half()) and torch.equal(pb, pool.to(BF))
        else:
            assert torch.equal(p16, pool.to(BF)) and plo.isnan().all() and pb.isnan().all()
    dpool = torch.randn(EB, EHT, device=DEV, generator=gen)
    g = (w / w.sum(1, keepdim=True))[:, :, None] * dpool.to(F64)[:, None, :]
    for acc in (0, 1):
        base = torch.randn(EB, ENT, EHT, device=DEV, generator=gen) if acc else torch.full((EB, ENT, EHT), NAN, device=DEV)
        dx = base.clone()
        L.check(lib.vb_masked_mean_bwd(dpool.data_ptr(), add.data_ptr(), dx.data_ptr(), acc, EB, ENT, EHT, _st()))
        torch.cuda.synchronize()
        r = g + (base.to(F64) if acc else 0)
        tol = 1e-6 * (g.abs() + (base.to(F64).abs() if acc else 0))
        assert ((dx.to(F64) - r).abs() <= tol).all(), ((dx.to(F64) - r).abs() - tol).max()
        if acc:
            assert torch.equal(dx[~m], base[~m])                         # masked tokens: + 0 exactly
        else:
            assert (dx[~m] == 0).all()


@pytest.mark.parametrize("mode", ["fp16", "fp16 hi+lo", "bf16"])
def test_gate_scale_fwd_bwd(mode):
    """vb_gate_scale_fwd in place on the Q | K columns of a [B * Nv, 3 * Hv] projection buffer (row pitch padded by 16 elements):
    hi within one 16-bit rounding of the float64 product, hi + lo within 2^-20; the V columns and the padding bitwise unchanged.
    vb_gate_scale_bwd: dqk = gate * dqk within bf16 rounding, dz = s (1 - s) / gate * sum_n dq q over the GATED buffer (bounded per
    column by 2e-5 of the sum of |terms|), dz16 = bf16(dz); with both dz outputs NULL only dqk changes."""
    fp16, split = mode != "bf16", mode == "fp16 hi+lo"
    dt = F16 if fp16 else BF
    u = 2.0 ** -11 if fp16 else 2.0 ** -8                                # unit roundoff of the 16-bit format
    gen = _gen("gate", mode)
    lib = L.lib()
    M, cols, ld = EB * ENV, 2 * EHV, 3 * EHV + 16
    x32 = torch.randn(M + 3, ld, device=DEV, generator=gen)              # 3 rows past the B * Nv rows: untouched too
    hi = x32.to(dt)
    lo = (x32 - hi.float()).to(dt) if split else None
    z = torch.randn(EB, cols, device=DEV, generator=gen) * 2
    hi0, lo0 = hi.clone(), (lo.clone() if split else None)
    L.check(lib.vb_gate_scale_fwd(hi.data_ptr(), _p(lo), ld, z.data_ptr(), EB, ENV, cols, int(fp16), _st()))
    torch.cuda.synchronize()
    gate = (1 + torch.sigmoid(z.to(F64))).repeat_interleave(ENV, 0)      # [M, cols]
    xin = hi0[:M, :cols].to(F64) + (lo0[:M, :cols].to(F64) if split else 0)
    ref = xin * gate
    assert torch.equal(hi[:M, cols:], hi0[:M, cols:]) and torch.equal(hi[M:], hi0[M:])
    tiny = 2.0 ** -24 if fp16 else 0.0                                   # fp16 subnormal spacing
    assert ((hi[:M, :cols].to(F64) - ref).abs() <= u * ref.abs() * (1 + 1e-2) + tiny).all()
    if split:
        assert torch.equal(lo[:M, cols:], lo0[:M, cols:]) and torch.equal(lo[M:], lo0[M:])
        e = (hi[:M, :cols].to(F64) + lo[:M, :cols].to(F64) - ref).abs()
        assert (e <= 2.0 ** -20 * ref.abs() + 2.0 ** -25).all(), (e / ref.abs()).max()

    # backward over the gated buffer
    ldd = 3 * EHV
    dq0 = torch.randn(M, ldd, device=DEV, generator=gen).to(BF)
    dq = dq0.clone()
    dz, dz16 = torch.full((EB, cols), NAN, device=DEV), torch.full((EB, cols), NAN, device=DEV, dtype=BF)
    L.check(lib.vb_gate_scale_bwd(dq.data_ptr(), ldd, hi.data_ptr(), _p(lo), ld, z.data_ptr(), dz.data_ptr(), dz16.data_ptr(), EB, ENV, cols,
                                  int(fp16), _st()))
    torch.cuda.synchronize()
    rq = dq0[:, :cols].to(F64) * gate
    assert ((dq[:, :cols].to(F64) - rq).abs() <= 2.0 ** -8 * rq.abs() * (1 + 1e-3)).all()
    assert torch.equal(dq[:, cols:], dq0[:, cols:])
    q = hi[:M, :cols].to(F64) + (lo[:M, :cols].to(F64) if split else 0)
    s = torch.sigmoid(z.to(F64))
    terms = (dq0[:, :cols].to(F64) * q).view(EB, ENV, cols)
    coef = s * (1 - s) / (1 + s)
    rz = coef * terms.sum(1)
    # the kernel forms s (1 - s) in fp32 as the header states it: 1 - s of a saturated gate (s near 1) carries 2^-24 / (1 - s) of
    # relative error, which the second term allows
    tol = 2e-5 * coef * terms.abs().sum(1) + 2.0 ** -22 * s / (1 + s) * terms.sum(1).abs()
    assert ((dz.to(F64) - rz).abs() <= tol).all(), ((dz.to(F64) - rz).abs() / tol).max()
    assert torch.equal(dz16, dz.to(BF))
    # both dz outputs NULL: dqk scaled bitwise as above, nothing else written
    dq2, hi2 = dq0.clone(), hi.clone()
    L.check(lib.vb_gate_scale_bwd(dq2.data_ptr(), ldd, hi.data_ptr(), _p(lo), ld, z.data_ptr(), None, None, EB, ENV, cols, int(fp16), _st()))
    torch.cuda.synchronize()
    assert torch.equal(dq2, dq) and torch.equal(hi, hi2)


@pytest.mark.parametrize("acc", [0, 1])
def test_sum_strided_in_batch_pairs(acc):
    """vb_sum_strided in both stride orders of the in_batch_pairs backward: pair p = i * b + j; a text item's gradient sums its b
    consecutive copies (stride_k = b * n, stride_r = n), an image item's the copies b * n apart (stride_k = n, stride_r = b * n). The
    buffer past b items holds NaN sentinels that must stay."""
    b = 8
    gen = _gen("sum_strided", acc)
    lib = L.lib()
    for N, Hh, text in ((ENT, EHT, True), (ENV, EHV, False)):
        n = N * Hh
        g = torch.randn(b * b, n, device=DEV, generator=gen)
        base = torch.randn(b + 1, n, device=DEV, generator=gen) if acc else torch.full((b + 1, n), 0.0, device=DEV)
        base[b] = NAN
        dst = base.clone()
        if text:
            L.check(lib.vb_sum_strided(g.data_ptr(), dst.data_ptr(), n, b, b * n, b, n, acc, _st()))
            terms = g.view(b, b, n)                                      # [i, j]: text i summed over j
        else:
            L.check(lib.vb_sum_strided(g.data_ptr(), dst.data_ptr(), n, b, n, b, b * n, acc, _st()))
            terms = g.view(b, b, n).transpose(0, 1)                       # image j summed over i
        torch.cuda.synchronize()
        t64 = terms.to(F64)
        r = t64.sum(1) + (base[:b].to(F64) if acc else 0)
        tol = 1e-6 * (t64.abs().sum(1) + (base[:b].to(F64).abs() if acc else 0))
        assert ((dst[:b].to(F64) - r).abs() <= tol).all(), ("text" if text else "image", ((dst[:b].to(F64) - r).abs() - tol).max())
        assert dst[b].isnan().all()


def test_broadcast_rows_relu_axpy_masks_counter_memset():
    """vb_broadcast_rows (fast_mode's text broadcast, bitwise), vb_relu_bwd (exact, y == 0 gives 0), vb_axpy_f32 (within 1 ulp of
    float64), vb_mask_concat_additive (exact), vb_step_counter_bump (incl. the wrap of 0xFFFFFFFF to 0), vb_memset_zero (a sub-range:
    the bytes on either side untouched), vb_device_info."""
    gen = _gen("misc")
    lib = L.lib()
    # broadcast: one caption's text states [Nt, Ht] to B rows of the batch, as fp32 and as 16-bit operand
    for dt in (torch.float32, F16):
        src = torch.randn(ENT, EHT, device=DEV, generator=gen).to(dt)
        dst = torch.full((EB + 1, ENT, EHT), NAN, device=DEV, dtype=dt)
        L.check(lib.vb_broadcast_rows(src.data_ptr(), dst.data_ptr(), src.numel() * src.element_size(), EB, _st()))
        torch.cuda.synchronize()
        assert torch.equal(dst[:EB], src.expand(EB, ENT, EHT)) and dst[EB].isnan().all()
    # relu backward: n not a multiple of 4, exact zeros (+0 and -0) in y
    n = EB * EHV + 3
    y = torch.randn(n, device=DEV, generator=gen); y[::7] = 0.0; y[1::11] = -0.0
    dy = torch.randn(n, device=DEV, generator=gen)
    dx16, dx32 = torch.full((n,), NAN, device=DEV, dtype=BF), torch.full((n,), NAN, device=DEV)
    L.check(lib.vb_relu_bwd(dy.data_ptr(), y.data_ptr(), dx16.data_ptr(), dx32.data_ptr(), n, _st()))
    torch.cuda.synchronize()
    r = torch.where(y > 0, dy, torch.zeros_like(dy))
    assert torch.equal(dx32, r) and torch.equal(dx16, r.to(BF)) and (dx32[y == 0] == 0).all()
    # axpy
    x = torch.randn(n, device=DEV, generator=gen); yy = torch.randn(n, device=DEV, generator=gen); y0 = yy.clone()
    L.check(lib.vb_axpy_f32(x.data_ptr(), yy.data_ptr(), n, 0.37, _st()))
    torch.cuda.synchronize()
    ref = y0.to(F64) + torch.tensor(0.37, dtype=torch.float32).item() * x.to(F64)
    assert ((yy.to(F64) - ref).abs() <= 2.0 ** -23 * ref.abs() + 2.0 ** -149).all()
    # single-stream masks: cat((1 - mask_t) * -10000, (1 - mask_v) * -10000)
    mt, _ = _prefix_mask(EB, ENT, gen)
    mv, _ = _prefix_mask(EB, ENV, gen)
    mt64, mv64 = mt.long(), mv.long()
    out = torch.full((EB * (ENT + ENV) + 5,), NAN, device=DEV)
    L.check(lib.vb_mask_concat_additive(mt64.data_ptr(), mv64.data_ptr(), out.data_ptr(), EB, ENT, ENV, _st()))
    torch.cuda.synchronize()
    ref = torch.cat([(1.0 - mt.float()) * -10000.0, (1.0 - mv.float()) * -10000.0], 1)
    assert torch.equal(out[:-5].view(EB, ENT + ENV), ref) and out[-5:].isnan().all()
    # step counter (uint32 held in an int32 tensor): 5 -> 6, 0xFFFFFFFF -> 0; neighbours untouched
    ctr = torch.tensor([11, 5, 11, -1, 11], dtype=torch.int32, device=DEV)
    L.check(lib.vb_step_counter_bump(ctr[1:].data_ptr(), _st()))
    L.check(lib.vb_step_counter_bump(ctr[3:].data_ptr(), _st()))
    torch.cuda.synchronize()
    assert ctr.tolist() == [11, 6, 11, 0, 11]
    # memset of an odd sub-range
    buf = torch.randint(1, 256, (4099,), dtype=torch.uint8, device=DEV, generator=gen)
    b0 = buf.clone()
    L.check(lib.vb_memset_zero(buf[3:].data_ptr(), 4001, _st()))
    torch.cuda.synchronize()
    assert (buf[3:4004] == 0).all() and torch.equal(buf[:3], b0[:3]) and torch.equal(buf[4004:], b0[4004:])
    # device info
    sm, cc = C.c_int(), C.c_int()
    L.check(lib.vb_device_info(C.byref(sm), C.byref(cc)))
    props = torch.cuda.get_device_properties(0)
    assert sm.value == props.multi_processor_count and cc.value == props.major * 10 + props.minor


# ============================================================================================ refusals
def test_limits_are_refused_not_launched():
    """Host-side checks that return before any launch, with their documented status and message: the two-kernel attention backward
    at D = 128 past 320 keys or (with dK / dV) 320 queries, LayerNorm widths that are not a multiple of 4 or above 2048, copies whose
    sizes are not multiples of 16 bytes, an odd gate column count. Nothing is written and no kernel runs."""
    lib = L.lib()
    H, D = 2, 128
    Hd = H * D

    def attn_bwd(Nq, Nk):
        q = torch.zeros(Nq, 3 * Hd, device=DEV, dtype=BF); k = torch.zeros(Nk, 3 * Hd, device=DEV, dtype=BF)
        dq = torch.full((Nq, 3 * Hd), NAN, device=DEV, dtype=BF); dk = torch.full((Nk, 3 * Hd), NAN, device=DEV, dtype=BF)
        o = torch.zeros(Nq, Hd, device=DEV, dtype=BF)
        lse, delta = torch.zeros(1, H, Nq, device=DEV), torch.full((1, H, Nq), NAN, device=DEV)
        a = L.AttnArgs()
        a.B, a.H, a.Nq, a.Nk, a.D = 1, H, Nq, Nk, D
        a.Q, a.ldq, a.K, a.ldk, a.V, a.ldv = q.data_ptr(), 3 * Hd, k[:, Hd:].data_ptr(), 3 * Hd, k[:, 2 * Hd:].data_ptr(), 3 * Hd
        a.scale, a.O, a.ldo, a.lse, a.dO, a.lddo, a.delta = 1.0, o.data_ptr(), Hd, lse.data_ptr(), o.data_ptr(), Hd, delta.data_ptr()
        a.dQ, a.lddq = dq.data_ptr(), 3 * Hd
        a.dK, a.dV, a.lddk, a.lddv = dk[:, Hd:].data_ptr(), dk[:, 2 * Hd:].data_ptr(), 3 * Hd, 3 * Hd
        st, names = launched(lambda: lib.vb_attention_bwd(C.byref(a), _st()))
        _refused(st, 2, r"sequence too long for the smem-resident panel")
        _no_kernel(names, r"attn_")
        assert dq.isnan().all() and dk.isnan().all() and delta.isnan().all()

    attn_bwd(36, 384)
    attn_bwd(384, 36)

    for Hbad in (2052, 130):
        x = torch.zeros(4, 2056, device=DEV); g = torch.zeros(2056, device=DEV)
        st, names = launched(lambda: lib.vb_layernorm_fwd(x.data_ptr(), 2056, g.data_ptr(), g.data_ptr(), 1e-12, x.data_ptr(), None, 2056,
                                                          None, None, 4, Hbad, None, 0, None, None, _st()))
        _refused(st, 1, r"need H % 4 == 0, H <= 2048")
        st2 = lib.vb_layernorm_bwd(x.data_ptr(), 2056, x.data_ptr(), 2056, g.data_ptr(), g.data_ptr(), g.data_ptr(), x.data_ptr(), None,
                                   2056, None, 0, None, None, None, 4, Hbad, None, None, _st())
        _refused(st2, 1, r"need H % 4 == 0, H <= 2048")
        _no_kernel(names, r"ln_")

    src = torch.zeros(64, device=DEV); dst = torch.full((256,), NAN, device=DEV)
    st, names = launched(lambda: lib.vb_broadcast_rows(src.data_ptr(), dst.data_ptr(), 24, 4, _st()))
    _refused(st, 1, r"vb_broadcast_rows: needs 16-byte aligned buffers and size")
    st = lib.vb_sum_strided(src.data_ptr(), dst.data_ptr(), 6, 2, 8, 2, 16, 0, _st())
    _refused(st, 1, r"vb_sum_strided: sizes / strides must be multiples of 4 floats")
    st = lib.vb_sum_strided(src.data_ptr(), dst.data_ptr(), 8, 2, 8, 2, 18, 0, _st())
    _refused(st, 1, r"vb_sum_strided: sizes / strides must be multiples of 4 floats")
    qk = torch.zeros(8, 12, device=DEV, dtype=F16); z = torch.zeros(2, 12, device=DEV); qk0 = qk.clone()
    st2 = lib.vb_gate_scale_fwd(qk.data_ptr(), None, 12, z.data_ptr(), 2, 4, 7, 1, _st())
    _refused(st2, 1, r"vb_gate_scale_fwd: bad arguments \(even cols")
    torch.cuda.synchronize()
    _no_kernel(names, r"broadcast_rows")
    assert dst.isnan().all() and torch.equal(qk, qk0)
