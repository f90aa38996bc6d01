"""Training-only kernel arguments against float64 references with the dropout mask applied explicitly (tests/_train_ref.py, pinned
by tests/test_train_kernels_cpu.py): every dropout site of the kernels (GEMM epilogue, attention probabilities, LayerNorm in / out,
add + LayerNorm, small linears, fused pooled vector, single-stream embeddings) and every fused bias-gradient sum (the GEMM's
out_colsum, the LayerNorm backward's dbias, the attention backward's dbias_q / dbias_k / dbias_v), at the shapes the engine launches.

Every case also recomputes its reference with a wrong mask (the next step's, and where a kernel computes an index of its own, the
index a plausible slip would give) and asserts that it misses by more than 10x the tolerance: the case would catch that slip.
Dropped elements of elementwise outputs are asserted exactly. Accumulated outputs start from a non-zero buffer. A bias sum is
bounded per column by c * sum_m |term_m| of that column (a column sum may cancel to about 0)."""
import ctypes as C
import math
import zlib

import pytest
import torch

import _train_ref as R
from vilbert_b200 import _lib as L
from vilbert_b200.engine import dropout_site_id

pytestmark = pytest.mark.gpu
BF, F16, F64 = torch.bfloat16, torch.float16, torch.float64
DEV = "cuda"
STEP = 123456           # step * 0x9E3779B9 wraps mod 2^32


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _step_tensor(step):
    """The device step counter (uint32) as an int32 tensor holding the same bits."""
    return torch.tensor([step - 2 ** 32 if step >= 2 ** 31 else step], dtype=torch.int32, device=DEV)


def _desc(step_t, site, p):
    d = L.Dropout()
    d.step, d.site, d.p = step_t.data_ptr(), site, p
    return d


def _gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def relmax(a, ref):
    a, ref = a.to(F64), ref.to(F64)
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()


def colsum_err(got, base, terms):
    """max over columns of |(got - base) - sum_m terms[m, col]| / sum_m |terms[m, col]|  (terms [M, cols])."""
    terms = terms.to(F64).reshape(terms.shape[0], -1)
    s, a = terms.sum(0), terms.abs().sum(0)
    return ((got.to(F64).flatten() - base.to(F64).flatten() - s).abs() / a.clamp_min(1e-300)).max().item()


def verdict(case, errs, tols, wrongs, dropped_frac=None, p=None):
    """errs / tols: {output: value}; wrongs: {label: {output: error of that wrong reference}}. Prints one line per case (the
    table of the pull request description comes from these lines), then asserts."""
    w = "  ".join(f"{lab}:" + ",".join(f"{k}={v:.2e}" for k, v in we.items()) for lab, we in wrongs.items())
    e = ",".join(f"{k}={v:.2e}/{tols[k]:.0e}" for k, v in errs.items())
    print(f"\n[train-kernels] {case} | err/tol {e} | wrong {w}" + (f" | dropped {dropped_frac:.4f} p={p}" if p else "")
          + f" | peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    for k, v in errs.items():
        assert v <= tols[k], (case, k, v, tols[k])
    for lab, we in wrongs.items():
        for k, v in we.items():
            assert v > 10 * tols[k], (case, lab, k, v, tols[k])
    if p is not None:
        assert abs(dropped_frac - p) < 0.05, (case, dropped_frac, p)


# ============================================================================================ attention
ATT_SITE = dropout_site_id("bert.encoder.c_layer.0.biattention.dropout1")
ATT_P = 0.1
# O of fp16 operands at fp16 accuracy; gradients against the attention of the bf16-rounded inputs (the backward contracts in bf16),
# the tolerances of tests/test_kernels_gpu.py::test_attention_fp16_operands
ATT_TOL = dict(O=2e-3, lse=1e-5, dQ=3e-2, dK=3e-2, dV=3e-2, dbias_q=2e-3, dbias_k=2e-3, dbias_v=2e-3,
               # dQ of a single-key row and dK of its key are 0 in exact arithmetic: relative to the largest dQ / dK of the case
               dQ_1key=1e-4, dK_1key=1e-4)


def _attn_setup(B, H, Nq, Nk, D, cross, gen, split=False):
    Hd = H * D
    q32 = torch.randn(B * Nq, 3 * Hd, device=DEV, generator=gen)
    k32 = torch.randn(B * Nk, 3 * Hd, device=DEV, generator=gen) if cross else q32
    qsrc, ksrc = q32.half(), k32.half()
    t = dict(q32=q32[:, :Hd], k32=k32[:, Hd:2 * Hd], v32=k32[:, 2 * Hd:], q=qsrc[:, :Hd], k=ksrc[:, Hd:2 * Hd], v=ksrc[:, 2 * Hd:])
    if split:
        qlo, klo = (q32 - qsrc.float()).half(), (k32 - ksrc.float()).half()
        t.update(qlo=qlo[:, :Hd], klo=klo[:, Hd:2 * Hd], vlo=klo[:, 2 * Hd:])
    lens = torch.randint(1, Nk + 1, (B,), device=DEV, generator=gen)
    lens[0] = Nk
    lens[1] = 1                                   # a row with a single valid key
    mask = (torch.arange(Nk, device=DEV)[None] >= lens[:, None]).float() * -10000.0
    mask[2] = -10000.0                            # a batch row with every key masked: its softmax is that of the unmasked scores
    t["mask"] = mask.contiguous()
    return t


def _attn_args(t, B, H, Nq, Nk, D, ld):
    a = L.AttnArgs()
    a.B, a.H, a.Nq, a.Nk, a.D = B, H, Nq, Nk, D
    a.Q, a.ldq, a.K, a.ldk, a.V, a.ldv = t["q"].data_ptr(), ld, t["k"].data_ptr(), ld, t["v"].data_ptr(), ld
    a.mask, a.scale = t["mask"].data_ptr(), 1.0 / math.sqrt(D)
    a.qkv_fp16 = 1
    return a


def _attn_ref(qq, kk, vv, mask, f, dO, B, H, Nq, Nk, D):
    """float64 attention with the dropout factor f [B, H, Nq, Nk] on the probabilities; returns O [B*Nq, H*D] and, when dO is
    given, dQ / dK / dV in [B*N, H*D] row layout."""
    sh = lambda x, N: x.to(F64).view(B, N, H, D).permute(0, 2, 1, 3).detach().requires_grad_(dO is not None)
    qf, kf, vf = sh(qq, Nq), sh(kk, Nk), sh(vv, Nk)
    s = qf @ kf.transpose(-1, -2) / math.sqrt(D) + mask.to(F64)[:, None, None, :]
    o = ((torch.softmax(s, -1) * f.to(F64)) @ vf).permute(0, 2, 1, 3).reshape(B * Nq, H * D)
    if dO is None:
        return o.detach(), None
    o.backward(dO.to(F64))
    back = lambda g, N: g.permute(0, 2, 1, 3).reshape(B * N, H * D)
    return o.detach(), (back(qf.grad, Nq), back(kf.grad, Nk), back(vf.grad, Nk))


def _attention_case(B, H, Nq, Nk, D, cross):
    """Forward + backward with dropout and dbias_q / k / v. Returns (errors, {wrong reference: errors}, dropped fraction,
    errors of dQ / dK on the batch rows with a single valid key, relative to the largest reference value of all rows)."""
    gen = _gen("attn", B, H, Nq, Nk, D)
    Hd = H * D
    t = _attn_setup(B, H, Nq, Nk, D, cross, gen)
    step_t = _step_tensor(STEP)
    a = _attn_args(t, B, H, Nq, Nk, D, 3 * Hd)
    O = torch.zeros(B * Nq, Hd, device=DEV, dtype=F16)
    Ob = torch.zeros(B * Nq, Hd, device=DEV, dtype=BF)
    lse, delta = torch.zeros(B, H, Nq, device=DEV), torch.zeros(B, H, Nq, device=DEV)
    dO = torch.randn(B * Nq, Hd, device=DEV, generator=gen).to(BF)
    dq = torch.zeros(B * Nq, 3 * Hd, device=DEV, dtype=BF)
    dkv = torch.zeros(B * Nk, 3 * Hd, device=DEV, dtype=BF)
    base = {k: torch.randn(Hd, device=DEV, generator=gen) for k in ("q", "k", "v")}
    db = {k: v.clone() for k, v in base.items()}
    a.O, a.ldo, a.lse, a.O_b16 = O.data_ptr(), Hd, lse.data_ptr(), Ob.data_ptr()
    a.dO, a.lddo, a.delta = dO.data_ptr(), Hd, delta.data_ptr()
    a.dQ, a.lddq = dq.data_ptr(), 3 * Hd
    a.dK, a.lddk, a.dV, a.lddv = dkv[:, Hd:].data_ptr(), 3 * Hd, dkv[:, 2 * Hd:].data_ptr(), 3 * Hd
    a.dbias_q, a.dbias_k, a.dbias_v = db["q"].data_ptr(), db["k"].data_ptr(), db["v"].data_ptr()
    a.dropout = _desc(step_t, ATT_SITE, ATT_P)
    L.check(L.lib().vb_attention_fwd(C.byref(a), _st()), "vb_attention_fwd")
    L.check(L.lib().vb_attention_bwd(C.byref(a), _st()), "vb_attention_bwd")
    torch.cuda.synchronize()
    got = dict(O=O, dQ=dq[:, :Hd], dK=dkv[:, Hd:2 * Hd], dV=dkv[:, 2 * Hd:])
    # batch rows whose mask leaves a single key (row 1, and any random length of 1)
    one = (t["mask"] == 0).sum(1) == 1
    qone, kone = one.repeat_interleave(Nq), one.repeat_interleave(Nk)
    single = {}

    def compare(f, keep_single=False):
        o_ref, _ = _attn_ref(t["q"], t["k"], t["v"], t["mask"], f, None, B, H, Nq, Nk, D)
        # the backward contracts bf16 panels (the fp16 Q / K / V rounded to bf16): its reference is the attention of those values
        _, (gq, gk, gv) = _attn_ref(t["q"].to(BF), t["k"].to(BF), t["v"].to(BF), t["mask"], f, dO, B, H, Nq, Nk, D)
        if keep_single:
            single.update(dQ_1key=((got["dQ"].to(F64) - gq)[qone].abs().max() / gq.abs().max()).item(),
                          dK_1key=((got["dK"].to(F64) - gk)[kone].abs().max() / gk.abs().max()).item())
        return dict(O=relmax(got["O"], o_ref), dQ=relmax(got["dQ"], gq), dK=relmax(got["dK"], gk), dV=relmax(got["dV"], gv),
                    dbias_q=colsum_err(db["q"], base["q"], gq), dbias_k=colsum_err(db["k"], base["k"], gk),
                    dbias_v=colsum_err(db["v"], base["v"], gv))

    f = R.keep_factor(ATT_SITE, STEP, ATT_P, R.attn_index(B, H, Nq, Nk, DEV))
    errs = compare(f, keep_single=True)
    s = (t["q"].to(F64).view(B, Nq, H, D).permute(0, 2, 1, 3) @ t["k"].to(F64).view(B, Nk, H, D).permute(0, 2, 3, 1)
         / math.sqrt(D) + t["mask"].to(F64)[:, None, None, :])
    live = torch.arange(B, device=DEV) != 2       # the fully masked row's lse sits near -10000: compare the others
    errs["lse"] = relmax((lse * math.log(2.0))[live], torch.logsumexp(s, -1)[live])
    wrongs = {"step+1": compare(R.keep_factor(ATT_SITE, STEP + 1, ATT_P, R.attn_index(B, H, Nq, Nk, DEV))),
              "k*Nq+q": compare(R.keep_factor(ATT_SITE, STEP, ATT_P, R.attn_index(B, H, Nq, Nk, DEV, transposed=True)))}
    # the key bias gradient is 0 in exact arithmetic whatever the mask (softmax shift invariance: sum_k dS[q, k] = 0 for every q), so
    # no wrong mask moves its reference: dbias_k is checked for accuracy only
    for w in wrongs.values():
        del w["dbias_k"]
    return errs, wrongs, (f == 0).double().mean().item(), single


@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", [
    # fused single-CTA backward (Nq <= 128, Nk <= 128, D >= 32 and the panels fit in shared memory)
    (64, 12, 36, 36, 64, False), (64, 8, 101, 101, 128, False), (64, 8, 36, 101, 128, True), (64, 8, 101, 36, 128, True),
    # two-kernel backward (dQ kernel, then dK / dV kernel): Nq > 128 or Nk > 128, or D == 16
    (32, 8, 200, 21, 128, True), (8, 8, 306, 257, 128, True), (8, 12, 257, 257, 64, False), (16, 4, 37, 33, 16, True)])
def test_attention_dropout_and_bias_sums(B, H, Nq, Nk, D, cross):
    errs, wrongs, dropped, single = _attention_case(B, H, Nq, Nk, D, cross)
    # single-key rows: their dQ / dK are 0 whatever the mask, so they take part in the tolerance but not in the wrong-mask checks
    verdict(f"attention {B}x{H}x{Nq}x{Nk}x{D}", dict(errs, **single), ATT_TOL, wrongs, dropped, ATT_P)


@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", [(64, 8, 101, 101, 128, False), (8, 8, 306, 257, 128, True), (16, 4, 37, 33, 16, True)])
def test_attention_dropout_single_key_row(B, H, Nq, Nk, D, cross):
    """A query row whose mask leaves one key: P = 1 on it, so dS = P (f dP - delta) = 0 and dQ of the row and dK of the key are 0 in
    exact arithmetic. The backward used to form delta from the bf16 copy of O, bf16(f V), against f (dO . bf16(V)) in dP: equal
    without dropout, but with it they differ by a bf16 rounding, and dK of that key reached 7e-2 of the largest dK at 306 x 257
    (1.3e-2 on the fused path at 101 x 101). delta is now formed from the P and f dP of dS itself, which cancel to fp32 rounding.
    One case per backward path: fused, two kernels, and two kernels at D = 16."""
    _, _, _, single = _attention_case(B, H, Nq, Nk, D, cross)
    verdict(f"attention single-key rows {B}x{H}x{Nq}x{Nk}x{D}", single, ATT_TOL, {})


@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", [(8, 8, 306, 306, 128, False), (8, 8, 257, 306, 128, True)])
def test_attention_split_forward_streamed_key_chunks(B, H, Nq, Nk, D, cross):
    """Split precision at D = 128: a key row of the hi + lo K and V panels takes (128 + 8) * 2 bytes * 2 parts = 544 B, so the
    query panels (64 rows), the padded mask and both K / V panels of all 320 padded keys need 64*544 + 320*4 + 2*320*544 = 384 KB
    > 227 KB of shared memory: vb_attention_fwd streams the keys in chunks of 128 (kchunk < nkp), and the mask index of a key is
    offset by its chunk start k0."""
    gen = _gen("split", B, H, Nq, Nk, D)
    Hd = H * D
    t = _attn_setup(B, H, Nq, Nk, D, cross, gen, split=True)
    step_t = _step_tensor(STEP)
    a = _attn_args(t, B, H, Nq, Nk, D, 3 * Hd)
    a.Q_lo, a.K_lo, a.V_lo = t["qlo"].data_ptr(), t["klo"].data_ptr(), t["vlo"].data_ptr()
    O, Olo = torch.zeros(B * Nq, Hd, device=DEV, dtype=F16), torch.zeros(B * Nq, Hd, device=DEV, dtype=F16)
    a.O, a.ldo, a.O_lo = O.data_ptr(), Hd, Olo.data_ptr()
    a.dropout = _desc(step_t, ATT_SITE, ATT_P)
    L.check(L.lib().vb_attention_fwd(C.byref(a), _st()), "vb_attention_fwd")
    torch.cuda.synchronize()
    o = O.double() + Olo.double()
    # batch row 2 has every key masked: its scores carry the -10000 * log2(e) offset in fp32, whose spacing (2^-10) bounds the
    # accuracy of its probabilities to ~7e-4, as in the fp32 reference model; every other row is held to the split-precision bound
    rows2 = torch.arange(B * Nq, device=DEV) // Nq == 2

    def err(f):   # split precision reconstructs the fp32 inputs: float64 reference of q32 / k32 / v32
        ref = _attn_ref(t["q32"], t["k32"], t["v32"], t["mask"], f, None, B, H, Nq, Nk, D)[0]
        scale_ = ref.abs().max()
        return dict(O_split=((o - ref)[~rows2].abs().max() / scale_).item(), O_masked_row=((o - ref)[rows2].abs().max() / scale_).item())

    f = R.keep_factor(ATT_SITE, STEP, ATT_P, R.attn_index(B, H, Nq, Nk, DEV))
    wrongs = {"step+1": err(R.keep_factor(ATT_SITE, STEP + 1, ATT_P, R.attn_index(B, H, Nq, Nk, DEV))),
              "k*Nq+q": err(R.keep_factor(ATT_SITE, STEP, ATT_P, R.attn_index(B, H, Nq, Nk, DEV, transposed=True)))}
    verdict(f"attention split fwd {B}x{H}x{Nq}x{Nk}x{D}", err(f), dict(O_split=2e-5, O_masked_row=2e-3), wrongs,
            (f == 0).double().mean().item(), ATT_P)


def test_attention_probs_export():
    """vb_attention_probs (config.visualization) at the largest co-attention, 306 queries x 257 keys, against the float64 softmax."""
    B, H, Nq, Nk, D = 4, 8, 306, 257, 128
    gen = _gen("probs")
    t = _attn_setup(B, H, Nq, Nk, D, True, gen)
    a = _attn_args(t, B, H, Nq, Nk, D, 3 * H * D)
    P = torch.full((B, H, Nq, Nk), float("nan"), device=DEV)
    L.check(L.lib().vb_attention_probs(C.byref(a), P.data_ptr(), _st()), "vb_attention_probs")
    torch.cuda.synchronize()
    s = (t["q"].to(F64).view(B, Nq, H, D).permute(0, 2, 1, 3) @ t["k"].to(F64).view(B, Nk, H, D).permute(0, 2, 3, 1) / math.sqrt(D))
    ref = torch.softmax(s + t["mask"].to(F64)[:, None, None, :], -1)
    verdict("attention probs 4x8x306x257x128", dict(P=relmax(P, ref)), dict(P=1e-4),
            {"no mask": dict(P=relmax(P, torch.softmax(s, -1)))})


# ============================================================================================ GEMM
def _pad8(n):
    return (n + 7) // 8 * 8


def _plan(g):
    bn, sp = C.c_int32(), C.c_int32()
    L.check(L.lib().vb_gemm_plan(C.byref(g), 0, C.byref(bn), C.byref(sp)), "vb_gemm_plan")
    return bn.value, sp.value


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K,aux_pad", [
    (2304, 3072, 768, 0), (6400, 1024, 1024, 0),      # config 2's text / image FFN dgrads: every chunk full -> fast column sum
    (1000, 520, 200, 0), (333, 1601, 1024, 0),        # ragged rows / columns: fast chunks plus the generic tail
    (1000, 520, 200, 1)])                             # ld_aux % 4 != 0: no vector aux loads -> generic column sum everywhere
def test_gemm_dgelu_colsum(M, N, K, aux_pad, block_n):
    """dgrad of the FFN intermediate: dx = (dy W) * gelu'(pre) as bf16, out_colsum += column sums (the intermediate bias
    gradient). B is the weight stored [K, N] (MN-major), operands bf16. EPI_DGELU: the fast path reduces each 16 x 32 chunk over
    its 4 row lanes by shuffles, then one atomic per column; ragged chunks and unaligned aux run the generic epilogue."""
    gen = _gen("dgelu", M, N, K, aux_pad)
    ld_ab = _pad8(K)
    A = torch.zeros(M, ld_ab, device=DEV, dtype=BF)
    A[:, :K] = (torch.randn(M, K, device=DEV, generator=gen) * 0.5).to(BF)
    ldn = _pad8(N)
    W = torch.zeros(K, ldn, device=DEV, dtype=BF)
    W[:, :N] = (torch.randn(K, N, device=DEV, generator=gen) * 0.5).to(BF)
    ld_aux = ldn + aux_pad
    aux = (torch.rand(M, ld_aux, device=DEV, generator=gen) * 1.2 - 0.1).to(BF)
    out = torch.full((M, ldn), float("nan"), device=DEV, dtype=BF)
    base = torch.randn(N, device=DEV, generator=gen)
    cs = base.clone()
    g = L.GemmArgs()
    g.M, g.N, g.K = M, N, K
    g.A, g.lda, g.B, g.ldb, g.b_mn_major = A.data_ptr(), ld_ab, W.data_ptr(), ldn, 1
    g.alpha, g.act = 1.0, L.VB_ACT_DGELU
    g.aux, g.ld_aux = aux.data_ptr(), ld_aux
    g.out_bf16, g.ld_out_bf16 = out.data_ptr(), ldn
    g.out_colsum = cs.data_ptr()
    g.block_n = block_n
    assert _plan(g) == (block_n, 1)
    L.check(L.lib().vb_gemm_bf16(C.byref(g), _st()), "vb_gemm_bf16")
    torch.cuda.synchronize()
    v = (A[:, :K].to(F64) @ W[:, :N].to(F64)) * aux[:, :N].to(F64)
    errs = dict(out=relmax(out[:, :N], v), colsum=colsum_err(cs, base, v))
    # a column sum that loses one 16-row epilogue chunk (the last one)
    wrongs = {"lost chunk": dict(colsum=colsum_err(cs, base, v[:M - 16]))}
    verdict(f"gemm dgelu colsum {M}x{N}x{K} bn{block_n} ld_aux%4={ld_aux % 4}", errs, dict(out=5e-3, colsum=1e-5), wrongs)


GEMM_SITE = dropout_site_id("bert.encoder.v_layer.2.output.dropout")


@pytest.mark.parametrize("M,N,K,ld_pad", [(6400, 1024, 1024, 0), (2304, 768, 768, 0), (6400, 1024, 1024, 3), (2304, 768, 768, 3)])
def test_gemm_f32_epilogue_dropout_residual(M, N, K, ld_pad):
    """EPI_F32 (act none, fp32 output only, no column sum) with bias + dropout + residual: LN(dropout(dense(x)) + residual).
    ld_pad = 3: the fp32 output pitch is N + 3 (not N, not a multiple of 4), so the fast path stores 32-bit words while the mask
    index stays m*N + n."""
    gen = _gen("f32drop", M, N, K, ld_pad)
    p = 0.1
    A = torch.randn(M, K, device=DEV, generator=gen).half()
    W = (torch.randn(N, K, device=DEV, generator=gen) * 0.05).half()
    bias, res = torch.randn(N, device=DEV, generator=gen), torch.randn(M, N, device=DEV, generator=gen)
    ld = N + ld_pad
    out = torch.full((M, ld), float("nan"), device=DEV)
    step_t = _step_tensor(STEP)
    g = L.GemmArgs()
    g.M, g.N, g.K = M, N, K
    g.A, g.lda, g.B, g.ldb = A.data_ptr(), K, W.data_ptr(), K
    g.alpha, g.bias = 1.0, bias.data_ptr()
    g.residual, g.ld_res = res.data_ptr(), N
    g.out_f32, g.ld_out_f32 = out.data_ptr(), ld
    g.a_fp16 = g.b_fp16 = 1
    g.dropout = _desc(step_t, GEMM_SITE, p)
    L.check(L.lib().vb_gemm_bf16(C.byref(g), _st()), "vb_gemm_bf16")
    torch.cuda.synchronize()
    o = out[:, :N]
    dense = A.to(F64) @ W.to(F64).t() + bias.to(F64)
    f = R.keep_factor(GEMM_SITE, STEP, p, R.rowmajor_index(M, N, DEV))
    drop = f == 0
    assert torch.equal(o[drop], res[drop])                        # a dropped value is exactly the residual
    err = lambda ff: dict(out=relmax(o, dense * ff.to(F64) + res.to(F64)))
    wrongs = {"step+1": err(R.keep_factor(GEMM_SITE, STEP + 1, p, R.rowmajor_index(M, N, DEV)))}
    if ld_pad:
        wrongs["m*ld+n"] = err(R.keep_factor(GEMM_SITE, STEP, p, R.rowmajor_index(M, N, DEV, ld=ld)))
    verdict(f"gemm f32 dropout+residual {M}x{N}x{K} ld={ld}", err(f), dict(out=2e-5), wrongs, drop.double().mean().item(), p)


@pytest.mark.parametrize("ld_pad", [0, 3])
@pytest.mark.parametrize("fmt", ["bf16", "fp16", "split"])
@pytest.mark.parametrize("M,N,K", [(64, 1536, 768), (130, 2048, 1024)])
def test_gemm_generic_relu_dropout(M, N, K, fmt, ld_pad):
    """The single-stream baseline's VQA head, Linear -> ReLU -> Dropout (SimpleClassifier): act ReLU with dropout has no
    specialised epilogue, so every chunk runs the generic one (index m*N + n), with the fp32 output and the 16-bit operand copy
    (bf16; fp16 + bf16 copy; split precision fp16 hi + lo + bf16 copy). ld_pad = 3: every output has pitch N + 3, and the mask
    index stays m*N + n."""
    gen = _gen("relu", M, N, K, fmt, ld_pad)
    ld = N + ld_pad
    p = 0.5
    site = dropout_site_id("vil_prediction.logit_fc.dropout")
    A32, W32 = torch.randn(M, K, device=DEV, generator=gen), torch.randn(N, K, device=DEV, generator=gen) * 0.05
    dt = BF if fmt == "bf16" else F16
    A, W = A32.to(dt), W32.to(dt)
    bias = torch.randn(N, device=DEV, generator=gen) * 0.1
    out_st = torch.full((M, ld), float("nan"), device=DEV)
    hi_st = torch.full((M, ld), float("nan"), device=DEV, dtype=dt)
    lo_st = torch.zeros(M, ld, device=DEV, dtype=F16) if fmt == "split" else None
    b16_st = torch.zeros(M, ld, device=DEV, dtype=BF) if fmt != "bf16" else None
    step_t = _step_tensor(STEP)
    g = L.GemmArgs()
    g.M, g.N, g.K = M, N, K
    g.A, g.lda, g.B, g.ldb = A.data_ptr(), K, W.data_ptr(), K
    g.alpha, g.bias, g.act = 1.0, bias.data_ptr(), L.VB_ACT_RELU
    g.out_f32, g.ld_out_f32, g.out_bf16, g.ld_out_bf16 = out_st.data_ptr(), ld, hi_st.data_ptr(), ld
    g.a_fp16 = g.b_fp16 = g.out_fp16 = int(fmt != "bf16")
    if fmt == "split":
        Alo, Wlo = (A32 - A.float()).half(), (W32 - W.float()).half()
        g.A_lo, g.B_lo, g.out_lo = Alo.data_ptr(), Wlo.data_ptr(), lo_st.data_ptr()
    g.out_b16 = _ptr(b16_st)
    g.dropout = _desc(step_t, site, p)
    L.check(L.lib().vb_gemm_bf16(C.byref(g), _st()), "vb_gemm_bf16")
    torch.cuda.synchronize()
    out, hi = out_st[:, :N], hi_st[:, :N]
    lo = lo_st[:, :N] if lo_st is not None else None
    b16 = b16_st[:, :N] if b16_st is not None else None
    # the 16-bit copies are the fp32 value rounded once (split: hi + the rounded remainder)
    assert torch.equal(hi, out.to(dt))
    if lo is not None:
        assert torch.equal(lo, (out - hi.float()).half())
    if b16 is not None:
        assert torch.equal(b16, out.to(BF))
    if fmt == "split":
        pre = (A32.to(F64) @ W32.to(F64).t() + bias.to(F64)).clamp_min(0)
    else:
        pre = (A.to(F64) @ W.to(F64).t() + bias.to(F64)).clamp_min(0)
    f = R.keep_factor(site, STEP, p, R.rowmajor_index(M, N, DEV))
    assert (out[f == 0] == 0).all()                               # dropped: exactly 0
    err = lambda ff: dict(out=relmax(out, pre * ff.to(F64)))
    wrongs = {"step+1": err(R.keep_factor(site, STEP + 1, p, R.rowmajor_index(M, N, DEV)))}
    if ld_pad:
        wrongs["m*ld+n"] = err(R.keep_factor(site, STEP, p, R.rowmajor_index(M, N, DEV, ld=ld)))
    pos = pre > 1e-3
    verdict(f"gemm generic relu+dropout {M}x{N}x{K} {fmt} ld={ld}", err(f), dict(out=2e-5 if fmt == "split" else 5e-5), wrongs,
            (out[pos] == 0).double().mean().item(), p)


# ============================================================================================ LayerNorm family
LN_SITE = dropout_site_id("bert.encoder.layer.5.output.dropout")
EMB_SITE = dropout_site_id("bert.embeddings.dropout")
LN_TOL = dict(x=0.0, y=1e-5, mean=1e-5, rstd=1e-5, dx32=1e-5, dx16=5e-3, dgamma=2e-5, dbeta=2e-5, dbias=2e-5)


def _ln64(x, gamma, beta):
    x = x.to(F64)
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + 1e-12)
    return (x - mean) * rstd * gamma.to(F64) + beta.to(F64), mean.squeeze(-1), rstd.squeeze(-1)


def _ln_bwd64(x, gamma, g):
    """float64 LayerNorm backward of the output gradient g: (dx, xhat)."""
    x = x.to(F64)
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + 1e-12)
    xh = (x - mean) * rstd
    gg = g.to(F64) * gamma.to(F64)
    dx = rstd * (gg - gg.mean(-1, keepdim=True) - xh * (gg * xh).mean(-1, keepdim=True))
    return dx, xh


@pytest.mark.parametrize("M,H", [(2304, 768), (6400, 1024), (303, 2048)])
def test_add_layernorm_dropout_and_dbias(M, H):
    """vb_add_layernorm_fwd: x = dropout(d) + residual (mask index row*H + col), LN(x); vb_add_layernorm_bwd of dy + dy2 with
    in_dropout: dx16 and dbias carry the mask, dx32 (the residual path) does not. M = 303, H = 2048: an odd row count (the last
    CTA's teams are partly idle) at the widest row."""
    gen = _gen("addln", M, H)
    p = 0.1
    lib = L.lib()
    d, r = torch.randn(M, H, device=DEV, generator=gen), torch.randn(M, H, device=DEV, generator=gen)
    gm, bt = torch.randn(H, device=DEV, generator=gen), torch.randn(H, device=DEV, generator=gen)
    step_t = _step_tensor(STEP)
    drop = _desc(step_t, LN_SITE, p)
    x = d.clone()
    y32, y16 = torch.empty(M, H, device=DEV), torch.empty(M, H, device=DEV, dtype=F16)
    mean, rstd = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    L.check(lib.vb_add_layernorm_fwd(x.data_ptr(), r.data_ptr(), H, C.byref(drop), x.data_ptr(), gm.data_ptr(), bt.data_ptr(), 1e-12,
                                     y32.data_ptr(), y16.data_ptr(), H, mean.data_ptr(), rstd.data_ptr(), M, H, 1, None, None, _st()))
    torch.cuda.synchronize()
    idx = R.rowmajor_index(M, H, DEV)
    f = R.keep_factor(LN_SITE, STEP, p, idx)
    drop_m = f == 0
    assert torch.equal(x[drop_m], r[drop_m])                      # dropped: the sum is exactly the residual
    assert torch.equal(y16, y32.half())

    def fwd_err(ff):
        xs = d * ff + r                                           # the one fp32 multiply and add of the kernel: bitwise
        y, mu, rs = _ln64(d.to(F64) * ff.to(F64) + r.to(F64), gm, bt)
        return dict(x=(x != xs).double().mean().item(), y=relmax(y32, y), mean=relmax(mean, mu), rstd=relmax(rstd, rs))

    # backward
    dy, dy2 = torch.randn(M, H, device=DEV, generator=gen), torch.randn(M, H, device=DEV, generator=gen)
    dx32, dx16 = torch.empty(M, H, device=DEV), torch.empty(M, H, device=DEV, dtype=BF)
    base = {k: torch.randn(H, device=DEV, generator=gen) for k in ("dgamma", "dbeta", "dbias")}
    acc = {k: v.clone() for k, v in base.items()}
    L.check(lib.vb_add_layernorm_bwd(dy.data_ptr(), dy2.data_ptr(), H, x.data_ptr(), H, gm.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                     dx32.data_ptr(), dx16.data_ptr(), H, None, 0, acc["dgamma"].data_ptr(), acc["dbeta"].data_ptr(),
                                     acc["dbias"].data_ptr(), M, H, None, C.byref(drop), _st()))
    torch.cuda.synchronize()
    assert (dx16[drop_m] == 0).all()                              # dropped: exactly 0
    g = dy.to(F64) + dy2.to(F64)
    dx, xh = _ln_bwd64(x, gm, g)

    def bwd_err(ff):
        dxm = dx * ff.to(F64)
        return dict(dx16=relmax(dx16, dxm), dbias=colsum_err(acc["dbias"], base["dbias"], dxm))

    errs = dict(fwd_err(f), dx32=relmax(dx32, dx), dgamma=colsum_err(acc["dgamma"], base["dgamma"], g * xh),
                dbeta=colsum_err(acc["dbeta"], base["dbeta"], g), **bwd_err(f))
    # x: fraction of elements that differ from the bitwise fp32 sum (tolerance 0)
    fw = R.keep_factor(LN_SITE, STEP + 1, p, idx)
    wrong = dict(fwd_err(fw), **bwd_err(fw))
    verdict(f"add_layernorm {M}x{H}", errs, LN_TOL, {"step+1": wrong}, drop_m.double().mean().item(), p)


@pytest.mark.parametrize("M,H", [(2304, 768), (6400, 1024)])
def test_layernorm_out_dropout(M, H):
    """The embeddings' dropout(LayerNorm(x)): vb_layernorm_fwd with out_dropout, vb_layernorm_bwd masking dy first."""
    gen = _gen("lnout", M, H)
    p = 0.1
    lib = L.lib()
    x = torch.randn(M, H, device=DEV, generator=gen) * 2 + 0.5
    gm, bt = torch.randn(H, device=DEV, generator=gen), torch.randn(H, device=DEV, generator=gen)
    step_t = _step_tensor(STEP)
    drop = _desc(step_t, EMB_SITE, p)
    y32, y16 = torch.empty(M, H, device=DEV), torch.empty(M, H, device=DEV, dtype=F16)
    mean, rstd = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    L.check(lib.vb_layernorm_fwd(x.data_ptr(), H, gm.data_ptr(), bt.data_ptr(), 1e-12, y32.data_ptr(), y16.data_ptr(), H, mean.data_ptr(),
                                 rstd.data_ptr(), M, H, C.byref(drop), 1, None, None, _st()))
    dy = torch.randn(M, H, device=DEV, generator=gen)
    dx32 = torch.empty(M, H, device=DEV)
    base = {k: torch.randn(H, device=DEV, generator=gen) for k in ("dgamma", "dbeta")}
    acc = {k: v.clone() for k, v in base.items()}
    L.check(lib.vb_layernorm_bwd(dy.data_ptr(), H, x.data_ptr(), H, gm.data_ptr(), mean.data_ptr(), rstd.data_ptr(), dx32.data_ptr(), None, H,
                                 None, 0, acc["dgamma"].data_ptr(), acc["dbeta"].data_ptr(), None, M, H, C.byref(drop), None, _st()))
    torch.cuda.synchronize()
    f = R.keep_factor(EMB_SITE, STEP, p, R.rowmajor_index(M, H, DEV))
    drop_m = f == 0
    assert (y32[drop_m] == 0).all() and (y16[drop_m] == 0).all()
    assert torch.equal(y16, y32.half())
    y, _, _ = _ln64(x, gm, bt)

    def err(ff):
        g = dy.to(F64) * ff.to(F64)
        dx, xh = _ln_bwd64(x, gm, g)
        return dict(y=relmax(y32, y * ff.to(F64)), dx32=relmax(dx32, dx), dgamma=colsum_err(acc["dgamma"], base["dgamma"], g * xh),
                    dbeta=colsum_err(acc["dbeta"], base["dbeta"], g))

    wrongs = {"step+1": err(R.keep_factor(EMB_SITE, STEP + 1, p, R.rowmajor_index(M, H, DEV)))}
    verdict(f"layernorm out_dropout {M}x{H}", err(f), LN_TOL, wrongs, drop_m.double().mean().item(), p)


def test_layernorm_gelu_pre_dbias():
    """Head transforms, Linear -> GELU -> LayerNorm: vb_layernorm_bwd multiplies dx16 by the saved gelu'(pre) and sums the product
    into dbias (the Linear's bias gradient). The wrong reference leaves the gelu' factor out of the sum."""
    M, H = 2304, 768
    gen = _gen("gelupre")
    lib = L.lib()
    x = torch.randn(M, H, device=DEV, generator=gen)
    gm, bt = torch.randn(H, device=DEV, generator=gen), torch.randn(H, device=DEV, generator=gen)
    pre = (torch.rand(M, H, device=DEV, generator=gen) * 1.2 - 0.1).to(BF)
    mean, rstd = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    L.check(lib.vb_layernorm_fwd(x.data_ptr(), H, gm.data_ptr(), bt.data_ptr(), 1e-12, None, None, H, mean.data_ptr(), rstd.data_ptr(),
                                 M, H, None, 0, None, None, _st()))
    dy = torch.randn(M, H, device=DEV, generator=gen)
    dx16 = torch.empty(M, H, device=DEV, dtype=BF)
    base = torch.randn(H, device=DEV, generator=gen)
    dbias = base.clone()
    L.check(lib.vb_layernorm_bwd(dy.data_ptr(), H, x.data_ptr(), H, gm.data_ptr(), mean.data_ptr(), rstd.data_ptr(), None, dx16.data_ptr(), H,
                                 pre.data_ptr(), H, None, None, dbias.data_ptr(), M, H, None, None, _st()))
    torch.cuda.synchronize()
    dx, _ = _ln_bwd64(x, gm, dy)
    err = lambda t: dict(dx16=relmax(dx16, t), dbias=colsum_err(dbias, base, t))
    verdict("layernorm gelu_pre dbias 2304x768", err(dx * pre.to(F64)), LN_TOL, {"no gelu'": err(dx)})


# ============================================================================================ small linears, pooled fusion
@pytest.mark.parametrize("M,K,N,accumulate", [(64, 1024, 1, 1), (64, 1024, 3, 1), (32, 2048, 2, 1), (6400, 1024, 1, 1), (64, 1024, 3, 0)])
def test_small_linear_in_dropout(M, K, N, accumulate):
    """vil_logit / vision_logit / linguisic_logit style heads: y = dropout(x) W^T + b (+ row addend), mask index m*K + k."""
    gen = _gen("small", M, K, N, accumulate)
    p = 0.1
    site = dropout_site_id("dropout.seq_v")
    lib = L.lib()
    x, W = torch.randn(M, K, device=DEV, generator=gen), torch.randn(N, K, device=DEV, generator=gen)
    b, add = torch.randn(N, device=DEV, generator=gen), torch.randn(M, device=DEV, generator=gen)
    step_t = _step_tensor(STEP)
    drop = _desc(step_t, site, p)
    y = torch.empty(M, N, device=DEV)
    L.check(lib.vb_small_linear_fwd(x.data_ptr(), K, W.data_ptr(), b.data_ptr(), add.data_ptr(), y.data_ptr(), M, K, N, C.byref(drop), _st()))
    dy = torch.randn(M, N, device=DEV, generator=gen)
    dx0 = torch.randn(M, K, device=DEV, generator=gen)
    dx = dx0.clone()
    dW0, db0 = torch.randn(N, K, device=DEV, generator=gen), torch.randn(N, device=DEV, generator=gen)
    dW, db = dW0.clone(), db0.clone()
    L.check(lib.vb_small_linear_bwd(dy.data_ptr(), x.data_ptr(), K, W.data_ptr(), dx.data_ptr(), K, accumulate, dW.data_ptr(), db.data_ptr(),
                                    M, K, N, C.byref(drop), _st()))
    torch.cuda.synchronize()
    f = R.keep_factor(site, STEP, p, R.rowmajor_index(M, K, DEV))
    drop_m = f == 0
    assert torch.equal(dx[drop_m], dx0[drop_m] if accumulate else torch.zeros_like(dx0[drop_m]))   # dropped: nothing added

    def err(ff):
        xd, dy64 = x.to(F64) * ff.to(F64), dy.to(F64)
        gx = (dy64 @ W.to(F64)) * ff.to(F64) + (dx0.to(F64) if accumulate else 0)
        # dW[j, k] = sum_m dy[m, j] xd[m, k]: a column sum per (j, k) over the M terms
        terms = (dy64.t()[:, :, None] * xd[None]).permute(1, 0, 2).reshape(M, N * K)
        return dict(y=relmax(y, xd @ W.to(F64).t() + b.to(F64) + add.to(F64)[:, None]), dx=relmax(dx - (dx0 if accumulate else 0), gx - (dx0.to(F64) if accumulate else 0)),
                    dW=colsum_err(dW, dW0, terms), db=colsum_err(db, db0, dy64))

    errs = err(f)
    wrong = {k: v for k, v in err(R.keep_factor(site, STEP + 1, p, R.rowmajor_index(M, K, DEV))).items() if k != "db"}   # db has no mask
    verdict(f"small_linear {M}x{K}x{N} acc={accumulate}", errs, dict(y=1e-5, dx=1e-5, dW=2e-5, db=2e-5), {"step+1": wrong},
            drop_m.double().mean().item(), p)


@pytest.mark.parametrize("mul", [1, 0])
def test_fuse_pooled_dropout(mul):
    """pooled_output = dropout(pooled_t * pooled_v) (fusion_method "mul") or of the sum, index i, with the fp16 hi / lo operand copy
    and the bf16 copy; backward accumulates the masked gradient into da / db."""
    n = 64 * 1024
    gen = _gen("fuse", mul)
    p = 0.1
    site = dropout_site_id("dropout.pooled")
    lib = L.lib()
    a, b = torch.randn(n, device=DEV, generator=gen), torch.randn(n, device=DEV, generator=gen)
    step_t = _step_tensor(STEP)
    drop = _desc(step_t, site, p)
    o32, hi, lo, b16 = (torch.empty(n, device=DEV), torch.empty(n, device=DEV, dtype=F16), torch.empty(n, device=DEV, dtype=F16),
                        torch.empty(n, device=DEV, dtype=BF))
    L.check(lib.vb_fuse_pooled_fwd(a.data_ptr(), b.data_ptr(), o32.data_ptr(), hi.data_ptr(), n, mul, C.byref(drop), 1, lo.data_ptr(),
                                   b16.data_ptr(), _st()))
    d = torch.randn(n, device=DEV, generator=gen)
    da0, db0 = torch.randn(n, device=DEV, generator=gen), torch.randn(n, device=DEV, generator=gen)
    da, db = da0.clone(), db0.clone()
    L.check(lib.vb_fuse_pooled_bwd(d.data_ptr(), a.data_ptr(), b.data_ptr(), da.data_ptr(), db.data_ptr(), n, mul, C.byref(drop), _st()))
    torch.cuda.synchronize()
    f = R.keep_factor(site, STEP, p, R.flat_index(n, DEV))
    drop_m = f == 0
    assert (o32[drop_m] == 0).all() and torch.equal(da[drop_m], da0[drop_m]) and torch.equal(db[drop_m], db0[drop_m])
    assert torch.equal(hi, o32.half()) and torch.equal(lo, (o32 - hi.float()).half()) and torch.equal(b16, o32.to(BF))

    def err(ff):
        f64 = ff.to(F64)
        v = (a.to(F64) * b.to(F64) if mul else a.to(F64) + b.to(F64)) * f64
        g = d.to(F64) * f64
        return dict(out=relmax(o32, v), da=relmax(da - da0, g * (b.to(F64) if mul else 1)), db=relmax(db - db0, g * (a.to(F64) if mul else 1)))

    wrongs = {"step+1": err(R.keep_factor(site, STEP + 1, p, R.flat_index(n, DEV)))}
    verdict(f"fuse_pooled mul={mul}", err(f), dict(out=1e-6, da=1e-6, db=1e-6), wrongs, drop_m.double().mean().item(), p)


# ============================================================================================ single-stream embeddings
def test_concat_embed_ln_dropout():
    """BaseBertForVLTasks' embeddings at the baseline's shapes (B = 64, 36 tokens, 101 regions, H = 768): each modality's LayerNorm
    and dropout (drop_t / drop_v, index = row within the modality * H + col), interleaved into one stream; the backward's dgamma /
    dbeta of both LayerNorms and the image column sum of dx (dcol_v: the region GEMM's bias, dcol_v2: token-type row 1)."""
    B, Nt, Nv, H = 64, 36, 101, 768
    gen = _gen("concat")
    p = 0.1
    st_, sv = dropout_site_id("bert.embeddings.dropout"), dropout_site_id("bert.v_embeddings.dropout")
    lib = L.lib()
    xt, xv = torch.randn(B * Nt, H, device=DEV, generator=gen), torch.randn(B * Nv, H, device=DEV, generator=gen)
    trow = torch.randn(H, device=DEV, generator=gen)
    gt, bt, gv, bv = (torch.randn(H, device=DEV, generator=gen) for _ in range(4))
    step_t = _step_tensor(STEP)
    dt_, dv_ = _desc(step_t, st_, p), _desc(step_t, sv, p)
    rows = B * (Nt + Nv)
    y32, y16 = torch.empty(rows, H, device=DEV), torch.empty(rows, H, device=DEV, dtype=F16)
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    L.check(lib.vb_concat_embed_ln_fwd(xt.data_ptr(), xv.data_ptr(), trow.data_ptr(), gt.data_ptr(), bt.data_ptr(), gv.data_ptr(), bv.data_ptr(),
                                       y32.data_ptr(), y16.data_ptr(), None, None, 1, mean.data_ptr(), rstd.data_ptr(), B, Nt, Nv, H,
                                       C.byref(dt_), C.byref(dv_), _st()))
    dy = torch.randn(rows, H, device=DEV, generator=gen)
    dxt, dxv, dxv16 = torch.empty(B * Nt, H, device=DEV), torch.empty(B * Nv, H, device=DEV), torch.empty(B * Nv, H, device=DEV, dtype=BF)
    names = ("dgamma_t", "dbeta_t", "dgamma_v", "dbeta_v", "dcol_v", "dcol_v2")
    base = {k: torch.randn(H, device=DEV, generator=gen) for k in names}
    acc = {k: v.clone() for k, v in base.items()}
    L.check(lib.vb_concat_embed_ln_bwd(dy.data_ptr(), xt.data_ptr(), xv.data_ptr(), trow.data_ptr(), gt.data_ptr(), gv.data_ptr(), mean.data_ptr(),
                                       rstd.data_ptr(), dxt.data_ptr(), dxv.data_ptr(), dxv16.data_ptr(), *(acc[k].data_ptr() for k in names),
                                       B, Nt, Nv, H, C.byref(dt_), C.byref(dv_), _st()))
    torch.cuda.synchronize()
    idx, text = R.concat_index(B, Nt, Nv, H, DEV)
    text_rows = text.reshape(rows)

    def factors(step, index):
        return torch.where(text[..., None], R.keep_factor(st_, step, p, index), R.keep_factor(sv, step, p, index)).reshape(rows, H)

    f = factors(STEP, idx)
    drop_m = f == 0
    assert (y32[drop_m] == 0).all() and torch.equal(y16, y32.half())
    xs = torch.empty(rows, H, device=DEV, dtype=F64)                 # the stream's pre-LayerNorm rows
    xs.view(B, Nt + Nv, H)[:, :Nt] = xt.to(F64).view(B, Nt, H)
    xs.view(B, Nt + Nv, H)[:, Nt:] = (xv.to(F64) + trow.to(F64)).view(B, Nv, H)
    gam = torch.where(text_rows[:, None], gt.to(F64), gv.to(F64))
    bet = torch.where(text_rows[:, None], bt.to(F64), bv.to(F64))
    y, _, _ = _ln64(xs, torch.ones(H, device=DEV), torch.zeros(H, device=DEV))
    y = y * gam + bet

    def err(ff):
        u = dy.to(F64) * ff.to(F64)
        xh = _ln_bwd64(xs, torch.ones(H, device=DEV), u)[1]
        gg = u * gam
        rs = 1.0 / torch.sqrt(((xs - xs.mean(-1, keepdim=True)) ** 2).mean(-1, keepdim=True) + 1e-12)
        dx = rs * (gg - gg.mean(-1, keepdim=True) - xh * (gg * xh).mean(-1, keepdim=True))
        t_, v_ = text_rows, ~text_rows
        dxv_ref = dx.view(B, Nt + Nv, H)[:, Nt:].reshape(B * Nv, H)
        return dict(y=relmax(y32, y * ff.to(F64)), dxt=relmax(dxt, dx.view(B, Nt + Nv, H)[:, :Nt].reshape(B * Nt, H)), dxv=relmax(dxv, dxv_ref),
                    dxv16=relmax(dxv16, dxv_ref),
                    dgamma_t=colsum_err(acc["dgamma_t"], base["dgamma_t"], (u * xh)[t_]), dbeta_t=colsum_err(acc["dbeta_t"], base["dbeta_t"], u[t_]),
                    dgamma_v=colsum_err(acc["dgamma_v"], base["dgamma_v"], (u * xh)[v_]), dbeta_v=colsum_err(acc["dbeta_v"], base["dbeta_v"], u[v_]),
                    dcol_v=colsum_err(acc["dcol_v"], base["dcol_v"], dxv_ref), dcol_v2=colsum_err(acc["dcol_v2"], base["dcol_v2"], dxv_ref))

    stream_idx = R.rowmajor_index(rows, H, DEV).view(B, Nt + Nv, H)   # the index a kernel would use if it numbered stream rows
    wrongs = {"step+1": err(factors(STEP + 1, idx)), "stream row": err(factors(STEP, stream_idx))}
    tols = dict(y=1e-5, dxt=1e-5, dxv=1e-5, dxv16=5e-3, dgamma_t=2e-5, dbeta_t=2e-5, dgamma_v=2e-5, dbeta_v=2e-5, dcol_v=2e-5, dcol_v2=2e-5)
    verdict("concat_embed_ln 64x(36+101)x768", err(f), tols, wrongs, drop_m.double().mean().item(), p)
