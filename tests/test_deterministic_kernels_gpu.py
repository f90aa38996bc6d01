"""The deterministic (_det) entry points and the split-K partials epilogue of vb_gemm_bf16 against float64 references at the
engine's shapes: ragged rows and columns, dropout masks applied explicitly (tests/_train_ref.py), the NaN conventions of the
losses, accumulation into non-zero buffers, and split-K partials through both the vectorised and the ragged (N % 4 != 0) epilogue.
Where a _det variant shares its non-reduced outputs with the default kernel (dx of the LayerNorm and small-linear backward, the
loss gradients), those are asserted bitwise equal to the default kernel's. A column sum is bounded per column by
c * sum_m |term_m| (a sum may cancel to about 0)."""
import ctypes as C

import pytest
import torch

import _train_ref as R
from vilbert_b200 import _lib as L
from vilbert_b200.engine import dropout_site_id

pytestmark = pytest.mark.gpu
BF, F64 = torch.bfloat16, torch.float64
DEV = "cuda"
STEP = 4242
TOL = 2e-5          # fp32 sums of up to a few thousand terms, relative to sum |term|


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else t.data_ptr()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ws(n):
    return torch.full((n,), float("nan"), device=DEV)     # a slice the kernel forgot to write would poison the sum


def colsum_err(got, base, terms):
    """max over columns of |(got - base) - sum_m terms[m, :]| / sum_m |terms[m, :]|  (terms [M, ...])."""
    terms = terms.to(F64).reshape(terms.shape[0], -1)
    s, a = terms.sum(0), terms.abs().sum(0)
    return ((got.to(F64).flatten() - base.to(F64).flatten() - s).abs() / a.clamp_min(1e-30)).max().item()


def _dropout(site, p):
    step_t = torch.tensor([STEP], dtype=torch.int32, device=DEV)
    d = L.Dropout()
    d.step, d.site, d.p = step_t.data_ptr(), site, p
    return d, step_t


def _keep(site, p, rows, cols):
    return R.keep_factor(site, STEP, p, R.rowmajor_index(rows, cols, device=DEV)).to(F64)


# ============================================================================================ ordered sum
def test_reduce_slices_is_the_ordered_fp32_sum():
    S, n, stride = 37, 1001, 1024
    ws = torch.randn(S, stride, device=DEV, generator=_gen(1)) * torch.logspace(-3, 3, S, device=DEV)[:, None]
    dst = torch.randn(n, device=DEV, generator=_gen(2))
    ref = torch.zeros(n, device=DEV)
    for k in range(S):      # fp32 adds in slice order, as the kernel does
        ref = ref + ws[k, :n]
    ref = dst + ref
    L.check(L.lib().vb_reduce_slices(ws.data_ptr(), stride, S, n, dst.data_ptr(), _st()))
    torch.cuda.synchronize()
    assert torch.equal(dst, ref)


# ============================================================================================ column sums
@pytest.mark.parametrize("M,N,ld,bf16", [(6400, 768, 2304, True), (6401, 1001, 1008, False), (64, 3129, 3129, False), (37, 5, 8, True)])
def test_colsum_det(M, N, ld, bf16):
    X = torch.randn(M, ld, device=DEV, generator=_gen(M + N))
    X = X.to(BF) if bf16 else X
    base = torch.randn(N, device=DEV, generator=_gen(3))
    out, ws = base.clone(), _ws(L.VB_DET_SLICES * N)
    L.check(L.lib().vb_colsum_det(X.data_ptr(), int(bf16), ld, out.data_ptr(), M, N, ws.data_ptr(), _st()))
    torch.cuda.synchronize()
    assert colsum_err(out, base, X[:, :N]) < TOL


# ============================================================================================ LayerNorm backward
LN_OUT_SITE, LN_IN_SITE = dropout_site_id("bert.embeddings.dropout"), dropout_site_id("bert.encoder.layer.0.output.dropout")


@pytest.mark.parametrize("M,H,mode", [(6400, 768, "out_drop"), (2368, 1024, "in_drop_pre_dbias"), (37 * 64, 1024, "dy2"),
                                      (37, 768, "plain")])
def test_layernorm_bwd_det(M, H, mode):
    lib, g = L.lib(), _gen(M + H)
    x = torch.randn(M, H, device=DEV, generator=g) * 2 + 0.5
    dy = torch.randn(M, H, device=DEV, generator=g)
    dy2 = torch.randn(M, H, device=DEV, generator=g) if mode == "dy2" else None
    gm = torch.rand(H, device=DEV, generator=g) + 0.5
    mean = x.mean(1)
    rstd = (x.var(1, unbiased=False) + 1e-12).rsqrt()
    pre = (torch.rand(M, H, device=DEV, generator=g) + 0.1).to(BF) if mode == "in_drop_pre_dbias" else None
    p = 0.1
    od, _s1 = _dropout(LN_OUT_SITE, p) if mode == "out_drop" else (None, None)
    idr, _s2 = _dropout(LN_IN_SITE, p) if mode == "in_drop_pre_dbias" else (None, None)
    bases = [torch.randn(H, device=DEV, generator=g) for _ in range(3)]
    want_bias = pre is not None

    def run(det):
        dx32 = torch.empty(M, H, device=DEV)
        dx16 = torch.empty(M, H, device=DEV, dtype=BF)
        dg, db, dbias = (b.clone() for b in bases)
        args = (x.data_ptr(), H, gm.data_ptr(), mean.data_ptr(), rstd.data_ptr(), dx32.data_ptr(), dx16.data_ptr(), H, _p(pre), H,
                dg.data_ptr(), db.data_ptr(), dbias.data_ptr() if want_bias else None, M, H, L.arg(od), L.arg(idr))
        if det:
            ws = _ws(3 * L.VB_DET_LN_SLICES * H)
            L.check(lib.vb_layernorm_bwd_det(dy.data_ptr(), _p(dy2), H, *args, ws.data_ptr(), _st()))
        elif dy2 is not None:
            L.check(lib.vb_add_layernorm_bwd(dy.data_ptr(), dy2.data_ptr(), H, *args, _st()))
        else:
            L.check(lib.vb_layernorm_bwd(dy.data_ptr(), H, *args, _st()))
        torch.cuda.synchronize()
        return dx32, dx16, dg, db, dbias

    dx32, dx16, dg, db, dbias = run(True)
    dx32_d, dx16_d, *_ = run(False)
    assert torch.equal(dx32, dx32_d) and torch.equal(dx16, dx16_d)      # the per-row part is the default kernel's body
    # float64 reference with the masks applied explicitly
    d = dy.to(F64) + (dy2.to(F64) if dy2 is not None else 0)
    if od is not None:
        d = d * _keep(LN_OUT_SITE, p, M, H)
    xh = (x.to(F64) - mean.to(F64)[:, None]) * rstd.to(F64)[:, None]
    gg = d * gm.to(F64)
    o = (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True)) * rstd.to(F64)[:, None]
    assert (dx32.to(F64) - o).abs().max().item() < 1e-4 * o.abs().max().item()
    assert colsum_err(dg, bases[0], d * xh) < TOL
    assert colsum_err(db, bases[1], d) < TOL
    if want_bias:
        ob = o * pre.to(F64) * _keep(LN_IN_SITE, p, M, H)
        assert colsum_err(dbias, bases[2], ob) < 1e-4        # the kernel sums the fp32 product, the reference its float64 value
    else:
        assert torch.equal(dbias, bases[2])


# ============================================================================================ text embeddings
@pytest.mark.parametrize("B,Nt,H,has_task,types", [(64, 36, 768, False, "zero"), (64, 36, 768, True, "random"), (3, 9, 64, True, "random"),
                                                   (32, 60, 1024, False, "random")])
def test_embed_text_bwd_det(B, Nt, H, has_task, types):
    g = _gen(B * Nt + H)
    V, P, T, K = 500, Nt, 2, 20
    ids = torch.randint(0, 40, (B, Nt), device=DEV, generator=g)         # many repeats and padding ids (0)
    ids[:, 0] = 101
    tt = torch.zeros(B, Nt, dtype=torch.long, device=DEV) if types == "zero" else torch.randint(0, T, (B, Nt), device=DEV, generator=g)
    task = torch.randint(0, K, (B,), device=DEV, generator=g) if has_task else None
    No = Nt + int(has_task)
    dout = torch.randn(B * No, H, device=DEV, generator=g)
    tabs = [torch.randn(n, H, device=DEV, generator=g) for n in (V, P, T, K)]
    got = [t.clone() for t in tabs]
    L.check(L.lib().vb_embed_text_bwd_det(dout.data_ptr(), ids.data_ptr(), tt.data_ptr(), _p(task), *(t.data_ptr() for t in got),
                                          B, Nt, H, _st()))
    torch.cuda.synchronize()
    # reference: the rows of d(out) each table row receives, summed in float64 on the host
    d = dout.to(F64).cpu().view(B, No, H)
    tok = torch.cat([d[:, :1], d[:, 2:]], 1) if has_task else d
    keys = [ids.cpu(), torch.arange(Nt).expand(B, Nt), tt.cpu()]
    for t, (base, out, key) in enumerate(zip(tabs, got, keys)):
        s = torch.zeros(base.shape, dtype=F64).index_add_(0, key.reshape(-1), tok.reshape(-1, H))
        a = torch.zeros(base.shape, dtype=F64).index_add_(0, key.reshape(-1), tok.reshape(-1, H).abs())
        if t == 0:      # padding_idx = 0 takes no gradient
            s[0] = a[0] = 0
        err = ((out.to(F64).cpu() - base.to(F64).cpu() - s).abs() - TOL * a).max().item()
        assert err <= 1e-6, (t, err)
    if has_task:
        s = torch.zeros(K, H, dtype=F64).index_add_(0, task.cpu(), d[:, 1])
        assert (got[3].to(F64).cpu() - tabs[3].to(F64).cpu() - s).abs().max().item() < 1e-4
    else:
        assert torch.equal(got[3], tabs[3])


# ============================================================================================ box projection
@pytest.mark.parametrize("M,H", [(6400, 1024), (2331, 768), (37, 1024)])
def test_loc_proj_bwd_det(M, H):
    g = _gen(M + H)
    dy = torch.randn(M, H, device=DEV, generator=g)
    loc = torch.rand(M, 5, device=DEV, generator=g)
    bW, bb = torch.randn(H, 5, device=DEV, generator=g), torch.randn(H, device=DEV, generator=g)
    dW, db, ws = bW.clone(), bb.clone(), _ws(L.VB_DET_SLICES * 6 * H)
    L.check(L.lib().vb_loc_proj_bwd_det(dy.data_ptr(), loc.data_ptr(), dW.data_ptr(), db.data_ptr(), M, H, ws.data_ptr(), _st()))
    torch.cuda.synchronize()
    terms = dy.to(F64)[:, :, None] * loc.to(F64)[:, None, :]
    assert colsum_err(dW, bW, terms) < TOL
    assert colsum_err(db, bb, dy) < TOL


# ============================================================================================ small linears
SL_SITE = dropout_site_id("vil_prediction.logit_fc.2")


@pytest.mark.parametrize("M,K,N,drop", [(64, 1024, 3, True), (6400, 1024, 1, True), (37, 768, 2, False), (2368, 768, 1, False)])
def test_small_linear_bwd_det(M, K, N, drop):
    lib, g = L.lib(), _gen(M + K + N)
    dy = torch.randn(M, N, device=DEV, generator=g)
    x = torch.randn(M, K, device=DEV, generator=g)
    W = torch.randn(N, K, device=DEV, generator=g)
    p = 0.5
    dd, _s = _dropout(SL_SITE, p) if drop else (None, None)
    bW, bb, bx = torch.randn(N, K, device=DEV, generator=g), torch.randn(N, device=DEV, generator=g), torch.randn(M, K, device=DEV, generator=g)

    def run(det):
        ws = _ws(L.VB_DET_SLICES * (N * K + N))
        dW, db, dx = bW.clone(), bb.clone(), bx.clone()
        args = (dy.data_ptr(), x.data_ptr(), K, W.data_ptr(), dx.data_ptr(), K, 1, dW.data_ptr(), db.data_ptr(), M, K, N, L.arg(dd))
        L.check(lib.vb_small_linear_bwd_det(*args, ws.data_ptr(), _st()) if det else lib.vb_small_linear_bwd(*args, _st()))
        torch.cuda.synchronize()
        return dW, db, dx

    dW, db, dx = run(True)
    _, _, dx_default = run(False)
    assert torch.equal(dx, dx_default)       # the input gradient is the default kernel's
    keep = _keep(SL_SITE, p, M, K) if drop else torch.ones(M, K, dtype=F64, device=DEV)
    xd = x.to(F64) * keep
    assert colsum_err(dW, bW, dy.to(F64)[:, :, None] * xd[:, None, :]) < TOL
    assert colsum_err(db, bb, dy) < TOL
    ref_dx = (dy.to(F64) @ W.to(F64)) * keep
    assert (dx.to(F64) - bx.to(F64) - ref_dx).abs().max().item() < 1e-5 * ref_dx.abs().max().item()


# ============================================================================================ losses
@pytest.mark.parametrize("rows,cols,frac,acc", [(2368, 30522, 0.15, 0), (64, 3129, 1.0, 1), (512, 2, 0.0, 0)])
def test_ce_loss_det(rows, cols, frac, acc):
    lib, g = L.lib(), _gen(rows + cols)
    z = torch.randn(rows, cols, device=DEV, generator=g) * 3
    lab = torch.randint(0, cols, (rows,), device=DEV, generator=g)
    lab[torch.rand(rows, device=DEV, generator=g) >= frac] = -1

    def run(det):
        loss = torch.full((1,), 0.75, device=DEV)
        ws = _ws(L.VB_DET_LOSS_SLICES)
        d16 = torch.empty(rows, cols, device=DEV, dtype=BF)
        args = (z.data_ptr(), cols, lab.data_ptr(), -1, loss.data_ptr(), None, 0, d16.data_ptr(), cols, rows, cols, 1.0, acc)
        L.check((lib.vb_ce_loss_det(*args, ws.data_ptr(), _st())) if det else lib.vb_ce_loss(*args, _st()))
        torch.cuda.synchronize()
        return loss, d16

    loss, d16 = run(True)
    _, d16_default = run(False)
    assert torch.equal(d16, d16_default)
    base = 0.75 if acc else 0.0
    if frac == 0.0:     # mean over no rows = nan (torch)
        assert torch.isnan(loss).all()
        return
    ref = torch.nn.functional.cross_entropy(z.to(F64), lab, ignore_index=-1)
    assert abs(loss.item() - base - ref.item()) < 1e-5 * abs(ref.item())


@pytest.mark.parametrize("B,Nv,C,none", [(64, 37, 1601, False), (8, 101, 1601, False), (4, 11, 21, True)])
def test_kl_masked_loss_det(B, Nv, C, none):
    lib, g = L.lib(), _gen(B + Nv + C)
    s = torch.randn(B * Nv, C, device=DEV, generator=g)
    t = torch.softmax(torch.randn(B, Nv - 1, C, device=DEV, generator=g), -1)
    lab = torch.full((B, Nv - 1), -1, dtype=torch.long, device=DEV)
    if not none:
        lab[torch.rand(B, Nv - 1, device=DEV, generator=g) < 0.15] = 1
        lab[:, 0] = 1

    def run(det):
        loss = torch.zeros(1, device=DEV)
        ws = _ws(L.VB_DET_LOSS_SLICES)
        d16 = torch.empty(B * Nv, C, device=DEV, dtype=BF)
        args = (s.data_ptr(), t.data_ptr(), lab.data_ptr(), loss.data_ptr(), None, d16.data_ptr(), C, B, Nv, C, 1.0, 0)
        L.check((lib.vb_kl_masked_loss_det(*args, ws.data_ptr(), _st())) if det else lib.vb_kl_masked_loss(*args, _st()))
        torch.cuda.synchronize()
        return loss, d16

    loss, d16 = run(True)
    assert torch.equal(d16, run(False)[1])
    if none:        # 0 / max(0, 0) in the reference
        assert torch.isnan(loss).all()
        return
    lp = torch.log_softmax(s.to(F64).view(B, Nv, C)[:, 1:], -1)
    tt = t.to(F64)
    kl = torch.where(tt > 0, tt * (tt.log() - lp), torch.zeros_like(tt)).sum(-1)
    m = (lab == 1).to(F64)
    ref = (kl * m).sum() / m.sum()
    assert abs(loss.item() - ref.item()) < 1e-5 * abs(ref.item())


@pytest.mark.parametrize("rows,cols", [(64, 3129), (3, 1533)])
def test_bce_logits_loss_det(rows, cols):
    lib, g = L.lib(), _gen(rows + cols)
    z = torch.randn(rows, cols, device=DEV, generator=g) * 3
    t = (torch.rand(rows, cols, device=DEV, generator=g) < 0.01).float()

    def run(det):
        loss = torch.full((1,), 5.0, device=DEV)
        ws = _ws(L.VB_DET_LOSS_SLICES)
        dz = torch.empty(rows, cols, device=DEV)
        args = (z.data_ptr(), t.data_ptr(), loss.data_ptr(), dz.data_ptr(), None, 0, rows, cols, 1.0)
        L.check((lib.vb_bce_logits_loss_det(*args, ws.data_ptr(), _st())) if det else lib.vb_bce_logits_loss(*args, _st()))
        torch.cuda.synchronize()
        return loss, dz

    loss, dz = run(True)
    assert torch.equal(dz, run(False)[1])
    ref = torch.nn.functional.binary_cross_entropy_with_logits(z.to(F64), t.to(F64)) * cols
    assert abs(loss.item() - ref.item()) < 1e-5 * ref.item()


# ============================================================================================ split-K partials of the GEMM
def _wgrad_args(M, N, K, ldb, g):
    """dW[M, N] = dy^T x with dy [K, M] (lda = M) and x [K, ldb] (its first N columns), both MN-major: the engine's wgrad."""
    dy = (torch.randn(K, M, device=DEV, generator=g) * 0.5).to(BF)
    x = (torch.randn(K, ldb, device=DEV, generator=g) * 0.5).to(BF)
    a = L.GemmArgs()
    a.M, a.N, a.K = M, N, K
    a.A, a.lda, a.a_mn_major = dy.data_ptr(), M, 1
    a.B, a.ldb, a.b_mn_major = x.data_ptr(), ldb, 1
    a.alpha, a.ld_out_f32, a.atomic_out, a.split_k = 1.0, N, L.VB_GEMM_PARTIALS, 0
    return a, dy, x


@pytest.mark.parametrize("M,N,K,ldb", [(768, 768, 6400, 768), (264, 770, 8192, 776), (1024, 3072, 2368, 3072), (64, 5, 4096, 8)])
def test_gemm_split_k_partials(M, N, K, ldb):
    lib, g = L.lib(), _gen(M + N + K)
    a, dy, x = _wgrad_args(M, N, K, ldb, g)
    bn, sp = C.c_int32(), C.c_int32()
    L.check(lib.vb_gemm_plan(C.byref(a), 0, C.byref(bn), C.byref(sp)))
    S = sp.value
    ws = _ws(S * M * N)
    base = torch.randn(M, N, device=DEV, generator=g)
    out = base.clone()
    a.out_f32, a.split_k = ws.data_ptr(), S
    L.check(lib.vb_gemm_bf16(C.byref(a), _st()))
    L.check(lib.vb_reduce_slices(ws.data_ptr(), M * N, S, M * N, out.data_ptr(), _st()))
    torch.cuda.synchronize()
    A, X = dy.to(F64), x[:, :N].to(F64)
    s, mag = A.t() @ X, A.abs().t() @ X.abs()            # sum over k of the terms, and of their magnitudes
    assert ((out.to(F64) - base.to(F64) - s).abs() / mag.clamp_min(1e-30)).max().item() < TOL
    if M >= 256 and N >= 256:
        assert S > 1, "the case should split K"
    # the partials mode takes a plain epilogue only
    bias = torch.zeros(N + 3, device=DEV)
    a.bias = bias.data_ptr()
    assert lib.vb_gemm_bf16(C.byref(a), _st()) != 0
