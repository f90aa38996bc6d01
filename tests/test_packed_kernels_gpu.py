"""The packed-row kernels against independent references: varlen attention (vb_attention_fwd / _bwd with q_off / q_len / k_off /
k_len) against float64 attention of the padded samples, the row-indexed dropout sites under a row map (vb_dropout.row_map) against
explicit-mask float64 references, and the pack, unpack and compaction kernels against plain torch, exactly.

The method is that of tests/test_train_kernels_gpu.py: masks come from tests/_train_ref.py at the indices tests/_packed_ref.py
gives, dropped elements are asserted exactly, accumulated outputs start from a non-zero buffer, a bias sum is bounded per column by
c * sum_m |term_m|, and every case recomputes its reference with a plausible wrong mask or map that must miss by more than 10x the
tolerance. Rows of no sample are filled with a sentinel before a call and asserted bitwise untouched after it."""
import ctypes as C
import math

import pytest
import torch

import _packed_ref as P
import _train_ref as R
from test_train_kernels_gpu import (ATT_P, ATT_SITE, ATT_TOL, EMB_SITE, LN_SITE, LN_TOL, STEP, _attn_ref, _gen, _ln64, _ln_bwd64,
                                    _st, _step_tensor, colsum_err, relmax)
from vilbert_b200 import _lib as L
from vilbert_b200.engine import PACKED_MASKED_LOGIT, dropout_site_id, pack_capacity

pytestmark = pytest.mark.gpu
BF, F16, F64, I32, I64 = torch.bfloat16, torch.float16, torch.float64, torch.int32, torch.int64
DEV = "cuda"
SENT = 7.0          # sentinel of the rows a kernel must not write (exact in every 16-bit format)
TAIL = 8            # rows of no sample behind a varlen attention batch


def _ptr(t):
    return None if t is None else t.data_ptr()


def _mdesc(step_t, site, p, row_map):
    d = L.Dropout()
    d.step, d.site, d.p, d.row_map = step_t.data_ptr(), site, p, _ptr(row_map)
    return d


def verdict(case, errs, tols, wrongs, dropped_frac=None, p=None):
    """As test_train_kernels_gpu.verdict: one line per case (error / tolerance, each wrong reference's error, peak memory), then
    the assertions."""
    w = "  ".join(f"{lab}:" + ",".join(f"{k}={v:.2e}" for k, v in we.items()) for lab, we in wrongs.items())
    e = ",".join(f"{k}={v:.2e}/{tols[k]:.0e}" for k, v in errs.items())
    print(f"\n[packed-kernels] {case} | err/tol {e} | wrong {w}" + (f" | dropped {dropped_frac:.4f} p={p}" if p else "")
          + f" | peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    for k, v in errs.items():
        assert v <= tols[k], (case, k, v, tols[k])
    for lab, we in wrongs.items():
        for k, v in we.items():
            assert v > 10 * tols[k], (case, lab, k, v, tols[k])
    if p is not None:
        assert abs(dropped_frac - p) < 0.05, (case, dropped_frac, p)


def _untouched(t, rows_from=None, where=None):
    """t (from row rows_from on, or at the bool `where`) still holds the sentinel, bitwise."""
    v = t[rows_from:] if where is None else t[where]
    return torch.equal(v, torch.full_like(v, SENT))


# ============================================================================================ varlen attention
def _lengths(B, N, gen, short=False):
    """Per-sample lengths in [1, N]: 1, N, N - 1, and ends inside a 16-row tile and a 64-key block (17, 63, 65) first, the rest
    random (in [1, min(N, 40)] when short: a batch whose padded maximum is far above most samples)."""
    lens = torch.randint(1, (min(N, 40) if short else N) + 1, (B,), device=DEV, generator=gen)
    for i, v in enumerate([1, N, N - 1, 17, 63, 65][:B]):
        lens[i] = max(1, min(v, N))
    return lens


def _layout(lens, N, extra):
    mask = (torch.arange(N, device=DEV)[None] < lens[:, None]).long()
    count = int(lens.sum())
    off, ln, mp = P.pack_layout(mask, 0, count + extra)
    return off.to(DEV), ln.to(DEV), mp.to(DEV), count


def _pad(x, mp, B, N):
    """Packed rows -> padded [B*N, C] float64 (zero rows where no packed row lands)."""
    out = torch.zeros(B * N, x.shape[1], dtype=F64, device=DEV)
    v = mp >= 0
    out[mp[v].long()] = x[:mp.numel()][v].to(F64)
    return out


class _Varlen:
    """One varlen attention problem: packed Q / K / V (self: one [R, 3*H*D] buffer; cross: a query and a key buffer), TAIL rows of
    no sample behind each, and the float64 reference of the padded samples."""

    def __init__(self, B, H, Nq, Nk, D, cross, mode, p, short=False):
        assert cross or Nq == Nk
        gen = _gen("varlen", B, H, Nq, Nk, D, cross, mode, p, short)
        self.B, self.H, self.Nq, self.Nk, self.D, self.cross, self.mode, self.p = B, H, Nq, Nk, D, cross, mode, p
        Hd = self.Hd = H * D
        lq = _lengths(B, Nq, gen, short)
        if cross:
            lk = _lengths(B, Nk, gen, short)
            lk[1:] = lk[1:].roll(2)
            lq[0] = Nq                                 # the single-key sample (k_len[0] = 1) has every query
        else:
            lk = lq
        self.lq, self.lk = lq, lk
        self.oq, self.lq32, self.mq, self.cq = _layout(lq, Nq, TAIL)
        self.ok, self.lk32, self.mk, self.ck = _layout(lk, Nk, TAIL) if cross else (self.oq, self.lq32, self.mq, self.cq)
        self.Rq, self.Rk = self.mq.numel(), self.mk.numel()
        dt = BF if mode == "bf16" else F16
        xq32 = torch.randn(self.Rq, 3 * Hd, device=DEV, generator=gen)
        xk32 = torch.randn(self.Rk, 3 * Hd, device=DEV, generator=gen) if cross else xq32
        xq, xk = xq32.to(dt), xk32.to(dt)
        self.t = dict(q32=xq32[:, :Hd], k32=xk32[:, Hd:2 * Hd], v32=xk32[:, 2 * Hd:], q=xq[:, :Hd], k=xk[:, Hd:2 * Hd], v=xk[:, 2 * Hd:])
        if mode == "split":
            lq_, lk_ = (xq32 - xq.float()).half(), (xk32 - xk.float()).half()
            self.t.update(qlo=lq_[:, :Hd], klo=lk_[:, Hd:2 * Hd], vlo=lk_[:, 2 * Hd:])
        self.dO = torch.randn(self.Rq, Hd, device=DEV, generator=gen).to(BF)
        self.base = {k: torch.randn(Hd, device=DEV, generator=gen) for k in ("q", "k", "v")}
        self.step_t = _step_tensor(STEP)
        # additive key mask of the padded reference: -inf past k_len
        self.kmask = torch.where(torch.arange(Nk, device=DEV)[None] < lk[:, None], 0.0, float("-inf")).to(F64)

    def args(self):
        a = L.AttnArgs()
        a.B, a.H, a.Nq, a.Nk, a.D, a.scale = self.B, self.H, self.Nq, self.Nk, self.D, 1.0 / math.sqrt(self.D)
        ld = 3 * self.Hd
        a.Q, a.ldq, a.K, a.ldk, a.V, a.ldv = self.t["q"].data_ptr(), ld, self.t["k"].data_ptr(), ld, self.t["v"].data_ptr(), ld
        a.qkv_fp16 = int(self.mode != "bf16")
        a.q_off, a.q_len, a.k_off, a.k_len = self.oq.data_ptr(), self.lq32.data_ptr(), self.ok.data_ptr(), self.lk32.data_ptr()
        if self.p:
            a.dropout.step, a.dropout.site, a.dropout.p = self.step_t.data_ptr(), ATT_SITE, self.p
        return a

    def forward(self):
        a = self.args()
        Hd = self.Hd
        odt = BF if self.mode == "bf16" else F16
        self.O = torch.full((self.Rq, Hd), SENT, device=DEV, dtype=odt)
        self.Ob = torch.full((self.Rq, Hd), SENT, device=DEV, dtype=BF) if self.mode != "bf16" else None
        self.Olo = torch.full((self.Rq, Hd), SENT, device=DEV, dtype=F16) if self.mode == "split" else None
        self.lse = torch.full((self.B, self.H, self.Nq), SENT, device=DEV)
        a.O, a.ldo, a.O_b16, a.O_lo, a.lse = self.O.data_ptr(), Hd, _ptr(self.Ob), _ptr(self.Olo), self.lse.data_ptr()
        if self.mode == "split":
            a.Q_lo, a.K_lo, a.V_lo = self.t["qlo"].data_ptr(), self.t["klo"].data_ptr(), self.t["vlo"].data_ptr()
        L.check(L.lib().vb_attention_fwd(C.byref(a), _st()), "vb_attention_fwd")

    def backward(self, dq=True, dkv=True):
        """One backward into fresh sentinel-filled buffers: {"dQ"/"dK"/"dV": gradient, "db_*": bias sums, "delta", "bufs"}."""
        a = self.args()
        Hd, ld = self.Hd, 3 * self.Hd
        a.O, a.ldo, a.O_b16, a.lse = self.O.data_ptr(), Hd, _ptr(self.Ob), self.lse.data_ptr()
        a.dO, a.lddo = self.dO.data_ptr(), Hd
        delta = torch.full((self.B, self.H, self.Nq), SENT, device=DEV)
        bq = torch.full((self.Rq, ld), SENT, device=DEV, dtype=BF)
        bk = torch.full((self.Rk, ld), SENT, device=DEV, dtype=BF) if self.cross else bq
        db = {k: v.clone() for k, v in self.base.items()}
        a.delta = delta.data_ptr()
        a.lddq, a.lddk, a.lddv = ld, ld, ld
        # every bias sum is passed: a partial backward ignores the sums of the side it does not compute
        a.dbias_q, a.dbias_k, a.dbias_v = db["q"].data_ptr(), db["k"].data_ptr(), db["v"].data_ptr()
        if dq:
            a.dQ = bq[:, :Hd].data_ptr()
        if dkv:
            a.dK, a.dV = bk[:, Hd:2 * Hd].data_ptr(), bk[:, 2 * Hd:].data_ptr()
        L.check(L.lib().vb_attention_bwd(C.byref(a), _st()), "vb_attention_bwd")
        torch.cuda.synchronize()
        return dict(dQ=bq[:, :Hd], dK=bk[:, Hd:2 * Hd], dV=bk[:, 2 * Hd:], db=db, delta=delta, bufs=[bq] + ([bk] if self.cross else []))

    def factor(self, step=STEP, extent="padded"):
        idx, _ = P.packed_attn_index(self.lq, self.lk, self.H, self.Nq, self.Nk, extent, q_off=self.oq)
        return R.keep_factor(ATT_SITE, step, self.p, idx) if self.p else torch.ones(1, device=DEV)

    def reference(self, f, grads=True, split=False):
        """float64 O (and dQ / dK / dV) of the valid packed rows, the dropout factor f at padded coordinates."""
        B, H, Nq, Nk, D = self.B, self.H, self.Nq, self.Nk, self.D
        pq = lambda x: _pad(x, self.mq, B, Nq)
        pk = lambda x: _pad(x, self.mk, B, Nk)
        vq, vk = self.mq[self.mq >= 0].long(), self.mk[self.mk >= 0].long()
        f = f.expand(B, H, Nq, Nk) if f.numel() == 1 else f
        if split:
            o, _ = _attn_ref(pq(self.t["q32"]), pk(self.t["k32"]), pk(self.t["v32"]), self.kmask, f, None, B, H, Nq, Nk, D)
            return o[vq], None
        o, _ = _attn_ref(pq(self.t["q"]), pk(self.t["k"]), pk(self.t["v"]), self.kmask, f, None, B, H, Nq, Nk, D)
        if not grads:
            return o[vq], None
        # the backward contracts bf16 panels: its reference is the attention of the bf16-rounded inputs; queries past q_len have dO 0
        _, (gq, gk, gv) = _attn_ref(pq(self.t["q"].to(BF)), pk(self.t["k"].to(BF)), pk(self.t["v"].to(BF)), self.kmask, f,
                                    pq(self.dO), B, H, Nq, Nk, D)
        return o[vq], (gq[vq], gk[vk], gv[vk])

    def lse_err(self):
        B, H, Nq, Nk, D = self.B, self.H, self.Nq, self.Nk, self.D
        q = _pad(self.t["q"], self.mq, B, Nq).view(B, Nq, H, D).permute(0, 2, 1, 3)
        k = _pad(self.t["k"], self.mk, B, Nk).view(B, Nk, H, D).permute(0, 2, 3, 1)
        ref = torch.logsumexp(q @ k / math.sqrt(D) + self.kmask[:, None, None, :], -1)
        qv = (torch.arange(Nq, device=DEV)[None] < self.lq[:, None])[:, None, :].expand(B, H, Nq)
        return relmax((self.lse * math.log(2.0))[qv], ref[qv]), qv

    def name(self):
        return f"{self.mode} {self.B}x{self.H}x{self.Nq}x{self.Nk}x{self.D}{' cross' if self.cross else ''} p={self.p}"


# O tolerance of bf16 operands: P is a bf16 MMA operand and O is stored in bf16, each a 2^-9 relative rounding (the bf16 attention
# bound of tests/test_kernels_gpu.py is 2e-2); the gradients and lse keep ATT_TOL
BF16_O_TOL = 1e-2


def _grad_errs(v, got, ref):
    gq, gk, gv = ref
    e = {}
    if got.get("q"):
        e.update(dQ=relmax(got["dQ"][:v.cq], gq), dbias_q=colsum_err(got["db"]["q"], v.base["q"], gq))
    if got.get("kv"):
        e.update(dK=relmax(got["dK"][:v.ck], gk), dV=relmax(got["dV"][:v.ck], gv),
                 dbias_k=colsum_err(got["db"]["k"], v.base["k"], gk), dbias_v=colsum_err(got["db"]["v"], v.base["v"], gv))
    return e


def _tails_untouched(v, got):
    """Rows past off[B] of every output, and lse / delta past q_len at padded coordinates, still hold the sentinel."""
    _, qv = v.lse_err()
    ok = dict(O=_untouched(v.O, v.cq), lse=_untouched(v.lse, where=~qv))
    if v.Ob is not None:
        ok["O_b16"] = _untouched(v.Ob, v.cq)
    if v.Olo is not None:
        ok["O_lo"] = _untouched(v.Olo, v.cq)
    if got is not None:
        ok.update(dQ=_untouched(got["bufs"][0], v.cq), dKV=_untouched(got["bufs"][-1], v.ck), delta=_untouched(got["delta"], where=~qv))
    return ok


def _varlen_full(v):
    """Forward + full backward: errors, wrong-reference errors, dropped fraction on the valid pairs, single-key errors."""
    v.forward()
    got = dict(v.backward(), q=True, kv=True)
    tols = dict(ATT_TOL, O=BF16_O_TOL) if v.mode == "bf16" else ATT_TOL
    one = v.lk == 1
    qone = one[(v.mq[:v.cq] // v.Nq).long()]
    kone = one[(v.mk[:v.ck] // v.Nk).long()]

    def compare(f, keep_single=False):
        o, grads = v.reference(f)
        e = dict(O=relmax(v.O[:v.cq], o), **_grad_errs(v, got, grads))
        if keep_single:
            gq, gk, _ = grads
            e.update(dQ_1key=((got["dQ"][:v.cq].to(F64) - gq)[qone].abs().max() / gq.abs().max()).item(),
                     dK_1key=((got["dK"][:v.ck].to(F64) - gk)[kone].abs().max() / gk.abs().max()).item())
        return e

    f = v.factor()
    errs = compare(f, keep_single=True)
    errs["lse"] = v.lse_err()[0]
    wrongs = {}
    if v.p:
        wrongs = {"step+1": compare(v.factor(STEP + 1)), "per-sample extents": compare(v.factor(extent="sample")),
                  "packed rows": compare(v.factor(extent="packed"))}
        for w in wrongs.values():     # sum_k dS[q, k] = 0: the key bias gradient is 0 whatever the mask
            del w["dbias_k"]
    _, valid = P.packed_attn_index(v.lq, v.lk, v.H, v.Nq, v.Nk)
    dropped = (f.expand(v.B, v.H, v.Nq, v.Nk)[valid.expand(v.B, v.H, v.Nq, v.Nk)] == 0).double().mean().item() if v.p else None
    tails = _tails_untouched(v, got)
    assert all(tails.values()), (v.name(), tails)
    return errs, tols, wrongs, dropped


VARLEN_SHAPES = [
    # fused single-CTA backward (padded Nq, Nk <= 128, D >= 32): text self-attention (12 and 16 heads), vision self, co-attention
    (64, 12, 37, 37, 64, False), (64, 16, 37, 37, 64, False), (64, 12, 21, 21, 64, False), (64, 8, 101, 101, 128, False),
    (64, 8, 37, 101, 128, True), (64, 8, 101, 37, 128, True),
    # two-kernel backward: Nq or Nk > 128, or D == 16
    (32, 8, 200, 21, 128, True), (16, 8, 306, 257, 128, True), (16, 8, 257, 306, 128, True), (16, 12, 257, 257, 64, False),
    (16, 4, 37, 21, 16, True)]


@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", VARLEN_SHAPES)
def test_varlen_attention_fp16_dropout(B, H, Nq, Nk, D, cross):
    """The engine's default: fp16 Q / K / V / O with the bf16 copy O_b16, dropout on the probabilities at padded coordinates,
    dbias_q / k / v over the valid rows, the single-key sample's dQ / dK at 0, and no write past off[B] or past q_len."""
    v = _Varlen(B, H, Nq, Nk, D, cross, "fp16", ATT_P)
    errs, tols, wrongs, dropped = _varlen_full(v)
    verdict(f"varlen attention {v.name()}", errs, tols, wrongs, dropped, ATT_P)


def test_varlen_attention_long_padded_short_samples():
    """A padded maximum of 200 (two-kernel backward) while most samples hold at most 40 rows: most query tiles of the grid lie
    past their sample's rows."""
    v = _Varlen(64, 8, 200, 200, 128, False, "fp16", ATT_P, short=True)
    errs, tols, wrongs, dropped = _varlen_full(v)
    verdict(f"varlen attention short samples {v.name()}", errs, tols, wrongs, dropped, ATT_P)


@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", [(64, 12, 37, 37, 64, False), (64, 8, 37, 101, 128, True), (16, 8, 306, 257, 128, True),
                                               (16, 4, 37, 21, 16, True)])
def test_varlen_attention_bf16_dropout(B, H, Nq, Nk, D, cross):
    v = _Varlen(B, H, Nq, Nk, D, cross, "bf16", ATT_P)
    errs, tols, wrongs, dropped = _varlen_full(v)
    verdict(f"varlen attention {v.name()}", errs, tols, wrongs, dropped, ATT_P)


@pytest.mark.parametrize("p", [ATT_P, 0.0])
@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", [(64, 12, 37, 37, 64, False), (64, 8, 101, 37, 128, True), (16, 8, 257, 306, 128, True)])
def test_varlen_attention_partial_backward(B, H, Nq, Nk, D, cross, p):
    """dQ-only and dK / dV-only backwards (a frozen stream): bitwise what the full backward writes, their bias sums against the
    reference, and nothing written past off[B]."""
    v = _Varlen(B, H, Nq, Nk, D, cross, "fp16", p)
    v.forward()
    full = v.backward()
    only_q = dict(v.backward(dkv=False), q=True)
    only_kv = dict(v.backward(dq=False), kv=True)
    assert torch.equal(only_q["dQ"], full["dQ"]) and torch.equal(only_kv["dK"], full["dK"]) and torch.equal(only_kv["dV"], full["dV"])
    assert torch.equal(only_q["db"]["k"], v.base["k"]) and torch.equal(only_kv["db"]["q"], v.base["q"])   # the other side's sums untouched
    for got in (only_q, only_kv):
        tails = _tails_untouched(v, got)
        assert all(tails.values()), (v.name(), tails)

    def errs_of(f):
        _, grads = v.reference(f)
        return dict(_grad_errs(v, only_q, grads), **_grad_errs(v, only_kv, grads))

    wrongs = {}
    if p:
        wrongs = {"step+1": errs_of(v.factor(STEP + 1)), "per-sample extents": errs_of(v.factor(extent="sample"))}
        for w in wrongs.values():
            del w["dbias_k"]
    verdict(f"varlen attention partial backward {v.name()}", errs_of(v.factor()), ATT_TOL, wrongs)


@pytest.mark.parametrize("B,H,Nq,Nk,D,cross", [(8, 8, 306, 306, 128, False), (8, 8, 257, 306, 128, True), (64, 8, 101, 101, 128, False),
                                               (64, 12, 37, 37, 64, False)])
def test_varlen_attention_split_forward(B, H, Nq, Nk, D, cross):
    """Split precision (Q_lo / K_lo / V_lo, O_lo): O + O_lo against float64 attention of the fp32 inputs at the 2e-5 bound of
    tests/test_kernels_gpu.py. At Nk = 306 the hi + lo panels do not fit in shared memory and the keys stream in chunks
    (kchunk < nkp), so a sample's keys are split across chunks."""
    v = _Varlen(B, H, Nq, Nk, D, cross, "split", ATT_P)
    v.forward()
    torch.cuda.synchronize()
    o = v.O[:v.cq].double() + v.Olo[:v.cq].double()
    err = lambda f: dict(O_split=relmax(o, v.reference(f, split=True)[0]))
    tails = _tails_untouched(v, None)
    assert all(tails.values()), (v.name(), tails)
    wrongs = {"step+1": err(v.factor(STEP + 1)), "per-sample extents": err(v.factor(extent="sample")),
              "packed rows": err(v.factor(extent="packed"))}
    f = v.factor()
    _, valid = P.packed_attn_index(v.lq, v.lk, v.H, v.Nq, v.Nk)
    dropped = (f[valid.expand_as(f)] == 0).double().mean().item()
    verdict(f"varlen attention split fwd {v.name()}", err(f), dict(O_split=2e-5), wrongs, dropped, ATT_P)


# ============================================================================================ row-mapped dropout sites
B_ROWS = 64
STREAMS = {768: (36, 1), 1024: (101, 0)}       # H -> (padded rows per sample before the task token, has_task): text, image


def _row_layout(H, seed):
    """Ragged prefix masks of B_ROWS samples, the capacity engine.pack_capacity gives them and the packed layout: (map [rows],
    count, rows). The capacity always leaves rows of no sample behind off[B]."""
    n_in, has_task = STREAMS[H]
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, n_in + 1, (B_ROWS,), generator=g)
    lens[0], lens[1] = 1, n_in
    count = int(lens.sum()) + B_ROWS * has_task
    if pack_capacity(count, B_ROWS * (n_in + has_task)) == count:
        lens[1] -= 1
        count -= 1
    rows = pack_capacity(count, B_ROWS * (n_in + has_task))
    mask = (torch.arange(n_in)[None] < lens[:, None]).long()
    _, _, mp = P.pack_layout(mask, has_task, rows)
    return mp.to(DEV), count, rows


def _rows_in(M, H, count, gen, scale=1.0, shift=0.0):
    """[M, H] fp32 with rows of no sample (past count) at zero, as the engine leaves them."""
    x = torch.randn(M, H, device=DEV, generator=gen) * scale + shift
    x[count:] = 0
    return x


def _ln_bwd_call(det, dy, dy2, x, gm, mean, rstd, dx32, dx16, pre, acc, M, H, dout, din):
    """vb_layernorm_bwd, vb_add_layernorm_bwd (dy2) or vb_layernorm_bwd_det (det) on the given rows."""
    lib = L.lib()
    tail = (H, x.data_ptr(), H, gm.data_ptr(), mean.data_ptr(), rstd.data_ptr(), _ptr(dx32), _ptr(dx16), H, _ptr(pre), H,
            _ptr(acc.get("dgamma")), _ptr(acc.get("dbeta")), _ptr(acc.get("dbias")), M, H, dout, din)
    if det:
        ws = torch.empty(3 * 256 * H, device=DEV)
        L.check(lib.vb_layernorm_bwd_det(dy.data_ptr(), _ptr(dy2), *tail, ws.data_ptr(), _st()), "vb_layernorm_bwd_det")
    elif dy2 is not None:
        L.check(lib.vb_add_layernorm_bwd(dy.data_ptr(), dy2.data_ptr(), *tail, _st()), "vb_add_layernorm_bwd")
    else:
        L.check(lib.vb_layernorm_bwd(dy.data_ptr(), *tail, _st()), "vb_layernorm_bwd")


def _tail_sums_zero(det, count, rows, H, site, p, mp, step_t, dy, dy2, x, gm, mean, rstd, pre, names, which):
    """The same backward on the rows of no sample alone (pointers and map offset to row count), every sum starting at 0: the rows
    contribute exactly nothing."""
    acc = {k: torch.zeros(H, device=DEV) for k in names}
    d = _mdesc(step_t, site, p, mp[count:])
    sl = lambda t: None if t is None else t[count:]
    dx16 = torch.empty(rows - count, H, device=DEV, dtype=BF) if "dbias" in names else None
    _ln_bwd_call(det, sl(dy), sl(dy2), sl(x), gm, sl(mean), sl(rstd), None, dx16, sl(pre), acc, rows - count, H,
                 C.byref(d) if which == "out" else None, C.byref(d) if which == "in" else None)
    torch.cuda.synchronize()
    return all(bool((v == 0).all()) for v in acc.values())


@pytest.mark.parametrize("det", [0, 1])
@pytest.mark.parametrize("H", [768, 1024])
def test_row_map_layernorm_out_dropout(H, det):
    """The embeddings' dropout(LayerNorm(x)) on a packed stream: vb_layernorm_fwd with out_dropout and a row map, then
    vb_layernorm_bwd (det: vb_layernorm_bwd_det) masking dy first. Packed row r draws padded row map[r]'s mask."""
    mp, count, rows = _row_layout(H, H + 1)
    gen = _gen("map-lnout", H, det)
    p, lib = 0.1, L.lib()
    x = _rows_in(rows, H, count, gen, 2.0, 0.5)
    gm, bt = torch.randn(H, device=DEV, generator=gen), torch.randn(H, device=DEV, generator=gen)
    step_t = _step_tensor(STEP)
    drop = _mdesc(step_t, EMB_SITE, p, mp)
    y32, y16 = torch.full((rows, H), SENT, device=DEV), torch.full((rows, H), SENT, device=DEV, dtype=F16)
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    L.check(lib.vb_layernorm_fwd(x.data_ptr(), H, gm.data_ptr(), bt.data_ptr(), 1e-12, y32.data_ptr(), y16.data_ptr(), H, mean.data_ptr(),
                                 rstd.data_ptr(), rows, H, C.byref(drop), 1, None, None, _st()))
    dy = _rows_in(rows, H, count, gen)
    dx32 = torch.full((rows, H), SENT, device=DEV)
    base = {k: torch.randn(H, device=DEV, generator=gen) for k in ("dgamma", "dbeta")}
    acc = {k: v.clone() for k, v in base.items()}
    _ln_bwd_call(det, dy, None, x, gm, mean, rstd, dx32, None, None, acc, rows, H, C.byref(drop), None)
    torch.cuda.synchronize()
    assert torch.isfinite(y32).all() and torch.isfinite(dx32).all()
    assert _tail_sums_zero(det, count, rows, H, EMB_SITE, p, mp, step_t, dy, None, x, gm, mean, rstd, None, ("dgamma", "dbeta"), "out")
    v = slice(0, count)
    f = R.keep_factor(EMB_SITE, STEP, p, P.packed_index(mp, H))[v]
    drop_m = f == 0
    assert (y32[v][drop_m] == 0).all() and (y16[v][drop_m] == 0).all() and torch.equal(y16, y32.half())
    y, _, _ = _ln64(x[v], gm, bt)

    def err(ff):
        g = dy[v].to(F64) * ff.to(F64)
        dx, xh = _ln_bwd64(x[v], gm, g)
        return dict(y=relmax(y32[v], y * ff.to(F64)), dx32=relmax(dx32[v], dx), dgamma=colsum_err(acc["dgamma"], base["dgamma"], g * xh),
                    dbeta=colsum_err(acc["dbeta"], base["dbeta"], g))

    wrongs = {"identity map": err(R.keep_factor(EMB_SITE, STEP, p, R.rowmajor_index(rows, H, DEV))[v]),
              "step+1": err(R.keep_factor(EMB_SITE, STEP + 1, p, P.packed_index(mp, H))[v])}
    verdict(f"row map layernorm out_dropout {rows}x{H} det={det}", err(f), LN_TOL, wrongs, drop_m.double().mean().item(), p)


@pytest.mark.parametrize("det", [0, 1])
@pytest.mark.parametrize("H", [768, 1024])
def test_row_map_layernorm_in_dropout_gelu_pre_dbias(H, det):
    """vb_layernorm_bwd with in_dropout under a row map, gelu_pre and dbias: dx16 = dx * gelu'(pre) * mask and dbias += its
    column sums over the valid rows; dgamma / dbeta carry no mask."""
    mp, count, rows = _row_layout(H, H + 2)
    gen = _gen("map-lnin", H, det)
    p, lib = 0.1, L.lib()
    x = _rows_in(rows, H, count, gen)
    gm, bt = torch.randn(H, device=DEV, generator=gen), torch.randn(H, device=DEV, generator=gen)
    pre = (torch.rand(rows, H, device=DEV, generator=gen) * 1.2 - 0.1).to(BF)
    pre[count:] = 0
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    L.check(lib.vb_layernorm_fwd(x.data_ptr(), H, gm.data_ptr(), bt.data_ptr(), 1e-12, None, None, H, mean.data_ptr(), rstd.data_ptr(),
                                 rows, H, None, 0, None, None, _st()))
    step_t = _step_tensor(STEP)
    drop = _mdesc(step_t, LN_SITE, p, mp)
    dy = _rows_in(rows, H, count, gen)
    dx16 = torch.full((rows, H), SENT, device=DEV, dtype=BF)
    base = {k: torch.randn(H, device=DEV, generator=gen) for k in ("dgamma", "dbeta", "dbias")}
    acc = {k: v.clone() for k, v in base.items()}
    _ln_bwd_call(det, dy, None, x, gm, mean, rstd, None, dx16, pre, acc, rows, H, None, C.byref(drop))
    torch.cuda.synchronize()
    assert torch.isfinite(dx16.float()).all()
    assert _tail_sums_zero(det, count, rows, H, LN_SITE, p, mp, step_t, dy, None, x, gm, mean, rstd, pre, ("dgamma", "dbeta", "dbias"), "in")
    v = slice(0, count)
    f = R.keep_factor(LN_SITE, STEP, p, P.packed_index(mp, H))[v]
    assert (dx16[v][f == 0] == 0).all()
    dx, xh = _ln_bwd64(x[v], gm, dy[v])

    def err(ff):
        t = dx * pre[v].to(F64) * ff.to(F64)
        return dict(dx16=relmax(dx16[v], t), dbias=colsum_err(acc["dbias"], base["dbias"], t))

    errs = dict(err(f), dgamma=colsum_err(acc["dgamma"], base["dgamma"], dy[v].to(F64) * xh),
                dbeta=colsum_err(acc["dbeta"], base["dbeta"], dy[v]))
    wrongs = {"identity map": err(R.keep_factor(LN_SITE, STEP, p, R.rowmajor_index(rows, H, DEV))[v]),
              "step+1": err(R.keep_factor(LN_SITE, STEP + 1, p, P.packed_index(mp, H))[v])}
    verdict(f"row map layernorm in_dropout gelu_pre dbias {rows}x{H} det={det}", errs, LN_TOL, wrongs, (f == 0).double().mean().item(), p)


@pytest.mark.parametrize("det", [0, 1])
@pytest.mark.parametrize("H", [768, 1024])
def test_row_map_add_layernorm(H, det):
    """The residual LayerNorm on a packed stream: vb_add_layernorm_fwd, x = dropout(d) + residual with the mask of padded row
    map[r], then vb_add_layernorm_bwd (det: vb_layernorm_bwd_det with dy2) with in_dropout: dx16 and dbias carry the mask."""
    mp, count, rows = _row_layout(H, H + 3)
    gen = _gen("map-addln", H, det)
    p, lib = 0.1, L.lib()
    d, r = _rows_in(rows, H, count, gen), _rows_in(rows, H, count, gen)
    gm, bt = torch.randn(H, device=DEV, generator=gen), torch.randn(H, device=DEV, generator=gen)
    step_t = _step_tensor(STEP)
    drop = _mdesc(step_t, LN_SITE, p, mp)
    x = d.clone()
    y32, y16 = torch.full((rows, H), SENT, device=DEV), torch.full((rows, H), SENT, device=DEV, dtype=F16)
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    L.check(lib.vb_add_layernorm_fwd(x.data_ptr(), r.data_ptr(), H, C.byref(drop), x.data_ptr(), gm.data_ptr(), bt.data_ptr(), 1e-12,
                                     y32.data_ptr(), y16.data_ptr(), H, mean.data_ptr(), rstd.data_ptr(), rows, H, 1, None, None, _st()))
    dy, dy2 = _rows_in(rows, H, count, gen), _rows_in(rows, H, count, gen)
    dx32, dx16 = torch.full((rows, H), SENT, device=DEV), torch.full((rows, H), SENT, device=DEV, dtype=BF)
    base = {k: torch.randn(H, device=DEV, generator=gen) for k in ("dgamma", "dbeta", "dbias")}
    acc = {k: v.clone() for k, v in base.items()}
    _ln_bwd_call(det, dy, dy2, x, gm, mean, rstd, dx32, dx16, None, acc, rows, H, None, C.byref(drop))
    torch.cuda.synchronize()
    assert torch.isfinite(y32).all() and torch.isfinite(dx32).all() and torch.isfinite(dx16.float()).all()
    assert _tail_sums_zero(det, count, rows, H, LN_SITE, p, mp, step_t, dy, dy2, x, gm, mean, rstd, None, ("dgamma", "dbeta", "dbias"), "in")
    v = slice(0, count)
    f = R.keep_factor(LN_SITE, STEP, p, P.packed_index(mp, H))[v]
    drop_m = f == 0
    assert torch.equal(x[v][drop_m], r[v][drop_m]) and (dx16[v][drop_m] == 0).all() and torch.equal(y16, y32.half())
    g = dy[v].to(F64) + dy2[v].to(F64)
    dx, xh = _ln_bwd64(x[v], gm, g)

    def err(ff):
        y, mu, rs = _ln64(d[v].to(F64) * ff.to(F64) + r[v].to(F64), gm, bt)
        dxm = dx * ff.to(F64)
        return dict(x=(x[v] != d[v] * ff + r[v]).double().mean().item(), y=relmax(y32[v], y), mean=relmax(mean[v], mu),
                    rstd=relmax(rstd[v], rs), dx16=relmax(dx16[v], dxm), dbias=colsum_err(acc["dbias"], base["dbias"], dxm))

    errs = dict(err(f), dx32=relmax(dx32[v], dx), dgamma=colsum_err(acc["dgamma"], base["dgamma"], g * xh),
                dbeta=colsum_err(acc["dbeta"], base["dbeta"], g))
    wrongs = {"identity map": err(R.keep_factor(LN_SITE, STEP, p, R.rowmajor_index(rows, H, DEV))[v]),
              "step+1": err(R.keep_factor(LN_SITE, STEP + 1, p, P.packed_index(mp, H))[v])}
    verdict(f"row map add_layernorm {rows}x{H} det={det}", errs, LN_TOL, wrongs, drop_m.double().mean().item(), p)


@pytest.mark.parametrize("det", [0, 1])
def test_row_map_small_linear_vision_logit(det):
    """The packed vision logit: vb_small_linear_fwd / _bwd (det: vb_small_linear_bwd_det) with in_dropout under the image row map,
    K = 1024, N = 1, dx accumulated onto a non-zero buffer, dW / db over the valid rows only."""
    K, N = 1024, 1
    mp, count, M = _row_layout(K, 7)
    gen = _gen("map-small", det)
    p, lib = 0.1, L.lib()
    site = dropout_site_id("dropout.seq_v")
    x, W = _rows_in(M, K, count, gen), torch.randn(N, K, device=DEV, generator=gen)
    b, add = torch.randn(N, device=DEV, generator=gen), torch.randn(M, device=DEV, generator=gen)
    step_t = _step_tensor(STEP)
    drop = _mdesc(step_t, site, p, mp)
    y = torch.full((M, N), SENT, device=DEV)
    L.check(lib.vb_small_linear_fwd(x.data_ptr(), K, W.data_ptr(), b.data_ptr(), add.data_ptr(), y.data_ptr(), M, K, N, C.byref(drop), _st()))
    dy = _rows_in(M, N, count, gen)
    dx0 = torch.randn(M, K, device=DEV, generator=gen)
    dx = dx0.clone()
    dW0, db0 = torch.randn(N, K, device=DEV, generator=gen), torch.randn(N, device=DEV, generator=gen)
    dW, db = dW0.clone(), db0.clone()

    def bwd(dy_, x_, dx_, dW_, db_, M_, d_):
        args = (dy_.data_ptr(), x_.data_ptr(), K, W.data_ptr(), dx_.data_ptr(), K, 1, dW_.data_ptr(), db_.data_ptr(), M_, K, N, C.byref(d_))
        if det:
            ws = torch.empty(64 * (N * K + N), device=DEV)
            L.check(lib.vb_small_linear_bwd_det(*args, ws.data_ptr(), _st()), "vb_small_linear_bwd_det")
        else:
            L.check(lib.vb_small_linear_bwd(*args, _st()), "vb_small_linear_bwd")

    bwd(dy, x, dx, dW, db, M, drop)
    # the rows of no sample alone, sums from 0: nothing
    tW, tb, tdx = torch.zeros(N, K, device=DEV), torch.zeros(N, device=DEV), torch.zeros(M - count, K, device=DEV)
    dtail = _mdesc(step_t, site, p, mp[count:])
    bwd(dy[count:], x[count:], tdx, tW, tb, M - count, dtail)
    torch.cuda.synchronize()
    assert (tW == 0).all() and (tb == 0).all() and torch.isfinite(y).all() and torch.isfinite(dx).all()
    v = slice(0, count)
    f = R.keep_factor(site, STEP, p, P.packed_index(mp, K))[v]
    assert torch.equal(dx[v][f == 0], dx0[v][f == 0])             # dropped: nothing added

    def err(ff):
        xd, dy64 = x[v].to(F64) * ff.to(F64), dy[v].to(F64)
        terms = (dy64.t()[:, :, None] * xd[None]).permute(1, 0, 2).reshape(count, N * K)
        return dict(y=relmax(y[v], xd @ W.to(F64).t() + b.to(F64) + add[v].to(F64)[:, None]),
                    dx=relmax(dx[v] - dx0[v], (dy64 @ W.to(F64)) * ff.to(F64)), dW=colsum_err(dW, dW0, terms))

    errs = dict(err(f), db=colsum_err(db, db0, dy[v]))
    wrongs = {"identity map": err(R.keep_factor(site, STEP, p, R.rowmajor_index(M, K, DEV))[v]),
              "step+1": err(R.keep_factor(site, STEP + 1, p, P.packed_index(mp, K))[v])}
    verdict(f"row map small_linear {M}x{K}x{N} det={det}", errs, dict(y=1e-5, dx=1e-5, dW=2e-5, db=2e-5), wrongs,
            (f == 0).double().mean().item(), p)


# ============================================================================================ pack / unpack / compaction (exact)
def _masks(B, N, gen):
    lens = torch.randint(1, N + 1, (B,), generator=gen)
    lens[0], lens[1] = 1, N
    return (torch.arange(N)[None] < lens[:, None]).long()


@pytest.mark.parametrize("clamp", [False, True])
@pytest.mark.parametrize("has_task", [0, 1])
def test_pack_build(has_task, clamp):
    """vb_pack_build against _packed_ref.pack_layout for both streams (B = 64, 36 tokens, 101 regions); clamp: capacities below
    the valid counts (the documented clamp: later samples keep what fits). map = -1 past off[B]."""
    B, Nt, Nv = 64, 36, 101
    g = torch.Generator().manual_seed(has_task * 2 + clamp)
    mt, mv = _masks(B, Nt, g), _masks(B, Nv, g)
    ct, cv = int(mt.sum()) + B * has_task, int(mv.sum())
    rt = ct - 50 if clamp else pack_capacity(ct, B * (Nt + has_task))
    rv = cv // 2 if clamp else pack_capacity(cv, B * Nv)
    out = [torch.full((n,), 12345, device=DEV, dtype=I32) for n in (B + 1, B, rt, B + 1, B, rv)]
    mt_d, mv_d = mt.to(DEV), mv.to(DEV)
    L.check(L.lib().vb_pack_build(mt_d.data_ptr(), Nt, has_task, mv_d.data_ptr(), Nv, B, rt, rv, *(o.data_ptr() for o in out), _st()),
            "vb_pack_build")
    torch.cuda.synchronize()
    for got, ref in zip(out, P.pack_layout(mt, has_task, rt) + P.pack_layout(mv, 0, rv)):
        assert torch.equal(got.cpu(), ref)
    if clamp:
        assert int(out[0][B]) == rt and int(out[3][B]) == rv
    else:
        assert int(out[0][B]) == ct and (out[2][ct:] == -1).all() and int(out[3][B]) == cv and (out[5][cv:] == -1).all()


def _vision_map(seed):
    B, Nv = 64, 101
    mv = _masks(B, Nv, torch.Generator().manual_seed(seed))
    cv = int(mv.sum())
    off, ln, mp = P.pack_layout(mv, 0, pack_capacity(cv, B * Nv))
    return off.to(DEV), ln.to(DEV), mp.to(DEV), cv, B, Nv


def _gather(src, mp):
    out = torch.zeros(mp.numel(), src.shape[1], device=DEV, dtype=src.dtype)
    v = mp >= 0
    out[v] = src[mp[v].long()]
    return out


@pytest.mark.parametrize("cols", [2048, 20, 1, 5])
def test_pack_rows_f32(cols):
    """dst[r] = src[map[r]], zeros where map[r] < 0: the float4 path (cols % 4 == 0) and the scalar path."""
    _, _, mp, cv, B, Nv = _vision_map(cols)
    gen = _gen("packrows", cols)
    src = torch.randn(B * Nv, cols, device=DEV, generator=gen)
    dst = torch.full((mp.numel(), cols), float("nan"), device=DEV)
    L.check(L.lib().vb_pack_rows_f32(src.data_ptr(), dst.data_ptr(), mp.data_ptr(), mp.numel(), cols, _st()), "vb_pack_rows_f32")
    torch.cuda.synchronize()
    assert torch.equal(dst, _gather(src, mp)) and (dst[cv:] == 0).all()


@pytest.mark.parametrize("lo,b16", [(0, 0), (1, 1), (0, 1)])
@pytest.mark.parametrize("fp16", [0, 1])
def test_pack_regions(fp16, lo, b16):
    """The packed region features as a tensor-core operand: bitwise vb_cast_f32_to_bf16 of the gathered padded rows (hi, split lo,
    bf16 copy) at cols = 2048, tail rows zero."""
    cols = 2048
    _, _, mp, cv, B, Nv = _vision_map(11)
    rows = mp.numel()
    gen = _gen("packreg", fp16, lo, b16)
    feat = torch.randn(B * Nv, cols, device=DEV, generator=gen) * 3
    mk = lambda on: torch.full((rows, cols), SENT, device=DEV, dtype=BF) if on else None
    hi, lo_t, bw = mk(True), mk(lo), mk(b16)
    L.check(L.lib().vb_pack_regions(feat.data_ptr(), mp.data_ptr(), rows, cols, fp16, hi.data_ptr(), _ptr(lo_t), _ptr(bw), _st()), "vb_pack_regions")
    gathered = _gather(feat, mp)
    rh, rl, rb = mk(True), mk(lo), mk(b16)
    L.check(L.lib().vb_cast_f32_to_bf16(gathered.data_ptr(), rh.data_ptr(), rows * cols, fp16, _ptr(rl), _ptr(rb), _st()), "vb_cast_f32_to_bf16")
    torch.cuda.synchronize()
    for got, ref in ((hi, rh), (lo_t, rl), (bw, rb)):
        if got is not None:
            assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
            assert (got[cv:].view(torch.int16) == 0).all()


@pytest.mark.parametrize("cols", [1, 1601])
@pytest.mark.parametrize("fill", [0.0, PACKED_MASKED_LOGIT])
def test_unpack_rows_f32(fill, cols):
    """dst[b*N + i] = src[off[b] + i] for i < len[b], else fill: per-region logits (cols 1) and per-region class scores (1601)."""
    off, ln, mp, cv, B, Nv = _vision_map(cols + (1 if fill else 0))
    gen = _gen("unpack", fill, cols)
    src = torch.randn(mp.numel(), cols, device=DEV, generator=gen)
    dst = torch.full((B * Nv, cols), float("nan"), device=DEV)
    L.check(L.lib().vb_unpack_rows_f32(src.data_ptr(), dst.data_ptr(), off.data_ptr(), ln.data_ptr(), B, Nv, cols, fill, _st()), "vb_unpack_rows_f32")
    torch.cuda.synchronize()
    ref = torch.full((B * Nv, cols), fill, device=DEV)
    ref[mp[:cv].long()] = src[:cv]
    assert torch.equal(dst, ref)


@pytest.mark.parametrize("cols", [768, 5])
def test_scatter_add_rows_f32(cols):
    """dst[idx[r]] += src[r] (distinct idx) onto a non-zero destination: one fp32 add per element, exact."""
    gen = _gen("scatadd", cols)
    rows, n = 2368, 64
    idx = torch.randperm(rows, device=DEV, generator=gen)[:n].to(I32)
    src = torch.randn(n, cols, device=DEV, generator=gen)
    dst0 = torch.randn(rows, cols, device=DEV, generator=gen)
    dst = dst0.clone()
    L.check(L.lib().vb_scatter_add_rows_f32(src.data_ptr(), dst.data_ptr(), idx.data_ptr(), n, cols, _st()), "vb_scatter_add_rows_f32")
    torch.cuda.synchronize()
    ref = dst0.clone()
    ref[idx.long()] += src
    assert torch.equal(dst, ref)


@pytest.mark.parametrize("n", [1, 2, 3])
def test_zero_tail_rows(n):
    """Rows [*first, rows) of one, two or three tensors zeroed over row_bytes; the rows before *first and the bytes between the row
    end and the pitch stay bitwise unchanged."""
    rows, H, ld = 2368, 768, 784                  # fp32 rows of 768 in a pitch of 784 (3072 of 3136 bytes)
    gen = _gen("zerotail", n)
    ts = [torch.randn(rows, ld, device=DEV, generator=gen) for _ in range(n)]
    before = [t.clone() for t in ts]
    first = torch.tensor([1531], device=DEV, dtype=I32)
    ptrs = [t.data_ptr() for t in ts] + [None] * (3 - n)
    L.check(L.lib().vb_zero_tail_rows(*ptrs, ld * 4, H * 4, first.data_ptr(), rows, _st()), "vb_zero_tail_rows")
    torch.cuda.synchronize()
    for t, b in zip(ts, before):
        ref = b.clone()
        ref[1531:, :H] = 0
        assert torch.equal(t.view(I32), ref.view(I32))


IGNORE = -1
VOCAB = 30522


def _compact_ref(sel_rows, labels_at, cap, ignore=IGNORE):
    """(idx [cap], labels_compact [cap], count) of a selection given as ascending row numbers."""
    n = sel_rows.numel()
    idx = torch.full((cap,), -1, dtype=I32, device=DEV)
    lab = torch.full((cap,), ignore, dtype=I64, device=DEV)
    k = min(n, cap)
    idx[:k] = sel_rows[:k].to(I32)
    lab[:k] = labels_at[:k]
    return idx, lab, n


def _no_carry(sel):
    """The idx a compaction would give that restarts its count in every 1024-row pass (a lost carry)."""
    r = torch.nonzero(sel).flatten()
    return r, (torch.cumsum(sel.long(), 0) - 1 - torch.cat([torch.zeros(1, dtype=I64, device=DEV), torch.cumsum(sel.long(), 0)])[
        (torch.arange(sel.numel(), device=DEV) // 1024) * 1024])[r]


def _compact_call(labels, mp, rows, cap):
    idx = torch.full((cap,), 777, device=DEV, dtype=I32)
    lab = torch.full((cap,), 777, device=DEV, dtype=I64)
    count = torch.full((1,), -5, device=DEV, dtype=I32)
    if mp is None:
        L.check(L.lib().vb_compact_rows(labels.data_ptr(), IGNORE, rows, cap, idx.data_ptr(), count.data_ptr(), lab.data_ptr(), _st()))
    else:
        L.check(L.lib().vb_compact_rows_mapped(labels.data_ptr(), IGNORE, mp.data_ptr(), rows, cap, idx.data_ptr(), count.data_ptr(),
                                               lab.data_ptr(), _st()))
    torch.cuda.synchronize()
    return idx, lab, int(count)


@pytest.mark.parametrize("capkind", ["room", "exact", "over", "empty"])
@pytest.mark.parametrize("rows", [2304, 6400])
def test_compact_rows(rows, capkind):
    """vb_compact_rows over more than 1024 rows (the scan carries its count across passes): count < cap, == cap, > cap (*count
    is the true count, idx truncated) and an empty selection."""
    gen = _gen("compact", rows, capkind)
    labels = torch.randint(0, VOCAB, (rows,), device=DEV, generator=gen)
    keep = torch.rand(rows, device=DEV, generator=gen) < (0.0 if capkind == "empty" else 0.15)
    labels[~keep] = IGNORE
    n = int(keep.sum())
    cap = dict(room=n + 37, exact=n, over=n - 9, empty=64)[capkind]
    idx, lab, count = _compact_call(labels, None, rows, cap)
    sel = torch.nonzero(keep).flatten()
    ridx, rlab, rn = _compact_ref(sel, labels[sel], cap)
    assert count == rn and torch.equal(idx, ridx) and torch.equal(lab, rlab)
    if n:
        r, pos = _no_carry(keep)
        wrong = torch.full((cap,), -1, dtype=I64, device=DEV)
        ok = pos < cap
        wrong[pos[ok]] = r[ok]
        assert not torch.equal(wrong.to(I32), idx)      # a lost carry would show


@pytest.mark.parametrize("capkind", ["room", "exact", "over", "empty"])
def test_compact_rows_mapped(capkind):
    """vb_compact_rows_mapped on a packed text stream of 64 x 37 rows (> 1024 packed rows): row r stands for padded row map[r];
    idx holds packed rows, in the order of their padded rows."""
    B, Nt = 64, 36
    g = torch.Generator().manual_seed(5)
    mt = _masks(B, Nt, g)
    ct = int(mt.sum()) + B
    _, _, mp = P.pack_layout(mt, 1, pack_capacity(ct, B * (Nt + 1)))
    mp = mp.to(DEV)
    rows = mp.numel()
    gen = _gen("compactmap", capkind)
    labels = torch.randint(0, VOCAB, (B * (Nt + 1),), device=DEV, generator=gen)
    on = torch.rand(B * (Nt + 1), device=DEV, generator=gen) < (0.0 if capkind == "empty" else 0.3)
    labels[~on] = IGNORE
    v = mp >= 0
    keep = torch.zeros(rows, dtype=torch.bool, device=DEV)
    keep[v] = labels[mp[v].long()] != IGNORE
    n = int(keep.sum())
    cap = dict(room=n + 37, exact=n, over=n - 9, empty=64)[capkind]
    idx, lab, count = _compact_call(labels, mp, rows, cap)
    sel = torch.nonzero(keep).flatten()
    ridx, rlab, rn = _compact_ref(sel, labels[mp[sel].long()], cap)
    assert rows > 1024 and count == rn and torch.equal(idx, ridx) and torch.equal(lab, rlab)
    if n:
        assert int(sel.max()) >= 1024                     # selected rows past the first pass
        unmapped, _, _ = _compact_call(labels, None, rows, cap)
        assert not torch.equal(unmapped, idx)             # the map is used


@pytest.mark.parametrize("capkind", ["room", "exact", "over"])
def test_masked_lm_chain(capkind):
    """The packed masked-LM head: vb_compact_rows_mapped -> vb_gather_rows16 (two sources) -> vb_ce_loss on the gathered
    [cap, 30522] rows (ld_d16 != cols, grad_scale != 1): its fp32 and bf16 gradients against float64 (softmax - onehot) * gs / n,
    ignored rows exactly 0 -> vb_scatter_rows_f32 back to the packed rows, NaN-poisoning the loss when count > cap."""
    B, Nt, H = 64, 36, 768
    g = torch.Generator().manual_seed(9)
    mt = _masks(B, Nt, g)
    _, _, mp = P.pack_layout(mt, 1, pack_capacity(int(mt.sum()) + B, B * (Nt + 1)))
    mp = mp.to(DEV)
    rows = mp.numel()
    gen = _gen("mlm", capkind)
    labels = torch.randint(0, VOCAB, (B * (Nt + 1),), device=DEV, generator=gen)
    labels[torch.rand(B * (Nt + 1), device=DEV, generator=gen) >= 0.15] = IGNORE
    v = mp >= 0
    keep = torch.zeros(rows, dtype=torch.bool, device=DEV)
    keep[v] = labels[mp[v].long()] != IGNORE
    n = int(keep.sum())
    cap = dict(room=n + 40, exact=n, over=n - 24)[capkind]
    idx, lab, count = _compact_call(labels, mp, rows, cap)
    assert count == n
    # gather: two 16-bit sources (the hidden rows and a second operand copy)
    hs = torch.randn(rows, H, device=DEV, generator=gen).to(BF)
    hs2 = torch.randn(rows, H, device=DEV, generator=gen).half()
    g1, g2 = torch.full((cap, H), SENT, device=DEV, dtype=BF), torch.full((cap, H), SENT, device=DEV, dtype=F16)
    L.check(L.lib().vb_gather_rows16(hs.data_ptr(), g1.data_ptr(), hs2.data_ptr(), g2.data_ptr(), idx.data_ptr(), cap, H, _st()))
    torch.cuda.synchronize()
    live = idx >= 0
    for got, src in ((g1, hs), (g2, hs2)):
        ref = torch.zeros_like(got)
        ref[live] = src[idx[live].long()]
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
    # the cross-entropy of the gathered rows
    gs = 0.37
    z = torch.randn(cap, VOCAB, device=DEV, generator=gen) * 2
    ld16 = VOCAB + 6
    d32 = torch.full((cap, VOCAB), SENT, device=DEV)
    d16 = torch.full((cap, ld16), SENT, device=DEV, dtype=BF)
    loss = torch.full((1,), SENT, device=DEV)
    L.check(L.lib().vb_ce_loss(z.data_ptr(), VOCAB, lab.data_ptr(), IGNORE, loss.data_ptr(), d32.data_ptr(), VOCAB, d16.data_ptr(), ld16,
                               cap, VOCAB, gs, 0, _st()), "vb_ce_loss")
    torch.cuda.synchronize()
    assert torch.equal(d16[:, VOCAB:].float(), torch.full((cap, 6), SENT, device=DEV))    # the pitch padding untouched
    rl = lab != IGNORE
    nv = int(rl.sum())
    assert nv == min(n, cap) and (d32[~rl] == 0).all() and (d16[~rl, :VOCAB] == 0).all()

    def ref_of(labs):
        z64 = z[rl].to(F64)
        sm = torch.softmax(z64, -1)
        oh = torch.zeros_like(sm)
        oh[torch.arange(nv, device=DEV), labs] = 1
        lse = torch.logsumexp(z64, -1)
        return (sm - oh) * gs / nv, (lse - z64[torch.arange(nv, device=DEV), labs]).mean()

    gref, lref = ref_of(lab[rl])
    err = lambda gr: dict(d32=relmax(d32[rl], gr), d16=relmax(d16[rl, :VOCAB], gr))
    errs = dict(err(gref), loss=abs(loss.item() - lref.item()) / abs(lref.item()))
    wrongs = {"next row's label": err(ref_of(lab[rl].roll(1))[0])}
    verdict(f"masked-LM chain cap={cap} count={n}", errs, dict(d32=1e-5, d16=4e-3, loss=1e-5), wrongs)
    # scatter the gathered rows' gradient back to the packed rows; count > cap poisons the loss
    src = torch.randn(cap, H, device=DEV, generator=gen)
    dst = torch.zeros(rows, H, device=DEV)
    poison = torch.full((1,), 1.5, device=DEV)
    cnt = torch.tensor([count], device=DEV, dtype=I32)
    L.check(L.lib().vb_scatter_rows_f32(src.data_ptr(), dst.data_ptr(), idx.data_ptr(), cap, H, cnt.data_ptr(), poison.data_ptr(), _st()),
            "vb_scatter_rows_f32")
    torch.cuda.synchronize()
    ref = torch.zeros(rows, H, device=DEV)
    ref[idx[live].long()] = src[live]
    assert torch.equal(dst, ref)
    assert math.isnan(poison.item()) if count > cap else poison.item() == 1.5


@pytest.mark.parametrize("det", [0, 1])
def test_ce_loss_out_of_range_label(det):
    """A label outside [0, cols) other than ignore_index (cols itself on an interior row, and a negative one) reads nothing: its
    row's gradient is exactly 0 and the loss is NaN; every other row keeps its gradient, averaged over all non-ignored rows."""
    rows, cols, gs = 16, VOCAB, 0.5
    gen = _gen("ce-oob", det)
    z = torch.randn(rows, cols, device=DEV, generator=gen)
    labels = torch.randint(0, cols, (rows,), device=DEV, generator=gen)
    labels[3], labels[5], labels[9] = IGNORE, cols, -7
    d32 = torch.full((rows, cols), SENT, device=DEV)
    d16 = torch.full((rows, cols), SENT, device=DEV, dtype=BF)
    loss = torch.zeros(1, device=DEV)
    args = (z.data_ptr(), cols, labels.data_ptr(), IGNORE, loss.data_ptr(), d32.data_ptr(), cols, d16.data_ptr(), cols, rows, cols, gs, 0)
    if det:
        ws = torch.empty(1024, device=DEV)
        L.check(L.lib().vb_ce_loss_det(*args, ws.data_ptr(), _st()), "vb_ce_loss_det")
    else:
        L.check(L.lib().vb_ce_loss(*args, _st()), "vb_ce_loss")
    torch.cuda.synchronize()
    assert math.isnan(loss.item())
    for r in (3, 5, 9):
        assert (d32[r] == 0).all() and (d16[r] == 0).all()
    ok = torch.ones(rows, dtype=torch.bool, device=DEV)
    ok[[3, 5, 9]] = False
    nv = rows - 1                                   # the out-of-range rows count as non-ignored
    z64 = z[ok].to(F64)
    oh = torch.zeros_like(z64)
    oh[torch.arange(int(ok.sum()), device=DEV), labels[ok]] = 1
    gref = (torch.softmax(z64, -1) - oh) * gs / nv
    verdict(f"ce_loss out-of-range label det={det}", dict(d32=relmax(d32[ok], gref)), dict(d32=1e-5),
            {"n without the bad rows": dict(d32=relmax(d32[ok], gref * nv / (nv - 2)))})
