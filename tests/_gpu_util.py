"""Shared GPU check helpers (used by the -m gpu tests and by the tools/ probe drivers).
Every check runs the CUDA path through the C ABI (ctypes) and compares with torch fp32 / the oracle."""
import ctypes as C
import gc
import math

import torch
import torch.nn.functional as F

from oracle import vilbert_oracle as O
from vilbert_b200 import _lib as L

BF = torch.bfloat16


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-20)).item()


def rel_l2(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-20)).item()


def launched(fn, *expect, tries=10, pad_cycles=2_000_000):
    """Runs fn() under torch.profiler (CUDA activity); returns (its result, the names of the recorded events). Kernel names are
    demangled, e.g. "void vb::ln_fwd_kernel<4, false>(float const*, ...)". The profiler now and then delivers a capture without its
    device records (only the runtime calls such as cudaLaunchKernelExC), most often for a capture that holds a single short launch
    late in a long-running process. So fn's launches are bracketed on the stream by two GPU busy-waits of `pad_cycles` clock cycles
    each (about 1 ms), which the capture records too. With expect
    (regular expressions), a capture in which one of them matches no name is taken again, up to `tries` captures, and then asserted:
    the launches are deterministic, so a kernel that is really not launched is missing from every capture. fn must be repeatable."""
    import re
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(pad_cycles)
            r = fn()
            torch.cuda._sleep(pad_cycles)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        if all(any(re.search(pat, n) for n in names) for pat in expect):
            break
    assert_launched(names, *expect)
    return r, names


def assert_launched(names, *patterns):
    """Every regular expression in patterns matches the name of a launched kernel (a boundary case stays on its variant)."""
    import re
    for pat in patterns:
        assert any(re.search(pat, n) for n in names), (pat, sorted(set(names)))


# ------------------------------------------------------------------------------------------ GEMM
# One float64 checker for every vb_gemm_bf16 test (GemmCase.errors). The reference is the epilogue value v of the 16-bit operands
# in float64; in split precision it is the kernel's three passes hi.hi + lo.hi + hi.lo (the header drops the lo.lo term, so the
# reference does too). Every bound is tied to the element's own magnitude S = |alpha| sum_k |a_mk b_nk| (+ |bias|, carried through
# the activation, times the dropout factor, + |residual|) and to the square root of n, the 16-deep k-steps accumulated into it:
#   fp32 outputs     |got - v| <= e = c 2^-24 sqrt(n) S, c = GEMM_C_ACC (GEMM_C_SPLIT in split precision), + GEMM_ERF |pre| for
#                    GELU (erf by A&S 7.1.26); atomic outputs add split 2^-24 (S + |base|) for the additions into the buffer
#   16-bit outputs   correctly rounded: got lies between RN16(fl32(v - e)) and RN16(fl32(v + e)), i.e. it is bitwise RN16(v) wherever
#                    no rounding midpoint lies within e of v, and either neighbour elsewhere; out_lo is held to RN16(v - hi) with hi
#                    the value written, out_b16 to RN_bf16(v), out_pre to RN_bf16(gelu'(pre)) with e' = 0.8 e(pre) + GEMM_ERF
#                    (|gelu''| <= 0.8); beside an fp32 output they must also be bitwise the rounding of the fp32 value written
#   column sums      added into a non-zero buffer: |got - base - sum_m v| <= 2^-24 (c sqrt(n) sum_m S + adds (|base| + sum_m |v|))
#   guard bands      every output has a leading gap, a row pitch past N and rows past M (past split * M for partials), all filled
#                    with a NaN sentinel; in-range elements must not hold it afterwards, everything else must be bitwise unchanged.
# Calibrated on an H100 80GB HBM3 (700 W power limit) over the 505 cases of test_gemm_float64_gpu.py, test_gemm_gpu.py and
# test_gemm_regsplit_gpu.py: the worst |got - v| / (2^-24 sqrt(n) S) of an fp32 output is 2.51 single-pass (a 300x200x136
# deterministic split-K slice; 0.78 with GELU) and 2.65 in split precision (130x30522x768). wgmma's fp32 accumulation error grows
# with K: as a multiple of 2^-24 S alone it reached 28 at K = 30522 and 54 at K = 3 x 4096 (split precision), so a constant
# multiple of 2^-24 S would be loose at small K or fail at large K.
U24 = 2.0 ** -24
GEMM_C_ACC, GEMM_C_SPLIT = 4.0, 8.0
GEMM_ERF = 5e-7
SENT32, SENT16 = 0x7FC5A5A5, 0x7FA5      # NaN bit patterns (fp32; bf16 and fp16 alike): no epilogue writes them
GUARD, XROWS = 64, 3                     # elements before and after each buffer; rows past the last row a call may write
F64 = torch.float64
GEMM_INPUTS = ("A", "B", "A_lo", "B_lo", "bias", "residual", "aux")
GEMM_OUTPUTS = ("out_f32", "out_bf16", "out_lo", "out_b16", "out_pre", "out_colsum")
EPI = dict(F32=0, BF16=1, GELU=2, DGELU=3, ATOMIC=4, GENERIC=5, PARTIAL=6)   # vb_gemm.cu's epilogue specialisations


def gemm_kernel_name(bn, epi, out16=0):
    """Regular expression of the demangled name of gemm_wgmma_kernel<BN, EPI, OUT16>."""
    return rf"gemm_wgmma_kernel<{bn}, {EPI.get(epi, epi)}, {out16}>"


def _bits(t):
    return t.view({4: torch.int32, 2: torch.int16}[t.element_size()])


def _sentinel(dt):
    return torch.tensor([SENT32 if dt == torch.float32 else SENT16], dtype=torch.int32 if dt == torch.float32 else torch.int16)


def rn16(x, dt):
    """float64 -> fp32 -> 16-bit, round to nearest even: what the epilogue does with its fp32 value."""
    return x.float().to(dt)


def rz16(x, dt):
    """float64 -> fp32 -> 16-bit rounded toward zero (a truncating epilogue)."""
    x32 = x.float()
    r = x32.to(dt)
    b = _bits(r).clone()
    b[r.float().abs() > x32.abs()] -= 1       # sign-magnitude: one pattern down is one ulp toward zero
    return b.view(dt)


def ulp_up(t):
    """The next 16-bit value away from zero."""
    return (_bits(t) + 1).view(t.dtype)


def keep_scale(M, N, site, ctr, p, device):
    """Dropout factor (0 or 1 / (1 - p), float64) of the GEMM epilogue's element (m, n): the kernel's hash of m * N + n."""
    def h(x):
        x = x & 0xFFFFFFFF
        x = x ^ (x >> 16); x = (x * 0x7FEB352D) & 0xFFFFFFFF
        x = x ^ (x >> 15); x = (x * 0x846CA68B) & 0xFFFFFFFF
        return x ^ (x >> 16)
    seed = h(torch.tensor(site + ctr * 0x9E3779B9, dtype=torch.int64))
    idx = (torch.arange(M, device=device, dtype=torch.int64)[:, None] * N + torch.arange(N, device=device, dtype=torch.int64)[None]) & 0xFFFFFFFF
    p32 = float(torch.tensor(p, dtype=torch.float32))   # the kernel's threshold and scale come from the float p
    keep = h(idx ^ seed.to(device)) >= int(p32 * 4294967296.0)
    return keep.double() * float(1.0 / (1.0 - torch.tensor(p32, dtype=torch.float32)))


def window16(got, v, e, dt, shift=0.0):
    """(distance of got outside [RN16(fl32(v - e) - shift), RN16(fl32(v + e) - shift)], float64 with NaN -> inf; mask where that
    window is one value, i.e. where got must be bitwise RN16(v - shift)). shift: the hi part already written (out_lo = RN16(v32 - hi),
    the subtraction exact in fp32)."""
    lo = rn16((v - e).float().double() - shift, dt).double()
    hi = rn16((v + e).float().double() - shift, dt).double()
    g = got.double()
    dist = torch.maximum(lo - g, g - hi).clamp_min(0)
    return torch.nan_to_num(dist, nan=math.inf), lo == hi


def _worst(d, e):
    """max of d / e, NaN (a NaN reference: a wrong one reading a sentinel) counted as infinite."""
    return torch.nan_to_num(d / e, nan=math.inf).max().item()


class GemmCase:
    """One vb_gemm_bf16 call on guarded buffers (see the comment above) and its float64 reference.

    outs: the output fields to pass. Operands are randn * scale rounded to the 16-bit format (fp16=True: fp16, else bf16); a_lo /
    b_lo add the low parts of the fp32 values (split precision). atomic: 0, 1 (red.add into a non-zero out_f32) or
    L.VB_GEMM_PARTIALS (split_k=0: the count vb_gemm_plan resolves). res_inplace: the residual is out_f32 itself. ld / align: a row
    pitch (elements) / base address modulo 256 (bytes) per field, defaults N + 8 and 0. Pitch padding, guard rows and the leading
    gaps of the inputs hold junk the kernel must not read. device="cpu" builds the buffers without the library (the CPU tests
    emulate the kernel into them)."""

    def __init__(self, M, N, K, outs=("out_f32",), a_mn=False, b_mn=False, fp16=False, out_fp16=False, alpha=1.0, bias=False, act=0,
                 res=False, res_inplace=False, drop=None, a_lo=False, b_lo=False, atomic=0, split_k=1, block_n=0, max_ctas=0,
                 ld=None, align=None, seed=0, scale=0.5, device="cuda"):
        self.M, self.N, self.K, self.alpha, self.act, self.atomic = M, N, K, alpha, act, atomic
        self.drop = drop
        self.dev = dev = torch.device(device)
        gen = torch.Generator(device=dev).manual_seed(seed)
        rnd = lambda *shape: torch.randn(*shape, device=dev, generator=gen)
        d16, o16 = (torch.float16 if fp16 else BF), (torch.float16 if out_fp16 else BF)
        self.dt = dict(A=d16, B=d16, A_lo=d16, B_lo=d16, aux=BF, out_bf16=o16, out_lo=o16, out_pre=BF, out_b16=BF)
        res = res or res_inplace
        fields = ["A", "B"] + (["A_lo"] if a_lo else []) + (["B_lo"] if b_lo else []) + (["bias"] if bias else []) \
            + (["residual"] if res else []) + (["aux"] if act == L.VB_ACT_DGELU else []) + list(outs)
        self.fields, self.outs = fields, [f for f in GEMM_OUTPUTS if f in outs]
        pad8 = lambda x: (x + 7) // 8 * 8
        self.ld = dict(A=pad8(M if a_mn else K), B=pad8(N if b_mn else K), bias=N, out_colsum=N)
        self.ld.update({f: N + 8 for f in ("residual", "aux", "out_f32", "out_bf16", "out_pre")})
        self.ld.update(ld or {})
        self.ld["A_lo"], self.ld["B_lo"] = self.ld["A"], self.ld["B"]
        self.ld["out_lo"] = self.ld["out_b16"] = self.ld["out_bf16"]
        if res_inplace:
            self.ld["residual"] = self.ld["out_f32"]
        self.res_inplace = res_inplace
        align = dict(align or {})

        g = self.g = L.GemmArgs()
        g.M, g.N, g.K, g.alpha, g.act = M, N, K, alpha, act
        g.a_mn_major, g.b_mn_major, g.lda, g.ldb = int(a_mn), int(b_mn), self.ld["A"], self.ld["B"]
        g.ld_res, g.ld_aux = (self.ld["residual"] if res else 0), (self.ld["aux"] if act == L.VB_ACT_DGELU else 0)
        g.ld_out_f32, g.ld_out_bf16, g.ld_out_pre = [self.ld[f] if f in outs else 0 for f in ("out_f32", "out_bf16", "out_pre")]
        g.atomic_out, g.split_k, g.block_n, g.max_ctas = atomic, split_k, block_n, max_ctas
        g.a_fp16 = g.b_fp16 = int(fp16)
        g.out_fp16 = int(out_fp16)
        self.bn, self.split = block_n or 128, max(split_k, 1)
        if dev.type == "cuda":
            for f in fields:
                setattr(g, f, 256)     # vb_gemm_plan reads only which pointers are set
            bn, sp = C.c_int32(), C.c_int32()
            L.check(L.lib().vb_gemm_plan(C.byref(g), 0, C.byref(bn), C.byref(sp)), "vb_gemm_plan")
            self.bn, self.split = bn.value, sp.value
            if atomic == L.VB_GEMM_PARTIALS and split_k == 0:
                g.split_k = self.split
        self.nslice = self.split if atomic == L.VB_GEMM_PARTIALS else 1

        # logical operands (float64 copies of the 16-bit values the kernel reads)
        A32, B32 = rnd(M, K) * scale, rnd(N, K) * scale
        A16, B16 = A32.to(d16), B32.to(d16)
        self.a, self.b = A16.double(), B16.double()
        self.a_lo = (A32 - A16.float()).to(d16) if a_lo else None
        self.b_lo = (B32 - B16.float()).to(d16) if b_lo else None
        rows = dict(A=K if a_mn else M, B=K if b_mn else N, bias=1, residual=M, aux=M, out_f32=M * self.nslice, out_bf16=M,
                    out_lo=M, out_b16=M, out_pre=M, out_colsum=1)
        rows["A_lo"], rows["B_lo"] = rows["A"], rows["B"]
        cols = dict(A=M if a_mn else K, B=N if b_mn else K)
        cols["A_lo"], cols["B_lo"] = cols["A"], cols["B"]
        logical = dict(A=A16.t() if a_mn else A16, B=B16.t() if b_mn else B16)
        if a_lo:
            logical["A_lo"] = self.a_lo.t() if a_mn else self.a_lo
        if b_lo:
            logical["B_lo"] = self.b_lo.t() if b_mn else self.b_lo
        if bias:
            logical["bias"] = rnd(1, N)
        if act == L.VB_ACT_DGELU:
            logical["aux"] = rnd(M, N).to(BF)
        self.raw, self.view, self.region, self.inside, self.off = {}, {}, {}, {}, {}
        for f in fields:
            if f == "residual" and res_inplace:
                continue
            dt = self.dt.get(f, torch.float32)
            el = torch.empty((), dtype=dt).element_size()
            nrows = rows[f] + XROWS
            raw = torch.empty(2 * GUARD + 256 // el + nrows * self.ld[f], device=dev, dtype=dt)
            o = self.off[f] = GUARD + ((align.get(f, 0) - raw.data_ptr() - GUARD * el) % 256) // el
            inside = torch.zeros(raw.numel(), dtype=torch.bool, device=dev)
            inside[o:o + nrows * self.ld[f]].view(nrows, self.ld[f])[:rows[f], :cols.get(f, N)] = True
            view = raw[o:o + nrows * self.ld[f]].view(nrows, self.ld[f])
            if f in GEMM_INPUTS:
                raw.copy_((rnd(raw.numel()) * 4).to(dt))                 # junk around the operand
                view[:rows[f], :cols.get(f, N)] = logical[f] if f in logical else rnd(rows[f], N)
            else:
                _bits(raw).fill_(_sentinel(dt).item())
            self.raw[f], self.view[f], self.region[f], self.inside[f] = raw, view, view[:rows[f], :cols.get(f, N)], inside
        if res_inplace:
            self.region["out_f32"].copy_(rnd(M, N))
            self.view["residual"] = self.view["out_f32"]
        if atomic == 1:
            self.region["out_f32"].copy_(rnd(M, N))                        # red.add into a non-zero buffer
        if "out_colsum" in outs:
            self.region["out_colsum"].copy_(rnd(1, N))
        self.init = {f: self.raw[f].clone() for f in self.outs}
        # the residual's rows, guard rows and pitch padding included (the wrong references read them)
        self.res0 = None if not res else self.init_view("out_f32") if res_inplace else self.view["residual"].clone()
        self.base32 = self.init["out_f32"] if "out_f32" in self.init else None
        for f in fields:
            setattr(g, f, (self.view["out_f32"] if f == "residual" and res_inplace else self.view[f]).data_ptr())
        if drop is not None:
            self.ctr = torch.ones(1, device=dev, dtype=torch.int32)
            if dev.type == "cuda":
                g.dropout.step, g.dropout.site, g.dropout.p = self.ctr.data_ptr(), drop[0], drop[1]

    # ---------------------------------------------------------------------------------- call
    def run(self, st=None):
        """Restores every output to its initial bits, then one vb_gemm_bf16 call (repeatable: launched() may run it again)."""
        for f in self.outs:
            self.raw[f].copy_(self.init[f])
        L.check(L.lib().vb_gemm_bf16(C.byref(self.g), st if st is not None else stream()), "vb_gemm_bf16")

    def init_view(self, f):
        """Output f's initial bits as the [rows, ld] view the call writes through."""
        v = self.view[f]
        return self.init[f][self.off[f]:self.off[f] + v.numel()].view(v.shape)

    def start(self, f):
        """The initial in-range values of output f (atomic base, column-sum base, in-place residual)."""
        i = self.init[f]
        return i[self.inside[f]].view(self.region[f].shape)

    # ---------------------------------------------------------------------------------- reference
    def passes(self, pass1_hi=False):
        """(A, B) float64 operands of each pass in the kernel's order: hi.hi, then lo.hi if A_lo, then hi.lo if B_lo."""
        ps = [(self.a, self.b)]
        if self.a_lo is not None:
            ps.append((self.a_lo.double(), self.b))
        if self.b_lo is not None:
            ps.append((self.a, self.b_lo.double()))
        if pass1_hi and len(ps) > 1:
            ps[1] = (self.a, self.b)
        return ps

    def kblocks(self, s=None):
        """Virtual 64-deep k-blocks (pass, k0, k1) of split s (None: all) in the kernel's split-K walk."""
        rk = -(-self.K // 64)
        nk = rk * len(self.passes())
        kps = -(-nk // self.split) if self.split > 1 else nk
        vb = range(nk) if s is None else range(s * kps, min((s + 1) * kps, nk))
        return [(v // rk, (v % rk) * 64, min((v % rk) * 64 + 64, self.K)) for v in vb]

    def contract(self, blocks, pass1_hi=False):
        """alpha * sum over blocks of A_p[:, k0:k1] B_p[:, k0:k1]^T and its magnitude |alpha| sum |a b| (float64)."""
        ps = self.passes(pass1_hi)
        x = torch.zeros(self.M, self.N, dtype=F64, device=self.dev)
        s = torch.zeros_like(x)
        merged = []
        for p, k0, k1 in blocks:
            if merged and merged[-1][0] == p and merged[-1][2] == k0:
                merged[-1][2] = k1
            else:
                merged.append([p, k0, k1])
        for p, k0, k1 in merged:
            A, B = ps[p][0][:, k0:k1], ps[p][1][:, k0:k1]
            x += A @ B.t()
            s += A.abs() @ B.abs().t()
        return self.alpha * x, abs(self.alpha) * s

    def c_acc(self, blocks):
        """GEMM_C_ACC (GEMM_C_SPLIT in split precision) times sqrt(16-deep k-steps accumulated over `blocks`)."""
        n = sum(-(-(k1 - k0) // 16) for _, k0, k1 in blocks)
        return (GEMM_C_ACC if len(self.passes()) == 1 else GEMM_C_SPLIT) * math.sqrt(max(n, 1))

    def reference(self, drop_last_lo_kblock=False, pass1_hi=False, no_bias=False, res_rows_down=0, res_ld=None, lose_last_chunk=False):
        """dict(y, ey, S) of the fp32 value (out_f32 region shape), plus pre / epre (gelu'(pre)) and col / ecol (column sums).
        The keyword arguments build the wrong references."""
        M, N = self.M, self.N
        r = {}
        if self.atomic == L.VB_GEMM_PARTIALS:
            ys = [self.contract(self.kblocks(s)) for s in range(self.split)]
            r["y"], S = torch.cat([y for y, _ in ys]), torch.cat([s for _, s in ys])
            r["cS"] = torch.cat([torch.full((self.M, 1), self.c_acc(self.kblocks(s)), dtype=F64, device=self.dev) for s in range(self.split)]) * S
            r["ey"], r["S"] = U24 * r["cS"], S
            return self._lose(r) if lose_last_chunk else r
        blocks = self.kblocks()
        c = self.c_acc(blocks)
        if drop_last_lo_kblock:
            rk = -(-self.K // 64)
            blocks = [b for i, b in enumerate(blocks) if i != 2 * rk - 1]
        x, S = self.contract(blocks, pass1_hi)
        extra = 0.0
        if "bias" in self.fields and not no_bias:
            bias = self.region["bias"].double()
            x, S = x + bias, S + bias.abs()
        if self.act == L.VB_ACT_GELU:
            cdf = 0.5 * (1 + torch.erf(x / math.sqrt(2)))
            r["pre"] = cdf + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
            r["epre"] = 0.8 * c * U24 * S + GEMM_ERF
            extra = GEMM_ERF * x.abs()
            x, S = x * cdf, 1.13 * S
        elif self.act == L.VB_ACT_RELU:
            x = x.clamp_min(0)
        elif self.act == L.VB_ACT_DGELU:
            aux = self.region["aux"].double()
            x, S = x * aux, S * aux.abs()
        if self.drop is not None:
            k = keep_scale(M, N, self.drop[0], int(self.ctr.item()), self.drop[1], self.dev)
            x, S, extra = x * k, S * k, extra * k
        if "out_colsum" in self.outs:
            base = self.start("out_colsum").double()[0]
            adds = -(-M // 16) + 8
            r["col"] = base + x.sum(0)
            r["ecol"] = U24 * (c * S.sum(0) + adds * (base.abs() + x.abs().sum(0)))
        if "residual" in self.fields:
            if res_ld is not None:
                res = self.res0.flatten()[:M * res_ld].view(M, res_ld)[:, :N].double()
            else:
                res = self.res0[res_rows_down:res_rows_down + M, :N].double()
            x, S = x + res, S + res.abs()
        if self.atomic == 1:
            base = self.start("out_f32").double()
            x, S = x + base, (S + base.abs()) * (1 + self.split / c)
        r["y"], r["S"], r["ey"] = x, S, c * U24 * S + extra
        r["cS"] = c * S
        return self._lose(r) if lose_last_chunk else r

    def _lose(self, r):
        """The last 16-row epilogue chunk of the last row block never written: the reference holds 0 there."""
        m0 = (self.M - 1) // 16 * 16
        for k in ("y", "pre"):
            if k in r:
                r[k] = r[k].clone()
                r[k][m0:self.M] = 0
        return r

    # ---------------------------------------------------------------------------------- verdict
    def errors(self, ref=None):
        """{check: value}, each to be <= its tolerance in GEMM_TOLS: fp32 and column sums as error / bound, 16-bit outputs as the
        largest distance outside the correctly rounded window in units of the bound (0 = correctly rounded everywhere),
        'unwritten' / 'guard' as element counts (in-range elements still holding the sentinel / out-of-range elements changed).
        Also 'c_f32' (|got - v| / (2^-24 S), the calibration figure) and 'exact' (share of 16-bit elements held bitwise)."""
        r = ref if ref is not None else self.reference()
        e, exact = {}, []
        y, ey = r["y"], r["ey"].clamp_min(1e-300)
        if "out_f32" in self.outs:
            d = torch.nan_to_num((self.region["out_f32"].double() - y).abs(), nan=math.inf)
            e["out_f32"] = _worst(d, ey)
            e["c_f32"] = (d / (U24 * r["cS"]).clamp_min(1e-300)).max().item() * (GEMM_C_ACC if len(self.passes()) == 1 else GEMM_C_SPLIT)
        # with an fp32 output beside them, the 16-bit outputs must also be bitwise the rounding of the fp32 value written
        v32 = self.region["out_f32"].double() if "out_f32" in self.outs and not self.atomic else None
        def held(f, dt, shift=0.0):
            dist, ex = window16(self.region[f], y, ey, dt, shift)
            if v32 is not None:
                dist = torch.maximum(dist, window16(self.region[f], v32, 0.0, dt, shift)[0])
            e[f] = _worst(dist, ey)
            return ex
        if "out_bf16" in self.outs:
            exact.append(held("out_bf16", self.dt["out_bf16"]))
            if "out_lo" in self.outs:
                held("out_lo", self.dt["out_bf16"], shift=self.region["out_bf16"].double())
        if "out_b16" in self.outs:
            exact.append(held("out_b16", BF))
        if "out_pre" in self.outs:
            dist, ex = window16(self.region["out_pre"], r["pre"], r["epre"], BF)
            e["out_pre"] = _worst(dist, r["epre"])
            exact.append(ex)
        if "out_colsum" in self.outs:
            d = torch.nan_to_num((self.region["out_colsum"].double()[0] - r["col"]).abs(), nan=math.inf)
            e["out_colsum"] = _worst(d, r["ecol"])
        e["unwritten"] = sum(int((_bits(self.region[f]) == _sentinel(self.dt.get(f, torch.float32)).to(self.dev)).sum())
                             for f in self.outs)
        e["guard"] = sum(int((_bits(self.raw[f]) != _bits(self.init[f]))[~self.inside[f]].sum()) for f in self.outs)
        if exact:
            e["exact"] = torch.cat([x.flatten() for x in exact]).double().mean().item()
        return e


GEMM_TOLS = dict(out_f32=1.0, out_bf16=0.0, out_lo=0.0, out_b16=0.0, out_pre=0.0, out_colsum=1.0, unwritten=0, guard=0)
GEMM_VALUE_CHECKS = ("out_f32", "out_bf16", "out_lo", "out_b16", "out_pre", "out_colsum")
REF_OF = dict(out_f32="y", out_bf16="y", out_lo="y", out_b16="y", out_pre="pre", out_colsum="col")


def gemm_wrongs(case):
    """The plausible wrong references that apply to a case: {label: reference}."""
    w = {"last 16-row chunk lost": case.reference(lose_last_chunk=True)}
    if "bias" in case.fields:
        w["bias omitted"] = case.reference(no_bias=True)
    if "residual" in case.fields:
        w["residual one row down"] = case.reference(res_rows_down=1)
        if case.ld["residual"] != case.N:
            w["residual at pitch N"] = case.reference(res_ld=case.N)
    if (case.a_lo is not None or case.b_lo is not None) and case.atomic != L.VB_GEMM_PARTIALS:
        w["pass 1 on the hi parts"] = case.reference(pass1_hi=True)
        if case.K <= 256:     # past that, one 64-deep k-block of a low part is within the accumulation error the bound admits
            w["last lo-pass k-block dropped"] = case.reference(drop_last_lo_kblock=True)
    return w


def gemm_verdict(case, label, expect=None, wrongs=True, quiet=False):
    """Runs the case (under the profiler when expect, a kernel-name pattern, is given, and asserts that kernel), checks it against
    its float64 reference and every applicable wrong reference (each must miss by more than 10x the tolerance; a 16-bit output
    must differ from the truncated (RZ) reference on at least a third of the elements held bitwise: RZ and RN agree where the
    dropped bits are below half an ulp, about half of them), prints one line and asserts. Returns the errors."""
    if expect:
        launched(case.run, expect)
    else:
        case.run()
    torch.cuda.synchronize()
    ref = case.reference()
    e = case.errors(ref)
    we = {}
    if wrongs:
        for lab, wr in gemm_wrongs(case).items():
            x = case.errors(wr)
            # the outputs whose reference this wrong one changes (a residual read elsewhere leaves the column sums alone)
            we[lab] = {k: x[k] for k in GEMM_VALUE_CHECKS if k in x and not torch.equal(wr[REF_OF[k]], ref[REF_OF[k]])}
    rz = None
    if wrongs and "out_bf16" in case.outs and "out_lo" not in case.outs:
        _, ex = window16(case.region["out_bf16"], ref["y"], ref["ey"], case.dt["out_bf16"])
        rzv = rz16(ref["y"], case.dt["out_bf16"])
        rz = (_bits(rzv) != _bits(case.region["out_bf16"]))[ex].double().mean().item() if ex.any() else 1.0
    if not quiet:
        chk = ",".join(f"{k}={e[k]:.2e}" for k in GEMM_VALUE_CHECKS if k in e)
        w = "  ".join(f"{lab}:" + ",".join(f"{k}={v:.1e}" for k, v in x.items()) for lab, x in we.items())
        print(f"\n[gemm] {label} | bn {case.bn} split {case.split} | err/tol {chk} c_f32={e.get('c_f32', 0):.2f} "
              f"exact={e.get('exact', 0):.2f} unwritten={e['unwritten']} guard={e['guard']}" + (f" rz-miss={rz:.2f}" if rz is not None else "")
              + f" | wrong {w}")
    for k, tol in GEMM_TOLS.items():
        if k in e:
            assert e[k] <= tol, (label, k, e[k], tol, e)
    for lab, x in we.items():
        for k, v in x.items():
            assert v > 10 * max(GEMM_TOLS[k], 1.0), (label, lab, k, v)
    if rz is not None:
        assert rz > 1 / 3, (label, "truncating reference agrees", rz)
    return e


def gemm_case(M, N, K, a_mn=False, b_mn=False, bias=False, res=False, act=0, out_bf16=False, atomic=False, split_k=1, block_n=0,
              alpha=1.0, check=True, iters=0, seed=0, both_outputs=False, a_fp16=False, b_fp16=False, out_fp16=False,
              split=False):
    """Returns (largest error past the correctly rounded result relative to max|v|, ms per launch or None). check=True runs the
    float64 checker (GemmCase, gemm_verdict) and asserts it, with the kernel width vb_gemm_plan resolves. a_fp16 / b_fp16 /
    out_fp16 pick fp16 instead of bf16 (wgmma takes one format for both operands); split=True stores A and B as hi + lo."""
    assert a_fp16 == b_fp16
    outs = []
    if (not out_bf16) or atomic or both_outputs:      # like the engine: a 16-bit-output GEMM has no fp32 output unless asked
        outs.append("out_f32")
    if out_bf16 and not atomic:
        outs.append("out_bf16")
        if split:
            outs.append("out_lo")
        if out_fp16:
            outs.append("out_b16")                    # the bf16 copy for the backward
        if act == L.VB_ACT_GELU and N % 8 == 0:
            outs.append("out_pre")
    case = GemmCase(M, N, K, outs=outs, a_mn=a_mn, b_mn=b_mn, fp16=a_fp16, out_fp16=out_fp16, alpha=alpha, bias=bias, act=act,
                    res=res, a_lo=split, b_lo=split, atomic=int(atomic), split_k=split_k, block_n=block_n, seed=seed)
    err = None
    if check:
        e = gemm_verdict(case, f"{M}x{N}x{K} {' '.join(f for f in case.fields if f not in ('A', 'B'))} act={act} "
                         f"{'fp16' if a_fp16 else 'bf16'}{' A^T' if a_mn else ''}{' B^T' if b_mn else ''}",
                         expect=rf"gemm_wgmma_kernel<{case.bn}, ")
        ref = case.reference()
        err = max(e.get(k, 0.0) for k in GEMM_VALUE_CHECKS) * ref["ey"].max().item() / (ref["y"].abs().max().item() + 1e-9)
    else:
        case.run()
    ms = None
    if iters:
        lib = L.lib()
        for _ in range(3): lib.vb_gemm_bf16(C.byref(case.g), stream())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        torch.cuda._sleep(int(4e6))          # hold the GPU so that the launches below are queued ahead (kernel time, not launch rate)
        e0.record()
        for _ in range(iters): lib.vb_gemm_bf16(C.byref(case.g), stream())
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
    return err, ms


# ------------------------------------------------------------------------------------------ attention
def attn_case(B, H, Nq, Nk, D, cross, peaked=1.0, iters=0, seed=0, fp16=False, split=False):
    """Returns (dict of relative errors of O, dQ, dK, dV, lse vs fp32 torch on the same 16-bit inputs, timing str).
    fp16: Q/K/V/O are fp16 (gradients stay bf16). split: Q/K/V given as hi + lo, O checked as hi + lo against the
    fp32 inputs (forward only carries the low parts)."""
    dev = torch.device("cuda"); lib = L.lib()
    g_ = torch.Generator(device=dev).manual_seed(seed)
    Hd = H * D
    DT = torch.float16 if fp16 else BF
    if cross:
        q32 = torch.randn(B * Nq, 3 * Hd, device=dev, generator=g_) * peaked
        k32 = torch.randn(B * Nk, 3 * Hd, device=dev, generator=g_) * peaked
        qsrc, ksrc = q32.to(DT), k32.to(DT)
    else:
        q32 = k32 = torch.randn(B * Nq, 3 * Hd, device=dev, generator=g_) * peaked
        qsrc = ksrc = q32.to(DT)
    q, k, v = qsrc[:, :Hd], ksrc[:, Hd:2 * Hd], ksrc[:, 2 * Hd:]
    if split:
        qlo_src, klo_src = (q32 - qsrc.float()).to(DT), (k32 - ksrc.float()).to(DT)
    lens = torch.randint(1, Nk + 1, (B,), device=dev, generator=g_); lens[0] = Nk
    if B > 1: lens[1] = 1                                                 # a row with a single valid key
    mask = ((torch.arange(Nk, device=dev)[None] >= lens[:, None]).float() * -10000.0).contiguous()
    Ot = torch.zeros(B * Nq, Hd, device=dev, dtype=DT); lse = torch.zeros(B, H, Nq, device=dev)
    Olo = torch.zeros(B * Nq, Hd, device=dev, dtype=DT) if split else None
    Ob = torch.zeros(B * Nq, Hd, device=dev, dtype=BF) if fp16 else None
    dO = torch.randn(B * Nq, Hd, device=dev, generator=g_).to(BF)
    dqb = torch.zeros(B * Nq, 3 * Hd, device=dev, dtype=BF); dkb = torch.zeros(B * Nk, 3 * Hd, device=dev, dtype=BF)
    delta = torch.zeros(B, H, Nq, device=dev)
    a = L.AttnArgs()
    a.B, a.H, a.Nq, a.Nk, a.D = B, H, Nq, Nk, D
    a.Q, a.ldq, a.K, a.ldk, a.V, a.ldv = q.data_ptr(), 3 * Hd, k.data_ptr(), 3 * Hd, v.data_ptr(), 3 * Hd
    a.mask, a.scale = mask.data_ptr(), 1.0 / math.sqrt(D)
    a.O, a.ldo, a.lse = Ot.data_ptr(), Hd, lse.data_ptr()
    a.dO, a.lddo = dO.data_ptr(), Hd
    a.dQ, a.lddq = dqb[:, :Hd].data_ptr(), 3 * Hd
    a.dK, a.lddk = dkb[:, Hd:2 * Hd].data_ptr(), 3 * Hd
    a.dV, a.lddv = dkb[:, 2 * Hd:].data_ptr(), 3 * Hd
    a.delta = delta.data_ptr()
    a.qkv_fp16 = int(fp16)
    if split:
        a.Q_lo, a.K_lo, a.V_lo = qlo_src[:, :Hd].data_ptr(), klo_src[:, Hd:2 * Hd].data_ptr(), klo_src[:, 2 * Hd:].data_ptr()
        a.O_lo = Olo.data_ptr()
    if Ob is not None:
        a.O_b16 = Ob.data_ptr()
    L.check(lib.vb_attention_fwd(C.byref(a), stream()), "vb_attention_fwd")
    L.check(lib.vb_attention_bwd(C.byref(a), stream()), "vb_attention_bwd")
    torch.cuda.synchronize()
    def ref(qq, kk, vv):
        qf = qq.float().view(B, Nq, H, D).permute(0, 2, 1, 3).detach().requires_grad_(True)
        kf = kk.float().view(B, Nk, H, D).permute(0, 2, 1, 3).detach().requires_grad_(True)
        vf = vv.float().view(B, Nk, H, D).permute(0, 2, 1, 3).detach().requires_grad_(True)
        s = qf @ kf.transpose(-1, -2) / math.sqrt(D) + mask[:, None, None, :]
        p = torch.softmax(s, -1)
        o = (p @ vf).permute(0, 2, 1, 3).reshape(B * Nq, Hd)
        o.backward(dO.float())
        return qf, kf, vf, s, o.detach()
    qf, kf, vf, s, o = ref(q, k, v)
    if fp16:
        # the backward kernels contract in bf16 (dO / dS are bf16 operands): their Q / K / V panels are the fp16 values rounded to
        # bf16, so the gradient reference is the attention of those rounded inputs; the forward reference keeps the fp16 values
        qf, kf, vf, _, _ = ref(q.to(BF), k.to(BF), v.to(BF))
    if split:
        # forward against the fp32 (hi + lo) inputs; the backward of split precision contracts the hi parts only
        qs = q32[:, :Hd].view(B, Nq, H, D).permute(0, 2, 1, 3); ks = k32[:, Hd:2 * Hd].view(B, Nk, H, D).permute(0, 2, 1, 3)
        vs = k32[:, 2 * Hd:].view(B, Nk, H, D).permute(0, 2, 1, 3)
        s32 = qs.double() @ ks.double().transpose(-1, -2) / math.sqrt(D) + mask[:, None, None, :].double()
        o32 = (torch.softmax(s32, -1) @ vs.double()).permute(0, 2, 1, 3).reshape(B * Nq, Hd).float()
        o_split = rel(Ot.float() + Olo.float(), o32)
    # dQ and dK are products of dS = P o (dP - delta), which is 0 in exact arithmetic when every row has one key (Nk = 1): their
    # error is measured against a floor of 1e-3 of the dV scale, so rounding residue of size ~1e-6 is not divided by ~0
    gfloor = 1e-3 * vf.grad.abs().max().item()
    relg = lambda a, b: ((a.float() - b.float()).abs().max() / max(b.float().abs().max().item(), gfloor, 1e-20)).item()
    errs = dict(O=rel(Ot, o), dQ=relg(dqb[:, :Hd].view(B, Nq, H, D).permute(0, 2, 1, 3), qf.grad),
                dK=relg(dkb[:, Hd:2 * Hd].view(B, Nk, H, D).permute(0, 2, 1, 3), kf.grad),
                dV=rel(dkb[:, 2 * Hd:].view(B, Nk, H, D).permute(0, 2, 1, 3), vf.grad),
                lse=rel(lse * math.log(2.0), torch.logsumexp(s, -1)))
    if split:
        errs["O_split"] = o_split
    if Ob is not None:
        errs["O_b16"] = max(rel(Ob, o) - 4e-3, 0.0)
    timing = ""
    if iters:
        for fn, nm in ((lib.vb_attention_fwd, "fwd"), (lib.vb_attention_bwd, "bwd")):
            e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
            for _ in range(3): fn(C.byref(a), stream())
            e0.record()
            for _ in range(iters): fn(C.byref(a), stream())
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / iters
            fl = 4.0 * B * H * Nq * Nk * D * (1 if nm == "fwd" else 2.5)
            timing += f" {nm} {ms*1e3:.1f}us {fl/ms/1e9:.1f}TF"
    return errs, timing


# ------------------------------------------------------------------------------------------ full model
def build_engine(cfgj, P, device, precision="fp16"):
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    eng = Engine(BertConfig.from_dict(cfgj), device, precision=precision)
    for k in eng.ps.entries:
        eng.ps.p(k).copy_(P[k])
    eng.refresh_weights()
    return eng


def oracle_args(inp):
    return (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
            inp["image_attention_mask"], inp["co_attention_mask"], inp["task_ids"])


def probe_loss(heads, names, tgt):
    """VQA loss on vil_prediction + a small quadratic on every other requested head (touches every grad path)."""
    l = 0
    for n, h in zip(O.HEAD_NAMES, heads):
        if n in names:
            l = l + (O.vqa_loss(h, tgt) if n == "vil_prediction" else 0.1 * h.float().clamp(-50, 50).pow(2).mean())
    return l


def model_case(cfgj, B, Nv, Nt, seed=0, qk_scale=1.0, names=None, grads=True, device="cuda", train_step=None, precision="fp16",
               oracle_modes=("fp32", "op"), head_dropout_prob=None):
    """Engine vs the oracle in fp32 and in the engine's operand-rounding mode ("op": fp16 forward / bf16 gradient operands for
    precision "fp16" and "fp32", all-bf16 for "bf16"). Returns dict(out_fp32, out_op, grad_fp32, grad_op, ...)
    where each is {tensor name: error}; gradient errors are (max-rel with floor, rel-L2).
    train_step=k runs the engine in TRAIN mode (every nn.Dropout of the reference active, dropout step counter = k) against
    the oracle with the same stateless masks (oracle.DropMasks(k))."""
    # engines and plans of earlier cases hold each other in reference cycles: collect them before building a new one, an 80 GB
    # card does not hold several full-size engines at once
    gc.collect()
    torch.cuda.empty_cache()
    dev = torch.device(device)
    cfg = O.make_config(cfgj)
    names = O.HEAD_NAMES if names is None else names
    P = O.synth_params(cfg, seed=seed, device=dev, qk_scale=qk_scale)
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=1234 + seed, device=dev)
    eng = build_engine(cfgj, P, dev, precision)
    if head_dropout_prob is not None:
        eng.head_dropout_prob = head_dropout_prob     # VILBertForVLTasks(dropout_prob=...)
    drop = None
    if train_step is not None:
        eng.drop_step.fill_(int(train_step))
        drop = O.DropMasks(train_step, head_p=eng.head_dropout_prob)
    plan = eng.plan(B, Nt, Nv, grad_outputs=names if grads else (), train=train_step is not None)
    plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                     inp["image_attention_mask"], inp["task_ids"])
    plan.run_forward()
    torch.cuda.synchronize()
    tgt = O.synth_vqa_target(B, 3129, device=dev)
    result = dict(plan=plan, engine=eng)
    mine_heads = [plan.outputs[n].detach().clone().requires_grad_(True) for n in O.HEAD_NAMES]
    if grads:
        lm = probe_loss(mine_heads, names, tgt); lm.backward()
        eng.zero_grad()
        for n, t in zip(O.HEAD_NAMES, mine_heads):
            if n in names:
                plan.gout[n].copy_(t.grad.reshape(plan.gout[n].shape))
        plan.run_backward()
        torch.cuda.synchronize()
        result["loss"] = lm.item()
    for mode in oracle_modes:
        Pg = {k: v.clone().requires_grad_(True) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
        Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
        if mode == "op":
            with (O.bf16_operand_mode() if precision == "bf16" else O.operand_mode()):
                bert_o, heads_o = O.vilbert_for_vl_tasks(Pg, cfg, *oracle_args(inp), drop=drop)
                if grads:
                    lo = probe_loss(heads_o, names, tgt); lo.backward()
        else:
            bert_o, heads_o = O.vilbert_for_vl_tasks(Pg, cfg, *oracle_args(inp), drop=drop)
            if grads:
                lo = probe_loss(heads_o, names, tgt); lo.backward()
        oe = {}
        for n, r in list(zip(O.BERT_OUT_NAMES, bert_o)) + list(zip(O.HEAD_NAMES, heads_o)):
            oe[n] = rel(plan.outputs[n].reshape(r.shape), r)
        result["out_" + mode] = oe
        if grads:
            result["loss_" + mode] = lo.item()
            gmax = max(v.grad.abs().max().item() for v in Pg.values() if v.grad is not None)
            ge = {}
            for k in eng.ps.entries:
                rg, mg = Pg[k].grad, eng.ps.g(k)
                if rg is None:
                    ge[k] = (0.0 if mg.abs().max().item() == 0 else float("inf"), 0.0)
                    continue
                # gradients that are ~0 in exact arithmetic (key biases: softmax shift invariance) are compared
                # against a floor of 1e-3 of the largest gradient in the model
                floor = 1e-3 * gmax
                ge[k] = (((mg - rg).abs().max() / max(rg.abs().max().item(), floor)).item(),
                         ((mg - rg).norm() / max(rg.norm().item(), floor * math.sqrt(rg.numel()) * 0.1)).item())
            result["grad_" + mode] = ge
    return result
