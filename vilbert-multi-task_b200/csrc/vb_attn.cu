// vb_attn.cu — fused QK^T * scale + additive key mask -> softmax -> PV for the three attention
// flavours of ViLBERT (text self-attention vilbert.py:424-460, image self-attention :571-619,
// cross-modal BertBiAttention :771-809), forward and backward.
//
// Problem sizes are tiny per (batch, head): Nq, Nk <= ~320, head dim 64/128, so a whole K/V panel
// lives in shared memory and S / P never touch HBM. One CTA = (64-row query tile, head, batch) with
// 4 warps x 16 rows; tensor-core work uses warp-level mma.sync m16n8k16 (bf16 -> fp32) with ldmatrix
// operand fetch, row statistics via warp-shuffle online softmax over 64-key blocks. 1.8 % of the
// model FLOPs live here (SURVEY.md §8d); the wgmma path is reserved for the dense contractions.
// Q/K/V are read in place from the packed QKV GEMM output (row stride = ld, head offset h*D), so the
// reference's permute().contiguous() copies (vilbert.py:416-422, 447) never materialise.
//
// Backward (FlashAttention-2 style recompute): P = exp2(S*c + mask*log2e - lse2),
//   delta = rowsum(dO o O), dS = P o (dO V^T - delta), dQ = scale dS K, dK = scale dS^T Q, dV = P^T dO.
// Kernel "dq" owns a query tile and loops over key blocks; kernel "dkv" owns a key tile and loops over
// query blocks with the transposed products so that no atomics are needed (deterministic).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>
#include <stdlib.h>

#include "vb_internal.h"
#include "vb_ptx.cuh"

namespace vb {

constexpr float LOG2E = 1.4426950408889634f;
constexpr int ATT_THREADS = 128;
constexpr int TQ = 64;  // rows per CTA tile (4 warps x 16)
constexpr int KB = 64;  // keys per online-softmax block

struct AttnParams {
  int B, H, Nq, Nk;
  const __nv_bfloat16 *Q, *K, *V;
  long long ldq, ldk, ldv;
  const float* mask;
  float scale;
  __nv_bfloat16* O;
  long long ldo;
  float* lse;  // [B,H,Nq], log2 domain
  const __nv_bfloat16* dO;
  long long lddo;
  __nv_bfloat16 *dQ, *dK, *dV;
  long long lddq, lddk, lddv;
  float* delta;  // [B,H,Nq]
  DropCfg drop;            // dropout on the attention probabilities (element index ((b*H + h)*Nq + q)*Nk + k)
  float *dbq, *dbk, *dbv;  // optional bias gradients [H*D] of the Q / K / V projections (+= column sums of dQ / dK / dV)
  int qkv_fp16;            // Q, K, V, O are fp16 (forward operands); gradients are always bf16
  const __nv_bfloat16 *Ql, *Kl, *Vl;   // split precision (forward): low parts of Q / K / V, or NULL
  __nv_bfloat16* Ol;                   // low part of O, or NULL
  __nv_bfloat16* Ob;                   // always-bf16 copy of O, or NULL
  int kchunk;                          // forward: keys resident in shared memory at a time (multiple of KB; >= padded Nk = one pass)
  // packed rows (varlen): sample b's queries are rows qoff[b] + i, i < qlen[b], its keys rows koff[b] + j, j < klen[b]; NULL = the
  // padded layout (rows b * Nq + i, b * Nk + j). Nq / Nk stay the maxima: lse, delta and the dropout index are at padded coordinates
  const int *qoff, *qlen, *koff, *klen;
};

__device__ __forceinline__ long long q_row0(const AttnParams& p, int b) { return p.qoff ? (long long)p.qoff[b] : (long long)b * p.Nq; }
__device__ __forceinline__ long long k_row0(const AttnParams& p, int b) { return p.koff ? (long long)p.koff[b] : (long long)b * p.Nk; }
__device__ __forceinline__ int q_count(const AttnParams& p, int b) { return p.qoff ? p.qlen[b] : p.Nq; }
__device__ __forceinline__ int k_count(const AttnParams& p, int b) { return p.koff ? p.klen[b] : p.Nk; }

// In-place fp16 -> bf16 conversion of a staged panel (rows x D at pitch D + 8): the backward kernels run their products in
// bf16 because dO / dS are bf16 (gradient range), while Q / K / V arrive as fp16 forward operands.
template <int D, int NTHREADS>
__device__ __forceinline__ void panel_f16_to_bf16(__nv_bfloat16* panel, int rows) {
  constexpr int LD = D + 8;
  constexpr int CH = D / 8;
  for (int idx = threadIdx.x; idx < rows * CH; idx += NTHREADS) {
    uint4* ptr = reinterpret_cast<uint4*>(panel + (idx / CH) * LD + (idx % CH) * 8);
    uint4 v = *ptr;
    uint32_t* w = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = unpack16(w[i], 1); w[i] = pack_bf16(f.x, f.y); }
    *ptr = v;
  }
}

// Copies `rows_valid` rows of D bf16 (row stride ld) into smem rows of stride D+8 with cp.async (16-byte LDGSTS, no
// register staging: every request of the panel is in flight at once); rows beyond rows_valid are zero-filled
// (src-size 0). Completion: cp_async_wait_all() + __syncthreads().
template <int D, int NTHREADS = ATT_THREADS>
__device__ __forceinline__ void load_panel(__nv_bfloat16* dst, const __nv_bfloat16* src, long long ld, int rows_valid,
                                           int rows_total) {
  constexpr int LD = D + 8;
  constexpr int CH = D / 8;  // 16-byte chunks per row
  for (int idx = threadIdx.x; idx < rows_total * CH; idx += NTHREADS) {
    const int r = idx / CH, c = idx % CH;
    const bool ok = r < rows_valid;
    const __nv_bfloat16* g = src + (long long)(ok ? r : 0) * ld + c * 8;
    const uint32_t d = smem_u32(dst + r * LD + c * 8);
    const int nbytes = ok ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(g), "r"(nbytes) : "memory");
  }
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// acc[nt][4] (16 x 64 block, 8 n-tiles) = A(16 x D from sA rows a_row0..) * B^T where B rows b_row0.. (64 rows) of sB.
template <int D, bool FP16 = false>
__device__ __forceinline__ void mma_a_bt(float (&acc)[8][4], const __nv_bfloat16* sA, int a_row0, const __nv_bfloat16* sB,
                                         int b_row0, int lane, int /*nb_valid*/) {
  constexpr int LD = D + 8;
#pragma unroll
  for (int kk = 0; kk < D / 16; ++kk) {
    uint32_t a[4];
    ldmatrix_x4(a, smem_u32(sA + (a_row0 + (lane & 15)) * LD + kk * 16 + (lane >> 4) * 8));
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b[4];
      const int mi = lane >> 3;
      ldmatrix_x4(b, smem_u32(sB + (b_row0 + np * 16 + (mi >> 1) * 8 + (lane & 7)) * LD + kk * 16 + (mi & 1) * 8));
      mma_16816<FP16>(acc[2 * np], a, b[0], b[1]);
      mma_16816<FP16>(acc[2 * np + 1], a, b[2], b[3]);
    }
  }
}

// acc[D/8][4] (16 x D) += P(16 x 64, given as C-fragments pf[8][4] converted to bf16) * B where B rows b_row0.. (64 rows, k index) of sB [row][D].
// FP16: operand format. SPLIT: P is split into hi + lo in registers and sBl holds the low part of B: acc += Ph B + Pl B + Ph Bl.
template <int D, bool FP16 = false, bool SPLIT = false>
__device__ __forceinline__ void mma_p_b(float (&acc)[D / 8][4], const float (&pf)[8][4], const __nv_bfloat16* sB, int b_row0,
                                        int lane, int /*nb_valid*/, const __nv_bfloat16* sBl = nullptr) {
  constexpr int LD = D + 8;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t a[4], al[4];
    if constexpr (SPLIT) {
      a[0] = pack16_split(pf[2 * kk][0], pf[2 * kk][1], FP16, al[0]);
      a[1] = pack16_split(pf[2 * kk][2], pf[2 * kk][3], FP16, al[1]);
      a[2] = pack16_split(pf[2 * kk + 1][0], pf[2 * kk + 1][1], FP16, al[2]);
      a[3] = pack16_split(pf[2 * kk + 1][2], pf[2 * kk + 1][3], FP16, al[3]);
    } else {
      a[0] = pack16(pf[2 * kk][0], pf[2 * kk][1], FP16);
      a[1] = pack16(pf[2 * kk][2], pf[2 * kk][3], FP16);
      a[2] = pack16(pf[2 * kk + 1][0], pf[2 * kk + 1][1], FP16);
      a[3] = pack16(pf[2 * kk + 1][2], pf[2 * kk + 1][3], FP16);
    }
#pragma unroll
    for (int dp = 0; dp < D / 16; ++dp) {
      uint32_t b[4];
      const int mi = lane >> 3;
      const int off = (b_row0 + kk * 16 + (mi & 1) * 8 + (lane & 7)) * LD + dp * 16 + (mi >> 1) * 8;
      ldmatrix_x4_trans(b, smem_u32(sB + off));
      mma_16816<FP16>(acc[2 * dp], a, b[0], b[1]);
      mma_16816<FP16>(acc[2 * dp + 1], a, b[2], b[3]);
      if constexpr (SPLIT) {
        mma_16816<FP16>(acc[2 * dp], al, b[0], b[1]);
        mma_16816<FP16>(acc[2 * dp + 1], al, b[2], b[3]);
        ldmatrix_x4_trans(b, smem_u32(sBl + off));
        mma_16816<FP16>(acc[2 * dp], a, b[0], b[1]);
        mma_16816<FP16>(acc[2 * dp + 1], a, b[2], b[3]);
      }
    }
  }
}

// Stores a 16 x D fp32 C-fragment tile (scaled) as bf16 rows; rows >= rows_valid are skipped. If colsum != nullptr the
// column sums of the stored (valid, scaled) values are accumulated there (bias gradient of the projection).
template <int D>
__device__ __forceinline__ void store_tile(__nv_bfloat16* dst, long long ld, const float (&acc)[D / 8][4], float s0, float s1,
                                           int row0, int rows_valid, int lane, float* colsum = nullptr, int fp16 = 0,
                                           __nv_bfloat16* dst_lo = nullptr) {
  const int g = lane >> 2, t = lane & 3;
  const bool v0 = row0 + g < rows_valid, v1 = row0 + g + 8 < rows_valid;
#pragma unroll
  for (int nt = 0; nt < D / 8; ++nt) {
    const int col = nt * 8 + 2 * t;
    const float a0 = acc[nt][0] * s0, a1 = acc[nt][1] * s0, a2 = acc[nt][2] * s1, a3 = acc[nt][3] * s1;
    uint32_t l01 = 0, l23 = 0;
    const uint32_t h01 = dst_lo ? pack16_split(a0, a1, fp16, l01) : pack16(a0, a1, fp16);
    const uint32_t h23 = dst_lo ? pack16_split(a2, a3, fp16, l23) : pack16(a2, a3, fp16);
    if (v0) *reinterpret_cast<uint32_t*>(dst + (long long)(row0 + g) * ld + col) = h01;
    if (v1) *reinterpret_cast<uint32_t*>(dst + (long long)(row0 + g + 8) * ld + col) = h23;
    if (dst_lo) {
      if (v0) *reinterpret_cast<uint32_t*>(dst_lo + (long long)(row0 + g) * ld + col) = l01;
      if (v1) *reinterpret_cast<uint32_t*>(dst_lo + (long long)(row0 + g + 8) * ld + col) = l23;
    }
    if (colsum) {
      float c0 = (v0 ? a0 : 0.f) + (v1 ? a2 : 0.f), c1 = (v0 ? a1 : 0.f) + (v1 ? a3 : 0.f);
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {   // reduce over the 8 row groups (lane bits 2..4)
        c0 += __shfl_xor_sync(0xffffffffu, c0, o);
        c1 += __shfl_xor_sync(0xffffffffu, c1, o);
      }
      if (g == 0) { atomicAdd(colsum + col, c0); atomicAdd(colsum + col + 1, c1); }
    }
  }
}

// ------------------------------------------------------------------------------------------ forward
template <int D, bool FP16, bool SPLIT>
__global__ void __launch_bounds__(ATT_THREADS) attn_fwd_kernel(const AttnParams p) {
  constexpr int LD = D + 8;
  extern __shared__ __align__(16) uint8_t smem_att[];
  pdl_entry();
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * TQ;
  const int nq = q_count(p, b), nk = k_count(p, b);
  if (q0 >= nq) return;   // a query tile past this sample's rows (packed rows)
  const long long qr = q_row0(p, b) + q0, kr = k_row0(p, b);
  const int nkp = (nk + KB - 1) / KB * KB;
  const int kch = min(p.kchunk, nkp);   // keys resident at a time: the whole (padded) key range unless it does not fit (long
                                        // sequences in split precision), then chunks streamed through the same panels
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_att);
  __nv_bfloat16* sK = sQ + TQ * LD;
  __nv_bfloat16* sV = sK + kch * LD;
  // split precision: low-part panels behind the hi ones
  __nv_bfloat16* sQl = sV + kch * LD;
  __nv_bfloat16* sKl = sQl + (SPLIT ? TQ * LD : 0);
  __nv_bfloat16* sVl = sKl + (SPLIT ? kch * LD : 0);
  float* sMask = reinterpret_cast<float*>(sVl + (SPLIT ? kch * LD : 0));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;

  load_panel<D>(sQ, p.Q + qr * p.ldq + h * D, p.ldq, min(TQ, nq - q0), TQ);
  if constexpr (SPLIT) load_panel<D>(sQl, p.Ql + qr * p.ldq + h * D, p.ldq, min(TQ, nq - q0), TQ);
  for (int j = threadIdx.x; j < nkp; j += ATT_THREADS)
    sMask[j] = (j < nk) ? (p.mask ? p.mask[(long long)b * p.Nk + j] * LOG2E : 0.f) : -CUDART_INF_F;

  const int r0 = warp * 16;
  const bool active = q0 + r0 < nq;   // a warp whose 16 query rows are all out of range only helps with the loads

  const float c = p.scale * LOG2E;
  const uint32_t dseed = p.drop.ctr ? drop_seed(p.drop) : 0u;
  float m[2] = {-CUDART_INF_F, -CUDART_INF_F}, l[2] = {0.f, 0.f};
  float o[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;

  for (int k0 = 0; k0 < nkp; k0 += kch) {
    const int kc = min(kch, nkp - k0);
    const int kvalid = max(0, min(kc, nk - k0));
    if (k0 > 0) __syncthreads();   // every warp is done with the previous chunk's panels
    load_panel<D>(sK, p.K + (kr + k0) * p.ldk + h * D, p.ldk, kvalid, kc);
    load_panel<D>(sV, p.V + (kr + k0) * p.ldv + h * D, p.ldv, kvalid, kc);
    if constexpr (SPLIT) {
      load_panel<D>(sKl, p.Kl + (kr + k0) * p.ldk + h * D, p.ldk, kvalid, kc);
      load_panel<D>(sVl, p.Vl + (kr + k0) * p.ldv + h * D, p.ldv, kvalid, kc);
    }
    cp_async_wait_all();
    __syncthreads();
    if (!active) continue;

    for (int kb = 0; kb < kc; kb += KB) {
      float s[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      mma_a_bt<D, FP16>(s, sQ, r0, sK, kb, lane, p.Nk);
      if constexpr (SPLIT) {   // S = Q K^T + Q_lo K^T + Q K_lo^T
        mma_a_bt<D, FP16>(s, sQl, r0, sK, kb, lane, p.Nk);
        mma_a_bt<D, FP16>(s, sQ, r0, sKl, kb, lane, p.Nk);
      }
      float mx0 = -CUDART_INF_F, mx1 = -CUDART_INF_F;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float mk0 = sMask[k0 + kb + nt * 8 + 2 * t], mk1 = sMask[k0 + kb + nt * 8 + 2 * t + 1];
        s[nt][0] = s[nt][0] * c + mk0; s[nt][1] = s[nt][1] * c + mk1;
        s[nt][2] = s[nt][2] * c + mk0; s[nt][3] = s[nt][3] * c + mk1;
        mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
        mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
      }
      mx0 = quad_max(mx0); mx1 = quad_max(mx1);
      const float mn0 = fmaxf(m[0], mx0), mn1 = fmaxf(m[1], mx1);
      const float al0 = exp2f(m[0] - mn0), al1 = exp2f(m[1] - mn1);
      m[0] = mn0; m[1] = mn1;
      float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        s[nt][0] = exp2f(s[nt][0] - mn0); s[nt][1] = exp2f(s[nt][1] - mn0);
        s[nt][2] = exp2f(s[nt][2] - mn1); s[nt][3] = exp2f(s[nt][3] - mn1);
        rs0 += s[nt][0] + s[nt][1]; rs1 += s[nt][2] + s[nt][3];
      }
      l[0] = l[0] * al0 + rs0; l[1] = l[1] * al1 + rs1;
#pragma unroll
      for (int i = 0; i < D / 8; ++i) { o[i][0] *= al0; o[i][1] *= al0; o[i][2] *= al1; o[i][3] *= al1; }
      if (p.drop.ctr) {   // nn.Dropout on the probabilities (vilbert.py:443, 604, 778, 800): the row sum above stays undropped
        const uint32_t e0 = (uint32_t)((((long long)b * p.H + h) * p.Nq + q0 + r0 + g) * p.Nk + k0 + kb + 2 * t);
        const uint32_t e1 = e0 + 8u * (uint32_t)p.Nk;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          s[nt][0] *= drop_factor(dseed, e0 + nt * 8, p.drop); s[nt][1] *= drop_factor(dseed, e0 + nt * 8 + 1, p.drop);
          s[nt][2] *= drop_factor(dseed, e1 + nt * 8, p.drop); s[nt][3] *= drop_factor(dseed, e1 + nt * 8 + 1, p.drop);
        }
      }
      mma_p_b<D, FP16, SPLIT>(o, s, sV, kb, lane, p.Nk, sVl);
    }
  }
  if (!active) return;
  l[0] = quad_sum(l[0]); l[1] = quad_sum(l[1]);
  const int rows_valid = nq - q0;
  store_tile<D>(p.O + qr * p.ldo + h * D, p.ldo, o, 1.f / l[0], 1.f / l[1], r0, rows_valid, lane, nullptr,
                FP16 ? 1 : 0, (SPLIT && p.Ol) ? p.Ol + qr * p.ldo + h * D : nullptr);
  if (p.Ob) store_tile<D>(p.Ob + qr * p.ldo + h * D, p.ldo, o, 1.f / l[0], 1.f / l[1], r0, rows_valid, lane);
  if (p.lse && t == 0) {
    float* lse = p.lse + ((long long)b * p.H + h) * p.Nq + q0;
    if (r0 + g < rows_valid) lse[r0 + g] = m[0] + log2f(l[0]);
    if (r0 + g + 8 < rows_valid) lse[r0 + g + 8] = m[1] + log2f(l[1]);
  }
}

// ------------------------------------------------------------------------------------------ backward: dQ
// DQ = false (dK / dV-only backward): the kernel writes delta, which the dK / dV kernel reads, and nothing else; without dropout it
// stages only dO.
template <int D, bool DQ = true>
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_dq_kernel(const AttnParams p) {
  constexpr int LD = D + 8;
  extern __shared__ __align__(16) uint8_t smem_att[];
  pdl_entry();
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * TQ;
  const int nq = q_count(p, b), nk = k_count(p, b);
  if (q0 >= nq) return;
  const long long qr = q_row0(p, b) + q0, kr = k_row0(p, b);
  const int nkp = (nk + KB - 1) / KB * KB;
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_att);
  __nv_bfloat16* sdO = sQ + TQ * LD;
  __nv_bfloat16* sK = sdO + TQ * LD;
  __nv_bfloat16* sV = sK + nkp * LD;
  float* sMask = reinterpret_cast<float*>(sV + nkp * LD);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int rows_valid = min(TQ, nq - q0);
  const bool stage_qkv = DQ || p.drop.ctr;   // with dropout, delta is formed from P and dP (below)

  if (stage_qkv) load_panel<D>(sQ, p.Q + qr * p.ldq + h * D, p.ldq, rows_valid, TQ);
  load_panel<D>(sdO, p.dO + qr * p.lddo + h * D, p.lddo, rows_valid, TQ);
  if (stage_qkv) {
    load_panel<D>(sK, p.K + kr * p.ldk + h * D, p.ldk, nk, nkp);
    load_panel<D>(sV, p.V + kr * p.ldv + h * D, p.ldv, nk, nkp);
    for (int j = threadIdx.x; j < nkp; j += ATT_THREADS)
      sMask[j] = (j < nk) ? (p.mask ? p.mask[(long long)b * p.Nk + j] * LOG2E : 0.f) : -CUDART_INF_F;
  }
  cp_async_wait_all();
  __syncthreads();
  if (stage_qkv && p.qkv_fp16) {
    panel_f16_to_bf16<D, ATT_THREADS>(sQ, TQ); panel_f16_to_bf16<D, ATT_THREADS>(sK, nkp); panel_f16_to_bf16<D, ATT_THREADS>(sV, nkp);
    __syncthreads();
  }

  const int r0 = warp * 16;
  if (r0 >= rows_valid) return;

  float ls[2] = {0.f, 0.f};
  {
    const float* lse = p.lse + ((long long)b * p.H + h) * p.Nq + q0;
    if (r0 + g < rows_valid) ls[0] = lse[r0 + g];
    if (r0 + g + 8 < rows_valid) ls[1] = lse[r0 + g + 8];
  }
  const float c = p.scale * LOG2E;
  const uint32_t dseed = p.drop.ctr ? drop_seed(p.drop) : 0u;

  // delta = rowsum(dO o O) for rows g, g+8 of this warp; each quad lane sums a quarter of the columns.
  float dl[2] = {0.f, 0.f};
  if (p.drop.ctr) {
    // With dropout, rowsum(dO o O_b16) no longer cancels f dP on a peaked row (bf16(f V) != f bf16(V)): form delta from the same P
    // and f dP as the dS below, delta = sum_k P f dP / sum_k P (one extra pass of the two products over the keys)
    float sp[2] = {0.f, 0.f}, sd[2] = {0.f, 0.f};
    for (int kb = 0; kb < nkp; kb += KB) {
      float s[8][4], dp[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
        dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
      }
      mma_a_bt<D>(s, sQ, r0, sK, kb, lane, p.Nk);
      mma_a_bt<D>(dp, sdO, r0, sV, kb, lane, p.Nk);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float mk0 = sMask[kb + nt * 8 + 2 * t], mk1 = sMask[kb + nt * 8 + 2 * t + 1];
        const float p0 = exp2f(s[nt][0] * c + mk0 - ls[0]), p1 = exp2f(s[nt][1] * c + mk1 - ls[0]);
        const float p2 = exp2f(s[nt][2] * c + mk0 - ls[1]), p3 = exp2f(s[nt][3] * c + mk1 - ls[1]);
        const uint32_t e0 = (uint32_t)((((long long)b * p.H + h) * p.Nq + q0 + r0 + g) * p.Nk + kb + nt * 8 + 2 * t);
        const uint32_t e1 = e0 + 8u * (uint32_t)p.Nk;
        sp[0] += p0 + p1; sp[1] += p2 + p3;
        sd[0] += p0 * (dp[nt][0] * drop_factor(dseed, e0, p.drop)) + p1 * (dp[nt][1] * drop_factor(dseed, e0 + 1, p.drop));
        sd[1] += p2 * (dp[nt][2] * drop_factor(dseed, e1, p.drop)) + p3 * (dp[nt][3] * drop_factor(dseed, e1 + 1, p.drop));
      }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      sp[hh] = quad_sum(sp[hh]); sd[hh] = quad_sum(sd[hh]);
      dl[hh] = sp[hh] > 0.f ? sd[hh] / sp[hh] : 0.f;
    }
  } else {
    // delta = rowsum(dO o O) must cancel against dP = dO V^T formed from the bf16-rounded V: use the bf16 copy of O when the
    // forward wrote one (an fp16 O differs from P V_bf16 by the bf16 rounding of V, which peaked rows do not forgive)
    const int o_fp16 = p.Ob ? 0 : p.qkv_fp16;
    const __nv_bfloat16* Og = (p.Ob ? p.Ob : p.O) + qr * p.ldo + h * D;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = r0 + g + hh * 8;
      if (r < rows_valid) {
        float acc = 0.f;
        for (int cidx = t * 8; cidx < D; cidx += 32) {
          const uint4 ov = __ldg(reinterpret_cast<const uint4*>(Og + (long long)r * p.ldo + cidx));
          const uint4 dv = *reinterpret_cast<const uint4*>(sdO + r * LD + cidx);
          const uint32_t* o2 = reinterpret_cast<const uint32_t*>(&ov);
          const __nv_bfloat162* d2 = reinterpret_cast<const __nv_bfloat162*>(&dv);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 of = unpack16(o2[i], o_fp16), df = __bfloat1622float2(d2[i]);
            acc += of.x * df.x + of.y * df.y;
          }
        }
        dl[hh] = acc;
      }
    }
    dl[0] = quad_sum(dl[0]); dl[1] = quad_sum(dl[1]);
  }
  if (t == 0) {
    float* dg = p.delta + ((long long)b * p.H + h) * p.Nq + q0;
    if (r0 + g < rows_valid) dg[r0 + g] = dl[0];
    if (r0 + g + 8 < rows_valid) dg[r0 + g + 8] = dl[1];
  }
  if constexpr (!DQ) return;

  float dq[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;

  for (int kb = 0; kb < nkp; kb += KB) {
    float s[8][4], dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    }
    mma_a_bt<D>(s, sQ, r0, sK, kb, lane, p.Nk);
    mma_a_bt<D>(dp, sdO, r0, sV, kb, lane, p.Nk);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float mk0 = sMask[kb + nt * 8 + 2 * t], mk1 = sMask[kb + nt * 8 + 2 * t + 1];
      const float p0 = exp2f(s[nt][0] * c + mk0 - ls[0]), p1 = exp2f(s[nt][1] * c + mk1 - ls[0]);
      const float p2 = exp2f(s[nt][2] * c + mk0 - ls[1]), p3 = exp2f(s[nt][3] * c + mk1 - ls[1]);
      if (p.drop.ctr) {   // dP = mask/(1-p) * (dO V^T); delta was formed from these products above
        const uint32_t e0 = (uint32_t)((((long long)b * p.H + h) * p.Nq + q0 + r0 + g) * p.Nk + kb + nt * 8 + 2 * t);
        const uint32_t e1 = e0 + 8u * (uint32_t)p.Nk;
        dp[nt][0] *= drop_factor(dseed, e0, p.drop); dp[nt][1] *= drop_factor(dseed, e0 + 1, p.drop);
        dp[nt][2] *= drop_factor(dseed, e1, p.drop); dp[nt][3] *= drop_factor(dseed, e1 + 1, p.drop);
      }
      s[nt][0] = p0 * (dp[nt][0] - dl[0]); s[nt][1] = p1 * (dp[nt][1] - dl[0]);
      s[nt][2] = p2 * (dp[nt][2] - dl[1]); s[nt][3] = p3 * (dp[nt][3] - dl[1]);
    }
    mma_p_b<D>(dq, s, sK, kb, lane, p.Nk);
  }
  store_tile<D>(p.dQ + qr * p.lddq + h * D, p.lddq, dq, p.scale, p.scale, r0, rows_valid, lane,
                p.dbq ? p.dbq + h * D : nullptr);
}

// ------------------------------------------------------------------------------------------ backward: dK, dV
template <int D>
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_dkv_kernel(const AttnParams p) {
  constexpr int LD = D + 8;
  extern __shared__ __align__(16) uint8_t smem_att[];
  pdl_entry();
  const int b = blockIdx.z, h = blockIdx.y, k0 = blockIdx.x * TQ;
  const int nq = q_count(p, b), nk = k_count(p, b);
  if (k0 >= nk) return;
  const long long qr = q_row0(p, b), kr = k_row0(p, b) + k0;
  const int nqp = (nq + KB - 1) / KB * KB;
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(smem_att);
  __nv_bfloat16* sV = sK + TQ * LD;
  __nv_bfloat16* sQ = sV + TQ * LD;
  __nv_bfloat16* sdO = sQ + nqp * LD;
  float* sLse = reinterpret_cast<float*>(sdO + nqp * LD);
  float* sDelta = sLse + nqp;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int rows_valid = min(TQ, nk - k0);

  load_panel<D>(sK, p.K + kr * p.ldk + h * D, p.ldk, rows_valid, TQ);
  load_panel<D>(sV, p.V + kr * p.ldv + h * D, p.ldv, rows_valid, TQ);
  load_panel<D>(sQ, p.Q + qr * p.ldq + h * D, p.ldq, nq, nqp);
  load_panel<D>(sdO, p.dO + qr * p.lddo + h * D, p.lddo, nq, nqp);
  {
    const float* lse = p.lse + ((long long)b * p.H + h) * p.Nq;
    const float* dg = p.delta + ((long long)b * p.H + h) * p.Nq;
    for (int i = threadIdx.x; i < nqp; i += ATT_THREADS) {
      sLse[i] = (i < nq) ? lse[i] : CUDART_INF_F;  // +inf -> P = 0 for padded query columns
      sDelta[i] = (i < nq) ? dg[i] : 0.f;
    }
  }
  cp_async_wait_all();
  __syncthreads();
  if (p.qkv_fp16) {
    panel_f16_to_bf16<D, ATT_THREADS>(sK, TQ); panel_f16_to_bf16<D, ATT_THREADS>(sV, TQ); panel_f16_to_bf16<D, ATT_THREADS>(sQ, nqp);
    __syncthreads();
  }

  const int r0 = warp * 16;
  if (r0 >= rows_valid) return;

  float mk[2];
  mk[0] = (r0 + g < rows_valid && p.mask) ? p.mask[(long long)b * p.Nk + k0 + r0 + g] * LOG2E : 0.f;
  mk[1] = (r0 + g + 8 < rows_valid && p.mask) ? p.mask[(long long)b * p.Nk + k0 + r0 + g + 8] * LOG2E : 0.f;

  const float c = p.scale * LOG2E;
  const uint32_t dseed = p.drop.ctr ? drop_seed(p.drop) : 0u;
  float dk[D / 8][4], dv[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) {
    dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
    dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  }

  for (int qb = 0; qb < nqp; qb += KB) {
    float st[8][4], dpt[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      st[i][0] = st[i][1] = st[i][2] = st[i][3] = 0.f;
      dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f;
    }
    mma_a_bt<D>(st, sK, r0, sQ, qb, lane, p.Nq);     // S^T  = K Q^T   (rows = keys, cols = queries)
    mma_a_bt<D>(dpt, sV, r0, sdO, qb, lane, p.Nq);   // dP^T = V dO^T
    // P^T, then dV += P^T dO ; overwrite st with dS^T afterwards
    float pt[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int q = qb + nt * 8 + 2 * t;
      const float l0 = sLse[q], l1 = sLse[q + 1];
      pt[nt][0] = exp2f(st[nt][0] * c + mk[0] - l0); pt[nt][1] = exp2f(st[nt][1] * c + mk[0] - l1);
      pt[nt][2] = exp2f(st[nt][2] * c + mk[1] - l0); pt[nt][3] = exp2f(st[nt][3] * c + mk[1] - l1);
      const float d0 = sDelta[q], d1 = sDelta[q + 1];
      float f0 = 1.f, f1 = 1.f, f2 = 1.f, f3 = 1.f;
      if (p.drop.ctr) {   // transposed tile: row = key (g, g+8), column = query (q, q+1)
        const uint32_t eq0 = (uint32_t)((((long long)b * p.H + h) * p.Nq + q) * p.Nk + k0 + r0 + g);
        const uint32_t eq1 = eq0 + (uint32_t)p.Nk;
        f0 = drop_factor(dseed, eq0, p.drop); f1 = drop_factor(dseed, eq1, p.drop);
        f2 = drop_factor(dseed, eq0 + 8, p.drop); f3 = drop_factor(dseed, eq1 + 8, p.drop);
      }
      st[nt][0] = pt[nt][0] * (dpt[nt][0] * f0 - d0); st[nt][1] = pt[nt][1] * (dpt[nt][1] * f1 - d1);
      st[nt][2] = pt[nt][2] * (dpt[nt][2] * f2 - d0); st[nt][3] = pt[nt][3] * (dpt[nt][3] * f3 - d1);
      pt[nt][0] *= f0; pt[nt][1] *= f1; pt[nt][2] *= f2; pt[nt][3] *= f3;   // dV = (mask/(1-p) P)^T dO
    }
    mma_p_b<D>(dv, pt, sdO, qb, lane, p.Nq);
    mma_p_b<D>(dk, st, sQ, qb, lane, p.Nq);
  }
  store_tile<D>(p.dV + kr * p.lddv + h * D, p.lddv, dv, 1.f, 1.f, r0, rows_valid, lane, p.dbv ? p.dbv + h * D : nullptr);
  store_tile<D>(p.dK + kr * p.lddk + h * D, p.lddk, dk, p.scale, p.scale, r0, rows_valid, lane, p.dbk ? p.dbk + h * D : nullptr);
}


// ------------------------------------------------------------------------------------------ backward: single pass (short sequences)
// acc (16 x D) += A^T B with A^T[m][k] = sA[k0 + k][m0 + m] (sA row-major [k][m], pitch lda elements: the 16 x 16 A fragment
// is fetched with ldmatrix.trans) and B = sB rows k0.. ([k][D], pitch D + 8).
template <int D>
__device__ __forceinline__ void mma_at_b(float (&acc)[D / 8][4], const __nv_bfloat16* sA, int lda, int m0,
                                         const __nv_bfloat16* sB, int k0, int lane) {
  constexpr int LD = D + 8;
  const int mi = lane >> 3;
  uint32_t a[4];
  ldmatrix_x4_trans(a, smem_u32(sA + (k0 + (mi >> 1) * 8 + (lane & 7)) * lda + m0 + (mi & 1) * 8));
#pragma unroll
  for (int dp = 0; dp < D / 16; ++dp) {
    uint32_t b[4];
    ldmatrix_x4_trans(b, smem_u32(sB + (k0 + (mi & 1) * 8 + (lane & 7)) * LD + dp * 16 + (mi >> 1) * 8));
    mma_bf16_16816(acc[2 * dp], a, b[0], b[1]);
    mma_bf16_16816(acc[2 * dp + 1], a, b[2], b[3]);
  }
}

// One CTA per (batch, head) when Nq, Nk <= 128 (every attention of ViLBERT: 36-38 tokens, 100-101 regions): Q, dO, K, V of the
// head live in shared memory, S and dP are computed ONCE. Phase 1: warp w owns query rows [16w, 16w+16): P, dS per 64-key
// block from registers, dQ += dS K, and P (with the dropout factor) / dS are parked as bf16 [query][key] tiles in shared
// memory. Phase 2: warp w owns key rows [16w, 16w+16): dV = P^T dO and dK = dS^T Q over all queries (A fragments by
// ldmatrix.trans). No recompute, no atomics, deterministic; the two-kernel path below remains for longer sequences.
// Partial backward (a frozen side of a co-attention): DQ = false skips the dQ accumulation and its store; DKV = false skips phase 2
// and the P / dS tiles parked for it (and their shared memory). Every output written is bitwise the full backward's.
constexpr int ATT1_THREADS = 256;
template <int D, bool DQ = true, bool DKV = true>
__global__ void __launch_bounds__(ATT1_THREADS) attn_bwd_fused_kernel(const AttnParams p) {
  constexpr int LD = D + 8;
  extern __shared__ __align__(16) uint8_t smem_att[];
  pdl_entry();
  const int b = blockIdx.y, h = blockIdx.x;
  const int nq = q_count(p, b), nk = k_count(p, b);
  const long long qr = q_row0(p, b), kr = k_row0(p, b);
  const int nqp = (nq + 15) / 16 * 16;        // query rows staged (16-row warp tiles)
  const int nkp = (nk + KB - 1) / KB * KB;    // key rows staged (64-key blocks)
  const int LDP = nkp + 8;
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_att);
  __nv_bfloat16* sdO = sQ + nqp * LD;
  __nv_bfloat16* sK = sdO + nqp * LD;
  __nv_bfloat16* sV = sK + nkp * LD;
  __nv_bfloat16* sP = sV + nkp * LD;
  __nv_bfloat16* sdS = sP + nqp * LDP;
  // the P / dS tiles are staged for phase 2, and with dropout also for phase 1 (see there)
  float* sMask = reinterpret_cast<float*>((DKV || p.drop.ctr) ? sdS + nqp * LDP : sP);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;

  load_panel<D, ATT1_THREADS>(sQ, p.Q + qr * p.ldq + h * D, p.ldq, nq, nqp);
  load_panel<D, ATT1_THREADS>(sdO, p.dO + qr * p.lddo + h * D, p.lddo, nq, nqp);
  load_panel<D, ATT1_THREADS>(sK, p.K + kr * p.ldk + h * D, p.ldk, nk, nkp);
  load_panel<D, ATT1_THREADS>(sV, p.V + kr * p.ldv + h * D, p.ldv, nk, nkp);
  for (int j = threadIdx.x; j < nkp; j += ATT1_THREADS)
    sMask[j] = (j < nk) ? (p.mask ? p.mask[(long long)b * p.Nk + j] * LOG2E : 0.f) : -CUDART_INF_F;
  cp_async_wait_all();
  __syncthreads();
  if (p.qkv_fp16) {
    panel_f16_to_bf16<D, ATT1_THREADS>(sQ, nqp); panel_f16_to_bf16<D, ATT1_THREADS>(sK, nkp); panel_f16_to_bf16<D, ATT1_THREADS>(sV, nkp);
    __syncthreads();
  }

  const float c = p.scale * LOG2E;
  const uint32_t dseed = p.drop.ctr ? drop_seed(p.drop) : 0u;
  const int r0 = warp * 16;
  if (r0 < nqp) {
    // ---- phase 1: this warp's 16 query rows
    float dl[2] = {0.f, 0.f};   // delta = rowsum(dO o O)
    if (!p.drop.ctr) {
      const int o_fp16 = p.Ob ? 0 : p.qkv_fp16;      // see attn_bwd_dq_kernel: the bf16 copy of O keeps delta consistent with dP
      const __nv_bfloat16* Og = (p.Ob ? p.Ob : p.O) + qr * p.ldo + h * D;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = r0 + g + hh * 8;
        if (r < nq) {
          float acc = 0.f;
          for (int cidx = t * 8; cidx < D; cidx += 32) {
            const uint4 ov = __ldg(reinterpret_cast<const uint4*>(Og + (long long)r * p.ldo + cidx));
            const uint4 dv = *reinterpret_cast<const uint4*>(sdO + r * LD + cidx);
            const uint32_t* o2 = reinterpret_cast<const uint32_t*>(&ov);
            const __nv_bfloat162* d2 = reinterpret_cast<const __nv_bfloat162*>(&dv);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float2 of = unpack16(o2[i], o_fp16), df = __bfloat1622float2(d2[i]);
              acc += of.x * df.x + of.y * df.y;
            }
          }
          dl[hh] = acc;
        }
      }
      dl[0] = quad_sum(dl[0]); dl[1] = quad_sum(dl[1]);
    }
    float ls[2] = {CUDART_INF_F, CUDART_INF_F};   // +inf -> P = 0 on padded query rows (their tiles must be zero for phase 2)
    {
      const float* lse = p.lse + ((long long)b * p.H + h) * p.Nq;
      if (r0 + g < nq) ls[0] = lse[r0 + g];
      if (r0 + g + 8 < nq) ls[1] = lse[r0 + g + 8];
    }
    float dq[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
    if (p.drop.ctr) {
      // With dropout, rowsum(dO o O_b16) no longer cancels f dP on a peaked row: bf16(f V) != f bf16(V), so dS of a row with one
      // valid key would be bf16 noise instead of 0. Pass A parks P and f dP as bf16 tiles and forms delta from those same values,
      // delta = sum_k P f dP / sum_k P (the recomputed P normalised); pass B forms dS = P (f dP - delta) from the parked values, which
      // cancel exactly, and replaces the tiles by P f and dS for phase 2.
      float sp[2] = {0.f, 0.f}, sd[2] = {0.f, 0.f};
      for (int kb = 0; kb < nkp; kb += KB) {
        float s[8][4], dp[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
          dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
        }
        mma_a_bt<D>(s, sQ, r0, sK, kb, lane, p.Nk);
        mma_a_bt<D>(dp, sdO, r0, sV, kb, lane, p.Nk);
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const int col = kb + nt * 8 + 2 * t;
          const float mk0 = sMask[col], mk1 = sMask[col + 1];
          const uint32_t e0 = (uint32_t)((((long long)b * p.H + h) * p.Nq + r0 + g) * p.Nk + col);
          const uint32_t e1 = e0 + 8u * (uint32_t)p.Nk;
          const uint32_t pa = pack_bf16(exp2f(s[nt][0] * c + mk0 - ls[0]), exp2f(s[nt][1] * c + mk1 - ls[0]));
          const uint32_t pb = pack_bf16(exp2f(s[nt][2] * c + mk0 - ls[1]), exp2f(s[nt][3] * c + mk1 - ls[1]));
          const uint32_t da = pack_bf16(dp[nt][0] * drop_factor(dseed, e0, p.drop), dp[nt][1] * drop_factor(dseed, e0 + 1, p.drop));
          const uint32_t db = pack_bf16(dp[nt][2] * drop_factor(dseed, e1, p.drop), dp[nt][3] * drop_factor(dseed, e1 + 1, p.drop));
          *reinterpret_cast<uint32_t*>(sP + (r0 + g) * LDP + col) = pa;
          *reinterpret_cast<uint32_t*>(sP + (r0 + g + 8) * LDP + col) = pb;
          *reinterpret_cast<uint32_t*>(sdS + (r0 + g) * LDP + col) = da;
          *reinterpret_cast<uint32_t*>(sdS + (r0 + g + 8) * LDP + col) = db;
          const float2 P0 = unpack16(pa, 0), P1 = unpack16(pb, 0), F0 = unpack16(da, 0), F1 = unpack16(db, 0);
          sp[0] += P0.x + P0.y; sd[0] += P0.x * F0.x + P0.y * F0.y;
          sp[1] += P1.x + P1.y; sd[1] += P1.x * F1.x + P1.y * F1.y;
        }
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        sp[hh] = quad_sum(sp[hh]); sd[hh] = quad_sum(sd[hh]);
        dl[hh] = sp[hh] > 0.f ? sd[hh] / sp[hh] : 0.f;
      }
      for (int kb = 0; kb < nkp; kb += KB) {
        float s[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {   // each lane reads back the elements it parked in pass A
          const int col = kb + nt * 8 + 2 * t;
          uint32_t* pp0 = reinterpret_cast<uint32_t*>(sP + (r0 + g) * LDP + col);
          uint32_t* pp1 = reinterpret_cast<uint32_t*>(sP + (r0 + g + 8) * LDP + col);
          uint32_t* ps0 = reinterpret_cast<uint32_t*>(sdS + (r0 + g) * LDP + col);
          uint32_t* ps1 = reinterpret_cast<uint32_t*>(sdS + (r0 + g + 8) * LDP + col);
          const float2 P0 = unpack16(*pp0, 0), P1 = unpack16(*pp1, 0), F0 = unpack16(*ps0, 0), F1 = unpack16(*ps1, 0);
          s[nt][0] = P0.x * (F0.x - dl[0]); s[nt][1] = P0.y * (F0.y - dl[0]);
          s[nt][2] = P1.x * (F1.x - dl[1]); s[nt][3] = P1.y * (F1.y - dl[1]);
          if constexpr (DKV) {
            const uint32_t e0 = (uint32_t)((((long long)b * p.H + h) * p.Nq + r0 + g) * p.Nk + col);
            const uint32_t e1 = e0 + 8u * (uint32_t)p.Nk;
            *pp0 = pack_bf16(P0.x * drop_factor(dseed, e0, p.drop), P0.y * drop_factor(dseed, e0 + 1, p.drop));
            *pp1 = pack_bf16(P1.x * drop_factor(dseed, e1, p.drop), P1.y * drop_factor(dseed, e1 + 1, p.drop));
            *ps0 = pack_bf16(s[nt][0], s[nt][1]);
            *ps1 = pack_bf16(s[nt][2], s[nt][3]);
          }
        }
        if constexpr (DQ) mma_p_b<D>(dq, s, sK, kb, lane, p.Nk);
      }
    } else
    for (int kb = 0; kb < nkp; kb += KB) {
      float s[8][4], dp[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
        dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
      }
      mma_a_bt<D>(s, sQ, r0, sK, kb, lane, p.Nk);
      mma_a_bt<D>(dp, sdO, r0, sV, kb, lane, p.Nk);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int col = kb + nt * 8 + 2 * t;
        const float mk0 = sMask[col], mk1 = sMask[col + 1];
        float p0 = exp2f(s[nt][0] * c + mk0 - ls[0]), p1 = exp2f(s[nt][1] * c + mk1 - ls[0]);
        float p2 = exp2f(s[nt][2] * c + mk0 - ls[1]), p3 = exp2f(s[nt][3] * c + mk1 - ls[1]);
        float f0 = 1.f, f1 = 1.f, f2 = 1.f, f3 = 1.f;
        if (p.drop.ctr) {   // element index of the reference's dropout on the probabilities: ((b*H + h)*Nq + q)*Nk + k
          const uint32_t e0 = (uint32_t)((((long long)b * p.H + h) * p.Nq + r0 + g) * p.Nk + col);
          const uint32_t e1 = e0 + 8u * (uint32_t)p.Nk;
          f0 = drop_factor(dseed, e0, p.drop); f1 = drop_factor(dseed, e0 + 1, p.drop);
          f2 = drop_factor(dseed, e1, p.drop); f3 = drop_factor(dseed, e1 + 1, p.drop);
        }
        // dS = P o (mask/(1-p) o dP - delta); the tile kept for dV is mask/(1-p) o P
        s[nt][0] = p0 * (dp[nt][0] * f0 - dl[0]); s[nt][1] = p1 * (dp[nt][1] * f1 - dl[0]);
        s[nt][2] = p2 * (dp[nt][2] * f2 - dl[1]); s[nt][3] = p3 * (dp[nt][3] * f3 - dl[1]);
        if constexpr (DKV) {
          *reinterpret_cast<uint32_t*>(sP + (r0 + g) * LDP + col) = pack_bf16(p0 * f0, p1 * f1);
          *reinterpret_cast<uint32_t*>(sP + (r0 + g + 8) * LDP + col) = pack_bf16(p2 * f2, p3 * f3);
          *reinterpret_cast<uint32_t*>(sdS + (r0 + g) * LDP + col) = pack_bf16(s[nt][0], s[nt][1]);
          *reinterpret_cast<uint32_t*>(sdS + (r0 + g + 8) * LDP + col) = pack_bf16(s[nt][2], s[nt][3]);
        }
      }
      if constexpr (DQ) mma_p_b<D>(dq, s, sK, kb, lane, p.Nk);
    }
    if constexpr (DQ)
      store_tile<D>(p.dQ + qr * p.lddq + h * D, p.lddq, dq, p.scale, p.scale, r0, nq, lane,
                    p.dbq ? p.dbq + h * D : nullptr);
  }
  if constexpr (!DKV) return;
  __syncthreads();
  // ---- phase 2: this warp's 16 key rows
  if (r0 < nk) {
    float dk[D / 8][4], dv[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
      dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
    }
    for (int q = 0; q < nqp; q += 16) {
      mma_at_b<D>(dv, sP, LDP, r0, sdO, q, lane);
      mma_at_b<D>(dk, sdS, LDP, r0, sQ, q, lane);
    }
    store_tile<D>(p.dV + kr * p.lddv + h * D, p.lddv, dv, 1.f, 1.f, r0, nk, lane, p.dbv ? p.dbv + h * D : nullptr);
    store_tile<D>(p.dK + kr * p.lddk + h * D, p.lddk, dk, p.scale, p.scale, r0, nk, lane, p.dbk ? p.dbk + h * D : nullptr);
  }
}

// ------------------------------------------------------------------------------------------ probability export (visualization)
// P[b, h, q, :] = softmax(Q K^T * scale + mask) as fp32 — the tensor the reference returns as attn_data["attn"] when
// config.visualization is set (vilbert.py:451-458, 610-617, 813-821). Inspection path: one warp per (b, h, q) row, fp32 SIMT.
__global__ void __launch_bounds__(256) attn_probs_kernel(const AttnParams p, float* __restrict__ P, int D) {
  pdl_entry();
  extern __shared__ float sq[];            // [8 warps][D] query rows
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rows = (long long)p.B * p.H * p.Nq;
  float* myq = sq + warp * D;
  for (long long r = (long long)blockIdx.x * 8 + warp; r < rows; r += (long long)gridDim.x * 8) {
    const int q = (int)(r % p.Nq), h = (int)((r / p.Nq) % p.H), b = (int)(r / ((long long)p.Nq * p.H));
    const uint16_t* qrow = reinterpret_cast<const uint16_t*>(p.Q) + ((long long)b * p.Nq + q) * p.ldq + h * D;
    for (int d = lane; d < D; d += 32) myq[d] = cvt16_to_f32(qrow[d], p.qkv_fp16);
    __syncwarp();
    float* prow = P + r * p.Nk;
    float mx = -CUDART_INF_F;
    for (int k = lane; k < p.Nk; k += 32) {
      const uint16_t* krow = reinterpret_cast<const uint16_t*>(p.K) + ((long long)b * p.Nk + k) * p.ldk + h * D;
      float acc = 0.f;
      for (int d = 0; d < D; d += 8) {
        const uint4 kv = *reinterpret_cast<const uint4*>(krow + d);
        const uint32_t* w = reinterpret_cast<const uint32_t*>(&kv);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack16(w[i], p.qkv_fp16);
          acc += myq[d + 2 * i] * f.x + myq[d + 2 * i + 1] * f.y;
        }
      }
      const float s = acc * p.scale + (p.mask ? p.mask[(long long)b * p.Nk + k] : 0.f);
      prow[k] = s;
      mx = fmaxf(mx, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int k = lane; k < p.Nk; k += 32) { const float e = __expf(prow[k] - mx); prow[k] = e; sum += e; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.f / sum;
    for (int k = lane; k < p.Nk; k += 32) prow[k] *= inv;
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------ host
static inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int validate(const vb_attn_args* a, bool bwd) {
  if (!a) return set_error(VB_ERR_INVALID, "vb_attention: null args");
  if (a->B <= 0 || a->H <= 0 || a->Nq <= 0 || a->Nk <= 0) return set_error(VB_ERR_INVALID, "vb_attention: empty problem");
  if (a->D != 16 && a->D != 32 && a->D != 64 && a->D != 128)
    return set_error(VB_ERR_UNSUPPORTED, "vb_attention: head dim %d not in {16,32,64,128}", a->D);
  if (!a->Q || !a->K || !a->V || !a->O) return set_error(VB_ERR_INVALID, "vb_attention: null tensor");
  if (!a->q_off != !a->q_len || !a->q_off != !a->k_off || !a->q_off != !a->k_len)
    return set_error(VB_ERR_INVALID, "vb_attention: packed rows need q_off, q_len, k_off and k_len together");
  if (a->q_off && a->mask) return set_error(VB_ERR_INVALID, "vb_attention: packed rows take no additive mask (the lengths exclude the keys)");
  if ((a->ldq % 8) || (a->ldk % 8) || (a->ldv % 8) || (a->ldo % 8) || !al16(a->Q) || !al16(a->K) || !al16(a->V) || !al16(a->O))
    return set_error(VB_ERR_INVALID, "vb_attention: tensors need ld %% 8 == 0 and 16-byte aligned bases");
  if (bwd) {
    // partial output sets: dQ alone, or dK and dV together (either side of a co-attention may be frozen)
    if (!a->dQ && !a->dK && !a->dV) return set_error(VB_ERR_INVALID, "vb_attention_bwd: dQ, dK and dV are all NULL");
    if (!a->dK != !a->dV) return set_error(VB_ERR_INVALID, "vb_attention_bwd: dK and dV are computed together (both or neither)");
    if (!a->dO || !a->lse || !a->delta) return set_error(VB_ERR_INVALID, "vb_attention_bwd: null tensor");
    if ((a->lddo % 8) || !al16(a->dO) || (a->dQ && ((a->lddq % 8) || !al16(a->dQ))) ||
        (a->dK && ((a->lddk % 8) || (a->lddv % 8) || !al16(a->dK) || !al16(a->dV))))
      return set_error(VB_ERR_INVALID, "vb_attention_bwd: gradient tensors need ld %% 8 == 0 and 16-byte aligned bases");
  }
  return VB_OK;
}

static AttnParams to_params(const vb_attn_args* a) {
  AttnParams p;
  p.B = a->B; p.H = a->H; p.Nq = a->Nq; p.Nk = a->Nk;
  p.Q = (const __nv_bfloat16*)a->Q; p.K = (const __nv_bfloat16*)a->K; p.V = (const __nv_bfloat16*)a->V;
  p.ldq = a->ldq; p.ldk = a->ldk; p.ldv = a->ldv;
  p.mask = a->mask; p.scale = a->scale;
  p.O = (__nv_bfloat16*)a->O; p.ldo = a->ldo; p.lse = a->lse;
  p.dO = (const __nv_bfloat16*)a->dO; p.lddo = a->lddo;
  p.dQ = (__nv_bfloat16*)a->dQ; p.dK = (__nv_bfloat16*)a->dK; p.dV = (__nv_bfloat16*)a->dV;
  p.lddq = a->lddq; p.lddk = a->lddk; p.lddv = a->lddv;
  p.delta = a->delta;
  p.dbq = a->dbias_q; p.dbk = a->dbias_k; p.dbv = a->dbias_v;
  const bool on = a->dropout.step && a->dropout.p > 0.f;
  p.drop.ctr = on ? a->dropout.step : nullptr;
  p.drop.site = a->dropout.site;
  p.drop.thresh = on ? (uint32_t)((double)a->dropout.p * 4294967296.0) : 0u;
  p.drop.scale = on && a->dropout.p < 1.f ? 1.f / (1.f - a->dropout.p) : 1.f;
  p.qkv_fp16 = a->qkv_fp16 ? 1 : 0;
  p.Ql = (const __nv_bfloat16*)a->Q_lo; p.Kl = (const __nv_bfloat16*)a->K_lo; p.Vl = (const __nv_bfloat16*)a->V_lo;
  p.Ol = (__nv_bfloat16*)a->O_lo;
  p.Ob = (__nv_bfloat16*)a->O_b16;
  p.kchunk = 1 << 30;
  p.qoff = a->q_off; p.qlen = a->q_len; p.koff = a->k_off; p.klen = a->k_len;
  return p;
}

template <typename Kern>
static int launch_att(Kern kern, dim3 grid, size_t smem, const AttnParams& p, cudaStream_t s, const char* what, int threads = ATT_THREADS) {
  if (smem > 227 * 1024) return set_error(VB_ERR_UNSUPPORTED, "%s: sequence too long for the smem-resident panel (%zu bytes)", what, smem);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
  }
  cudaError_t e = launch_pdl(kern, grid, dim3(threads), smem, s, p);
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return VB_OK;
}

}  // namespace vb

extern "C" vb_status vb_attention_fwd(const vb_attn_args* a, void* stream) {
  using namespace vb;
  if (int s = validate(a, false)) return s;
  const AttnParams p = to_params(a);
  const int nkp = (a->Nk + KB - 1) / KB * KB;
  const bool split = a->Q_lo || a->K_lo || a->V_lo;
  if (split && !(a->Q_lo && a->K_lo && a->V_lo)) return set_error(VB_ERR_INVALID, "vb_attention_fwd: split precision needs Q_lo, K_lo and V_lo");
  if (split && (!al16(a->Q_lo) || !al16(a->K_lo) || !al16(a->V_lo) || (a->O_lo && !al16(a->O_lo))))
    return set_error(VB_ERR_INVALID, "vb_attention_fwd: low-part tensors need 16-byte aligned bases");
  // keys resident at a time: all of them when the panels fit, else the largest multiple of KB that does (streamed chunks)
  const size_t row_bytes = (size_t)(a->D + 8) * 2 * (split ? 2 : 1);
  const size_t fixed = (size_t)TQ * row_bytes + (size_t)nkp * 4;
  int kchunk = nkp;
  while (kchunk > KB && fixed + 2 * (size_t)kchunk * row_bytes > 227 * 1024) kchunk -= KB;
  const size_t smem = fixed + 2 * (size_t)kchunk * row_bytes;
  AttnParams& pm = const_cast<AttnParams&>(p);
  pm.kchunk = kchunk;
  dim3 grid((a->Nq + TQ - 1) / TQ, a->H, a->B);
  cudaStream_t st = (cudaStream_t)stream;
#define VB_FWD(DD)                                                                                                     \
  if (split) return a->qkv_fp16 ? launch_att(attn_fwd_kernel<DD, true, true>, grid, smem, p, st, "vb_attention_fwd")   \
                                : launch_att(attn_fwd_kernel<DD, false, true>, grid, smem, p, st, "vb_attention_fwd"); \
  return a->qkv_fp16 ? launch_att(attn_fwd_kernel<DD, true, false>, grid, smem, p, st, "vb_attention_fwd")             \
                     : launch_att(attn_fwd_kernel<DD, false, false>, grid, smem, p, st, "vb_attention_fwd");
  switch (a->D) {
    case 16: VB_FWD(16)
    case 32: VB_FWD(32)
    case 64: VB_FWD(64)
    default: VB_FWD(128)
  }
#undef VB_FWD
}

extern "C" vb_status vb_attention_bwd(const vb_attn_args* a, void* stream) {
  using namespace vb;
  if (int s = validate(a, true)) return s;
  const AttnParams p = to_params(a);
  cudaStream_t st = (cudaStream_t)stream;
  const bool want_dq = a->dQ != nullptr, want_dkv = a->dK != nullptr;
  const int nkp = (a->Nk + KB - 1) / KB * KB, nqp = (a->Nq + KB - 1) / KB * KB;
  // short sequences (all of ViLBERT's): one CTA per (batch, head) computes dQ, dK and dV in a single pass
  static const bool two_kernels_forced = getenv("VB_ATTN_BWD_TWO_KERNELS") != nullptr;   // development switch (tools/attn_probe.py)
  if (a->Nq <= 128 && a->Nk <= 128 && a->D >= 32 && !two_kernels_forced) {
    const int nq16 = (a->Nq + 15) / 16 * 16;
    const size_t smem_f = (size_t)(2 * nq16 + 2 * nkp) * (a->D + 8) * 2 + (size_t)2 * nq16 * (nkp + 8) * 2 + (size_t)nkp * 4;
    if (smem_f <= 227 * 1024) {
      dim3 gf(a->H, a->B);
      const char* what = "vb_attention_bwd(fused)";
      // the dQ-only variant keeps no P / dS tiles, except with dropout (phase 1 stages P and dP there)
      const size_t smem_q = p.drop.ctr ? smem_f : smem_f - (size_t)2 * nq16 * (nkp + 8) * 2;
#define VB_BWD_FUSED(DD)                                                                                            \
  if (!want_dkv) return launch_att(attn_bwd_fused_kernel<DD, true, false>, gf, smem_q, p, st, what, ATT1_THREADS); \
  if (!want_dq) return launch_att(attn_bwd_fused_kernel<DD, false, true>, gf, smem_f, p, st, what, ATT1_THREADS);  \
  return launch_att(attn_bwd_fused_kernel<DD>, gf, smem_f, p, st, what, ATT1_THREADS);
      switch (a->D) {
        case 32: VB_BWD_FUSED(32)
        case 64: VB_BWD_FUSED(64)
        default: VB_BWD_FUSED(128)
      }
#undef VB_BWD_FUSED
    }
  }
  // two kernels: dQ (which also writes delta), then dK / dV. Without dQ the first kernel only writes delta; without dK / dV the
  // second is not launched.
  const size_t smem_q = (size_t)(2 * TQ + 2 * nkp) * (a->D + 8) * 2 + (size_t)nkp * 4;
  const size_t smem_delta = p.drop.ctr ? smem_q : (size_t)(2 * TQ) * (a->D + 8) * 2;   // with dropout delta needs Q / K / V
  const size_t smem_k = (size_t)(2 * TQ + 2 * nqp) * (a->D + 8) * 2 + (size_t)nqp * 8;
  dim3 gq((a->Nq + TQ - 1) / TQ, a->H, a->B), gk((a->Nk + TQ - 1) / TQ, a->H, a->B);
  // refuse a query range the dK / dV panels cannot hold before the dQ kernel runs: a refused call writes nothing
  if (want_dkv && smem_k > 227 * 1024)
    return set_error(VB_ERR_UNSUPPORTED, "vb_attention_bwd(dkv): sequence too long for the smem-resident panel (%zu bytes)", smem_k);
  int s;
#define VB_BWD_TWO(DD)                                                                                                         \
  s = want_dq ? launch_att(attn_bwd_dq_kernel<DD>, gq, smem_q, p, st, "vb_attention_bwd(dq)")                                  \
              : launch_att(attn_bwd_dq_kernel<DD, false>, gq, smem_delta, p, st, "vb_attention_bwd(delta)");                  \
  if (s || !want_dkv) return s;                                                                                                \
  return launch_att(attn_bwd_dkv_kernel<DD>, gk, smem_k, p, st, "vb_attention_bwd(dkv)");
  switch (a->D) {
    case 16: VB_BWD_TWO(16)
    case 32: VB_BWD_TWO(32)
    case 64: VB_BWD_TWO(64)
    default: VB_BWD_TWO(128)
  }
#undef VB_BWD_TWO
}

extern "C" vb_status vb_attention_probs(const vb_attn_args* a, float* probs, void* stream) {
  using namespace vb;
  if (!a || !probs || !a->Q || !a->K) return set_error(VB_ERR_INVALID, "vb_attention_probs: null argument");
  if (a->q_off) return set_error(VB_ERR_UNSUPPORTED, "vb_attention_probs: the probability export reads the padded layout only");
  if (a->B <= 0 || a->H <= 0 || a->Nq <= 0 || a->Nk <= 0 || (a->D % 8) || a->D > 512) return set_error(VB_ERR_INVALID, "vb_attention_probs: bad shape");
  if ((a->ldq % 8) || (a->ldk % 8) || !al16(a->Q) || !al16(a->K)) return set_error(VB_ERR_INVALID, "vb_attention_probs: Q / K need ld %% 8 == 0 and 16-byte aligned bases");
  AttnParams p = to_params(a);
  const long long rows = (long long)a->B * a->H * a->Nq;
  long long blocks = (rows + 7) / 8;
  int cap = sm_count() * 8; if (cap <= 0) cap = 132 * 8;
  const int grid = (int)(blocks < cap ? blocks : cap);
  cudaError_t e = launch_pdl(attn_probs_kernel, dim3(grid), dim3(256), (size_t)(8 * a->D * sizeof(float)), (cudaStream_t)stream, p, probs, (int)a->D);
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_attention_probs: %s", cudaGetErrorString(e));
  return VB_OK;
}
