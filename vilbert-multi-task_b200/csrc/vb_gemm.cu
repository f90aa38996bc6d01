// vb_gemm.cu — persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] = alpha * A[M,K] . B[N,K]^T  (16-bit operands, fp32 accumulation in registers) + fused epilogue.
//
// Replaces the aten addmm behind every nn.Linear on the ViLBERT hot path and its autograd
// (reference: vilbert/vilbert.py:410-412,466,492,509,553-555,625,653,670,716-725,830,837,865-869 and
// SURVEY.md appendix A). Design:
//   warpgroup 0      TMA producer: one elected lane of warp 0 issues cp.async.bulk.tensor 2D boxes (64 x rows, 128B swizzle)
//                    into a NUM_STAGES-deep smem ring, completion on mbarriers (complete_tx); warps 1..3 only hold the
//                    warpgroup slot so that the consumers start at a warpgroup boundary; the warpgroup keeps 40 registers
//                    per thread and hands the rest to the consumers (setmaxnreg);
//   warpgroups 1, 2  consumers, 64 rows of the 128 x BN tile each: wgmma.mma_async (m64 nBN k16)
//                    from the swizzled stages into fp32 register accumulators; a stage is released once the wgmma group
//                    reading it has retired (one group stays in flight). Then the epilogue of the warp's 16 rows: registers ->
//                    XOR-swizzled smem tile -> row-wise, 128-bit coalesced pass doing bias / erf-GELU / GELU' / residual /
//                    16-bit conversion, while the producer already loads the next tile's stages.
// Operands may be K-major (nn.Linear forward) or MN-major (dgrad / wgrad operands read in place, no transposed copies); both
// are the canonical SWIZZLE_128B layouts TMA writes, wgmma reads the MN-major ones with its transpose flag.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "vb_internal.h"
#include "vb_ptx.cuh"

namespace vb {

constexpr int BM = 128;          // rows of a CTA tile: two consumer warpgroups x wgmma M = 64
constexpr int BK = 64;           // one 128-byte swizzle span of a 16-bit operand
constexpr int UK = 16;           // wgmma K for 16-bit inputs
constexpr int CONSUMER_WARPS = 8;
constexpr int GEMM_THREADS = 128 + CONSUMER_WARPS * 32;
constexpr int EPI_ROWS = 16;              // rows of the tile whose accumulators one consumer warp holds
constexpr int EPI_PS = EPI_ROWS / 4;      // passes of the coalesced epilogue (4 rows per pass)
// Epilogue staging tile per warp: 16 rows x 32 fp32, dense 128-byte rows whose 16-byte chunks are XOR-swizzled with the
// row index (chunk ^ (row & 7)): the fragment stores and the row-wise 128-bit loads spread over all banks without padding
// (2 KB per warp).
constexpr int STAGING_BYTES_PER_WARP = EPI_ROWS * 32 * 4;
__device__ __forceinline__ int stg_off(int row, int col) { return row * 32 + ((((col >> 2) ^ (row & 7)) << 2) | (col & 3)); }

// One stage = the 128 x 64 A box and the BN x 64 B box. 192 KB of stages leave room for the staging tiles within the 227 KB of
// an H100 block.
template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int NUM_STAGES = (192 * 1024) / STAGE_BYTES;   // 6 (BN 128) / 4 (BN 256)
  static constexpr int SMEM_BYTES = NUM_STAGES * STAGE_BYTES + CONSUMER_WARPS * STAGING_BYTES_PER_WARP + 256 /*barriers*/;
};

struct GemmKernelParams {
  int M, N, K;
  int num_m_blocks, num_n_blocks, num_k_blocks;   // num_k_blocks counts VIRTUAL k-blocks: npass x real_k_blocks
  int real_k_blocks;         // ceil(K / 64)
  int npass;                 // 1, or 2..3 in split precision: pass_sel[i] bit 0 = A_lo, bit 1 = B_lo
  int pass_sel[3];
  int out_fp16;              // format of out_bf16 / out_lo: 0 = bf16, 1 = fp16
  __nv_bfloat16* out_lo;     // split precision: low part of the value written to out_bf16 (same pitch), or NULL
  __nv_bfloat16* out_b16;    // always-bf16 copy of the value written to out_bf16 (same pitch), or NULL
  int split_k, k_blocks_per_split;
  float alpha;
  const float* bias;
  const float* residual;
  long long ld_res;
  const __nv_bfloat16* aux;
  long long ld_aux;
  int act;
  float* out_f32;
  long long ld_of;
  __nv_bfloat16* out_bf16;
  long long ld_ob;
  __nv_bfloat16* out_pre;
  long long ld_op;
  int atomic_out;
  float* out_colsum;
  int vec_f32, vec_bf16, vec_pre, vec_res, vec_aux;  // 128/64-bit access legal for that buffer
  uint64_t desc_base_a, desc_base_b;                 // smem descriptor without the address field
  int mma_kind;              // bit 0: B MN-major, bit 1: A MN-major, bit 2: fp16 operands (else bf16)
  DropCfg drop;              // dropout on the epilogue value before the residual add (EPI_F32 / generic)
  int a_mn, b_mn;            // operand majors
  int fast_ok;               // every buffer the specialised epilogue touches allows 128/64-bit accesses
  unsigned long long* dbg;   // optional per-CTA timeline [grid][10] (8 x clock64 + 2 x globaltimer ns), NULL in production
};

// Epilogue specialisations. Each instantiation keeps ONE compact, fully unrolled fast path (whole 16x32 chunk inside
// the matrix, 128/64-bit aligned buffers) plus a shared non-inlined generic path for ragged edges / odd layouts, so that
// the epilogue code of a kernel stays small enough for the instruction cache.
enum { EPI_F32 = 0,     // v = alpha*acc (+bias) (ReLU) (+fp32 residual) -> out_f32 (+ 16-bit copy)   (out-proj / FFN2 / dgrad-into-residual / logits / poolers)
       EPI_BF16 = 1,    // v = alpha*acc (+bias) -> out_bf16                                 (QKV, plain dgrads)
       EPI_GELU = 2,    // pre = acc + bias; gelu(pre) -> out_bf16 / out_f32; gelu'(pre) -> out_pre (bf16, saved for backward)
       EPI_DGELU = 3,   // v = acc * aux (aux = saved gelu'(pre)) -> out_bf16 (+ column sums)
       EPI_ATOMIC = 4,  // red.global.add.v4.f32 into out_f32 (split-K wgrad)
       EPI_GENERIC = 5, // runtime flags only (ReLU poolers, unusual output combinations)
       EPI_PARTIAL = 6, // deterministic split-K wgrad: split s stores its fp32 tile into rows [s*M, s*M + M) of out_f32 (a workspace)
       EPI_COUNT = 7 };

// Generic, compact (non-unrolled) path: any flags, any alignment, ragged rows / columns.
__device__ __noinline__ void epi_generic_chunk(const GemmKernelParams& p, const float* stg, int m_base, int n, int rr, int cc) {
  const int nv = min(4, p.N - n);
  if (nv <= 0) return;
  float cs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
  for (int ps = 0; ps < EPI_PS; ++ps) {
    const int row = ps * 4 + rr;
    const long long m = m_base + row;
    if (m >= p.M) break;
#pragma unroll 1
    for (int j = 0; j < nv; ++j) {
      float v = stg[stg_off(row, cc + j)] * p.alpha;
      if (p.bias) v += p.bias[n + j];
      if (p.act == VB_ACT_GELU) {
        float gg, dg;
        gelu_erf_and_grad(v, gg, dg);
        if (p.out_pre) p.out_pre[m * p.ld_op + n + j] = __float2bfloat16(dg);   // saved for backward: gelu'(pre)
        v = gg;
      } else if (p.act == VB_ACT_RELU) {
        v = fmaxf(v, 0.f);
      } else if (p.act == VB_ACT_DGELU) {
        v *= __bfloat162float(p.aux[m * p.ld_aux + n + j]);                      // aux = saved gelu'(pre)
      }
      if (p.drop.ctr) v = drop_apply(v, drop_seed(p.drop), (uint32_t)(m * p.N + n + j), p.drop);
      cs[j] += v;
      if (p.residual) v += p.residual[m * p.ld_res + n + j];
      if (p.out_f32) {
        if (p.atomic_out) atomicAdd(p.out_f32 + m * p.ld_of + n + j, v);
        else p.out_f32[m * p.ld_of + n + j] = v;
      }
      if (p.out_bf16) {
        const uint16_t hi = cvt16(v, p.out_fp16);
        reinterpret_cast<uint16_t*>(p.out_bf16)[m * p.ld_ob + n + j] = hi;
        if (p.out_lo) reinterpret_cast<uint16_t*>(p.out_lo)[m * p.ld_ob + n + j] = cvt16(v - cvt16_to_f32(hi, p.out_fp16), p.out_fp16);
        if (p.out_b16) p.out_b16[m * p.ld_ob + n + j] = __float2bfloat16(v);
      }
    }
  }
  if (p.out_colsum) {
#pragma unroll 1
    for (int j = 0; j < nv; ++j) atomicAdd(p.out_colsum + n + j, cs[j]);
  }
}

// Ragged chunks of EPI_PARTIAL: plain stores of alpha * acc into the split's slice (row m + slice_row), bounds-checked.
__device__ __noinline__ void epi_partial_chunk(const GemmKernelParams& p, const float* stg, int m_base, int n, int rr, int cc, long long slice_row) {
  const int nv = min(4, p.N - n);
  if (nv <= 0) return;
#pragma unroll 1
  for (int ps = 0; ps < EPI_PS; ++ps) {
    const int row = ps * 4 + rr;
    const long long m = m_base + row;
    if (m >= p.M) break;
#pragma unroll 1
    for (int j = 0; j < nv; ++j) p.out_f32[(m + slice_row) * p.ld_of + n + j] = stg[stg_off(row, cc + j)] * p.alpha;
  }
}

// 16-bit output variants of the specialised epilogues (template parameter OUT16; kept out of line / out of the kernels that do
// not need them: the fast paths are 8x unrolled and the epilogue time follows the instruction footprint, see the note above):
//   0 = bf16 (gradient operands, bf16 precision)   1 = fp16 (forward operands)   2 = fp16 + an always-bf16 copy (forward
//   operands the backward's weight-gradient GEMM reads)   3 = split precision: fp16 hi + lo (+ bf16 copy at run time).
__device__ __noinline__ void store16x4_slow(const GemmKernelParams& p, long long off, float v0, float v1, float v2, float v3) {
  if (p.out_lo) {
    uint32_t l01, l23;
    const uint32_t h01 = pack16_split(v0, v1, p.out_fp16, l01), h23 = pack16_split(v2, v3, p.out_fp16, l23);
    *reinterpret_cast<uint2*>(p.out_bf16 + off) = make_uint2(h01, h23);
    *reinterpret_cast<uint2*>(p.out_lo + off) = make_uint2(l01, l23);
  } else {
    *reinterpret_cast<uint2*>(p.out_bf16 + off) = make_uint2(pack16(v0, v1, p.out_fp16), pack16(v2, v3, p.out_fp16));
  }
  if (p.out_b16) *reinterpret_cast<uint2*>(p.out_b16 + off) = make_uint2(pack_bf16(v0, v1), pack_bf16(v2, v3));
}
template <int OUT16>
__device__ __forceinline__ void store16x4(const GemmKernelParams& p, long long off, float v0, float v1, float v2, float v3) {
  if (OUT16 == 0) {
    *reinterpret_cast<uint2*>(p.out_bf16 + off) = make_uint2(pack_bf16(v0, v1), pack_bf16(v2, v3));
  } else if (OUT16 == 3) {   // split precision: fp16 hi + lo (+ the bf16 copy when asked for)
    uint32_t l01, l23;
    const uint32_t h01 = pack16_split(v0, v1, 1, l01), h23 = pack16_split(v2, v3, 1, l23);
    *reinterpret_cast<uint2*>(p.out_bf16 + off) = make_uint2(h01, h23);
    *reinterpret_cast<uint2*>(p.out_lo + off) = make_uint2(l01, l23);
    if (p.out_b16) *reinterpret_cast<uint2*>(p.out_b16 + off) = make_uint2(pack_bf16(v0, v1), pack_bf16(v2, v3));
  } else {
    *reinterpret_cast<uint2*>(p.out_bf16 + off) = make_uint2(pack_f16(v0, v1), pack_f16(v2, v3));
    if (OUT16 == 2) *reinterpret_cast<uint2*>(p.out_b16 + off) = make_uint2(pack_bf16(v0, v1), pack_bf16(v2, v3));
  }
}

// Poolers (vilbert.py:1116-1122, 1131-1137): relu(acc + bias) -> fp32 and a 16-bit operand copy. Two tiny launches per step: one
// compact out-of-line routine selected per chunk inside the F32 kernel, so that kernel's unrolled fast path stays as small as it was.
__device__ __noinline__ void epi_pool_chunk(const GemmKernelParams& p, const float* stg, int m_base, int n, int rr, int cc, const float4 b4) {
#pragma unroll 1
  for (int ps = 0; ps < EPI_PS; ++ps) {
    const int row = ps * 4 + rr;
    const long long m = m_base + row;
    const float4 a4 = *reinterpret_cast<const float4*>(stg + stg_off(row, cc));
    const float v0 = fmaxf(fmaf(a4.x, p.alpha, b4.x), 0.f), v1 = fmaxf(fmaf(a4.y, p.alpha, b4.y), 0.f);
    const float v2 = fmaxf(fmaf(a4.z, p.alpha, b4.z), 0.f), v3 = fmaxf(fmaf(a4.w, p.alpha, b4.w), 0.f);
    *reinterpret_cast<float4*>(p.out_f32 + m * p.ld_of + n) = make_float4(v0, v1, v2, v3);
    if (p.out_bf16) store16x4_slow(p, m * p.ld_ob + n, v0, v1, v2, v3);
  }
}

template <int EPI, int OUT16>
__device__ __forceinline__ void epi_fast_chunk(const GemmKernelParams& p, const float* stg, int m_base, int n, int rr, int cc,
                                               const float4 (&resv)[EPI_PS], const uint2 (&auxv)[EPI_PS], const float4 b4) {
  float cs0 = 0.f, cs1 = 0.f, cs2 = 0.f, cs3 = 0.f;
  const uint32_t dseed = (EPI == EPI_F32 && p.drop.ctr) ? drop_seed(p.drop) : 0u;
#pragma unroll
  for (int ps = 0; ps < EPI_PS; ++ps) {
    const int row = ps * 4 + rr;
    const long long m = m_base + row;
    const float4 a4 = *reinterpret_cast<const float4*>(stg + stg_off(row, cc));
    float v0 = fmaf(a4.x, p.alpha, b4.x), v1 = fmaf(a4.y, p.alpha, b4.y), v2 = fmaf(a4.z, p.alpha, b4.z), v3 = fmaf(a4.w, p.alpha, b4.w);
    if (EPI == EPI_GELU) {
      float d0, d1, d2, d3;
      gelu_erf_and_grad(v0, v0, d0); gelu_erf_and_grad(v1, v1, d1); gelu_erf_and_grad(v2, v2, d2); gelu_erf_and_grad(v3, v3, d3);
      *reinterpret_cast<uint2*>(p.out_pre + m * p.ld_op + n) = make_uint2(pack_bf16(d0, d1), pack_bf16(d2, d3));   // gelu'(pre) for backward
      if (p.out_f32) *reinterpret_cast<float4*>(p.out_f32 + m * p.ld_of + n) = make_float4(v0, v1, v2, v3);
      if (p.out_bf16) store16x4<OUT16>(p, m * p.ld_ob + n, v0, v1, v2, v3);
    } else if (EPI == EPI_DGELU) {
      const float2 x01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&auxv[ps].x));
      const float2 x23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&auxv[ps].y));
      v0 *= x01.x; v1 *= x01.y; v2 *= x23.x; v3 *= x23.y;   // aux = gelu'(pre) saved by the forward epilogue
      cs0 += v0; cs1 += v1; cs2 += v2; cs3 += v3;
      store16x4<0>(p, m * p.ld_ob + n, v0, v1, v2, v3);   // a gradient operand: always bf16
    } else if (EPI == EPI_F32) {
      if (p.drop.ctr) {   // LN(dropout(dense(x)) + residual): mask the dense output, element index m*N + n
        const uint32_t e0 = (uint32_t)(m * p.N + n);
        v0 = drop_apply(v0, dseed, e0, p.drop); v1 = drop_apply(v1, dseed, e0 + 1, p.drop);
        v2 = drop_apply(v2, dseed, e0 + 2, p.drop); v3 = drop_apply(v3, dseed, e0 + 3, p.drop);
      }
      if (p.residual) { v0 += resv[ps].x; v1 += resv[ps].y; v2 += resv[ps].z; v3 += resv[ps].w; }
      float* dst = p.out_f32 + m * p.ld_of + n;
      if (p.vec_f32) {
        *reinterpret_cast<float4*>(dst) = make_float4(v0, v1, v2, v3);
      } else {   // row pitch not a multiple of 4 floats (30522-/1601-/3129-wide logits): same bytes, 32-bit stores
        dst[0] = v0; dst[1] = v1; dst[2] = v2; dst[3] = v3;
      }
    } else if (EPI == EPI_BF16) {
      store16x4<OUT16>(p, m * p.ld_ob + n, v0, v1, v2, v3);
    } else if (EPI == EPI_ATOMIC) {
      asm volatile("red.global.v4.f32.add [%0], {%1, %2, %3, %4};" ::"l"(p.out_f32 + m * p.ld_of + n), "f"(v0), "f"(v1), "f"(v2), "f"(v3) : "memory");
    } else if (EPI == EPI_PARTIAL) {   // m already points into the split's slice
      *reinterpret_cast<float4*>(p.out_f32 + m * p.ld_of + n) = make_float4(v0, v1, v2, v3);
    }
  }
  if (EPI == EPI_DGELU && p.out_colsum) {
    // reduce over the 4 row-lanes sharing these columns (lane bits 3,4), then one atomic per column
    cs0 += __shfl_xor_sync(0xffffffffu, cs0, 8);  cs1 += __shfl_xor_sync(0xffffffffu, cs1, 8);
    cs2 += __shfl_xor_sync(0xffffffffu, cs2, 8);  cs3 += __shfl_xor_sync(0xffffffffu, cs3, 8);
    cs0 += __shfl_xor_sync(0xffffffffu, cs0, 16); cs1 += __shfl_xor_sync(0xffffffffu, cs1, 16);
    cs2 += __shfl_xor_sync(0xffffffffu, cs2, 16); cs3 += __shfl_xor_sync(0xffffffffu, cs3, 16);
    if (rr == 0) {
      atomicAdd(p.out_colsum + n, cs0); atomicAdd(p.out_colsum + n + 1, cs1);
      atomicAdd(p.out_colsum + n + 2, cs2); atomicAdd(p.out_colsum + n + 3, cs3);
    }
  }
}

// One 64-deep k-block of a consumer warpgroup: 4 k steps of one wgmma each (m64 n128 or n256), committed as one group.
// MN-major operands advance 16 k rows = two 8-row groups (2 KB) per step, K-major ones 32 bytes inside the swizzle span.
// The n256 B operand continues the n128 layout: K-major rows 16 KB on, MN-major 64-wide boxes LBO = BK * 128 apart.
template <int BN, int F16, int TA, int TB>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint32_t sa, uint32_t sb, uint64_t desc_base_a, uint64_t desc_base_b,
                                           bool accumulate) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < BK / UK; ++k) {
    const uint64_t da = gmma_desc_at(desc_base_a, sa + k * (TA ? 2048 : UK * 2));
    const uint64_t db = gmma_desc_at(desc_base_b, sb + k * (TB ? 2048 : UK * 2));
    if constexpr (BN == 256) wgmma_m64n256k16<F16, TA, TB>(acc, da, db, (accumulate || k > 0) ? 1u : 0u);
    else                     wgmma_m64n128k16<F16, TA, TB>(acc, da, db, (accumulate || k > 0) ? 1u : 0u);
  }
  wgmma_commit();
}

// Columns [32 c4, +32) of the accumulator fragment -> the warp's staging tile (row = fragment row within the warp's 16).
template <int NR>
__device__ __forceinline__ void stage_chunk(const float (&d)[NR], int c4, float* stg, int lane) {
  const int r0 = lane >> 2, c0 = 2 * (lane & 3);
#pragma unroll
  for (int ii = 0; ii < 4; ++ii) {
    const int i = c4 * 4 + ii;
    *reinterpret_cast<float2*>(stg + stg_off(r0, ii * 8 + c0)) = make_float2(d[4 * i], d[4 * i + 1]);
    *reinterpret_cast<float2*>(stg + stg_off(r0 + 8, ii * 8 + c0)) = make_float2(d[4 * i + 2], d[4 * i + 3]);
  }
}

template <int BN, int EPI, int OUT16>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_a_lo, const __grid_constant__ CUtensorMap tmap_b_lo,
                  const __grid_constant__ GemmKernelParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int NUM_STAGES = Cfg::NUM_STAGES;

  // SWIZZLE_128B tiles need 1024-byte alignment: the kernel has no static shared memory, so the dynamic window starts at
  // the CTA's (1024-aligned) shared base; checked once below.
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* smem_tiles = smem;
  float* staging = reinterpret_cast<float*>(smem + NUM_STAGES * Cfg::STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NUM_STAGES * Cfg::STAGE_BYTES + CONSUMER_WARPS * STAGING_BYTES_PER_WARP);
  uint64_t* full_bar = bars;                       // [NUM_STAGES]
  uint64_t* empty_bar = bars + NUM_STAGES;         // [NUM_STAGES]

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
#define VB_DBG(slot) do { if (p.dbg) p.dbg[blockIdx.x * 10 + (slot)] = clock64(); } while (0)
#define VB_DBG_NS(slot) do { if (p.dbg) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); p.dbg[blockIdx.x * 10 + (slot)] = t_; } } while (0)
  if (threadIdx.x == 0) { VB_DBG(0); VB_DBG_NS(8); }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (p.npass > 1) { tma_prefetch_desc(&tmap_a_lo); tma_prefetch_desc(&tmap_b_lo); }
    for (int s = 0; s < NUM_STAGES; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), CONSUMER_WARPS);   // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_entry();   // everything above (barrier init, descriptor prefetch) overlapped the previous kernel's tail
  if (threadIdx.x == 0) VB_DBG(1);

  // work items = (row block, column block, k split), walked by the persistent CTAs in grid-stride order
  const int group = blockIdx.x;
  const int num_groups = gridDim.x;
  const int total_work = p.num_m_blocks * p.num_n_blocks * p.split_k;

  // Register split: one lane of the producer warpgroup issues the loads, the consumers hold the accumulators (BN / 2 per thread
  // at BN = 256). 128 x 40 + 256 x 232 = 64512 of the 65536 registers the launch bounds give the CTA (168 per thread). Each
  // setmaxnreg sits inside its role's branch (ptxas ignores it if code needing more registers is reachable after it), and all
  // four warps of a warpgroup execute it.
  if (warp_idx < 4) setmaxnreg_dec<40>();
  if (warp_idx == 0) {
    // ================================================================ TMA producer (one elected lane issues; the warp stays converged)
    int stage = 0;
    uint32_t phase = 0;
    for (int w = group; w < total_work; w += num_groups) {
      const int split = w % p.split_k;
      const int t2 = w / p.split_k;
      const int m_blk = t2 % p.num_m_blocks;
      const int n_blk = t2 / p.num_m_blocks;
      const int kb0 = split * p.k_blocks_per_split;
      const int kb1 = min(kb0 + p.k_blocks_per_split, p.num_k_blocks);
      // loads of one (real) k-block from the given tensor maps; split precision selects hi / lo maps per pass
      auto issue_loads = [&](const CUtensorMap* tma_a, const CUtensorMap* tma_b, int kb) {
        mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1);
        const uint32_t sa = smem_u32(smem_tiles + stage * Cfg::STAGE_BYTES);
        const uint32_t sb = sa + Cfg::A_BYTES;
        const uint32_t fb = smem_u32(&full_bar[stage]);
        mbar_arrive_expect_tx(fb, Cfg::STAGE_BYTES);
        if (p.a_mn) {
#pragma unroll
          for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * (BK * 128), tma_a, m_blk * BM + j * 64, kb * BK, fb);
        } else {
          tma_load_2d(sa, tma_a, kb * BK, m_blk * BM, fb);
        }
        if (p.b_mn) {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * (BK * 128), tma_b, n_blk * BN + j * 64, kb * BK, fb);
        } else {
          tma_load_2d(sb, tma_b, kb * BK, n_blk * BN, fb);
        }
      };
      for (int kbv = kb0; kbv < kb1; ++kbv) {
        if (elect_one()) {
          if (p.npass == 1) {
            issue_loads(&tmap_a, &tmap_b, kbv);
          } else {
            // virtual k-block -> (pass, real k-block): split precision walks K once per pass with the hi / lo tensor maps
            const int ps = kbv / p.real_k_blocks;
            const int sel = p.pass_sel[ps];
            issue_loads((sel & 1) ? &tmap_a_lo : &tmap_a, (sel & 2) ? &tmap_b_lo : &tmap_b, kbv - ps * p.real_k_blocks);
          }
          if (kbv == kb0 && w == group) VB_DBG(2);
        }
        __syncwarp();
        if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp_idx >= 4) {
    // ================================================================ consumers (warps 4..11 = warpgroups 1, 2)
    setmaxnreg_inc<232>();
    const int cw = warp_idx - 4;
    const int wg = cw >> 2;                 // rows [64 wg, +64) of the tile
    float* stg = staging + cw * (EPI_ROWS * 32);
    const int rr = lane >> 3;               // row within a 4-row group of the coalesced pass
    const int cc = (lane & 7) * 4;          // first of 4 columns handled by this lane
    // 64 rows of A start 8 KB into the stage in both majors (K-major: 64 rows x 128 B; MN-major: the second 64-wide box)
    const uint32_t a_off = wg * (64 * 128);
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&empty_bar[s]));
    };
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    const int mma_kind = p.mma_kind;
    const uint64_t desc_base_a = p.desc_base_a, desc_base_b = p.desc_base_b;
    for (int w = group; w < total_work; w += num_groups) {
      const int split = w % p.split_k;
      const int t2 = w / p.split_k;
      const int m_blk = t2 % p.num_m_blocks;
      const int n_blk = t2 / p.num_m_blocks;
      const int kb0 = split * p.k_blocks_per_split;
      const int kb1 = min(kb0 + p.k_blocks_per_split, p.num_k_blocks);
      int prev = -1;
      // the k-loop of the tile, one copy per operand kind (formats and majors are wgmma immediates)
      auto kloop = [&](auto kind) {
        constexpr int KIND = decltype(kind)::value;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(smem_u32(&full_bar[stage]), phase);
          if (kb == kb0 && w == group && threadIdx.x == 128) VB_DBG(3);
          const uint32_t sa = smem_u32(smem_tiles + stage * Cfg::STAGE_BYTES) + a_off;
          const uint32_t sb = smem_u32(smem_tiles + stage * Cfg::STAGE_BYTES) + Cfg::A_BYTES;
          mma_kblock<BN, (KIND >> 2) & 1, (KIND >> 1) & 1, KIND & 1>(acc, sa, sb, desc_base_a, desc_base_b, kb > kb0);
          // the group of the previous k-block has retired: its stage may be refilled
          wgmma_wait<1>();
          if (prev >= 0) release(prev);
          prev = stage;
          if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
        }
      };
      switch (mma_kind) {
        case 0: kloop(std::integral_constant<int, 0>{}); break;
        case 1: kloop(std::integral_constant<int, 1>{}); break;
        case 2: kloop(std::integral_constant<int, 2>{}); break;
        case 3: kloop(std::integral_constant<int, 3>{}); break;
        case 4: kloop(std::integral_constant<int, 4>{}); break;
        case 5: kloop(std::integral_constant<int, 5>{}); break;
        case 6: kloop(std::integral_constant<int, 6>{}); break;
        default: kloop(std::integral_constant<int, 7>{}); break;
      }
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
      if (prev >= 0) release(prev);
      if (w == group && threadIdx.x == 128) VB_DBG(5);

      // ---- epilogue of the warp's 16 rows, 32 columns at a time
      const int m_base = m_blk * BM + wg * 64 + (cw & 3) * EPI_ROWS;
      const bool rows_full = (m_base + EPI_ROWS <= p.M);
      if (m_base < p.M) {
        constexpr int NC = BN / 32;
#pragma unroll 1
        for (int c = 0; c < NC; ++c) {
          const int n_chunk = n_blk * BN + c * 32;
          if (n_chunk >= p.N) break;   // warp-uniform
          const bool fast = (EPI != EPI_GENERIC) && p.fast_ok && rows_full && (n_chunk + 32 <= p.N);
          const int n = n_chunk + cc;
          // global operands of the chunk first, so that their latency overlaps the staging
          float4 resv[EPI_PS];
          uint2 auxv[EPI_PS];
          float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
          if (fast) {
            if (EPI == EPI_F32 && p.residual) {
#pragma unroll
              for (int ps = 0; ps < EPI_PS; ++ps) {
                const float* src = p.residual + (long long)(m_base + ps * 4 + rr) * p.ld_res + n;
                if (p.vec_res) resv[ps] = *reinterpret_cast<const float4*>(src);
                else resv[ps] = make_float4(src[0], src[1], src[2], src[3]);
              }
            }
            if (EPI == EPI_DGELU) {
#pragma unroll
              for (int ps = 0; ps < EPI_PS; ++ps)
                auxv[ps] = *reinterpret_cast<const uint2*>(p.aux + (long long)(m_base + ps * 4 + rr) * p.ld_aux + n);
            }
            if (p.bias) b4 = *reinterpret_cast<const float4*>(p.bias + n);
          }
          // registers -> staging tile: the 32-column chunk of the fragment must be a compile-time index
#pragma unroll
          for (int c2 = 0; c2 < NC; ++c2)
            if (c2 == c) stage_chunk(acc, c2, stg, lane);
          __syncwarp();
          if (EPI == EPI_PARTIAL) {
            if (fast) epi_fast_chunk<EPI, OUT16>(p, stg, m_base + split * p.M, n, rr, cc, resv, auxv, b4);
            else      epi_partial_chunk(p, stg, m_base, n, rr, cc, (long long)split * p.M);
          }
          else if (EPI == EPI_F32 && p.act == VB_ACT_RELU && fast) epi_pool_chunk(p, stg, m_base, n, rr, cc, b4);
          else if (fast) epi_fast_chunk<EPI, OUT16>(p, stg, m_base, n, rr, cc, resv, auxv, b4);
          else           epi_generic_chunk(p, stg, m_base, n, rr, cc);
          __syncwarp();
        }
      }
      if (w == group && threadIdx.x == 128) VB_DBG(6);
    }
  }

  if (threadIdx.x == 0) { VB_DBG(7); VB_DBG_NS(9); }
#undef VB_DBG
#undef VB_DBG_NS
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

// 2D bf16 tensor map: inner extent `inner` (contiguous), outer extent `outer` with row pitch ld elements.
static int make_tmap(CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld,
                     uint32_t box_inner, uint32_t box_outer) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return set_error(VB_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(VB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return VB_OK;
}

template <int BN, int EPI, int OUT16 = 0>
static int launch_gemm(const CUtensorMap* tm, GemmKernelParams& p, long long total_work, int max_ctas,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_wgmma_kernel<BN, EPI, OUT16>;
  static bool attr_set = false;  // per template instantiation
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  // persistent grid: one CTA per SM, fewer when there are fewer work items
  const int grid = (int)(total_work < max_ctas ? total_work : max_ctas);
  cudaError_t e = launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), (size_t)Cfg::SMEM_BYTES, stream, tm[0], tm[1], tm[2], tm[3], p);
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "gemm launch: %s", cudaGetErrorString(e));
  return VB_OK;
}

template <int BN>
static int launch_gemm_epi(int epi, int out16, const CUtensorMap* tm, GemmKernelParams& p, long long work, int max_ctas,
                           cudaStream_t stream) {
  switch (epi) {
    case EPI_F32: return launch_gemm<BN, EPI_F32>(tm, p, work, max_ctas, stream);
    case EPI_BF16:
      if (out16 == 1) return launch_gemm<BN, EPI_BF16, 1>(tm, p, work, max_ctas, stream);
      if (out16 == 2) return launch_gemm<BN, EPI_BF16, 2>(tm, p, work, max_ctas, stream);
      if (out16 == 3) return launch_gemm<BN, EPI_BF16, 3>(tm, p, work, max_ctas, stream);
      return launch_gemm<BN, EPI_BF16, 0>(tm, p, work, max_ctas, stream);
    case EPI_GELU:
      if (out16 == 1) return launch_gemm<BN, EPI_GELU, 1>(tm, p, work, max_ctas, stream);
      if (out16 == 2) return launch_gemm<BN, EPI_GELU, 2>(tm, p, work, max_ctas, stream);
      if (out16 == 3) return launch_gemm<BN, EPI_GELU, 3>(tm, p, work, max_ctas, stream);
      return launch_gemm<BN, EPI_GELU, 0>(tm, p, work, max_ctas, stream);
    case EPI_DGELU: return launch_gemm<BN, EPI_DGELU>(tm, p, work, max_ctas, stream);
    case EPI_ATOMIC: return launch_gemm<BN, EPI_ATOMIC>(tm, p, work, max_ctas, stream);
    case EPI_PARTIAL: return launch_gemm<BN, EPI_PARTIAL>(tm, p, work, max_ctas, stream);
    default: return launch_gemm<BN, EPI_GENERIC>(tm, p, work, max_ctas, stream);
  }
}

static inline bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

// Chooses (tile width, k splits) for a problem; honours the values the caller fixed. Pure host code.
static int choose_config(const vb_gemm_args* a, int max_ctas, int* bn_out, int* split_out) {
  const int num_m = (a->M + BM - 1) / BM;
  const int num_k = (a->K + BK - 1) / BK * (1 + (a->A_lo ? 1 : 0) + (a->B_lo ? 1 : 0));   // virtual k-blocks (split precision passes)
  // Tile configuration = (tile width bn, k splits): minimise the modelled time of the busiest CTA,
  // in SM cycles. The constants are estimates, not measurements: a 64-deep k-block of a 128 x 128 tile is 2.1 MFLOP, ~512
  // cycles at the dense BF16 / FP16 rate of an H100 SM (4096 FLOP per cycle), plus ~10 % for barrier waits and wgmma issue
  // (128 x 256: twice that); the epilogue of a tile follows its main loop (the accumulators live in the consumers' registers)
  // while the producer already loads the next tile; ~3k cycles of prologue + first-load latency per launch.
  if (a->block_n != 0 && a->block_n != 128 && a->block_n != 256) return set_error(VB_ERR_INVALID, "vb_gemm_bf16: block_n must be 0, 128 or 256");
  if (a->split_k > 1 && (!a->atomic_out || a->act != VB_ACT_NONE || a->bias || a->residual || a->out_colsum))
    return set_error(VB_ERR_INVALID, "vb_gemm_bf16: split_k > 1 needs atomic_out and a plain epilogue");
  const bool can_split = a->atomic_out && a->act == VB_ACT_NONE && !a->bias && !a->residual && !a->out_colsum;
  long long epi_base = 9000;   // generic epilogue
  if (a->atomic_out) epi_base = 3000;
  else if (a->act == VB_ACT_GELU || a->act == VB_ACT_DGELU) epi_base = 4200;
  else if (a->act == VB_ACT_NONE && a->out_f32 && !a->out_bf16) epi_base = a->residual ? 4800 : 3000;
  else if (a->act == VB_ACT_NONE && a->out_bf16 && !a->out_f32) epi_base = 3000;
  int bn = 128, split_k = 1;
  {
    long long best = -1;
    static const int split_cand[] = {1, 2, 3, 4, 5, 6, 8, 10, 12, 16, 24, 32};
    for (int w = 128; w <= 256; w += 128) {
      if (a->block_n && a->block_n != w) continue;
      if (!a->block_n && w == 256 && a->N <= 128) continue;
      const long long t_kb = (w == 128) ? 560 : 1100;
      const long long epi = epi_base * (w / 128);
      const long long tiles = (long long)num_m * ((a->N + w - 1) / w);
      for (int sc : split_cand) {
        if (a->split_k > 0 && sc != 1) break;
        int sp = a->split_k > 0 ? a->split_k : sc;
        if (sp > 1 && !can_split) break;
        if (sp > num_k) { if (a->split_k > 0) sp = num_k; else break; }
        const long long kps_ = (num_k + sp - 1) / sp;
        sp = (int)((num_k + kps_ - 1) / kps_);   // no empty splits
        const long long rounds = (tiles * sp + max_ctas - 1) / max_ctas;
        const long long ml = kps_ * t_kb;
        const long long c = 3000 + rounds * (ml + epi);
        if (best < 0 || c < best) { best = c; bn = w; split_k = sp; }
      }
    }
    if (best < 0) return set_error(VB_ERR_INVALID, "vb_gemm_bf16: no tile configuration for block_n=%d split_k=%d", a->block_n, a->split_k);
  }
  *bn_out = bn; *split_out = split_k;
  return VB_OK;
}

}  // namespace vb

extern "C" vb_status vb_gemm_bf16(const vb_gemm_args* a, void* stream_) {
  using namespace vb;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!a) return set_error(VB_ERR_INVALID, "vb_gemm_bf16: null args");
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return set_error(VB_ERR_INVALID, "vb_gemm_bf16: empty problem %dx%dx%d", a->M, a->N, a->K);
  if (!a->A || !a->B) return set_error(VB_ERR_INVALID, "vb_gemm_bf16: null operand");
  if ((a->lda % 8) || (a->ldb % 8) || !aligned(a->A, 16) || !aligned(a->B, 16))
    return set_error(VB_ERR_INVALID, "vb_gemm_bf16: operands need ld %% 8 == 0 and 16-byte aligned bases (lda=%lld ldb=%lld)",
                     (long long)a->lda, (long long)a->ldb);
  if (!a->out_f32 && !a->out_bf16) return set_error(VB_ERR_INVALID, "vb_gemm_bf16: no output");
  if (a->act == VB_ACT_DGELU && !a->aux) return set_error(VB_ERR_INVALID, "vb_gemm_bf16: DGELU needs aux");
  if (a->bias && !aligned(a->bias, 16)) return set_error(VB_ERR_INVALID, "vb_gemm_bf16: bias must be 16-byte aligned");
  if (a->atomic_out && (!a->out_f32 || a->out_bf16 || a->out_pre))
    return set_error(VB_ERR_INVALID, "vb_gemm_bf16: atomic_out supports only out_f32");
  if (a->atomic_out != 0 && a->atomic_out != 1 && a->atomic_out != VB_GEMM_PARTIALS)
    return set_error(VB_ERR_INVALID, "vb_gemm_bf16: atomic_out must be 0, 1 or VB_GEMM_PARTIALS");
  if ((a->A_lo && !aligned(a->A_lo, 16)) || (a->B_lo && !aligned(a->B_lo, 16)))
    return set_error(VB_ERR_INVALID, "vb_gemm_bf16: A_lo / B_lo must be 16-byte aligned");
  if ((a->out_lo || a->out_b16) && !a->out_bf16) return set_error(VB_ERR_INVALID, "vb_gemm_bf16: out_lo / out_b16 need out_bf16");
  if ((a->a_fp16 != 0) != (a->b_fp16 != 0))
    return set_error(VB_ERR_UNSUPPORTED, "vb_gemm_bf16: A and B must have the same 16-bit format (wgmma takes one operand type for both)");
  int dev_sms = 0, cc = 0;
  if (int s = vb_device_info(&dev_sms, &cc)) return s;
  if (cc != 90) return set_error(VB_ERR_UNSUPPORTED, "vb_gemm_bf16: needs an sm_90 device (found sm_%d)", cc);

  const int num_m = (a->M + BM - 1) / BM;
  const int real_k = (a->K + BK - 1) / BK;
  const int npass = 1 + (a->A_lo ? 1 : 0) + (a->B_lo ? 1 : 0);
  const int num_k = real_k * npass;   // virtual k-blocks (split precision: K is walked once per pass)
  int max_ctas = a->max_ctas > 0 ? a->max_ctas : dev_sms;

  int bn = 128, split_k = 1;
  if (int st = choose_config(a, max_ctas, &bn, &split_k)) return st;
  const int num_n = (a->N + bn - 1) / bn;
  const int kps = (num_k + split_k - 1) / split_k;

  GemmKernelParams p;
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.num_m_blocks = num_m; p.num_n_blocks = num_n; p.num_k_blocks = num_k;
  p.real_k_blocks = real_k; p.npass = npass;
  p.pass_sel[0] = 0; p.pass_sel[1] = a->A_lo ? 1 : 2; p.pass_sel[2] = 2;
  p.out_fp16 = a->out_fp16 ? 1 : 0;
  p.out_lo = static_cast<__nv_bfloat16*>(a->out_lo);
  p.out_b16 = static_cast<__nv_bfloat16*>(a->out_b16);
  p.split_k = split_k; p.k_blocks_per_split = kps;
  p.alpha = a->alpha;
  p.bias = a->bias;
  p.residual = a->residual; p.ld_res = a->ld_res;
  p.aux = static_cast<const __nv_bfloat16*>(a->aux); p.ld_aux = a->ld_aux;
  p.act = a->act;
  p.out_f32 = a->out_f32; p.ld_of = a->ld_out_f32;
  p.out_bf16 = static_cast<__nv_bfloat16*>(a->out_bf16); p.ld_ob = a->ld_out_bf16;
  p.out_pre = static_cast<__nv_bfloat16*>(a->out_pre); p.ld_op = a->ld_out_pre;
  p.atomic_out = a->atomic_out;
  p.out_colsum = a->out_colsum;
  p.vec_f32 = a->out_f32 && aligned(a->out_f32, 16) && (a->ld_out_f32 % 4 == 0);
  p.vec_bf16 = a->out_bf16 && aligned(a->out_bf16, 8) && (a->ld_out_bf16 % 4 == 0) && (!a->out_lo || aligned(a->out_lo, 8)) &&
               (!a->out_b16 || aligned(a->out_b16, 8));
  p.vec_pre = a->out_pre && aligned(a->out_pre, 8) && (a->ld_out_pre % 4 == 0);
  p.vec_res = a->residual && aligned(a->residual, 16) && (a->ld_res % 4 == 0);
  p.vec_aux = a->aux && aligned(a->aux, 8) && (a->ld_aux % 4 == 0);

  // smem matrix descriptors (see vb_ptx.cuh). K-major: rows of 128 B, 8-row groups 1024 B apart (SBO),
  // K advance of 16 elements = 32 B inside the swizzle span. MN-major: 64-element (128 B) rows indexed
  // by k, 8-k groups 1024 B apart (SBO), next 64 MN elements BK*128 B further (LBO); K advance of 16 = 2 groups.
  p.desc_base_a = gmma_desc_base(a->a_mn_major ? BK * 128 : 16, 1024);
  p.desc_base_b = gmma_desc_base(a->b_mn_major ? BK * 128 : 16, 1024);
  p.mma_kind = (a->b_mn_major ? 1 : 0) | (a->a_mn_major ? 2 : 0) | (a->a_fp16 ? 4 : 0);
  p.dbg = reinterpret_cast<unsigned long long*>(a->dbg_timeline);
  p.a_mn = a->a_mn_major ? 1 : 0;
  p.b_mn = a->b_mn_major ? 1 : 0;
  p.fast_ok = 0;
  p.drop.ctr = (a->dropout.step && a->dropout.p > 0.f) ? a->dropout.step : nullptr;
  p.drop.site = a->dropout.site;
  p.drop.thresh = (uint32_t)((double)a->dropout.p * 4294967296.0);
  p.drop.scale = a->dropout.p < 1.f ? 1.f / (1.f - a->dropout.p) : 0.f;

  CUtensorMap tm[4];   // A, B, A_lo, B_lo (the lo maps alias the hi ones when a low part is absent)
  int st;
  for (int i = 0; i < 4; ++i) {
    const bool is_a = (i & 1) == 0;
    const void* ptr = is_a ? (i < 2 ? a->A : a->A_lo) : (i < 2 ? a->B : a->B_lo);
    if (!ptr) { tm[i] = tm[i - 2]; continue; }
    if (is_a) {
      if (a->a_mn_major) st = make_tmap(&tm[i], ptr, (uint64_t)a->M, (uint64_t)a->K, (uint64_t)a->lda, 64, BK);
      else               st = make_tmap(&tm[i], ptr, (uint64_t)a->K, (uint64_t)a->M, (uint64_t)a->lda, BK, BM);
    } else {
      if (a->b_mn_major) st = make_tmap(&tm[i], ptr, (uint64_t)a->N, (uint64_t)a->K, (uint64_t)a->ldb, 64, BK);
      else               st = make_tmap(&tm[i], ptr, (uint64_t)a->K, (uint64_t)a->N, (uint64_t)a->ldb, BK, (uint32_t)bn);
    }
    if (st) return st;
  }

  const long long total_work = (long long)num_m * num_n * split_k;
  // pick the epilogue specialisation; anything unusual runs the generic one
  int epi = EPI_GENERIC;
  const bool no_extra = !a->out_colsum;
  const bool has_drop = p.drop.ctr != nullptr;   // only the F32 specialisation (and the generic path) implement it
  if (a->atomic_out == VB_GEMM_PARTIALS) {
    // split s owns rows [s*M, s*M + M) of out_f32; the caller reduces them (vb_reduce_slices) and must know the split count
    if (a->act != VB_ACT_NONE || a->bias || a->residual || !no_extra || has_drop || a->split_k != split_k)
      return set_error(VB_ERR_INVALID, "vb_gemm_bf16: VB_GEMM_PARTIALS needs a plain epilogue and split_k as vb_gemm_plan resolves it "
                       "(asked %d, resolved %d)", a->split_k, split_k);
    epi = EPI_PARTIAL; p.fast_ok = p.vec_f32;
  } else if (a->atomic_out) {
    if (a->act == VB_ACT_NONE && !a->bias && !a->residual && no_extra && !has_drop) { epi = EPI_ATOMIC; p.fast_ok = p.vec_f32; }
  } else if (a->act == VB_ACT_GELU) {
    if (a->out_pre && !a->residual && no_extra && !has_drop && (a->out_bf16 || a->out_f32)) {
      epi = EPI_GELU; p.fast_ok = p.vec_pre && (!a->out_bf16 || p.vec_bf16) && (!a->out_f32 || p.vec_f32);
    }
  } else if (a->act == VB_ACT_DGELU) {
    if (a->out_bf16 && !a->out_f32 && !a->residual && !a->bias && !has_drop) { epi = EPI_DGELU; p.fast_ok = p.vec_bf16 && p.vec_aux; }
  } else if (a->act == VB_ACT_RELU) {
    if (a->out_f32 && no_extra && !a->residual && !has_drop) { epi = EPI_F32; p.fast_ok = p.vec_f32 && (!a->out_bf16 || p.vec_bf16); }   // poolers: fp32 + operand copy
  } else if (a->act == VB_ACT_NONE) {
    if (a->out_f32 && !a->out_bf16 && no_extra) { epi = EPI_F32; p.fast_ok = 1; }   // unaligned pitches use 32-bit accesses
    else if (a->out_bf16 && !a->out_f32 && !a->residual && no_extra && !has_drop) { epi = EPI_BF16; p.fast_ok = p.vec_bf16; }
  }
  // 16-bit output variant of the BF16 / GELU specialisations; split precision (out_lo) and other combinations run the generic epilogue
  int out16 = 0;
  if (epi == EPI_BF16 || epi == EPI_GELU) {
    if ((a->out_lo || a->out_b16) && !a->out_fp16) epi = EPI_GENERIC;     // bf16 hi + lo: not a combination the engine uses
    else out16 = a->out_lo ? 3 : (a->out_fp16 ? (a->out_b16 ? 2 : 1) : 0);
  } else if (epi == EPI_DGELU && (a->out_fp16 || a->out_lo || a->out_b16)) {
    epi = EPI_GENERIC;
  }
  if (bn == 256) return launch_gemm_epi<256>(epi, out16, tm, p, total_work, max_ctas, stream);
  return launch_gemm_epi<128>(epi, out16, tm, p, total_work, max_ctas, stream);
}

extern "C" vb_status vb_gemm_plan(const vb_gemm_args* a, int32_t sm_count_, int32_t* block_n, int32_t* split_k) {
  using namespace vb;
  if (!a || !block_n || !split_k) return set_error(VB_ERR_INVALID, "vb_gemm_plan: null argument");
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return set_error(VB_ERR_INVALID, "vb_gemm_plan: empty problem %dx%dx%d", a->M, a->N, a->K);
  int sms = sm_count_;
  if (sms <= 0) {
    int cc = 0;
    if (int s = vb_device_info(&sms, &cc)) return s;
  }
  const int max_ctas = a->max_ctas > 0 ? a->max_ctas : sms;
  int bn, sp;
  if (int s = choose_config(a, max_ctas, &bn, &sp)) return s;
  *block_n = bn; *split_k = sp;
  return VB_OK;
}
