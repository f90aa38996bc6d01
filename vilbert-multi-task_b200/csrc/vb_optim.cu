// vb_optim.cu — fused multi-tensor AdamW and RAdam on the engine's flat buffers (SURVEY.md §8 f2).
//
// Reference semantics: pytorch_transformers==1.0.0 AdamW as constructed at train_tasks.py:425-426
// (AdamW(optimizer_grouped_parameters, lr=base_lr, correct_bias=False), one param group PER TENSOR with its own
// lr / weight_decay, train_tasks.py:401-421), stepped at train_tasks.py:550-551 followed by model.zero_grad():
//     m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g g;  p -= step_size m / (sqrt(v) + eps);  p -= lr wd p
// with step_size = lr (correct_bias False) or lr sqrt(1 - b2^t) / (1 - b1^t). The decoupled weight decay is applied
// AFTER the Adam update and uses the updated p, like the reference.
//
// Hyper-parameters enter as the reference's fp32 torch ops see its Python floats: b and fp32(1 - b) as the moment factors
// (the host forms 1 - b in float64: 1 - fp32(0.999) would be 0.00099998713, 1.3e-5 low), and the step sizes in float64
// (fp32 1 - b2^t loses ~1e-5 to cancellation at small t, and fast-math powf adds its approximation on top).
//
// All parameters live in ONE flat fp32 buffer (engine.ParamStore), so the whole optimizer step is one HBM-bound
// launch: per element read p, g, m, v (16 B), write p, m, v (12 B) + the 16-bit tensor-core operand copy of the new
// weight (2 B, + 2 B low part in split precision) + the zeroed gradient (4 B). That removes the separate weight
// cast and gradient memset kernels of the training step. Work is described by a chunk table (contiguous ranges that
// do not cross tensor boundaries, each pointing at its hyper-parameter group).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "vb_internal.h"
#include "vb_ptx.cuh"

namespace vb {

constexpr int OPT_THREADS = 256;

// The 16-bit tensor-core operand copies of four updated weights at float4 index i of the chunk starting at s0: hi (and its
// split-precision low part when p16_lo) in fp16 or bf16, and the always-bf16 backward copy when p16_b.
__device__ __forceinline__ void store_copies4(uint16_t* __restrict__ p16, uint16_t* __restrict__ p16_lo, __nv_bfloat16* __restrict__ p16_b,
                                              int fp16, long long s0, int i, float4 pv) {
  if (p16) {
    if (p16_lo) {
      uint32_t l01, l23;
      const uint32_t h01 = pack16_split(pv.x, pv.y, fp16, l01), h23 = pack16_split(pv.z, pv.w, fp16, l23);
      reinterpret_cast<uint2*>(p16 + s0)[i] = make_uint2(h01, h23);
      reinterpret_cast<uint2*>(p16_lo + s0)[i] = make_uint2(l01, l23);
    } else {
      reinterpret_cast<uint2*>(p16 + s0)[i] = make_uint2(pack16(pv.x, pv.y, fp16), pack16(pv.z, pv.w, fp16));
    }
  }
  if (p16_b) reinterpret_cast<uint2*>(p16_b + s0)[i] = make_uint2(pack_bf16(pv.x, pv.y), pack_bf16(pv.z, pv.w));
}

// The same for one weight at flat element e (the ragged tail of a tensor).
__device__ __forceinline__ void store_copies1(uint16_t* __restrict__ p16, uint16_t* __restrict__ p16_lo, __nv_bfloat16* __restrict__ p16_b,
                                              int fp16, long long e, float pv) {
  if (p16) {
    const uint16_t hi = cvt16(pv, fp16);
    p16[e] = hi;
    if (p16_lo) p16_lo[e] = cvt16(pv - cvt16_to_f32(hi, fp16), fp16);
  }
  if (p16_b) p16_b[e] = __float2bfloat16(pv);
}

// Sum over the CTA in a fixed order (warp trees, then the warp sums in warp order); valid in thread 0. Ends with a barrier so
// that `red` may be reused by the next call.
__device__ __forceinline__ double block_sum_f64(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = threadIdx.x < OPT_THREADS / 32 ? red[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  }
  __syncthreads();
  return v;
}

__device__ __forceinline__ double add_squares4(double acc, float4 x) {
  acc = fma((double)x.x, (double)x.x, acc); acc = fma((double)x.y, (double)x.y, acc);
  acc = fma((double)x.z, (double)x.z, acc); return fma((double)x.w, (double)x.w, acc);
}

// Gradient norm for clipping and non-finite step skipping, pass 1: partials[c] = sum of g^2 over chunk c in float64. One CTA
// reduces a whole chunk in a fixed thread order, so each partial, and the norm the finalize forms from them, is bitwise the same
// whatever the grid size. The square of an fp32 value is exact in float64 and 2^28 of them cannot overflow it: the sum is
// finite unless some gradient element is NaN or +-inf. 4 B of HBM traffic per element, four 128-bit loads in flight per thread.
__global__ void __launch_bounds__(OPT_THREADS)
grad_sq_partials_kernel(const float* __restrict__ g, const long long* __restrict__ chunk_start, const int* __restrict__ chunk_count,
                        int n_chunks, double* __restrict__ partials) {
  __shared__ double red[OPT_THREADS / 32];
  pdl_entry();
  for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const long long s0 = chunk_start[c];
    const int n = chunk_count[c];
    const int n4 = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g + s0);
    double acc = 0.0;
    for (int i0 = threadIdx.x; i0 < n4; i0 += 4 * OPT_THREADS) {
      float4 x[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * OPT_THREADS;
        x[u] = i < n4 ? g4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) acc = add_squares4(acc, x[u]);
    }
    for (int i = (n4 << 2) + threadIdx.x; i < n; i += OPT_THREADS) {
      const double x = g[s0 + i];
      acc = fma(x, x, acc);
    }
    acc = block_sum_f64(acc, red);
    if (threadIdx.x == 0) partials[c] = acc;
  }
}

// The record the clipped optimizer launches read, from the float64 sum of squares s (one thread). The clip coefficient is
// torch.nn.utils.clip_grad_norm_'s fp32 arithmetic, clamp(max_norm * reciprocal(norm + 1e-6), max=1) (torch evaluates
// `max_norm / tensor` as reciprocal times max_norm), with IEEE rounding whatever the fast-math flags.
__device__ __forceinline__ void write_clip_record(double s, float grad_scale, float max_norm, vb_clip_record* __restrict__ rec,
                                                  int* __restrict__ step) {
  const int skip = isfinite(s) ? 0 : 1;
  const float norm = (float)(fabs((double)grad_scale) * sqrt(s));
  rec->norm = norm;
  rec->coef = skip ? 0.f : fminf(__fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), max_norm), 1.f);
  rec->skip = skip;
  rec->skipped += skip;
  if (step && !skip) *step += 1;
}

// Pass 2 (one CTA): adds the partials in a fixed order and writes the record.
__global__ void __launch_bounds__(OPT_THREADS)
grad_norm_finalize_kernel(const double* __restrict__ partials, int n_chunks, float grad_scale, float max_norm,
                          vb_clip_record* __restrict__ rec, int* __restrict__ step) {
  __shared__ double red[OPT_THREADS / 32];
  pdl_entry();
  double s = 0.0;
  for (int c = threadIdx.x; c < n_chunks; c += OPT_THREADS) s += partials[c];
  s = block_sum_f64(s, red);
  if (threadIdx.x == 0) write_clip_record(s, grad_scale, max_norm, rec, step);
}

// vb_grad_norm_partial, pass 2 (one CTA): *sum = the partials added in grad_norm_finalize_kernel's fixed order.
__global__ void __launch_bounds__(OPT_THREADS)
grad_sq_sum_kernel(const double* __restrict__ partials, int n_chunks, double* __restrict__ sum) {
  __shared__ double red[OPT_THREADS / 32];
  pdl_entry();
  double s = 0.0;
  for (int c = threadIdx.x; c < n_chunks; c += OPT_THREADS) s += partials[c];
  s = block_sum_f64(s, red);
  if (threadIdx.x == 0) *sum = s;
}

// vb_clip_finish (one thread): the record from a sum of squares reduced over the ranks.
__global__ void clip_finish_kernel(const double* __restrict__ sum, float grad_scale, float max_norm, vb_clip_record* __restrict__ rec,
                                   int* __restrict__ step) {
  pdl_entry();
  write_clip_record(*sum, grad_scale, max_norm, rec, step);
}

// What a skipped step still does: zero the gradient over the chunk table (keeps the caller's "gradient is clean" bookkeeping).
__device__ void zero_chunks(float* __restrict__ g, const long long* __restrict__ chunk_start, const int* __restrict__ chunk_count,
                            int n_chunks) {
  for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const long long s0 = chunk_start[c];
    const int n = chunk_count[c];
    const int n4 = n >> 2;
    float4* g4 = reinterpret_cast<float4*>(g + s0);
    for (int i = threadIdx.x; i < n4; i += OPT_THREADS) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = (n4 << 2) + threadIdx.x; i < n; i += OPT_THREADS) g[s0 + i] = 0.f;
  }
}

// The effective gradient multiplier of an optimizer launch: grad_scale, times the clip coefficient when a record is given.
// Returns false when the record says to skip the step (the caller then only zeroes the gradient).
__device__ __forceinline__ bool step_scale(const vb_clip_record* __restrict__ rec, float grad_scale, float& gs) {
  gs = grad_scale;
  if (!rec) return true;
  if (rec->skip) return false;
  gs = grad_scale * rec->coef;
  return true;
}

// 1 - b^t in float64 for b = 1 - om, without the cancellation of forming b^t first.
__device__ __forceinline__ double one_minus_pow(float om, double t) { return -expm1(t * log1p(-(double)om)); }

// COMPACT: the moments of chunk c start at state_start[c] of m / v (a rank's slice of the optimizer state, vb_*_step_sharded)
// instead of at the weight's flat offset; the per-element arithmetic is the same.
template <bool COMPACT>
__global__ void __launch_bounds__(OPT_THREADS)
adamw_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
             uint16_t* __restrict__ p16, uint16_t* __restrict__ p16_lo, __nv_bfloat16* __restrict__ p16_b, int fp16,
             const long long* __restrict__ chunk_start, const long long* __restrict__ state_start,
             const int* __restrict__ chunk_count, const int* __restrict__ chunk_group, int n_chunks,
             const vb_adamw_group* __restrict__ groups, const int* __restrict__ step, float grad_scale, int zero_grad,
             const vb_clip_record* __restrict__ rec) {
  pdl_entry();
  float gs;
  if (!step_scale(rec, grad_scale, gs)) {
    if (zero_grad) zero_chunks(g, chunk_start, chunk_count, n_chunks);
    return;
  }
  // a counter still at 0 steps like t = 1 (the counter is advanced before the first step; 1 - b1^0 would divide by zero)
  const double t = step ? (double)max(*step, 1) : 1.0;
  for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const long long s0 = chunk_start[c];
    const int n = chunk_count[c];
    const vb_adamw_group G = groups[chunk_group[c]];
    const float step_size = G.correct_bias ? (float)((double)G.lr * sqrt(one_minus_pow(G.one_minus_beta2, t)) / one_minus_pow(G.one_minus_beta1, t))
                                           : G.lr;
    const float decay = 1.f - G.lr * G.weight_decay;   // p <- p - lr wd p  (weight_decay > 0 only)
    const float ob1 = G.one_minus_beta1, ob2 = G.one_minus_beta2;
    auto upd = [&](float pv, float gv, float& mv, float& vv) -> float {
      gv *= gs;
      mv = G.beta1 * mv + ob1 * gv;
      vv = G.beta2 * vv + ob2 * gv * gv;
      pv = pv - step_size * (mv / (sqrtf(vv) + G.eps));
      if (G.weight_decay > 0.f) pv *= decay;
      return pv;
    };
    const int n4 = n >> 2;   // chunk starts are multiples of 4 elements (tensors start on 8-element boundaries)
    const long long m0 = COMPACT ? state_start[c] : s0;   // the chunk's first moment element
    float4* p4 = reinterpret_cast<float4*>(p + s0);
    float4* g4 = reinterpret_cast<float4*>(g + s0);
    float4* m4 = reinterpret_cast<float4*>(m + m0);
    float4* v4 = reinterpret_cast<float4*>(v + m0);
    for (int i = threadIdx.x; i < n4; i += OPT_THREADS) {
      float4 pv = p4[i], mv = m4[i], vv = v4[i];
      const float4 gv = g4[i];
      pv.x = upd(pv.x, gv.x, mv.x, vv.x); pv.y = upd(pv.y, gv.y, mv.y, vv.y);
      pv.z = upd(pv.z, gv.z, mv.z, vv.z); pv.w = upd(pv.w, gv.w, mv.w, vv.w);
      p4[i] = pv; m4[i] = mv; v4[i] = vv;
      if (zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      store_copies4(p16, p16_lo, p16_b, fp16, s0, i, pv);
    }
    for (int i = (n4 << 2) + threadIdx.x; i < n; i += OPT_THREADS) {   // ragged tail of a tensor (e.g. a 3129-entry bias)
      const long long e = s0 + i, f = m0 + i;
      float mv = m[f], vv = v[f];
      const float pv = upd(p[e], g[e], mv, vv);
      p[e] = pv; m[f] = mv; v[f] = vv;
      if (zero_grad) g[e] = 0.f;
      store_copies1(p16, p16_lo, p16_b, fp16, e, pv);
    }
  }
}

// RAdam as vilbert/optimization.py:16-100 defines it (the reference's `--optim RAdam`, train_tasks.py:427-428), per element:
//     v = b2 v + (1 - b2) g g;  m = b1 m + (1 - b1) g;  p -= wd lr p   (own group's betas, lr, wd; decay FIRST, on the old p)
//     p -= step_size m / (sqrt(v) + eps)   if N_sma >= 5,   else   p -= step_size m
// with, at step t,  N_sma_max = 2 / (1 - b2) - 1,  N_sma = N_sma_max - 2 t b2^t / (1 - b2^t)  and
//     step_size = lr sqrt((1 - b2^t) (N_sma - 4) / (N_sma_max - 4) (N_sma - 2) / N_sma N_sma_max / (N_sma_max - 2)) / (1 - b1^t)
//     (N_sma >= 5),  lr / (1 - b1^t) otherwise.
// The reference caches (N_sma, step_size) per step in one buffer shared by all param groups (optimization.py:59-86), so
// within a step every tensor uses the values computed from the FIRST tensor's group: the lr, b1 and b2 of the leader group
// `leader` drive the rectified step of all tensors. Both scalars are computed in float64 like the reference's Python floats:
// in fp32, 1 - b2^t cancels (at b2 = 0.999 N_sma(6) comes out 6.0005 instead of 5.994). b = 1 - one_minus_beta, not the fp32 b:
// 2 / (1 - fp32(0.999)) - 1 is N_sma_max = 1999.03 instead of 1999. COMPACT as adamw_kernel.
template <bool COMPACT>
__global__ void __launch_bounds__(OPT_THREADS)
radam_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
             uint16_t* __restrict__ p16, uint16_t* __restrict__ p16_lo, __nv_bfloat16* __restrict__ p16_b, int fp16,
             const long long* __restrict__ chunk_start, const long long* __restrict__ state_start,
             const int* __restrict__ chunk_count, const int* __restrict__ chunk_group,
             int n_chunks, const vb_adamw_group* __restrict__ groups, int leader, const int* __restrict__ step, float grad_scale,
             int zero_grad, const vb_clip_record* __restrict__ rec) {
  __shared__ float s_step_size;
  __shared__ int s_rect;
  pdl_entry();
  float gs;
  if (!step_scale(rec, grad_scale, gs)) {   // uniform over the CTA: no thread reaches the barrier below
    if (zero_grad) zero_chunks(g, chunk_start, chunk_count, n_chunks);
    return;
  }
  if (threadIdx.x == 0) {
    const vb_adamw_group L = groups[leader];
    const double t = (double)max(*step, 1);   // the counter is advanced before the first step; 0 would divide by zero
    const double lr = L.lr, ob2 = L.one_minus_beta2;
    const double obt1 = one_minus_pow(L.one_minus_beta1, t), obt2 = one_minus_pow(L.one_minus_beta2, t);   // 1 - b1^t, 1 - b2^t
    const double n_max = 2.0 / ob2 - 1.0;
    const double n_sma = n_max - 2.0 * t * (1.0 - obt2) / obt2;
    const int rect = n_sma >= 5.0;
    const double ss = rect ? lr * sqrt(obt2 * (n_sma - 4.0) / (n_max - 4.0) * (n_sma - 2.0) / n_sma * n_max / (n_max - 2.0)) / obt1
                           : lr / obt1;
    s_step_size = (float)ss;
    s_rect = rect;
  }
  __syncthreads();
  const float step_size = s_step_size;
  const bool rect = s_rect != 0;
  for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const long long s0 = chunk_start[c];
    const int n = chunk_count[c];
    const vb_adamw_group G = groups[chunk_group[c]];
    const float decay = G.weight_decay * G.lr;
    const float ob1 = G.one_minus_beta1, ob2 = G.one_minus_beta2;
    auto upd = [&](float pv, float gv, float& mv, float& vv) -> float {
      gv *= gs;
      vv = G.beta2 * vv + ob2 * gv * gv;
      mv = G.beta1 * mv + ob1 * gv;
      if (G.weight_decay != 0.f) pv = pv - decay * pv;
      return rect ? pv - step_size * (mv / (sqrtf(vv) + G.eps)) : pv - step_size * mv;
    };
    const int n4 = n >> 2;
    const long long m0 = COMPACT ? state_start[c] : s0;   // the chunk's first moment element
    float4* p4 = reinterpret_cast<float4*>(p + s0);
    float4* g4 = reinterpret_cast<float4*>(g + s0);
    float4* m4 = reinterpret_cast<float4*>(m + m0);
    float4* v4 = reinterpret_cast<float4*>(v + m0);
    for (int i = threadIdx.x; i < n4; i += OPT_THREADS) {
      float4 pv = p4[i], mv = m4[i], vv = v4[i];
      const float4 gv = g4[i];
      pv.x = upd(pv.x, gv.x, mv.x, vv.x); pv.y = upd(pv.y, gv.y, mv.y, vv.y);
      pv.z = upd(pv.z, gv.z, mv.z, vv.z); pv.w = upd(pv.w, gv.w, mv.w, vv.w);
      p4[i] = pv; m4[i] = mv; v4[i] = vv;
      if (zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      store_copies4(p16, p16_lo, p16_b, fp16, s0, i, pv);
    }
    for (int i = (n4 << 2) + threadIdx.x; i < n; i += OPT_THREADS) {
      const long long e = s0 + i, f = m0 + i;
      float mv = m[f], vv = v[f];
      const float pv = upd(p[e], g[e], mv, vv);
      p[e] = pv; m[f] = mv; v[f] = vv;
      if (zero_grad) g[e] = 0.f;
      store_copies1(p16, p16_lo, p16_b, fp16, e, pv);
    }
  }
}

// Grid of the optimizer kernels: up to 8 CTAs per SM, at most max_ctas when max_ctas > 0, never more CTAs than chunks. The
// CTAs stride over the chunk table, so the grid decides only which CTA updates an element, never how.
static int opt_grid(int n_chunks, int max_ctas = 0) {
  int grid = sm_count() * 8;
  if (grid <= 0) grid = 132 * 8;
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  return grid > n_chunks ? n_chunks : grid;
}

static bool opt_buffers_aligned(const void* p, const void* g, const void* m, const void* v, const void* p16, const void* p16_lo,
                                const void* p16_b) {
  auto al = [](const void* q, uintptr_t a) { return (reinterpret_cast<uintptr_t>(q) % a) == 0; };
  return al(p, 16) && al(g, 16) && al(m, 16) && al(v, 16) && (!p16 || al(p16, 8)) && (!p16_lo || (al(p16_lo, 8) && p16)) && al(p16_b, 8);
}

// The two step calls share their launch code with their clipped variants; rec == NULL is the plain step.
static vb_status adamw_launch(const char* name, float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b,
                              int32_t p16_fp16, const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group,
                              int32_t n_chunks, const vb_adamw_group* groups, const int32_t* step, float grad_scale, int32_t zero_grad,
                              const vb_clip_record* rec, int32_t max_ctas, void* stream, const int64_t* state_start = nullptr) {
  if (max_ctas < 0) return set_error(VB_ERR_INVALID, "%s: max_ctas must be >= 0 (0: no cap)", name);
  if (n_chunks <= 0) return VB_OK;
  if (!p || !g || !m || !v || !chunk_start || !chunk_count || !chunk_group || !groups)
    return set_error(VB_ERR_INVALID, "%s: null argument", name);
  if (!opt_buffers_aligned(p, g, m, v, p16, p16_lo, p16_b))
    return set_error(VB_ERR_INVALID, "%s: buffers must be 16-byte aligned (16-bit copies 8-byte)", name);
  cudaError_t e = launch_pdl(state_start ? adamw_kernel<true> : adamw_kernel<false>, dim3(opt_grid(n_chunks, max_ctas)), dim3(OPT_THREADS), (size_t)0,
                             static_cast<cudaStream_t>(stream), p, g, m, v,
                             static_cast<uint16_t*>(p16), static_cast<uint16_t*>(p16_lo), static_cast<__nv_bfloat16*>(p16_b), (int)(p16_fp16 ? 1 : 0),
                             reinterpret_cast<const long long*>(chunk_start), reinterpret_cast<const long long*>(state_start), chunk_count,
                             chunk_group, (int)n_chunks, groups, step, grad_scale, (int)(zero_grad ? 1 : 0), rec);
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "%s: %s", name, cudaGetErrorString(e));
  return VB_OK;
}

static vb_status radam_launch(const char* name, float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b,
                              int32_t p16_fp16, const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group,
                              int32_t n_chunks, const vb_adamw_group* groups, int32_t leader_group, int32_t* step, int32_t advance_step,
                              float grad_scale, int32_t zero_grad, const vb_clip_record* rec, int32_t max_ctas, void* stream,
                              const int64_t* state_start = nullptr) {
  if (!step || leader_group < 0) return set_error(VB_ERR_INVALID, "%s: null step counter or negative leader group", name);
  if (max_ctas < 0) return set_error(VB_ERR_INVALID, "%s: max_ctas must be >= 0 (0: no cap)", name);
  // every argument is checked before the counter moves: a refused call changes nothing
  if (n_chunks > 0) {
    if (!p || !g || !m || !v || !chunk_start || !chunk_count || !chunk_group || !groups)
      return set_error(VB_ERR_INVALID, "%s: null argument", name);
    if (!opt_buffers_aligned(p, g, m, v, p16, p16_lo, p16_b))
      return set_error(VB_ERR_INVALID, "%s: buffers must be 16-byte aligned (16-bit copies 8-byte)", name);
  }
  if (advance_step) {
    const vb_status st = vb_step_counter_bump(reinterpret_cast<uint32_t*>(step), stream);
    if (st != VB_OK) return st;
  }
  if (n_chunks <= 0) return VB_OK;
  cudaError_t e = launch_pdl(state_start ? radam_kernel<true> : radam_kernel<false>, dim3(opt_grid(n_chunks, max_ctas)), dim3(OPT_THREADS), (size_t)0,
                             static_cast<cudaStream_t>(stream), p, g, m, v,
                             static_cast<uint16_t*>(p16), static_cast<uint16_t*>(p16_lo), static_cast<__nv_bfloat16*>(p16_b), (int)(p16_fp16 ? 1 : 0),
                             reinterpret_cast<const long long*>(chunk_start), reinterpret_cast<const long long*>(state_start), chunk_count,
                             chunk_group, (int)n_chunks, groups, (int)leader_group,
                             static_cast<const int*>(step), grad_scale, (int)(zero_grad ? 1 : 0), rec);
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "%s: %s", name, cudaGetErrorString(e));
  return VB_OK;
}

}  // namespace vb

extern "C" vb_status vb_adamw_step(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                   const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group, int32_t n_chunks,
                                   const vb_adamw_group* groups, const int32_t* step, float grad_scale, int32_t zero_grad, void* stream) {
  return vb::adamw_launch("vb_adamw_step", p, g, m, v, p16, p16_lo, p16_b, p16_fp16, chunk_start, chunk_count, chunk_group, n_chunks,
                          groups, step, grad_scale, zero_grad, nullptr, 0, stream);
}

extern "C" vb_status vb_radam_step(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                   const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group, int32_t n_chunks,
                                   const vb_adamw_group* groups, int32_t leader_group, int32_t* step, int32_t advance_step, float grad_scale,
                                   int32_t zero_grad, void* stream) {
  return vb::radam_launch("vb_radam_step", p, g, m, v, p16, p16_lo, p16_b, p16_fp16, chunk_start, chunk_count, chunk_group, n_chunks,
                          groups, leader_group, step, advance_step, grad_scale, zero_grad, nullptr, 0, stream);
}

// The same steps on at most max_ctas CTAs, for a step that shares the SMs with the backward's GEMMs (DESIGN.md §4d).
extern "C" vb_status vb_adamw_step_capped(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                          const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group,
                                          int32_t n_chunks, const vb_adamw_group* groups, const int32_t* step, float grad_scale,
                                          int32_t zero_grad, int32_t max_ctas, void* stream) {
  return vb::adamw_launch("vb_adamw_step_capped", p, g, m, v, p16, p16_lo, p16_b, p16_fp16, chunk_start, chunk_count, chunk_group,
                          n_chunks, groups, step, grad_scale, zero_grad, nullptr, max_ctas, stream);
}

extern "C" vb_status vb_radam_step_capped(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                          const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group,
                                          int32_t n_chunks, const vb_adamw_group* groups, int32_t leader_group, int32_t* step,
                                          int32_t advance_step, float grad_scale, int32_t zero_grad, int32_t max_ctas, void* stream) {
  return vb::radam_launch("vb_radam_step_capped", p, g, m, v, p16, p16_lo, p16_b, p16_fp16, chunk_start, chunk_count, chunk_group,
                          n_chunks, groups, leader_group, step, advance_step, grad_scale, zero_grad, nullptr, max_ctas, stream);
}

extern "C" vb_status vb_grad_norm(const float* g, const int64_t* chunk_start, const int32_t* chunk_count, int32_t n_chunks, float grad_scale,
                                  float max_norm, double* partials, vb_clip_record* record, int32_t* step, void* stream) {
  using namespace vb;
  if (!record) return set_error(VB_ERR_INVALID, "vb_grad_norm: null record");
  if (!(max_norm > 0.f)) return set_error(VB_ERR_INVALID, "vb_grad_norm: max_norm must be > 0 (inf: skip without clipping)");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n_chunks > 0) {
    if (!g || !chunk_start || !chunk_count || !partials) return set_error(VB_ERR_INVALID, "vb_grad_norm: null argument");
    if (reinterpret_cast<uintptr_t>(g) % 16) return set_error(VB_ERR_INVALID, "vb_grad_norm: g must be 16-byte aligned");
    cudaError_t e = launch_pdl(grad_sq_partials_kernel, dim3(opt_grid(n_chunks)), dim3(OPT_THREADS), (size_t)0, st, g,
                               reinterpret_cast<const long long*>(chunk_start), chunk_count, (int)n_chunks, partials);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_grad_norm: %s", cudaGetErrorString(e));
  }
  cudaError_t e = launch_pdl(grad_norm_finalize_kernel, dim3(1), dim3(OPT_THREADS), (size_t)0, st, (const double*)partials,
                             (int)(n_chunks > 0 ? n_chunks : 0), grad_scale, max_norm, record, static_cast<int*>(step));
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_grad_norm: %s", cudaGetErrorString(e));
  return VB_OK;
}

extern "C" vb_status vb_adamw_step_clipped(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                           const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group,
                                           int32_t n_chunks, const vb_adamw_group* groups, const int32_t* step, float grad_scale,
                                           int32_t zero_grad, const vb_clip_record* record, void* stream) {
  if (!record) return vb::set_error(VB_ERR_INVALID, "vb_adamw_step_clipped: null record");
  return vb::adamw_launch("vb_adamw_step_clipped", p, g, m, v, p16, p16_lo, p16_b, p16_fp16, chunk_start, chunk_count, chunk_group,
                          n_chunks, groups, step, grad_scale, zero_grad, record, 0, stream);
}

extern "C" vb_status vb_radam_step_clipped(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                           const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group,
                                           int32_t n_chunks, const vb_adamw_group* groups, int32_t leader_group, int32_t* step,
                                           int32_t advance_step, float grad_scale, int32_t zero_grad, const vb_clip_record* record,
                                           void* stream) {
  if (!record) return vb::set_error(VB_ERR_INVALID, "vb_radam_step_clipped: null record");
  return vb::radam_launch("vb_radam_step_clipped", p, g, m, v, p16, p16_lo, p16_b, p16_fp16, chunk_start, chunk_count, chunk_group,
                          n_chunks, groups, leader_group, step, advance_step, grad_scale, zero_grad, record, 0, stream);
}

// One rank's slice of a sharded optimizer state (optim shard_state=True): the same kernels with the moments of chunk c at
// state_start[c] of m / v; record may be NULL (no clipping), max_ctas 0 (no cap).
extern "C" vb_status vb_adamw_step_sharded(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                           const int64_t* chunk_start, const int64_t* state_start, const int32_t* chunk_count,
                                           const int32_t* chunk_group, int32_t n_chunks, const vb_adamw_group* groups, const int32_t* step,
                                           float grad_scale, int32_t zero_grad, const vb_clip_record* record, int32_t max_ctas,
                                           void* stream) {
  if (n_chunks > 0 && !state_start) return vb::set_error(VB_ERR_INVALID, "vb_adamw_step_sharded: null state_start");
  return vb::adamw_launch("vb_adamw_step_sharded", p, g, m, v, p16, p16_lo, p16_b, p16_fp16, chunk_start, chunk_count, chunk_group,
                          n_chunks, groups, step, grad_scale, zero_grad, record, max_ctas, stream, state_start);
}

extern "C" vb_status vb_radam_step_sharded(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                           const int64_t* chunk_start, const int64_t* state_start, const int32_t* chunk_count,
                                           const int32_t* chunk_group, int32_t n_chunks, const vb_adamw_group* groups, int32_t leader_group,
                                           int32_t* step, int32_t advance_step, float grad_scale, int32_t zero_grad,
                                           const vb_clip_record* record, int32_t max_ctas, void* stream) {
  if (n_chunks > 0 && !state_start) return vb::set_error(VB_ERR_INVALID, "vb_radam_step_sharded: null state_start");
  return vb::radam_launch("vb_radam_step_sharded", p, g, m, v, p16, p16_lo, p16_b, p16_fp16, chunk_start, chunk_count, chunk_group,
                          n_chunks, groups, leader_group, step, advance_step, grad_scale, zero_grad, record, max_ctas, stream, state_start);
}

extern "C" vb_status vb_grad_norm_partial(const float* g, const int64_t* chunk_start, const int32_t* chunk_count, int32_t n_chunks,
                                          double* partials, double* sum, void* stream) {
  using namespace vb;
  if (!sum) return set_error(VB_ERR_INVALID, "vb_grad_norm_partial: null sum");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n_chunks > 0) {
    if (!g || !chunk_start || !chunk_count || !partials) return set_error(VB_ERR_INVALID, "vb_grad_norm_partial: null argument");
    if (reinterpret_cast<uintptr_t>(g) % 16) return set_error(VB_ERR_INVALID, "vb_grad_norm_partial: g must be 16-byte aligned");
    cudaError_t e = launch_pdl(grad_sq_partials_kernel, dim3(opt_grid(n_chunks)), dim3(OPT_THREADS), (size_t)0, st, g,
                               reinterpret_cast<const long long*>(chunk_start), chunk_count, (int)n_chunks, partials);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_grad_norm_partial: %s", cudaGetErrorString(e));
  }
  cudaError_t e = launch_pdl(grad_sq_sum_kernel, dim3(1), dim3(OPT_THREADS), (size_t)0, st, (const double*)partials,
                             (int)(n_chunks > 0 ? n_chunks : 0), sum);
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_grad_norm_partial: %s", cudaGetErrorString(e));
  return VB_OK;
}

extern "C" vb_status vb_clip_finish(const double* sum, float grad_scale, float max_norm, vb_clip_record* record, int32_t* step,
                                    void* stream) {
  using namespace vb;
  if (!sum || !record) return set_error(VB_ERR_INVALID, "vb_clip_finish: null sum or record");
  if (!(max_norm > 0.f)) return set_error(VB_ERR_INVALID, "vb_clip_finish: max_norm must be > 0 (inf: skip without clipping)");
  cudaError_t e = launch_pdl(clip_finish_kernel, dim3(1), dim3(1), (size_t)0, static_cast<cudaStream_t>(stream), sum, grad_scale,
                             max_norm, record, static_cast<int*>(step));
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_clip_finish: %s", cudaGetErrorString(e));
  return VB_OK;
}
