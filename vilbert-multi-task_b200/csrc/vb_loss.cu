// vb_loss.cu — objectives of the ViLBERT heads as single fused kernels (SURVEY.md §8 f1): softmax cross-entropy with
// ignore_index (masked-LM over the 30522-way tied decoder, alignment / VL-logit / tri / binary heads; vilbert.py:1578-1590,
// task_utils.py:339-374) and the masked-region KL divergence of the pre-training objective (vilbert.py:1506-1525). Each reads
// the fp32 logits ONCE more than strictly needed (max, then exp-sum + gradient from the row kept in registers / L2) and writes
// the gradient of the logits directly as the bf16 GEMM operand of the head's backward (and optionally fp32): no separate
// log_softmax / nll / kl_div / masking / cast kernels, no fp32 probability tensor.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "vb_internal.h"
#include "vb_ptx.cuh"

namespace vb {

constexpr int LOSS_THREADS = 256;

__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, w) : v + w;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = (threadIdx.x < LOSS_THREADS / 32) ? red[threadIdx.x] : (is_max ? -CUDART_INF_F : 0.f);
  if (threadIdx.x < 32) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float w = __shfl_xor_sync(0xffffffffu, r, o);
      r = is_max ? fmaxf(r, w) : r + w;
    }
    if (threadIdx.x == 0) red[0] = r;
  }
  __syncthreads();
  return red[0];
}

// number of entries of labels[0..n) for which pred holds, computed redundantly by every CTA (n is a few thousand at most)
template <typename Pred>
__device__ __forceinline__ float block_count(const long long* labels, int n, float* red, Pred pred) {
  float c = 0.f;
  for (int i = threadIdx.x; i < n; i += LOSS_THREADS) c += pred(labels[i]) ? 1.f : 0.f;
  return block_reduce(c, red, false);
}

// F.cross_entropy(logits [rows, cols], labels [rows], ignore_index), reduction = mean over the non-ignored rows.
// One CTA per row (grid-stride). loss += sum over its rows of (lse - z[label]) / n_valid; dlogits = (softmax - onehot) * gs / n_valid.
__global__ void __launch_bounds__(LOSS_THREADS)
ce_loss_kernel(const float* __restrict__ z, long long ldz, const long long* __restrict__ labels, long long ignore_index,
               float* __restrict__ loss, float* __restrict__ d32, long long ldd32, __nv_bfloat16* __restrict__ d16, long long ldd16,
               int rows, int cols, float grad_scale) {
  pdl_entry();
  __shared__ float red[LOSS_THREADS / 32];
  const float n_valid = block_count(labels, rows, red, [&](long long l) { return l != ignore_index; });
  const float inv = n_valid > 0.f ? 1.f / n_valid : 0.f;
  float local = 0.f;
  for (int r = blockIdx.x; r < rows; r += gridDim.x) {
    const long long lab = labels[r];
    const float* zr = z + (long long)r * ldz;
    const bool live = lab != ignore_index;
    if (!live) {   // ignored row: zero gradient
      for (int c = threadIdx.x; c < cols; c += LOSS_THREADS) {
        if (d32) d32[(long long)r * ldd32 + c] = 0.f;
        if (d16) d16[(long long)r * ldd16 + c] = __float2bfloat16(0.f);
      }
      continue;
    }
    float mx = -CUDART_INF_F;
    for (int c = threadIdx.x; c < cols; c += LOSS_THREADS) mx = fmaxf(mx, zr[c]);
    mx = block_reduce(mx, red, true);
    float s = 0.f;
    for (int c = threadIdx.x; c < cols; c += LOSS_THREADS) s += __expf(zr[c] - mx);
    s = block_reduce(s, red, false);
    const float lse = mx + __logf(s);
    const float gs = grad_scale * inv;
    for (int c = threadIdx.x; c < cols; c += LOSS_THREADS) {
      float g = __expf(zr[c] - lse);
      if (c == lab) g -= 1.f;
      g *= gs;
      if (d32) d32[(long long)r * ldd32 + c] = g;
      if (d16) d16[(long long)r * ldd16 + c] = __float2bfloat16(g);
    }
    if (threadIdx.x == 0) local += (lse - zr[lab]) * inv;
  }
  if (threadIdx.x == 0 && local != 0.f) atomicAdd(loss, local);
  if (threadIdx.x == 0 && blockIdx.x == 0 && n_valid == 0.f) atomicAdd(loss, CUDART_NAN_F);   // torch: mean over no rows = nan
}

// Masked-region objective (vilbert.py:1506-1525, visual_target == 0):
//   scores = prediction_scores_v[:, 1:]            (the global region 0 is dropped)
//   loss   = sum_{b,r: label[b,r] == 1} sum_c t * (log t - log_softmax(scores)_c)  /  max(#(label == 1), 0)
// scores: f32 [B, Nv, C] (ld = C between regions), target f32 [B, Nv-1, C], label int64 [B, Nv-1]. One CTA per (b, r) row.
// d scores_c = ((sum_c t) * softmax_c - t_c) * gs / n_pos on masked rows, 0 elsewhere (incl. region 0).
__global__ void __launch_bounds__(LOSS_THREADS)
kl_masked_loss_kernel(const float* __restrict__ scores, const float* __restrict__ target, const long long* __restrict__ label,
                      float* __restrict__ loss, float* __restrict__ d32, __nv_bfloat16* __restrict__ d16, long long ldd16, int B, int Nv,
                      int C, float grad_scale) {
  pdl_entry();
  __shared__ float red[LOSS_THREADS / 32];
  const int rows_t = B * (Nv - 1);
  const float n_pos = block_count(label, rows_t, red, [](long long l) { return l == 1; });
  const float inv = n_pos > 0.f ? 1.f / n_pos : 0.f;
  float local = 0.f;
  const int rows = B * Nv;
  for (int rr = blockIdx.x; rr < rows; rr += gridDim.x) {
    const int b = rr / Nv, reg = rr % Nv;
    const bool live = reg > 0 && label[(long long)b * (Nv - 1) + reg - 1] == 1;
    if (!live) {
      for (int c = threadIdx.x; c < C; c += LOSS_THREADS) {
        if (d32) d32[(long long)rr * C + c] = 0.f;
        if (d16) d16[(long long)rr * ldd16 + c] = __float2bfloat16(0.f);
      }
      continue;
    }
    const float* zr = scores + (long long)rr * C;
    const float* tr = target + ((long long)b * (Nv - 1) + reg - 1) * C;
    float mx = -CUDART_INF_F;
    for (int c = threadIdx.x; c < C; c += LOSS_THREADS) mx = fmaxf(mx, zr[c]);
    mx = block_reduce(mx, red, true);
    float s = 0.f, ts = 0.f;
    for (int c = threadIdx.x; c < C; c += LOSS_THREADS) { s += __expf(zr[c] - mx); ts += tr[c]; }
    s = block_reduce(s, red, false);
    ts = block_reduce(ts, red, false);
    const float lse = mx + __logf(s);
    float acc = 0.f;
    const float gs = grad_scale * inv;
    for (int c = threadIdx.x; c < C; c += LOSS_THREADS) {
      const float t = tr[c], lp = zr[c] - lse;
      if (t > 0.f) acc += t * (__logf(t) - lp);      // F.kl_div: t * (log t - input), 0 where t == 0
      const float g = (ts * __expf(lp) - t) * gs;
      if (d32) d32[(long long)rr * C + c] = g;
      if (d16) d16[(long long)rr * ldd16 + c] = __float2bfloat16(g);
    }
    acc = block_reduce(acc, red, false);
    if (threadIdx.x == 0) local += acc * inv;
  }
  if (threadIdx.x == 0 && local != 0.f) atomicAdd(loss, local);
  if (threadIdx.x == 0 && blockIdx.x == 0 && n_pos == 0.f) atomicAdd(loss, CUDART_NAN_F);   // 0 / max(0, 0) in the reference
}

// ------------------------------------------------------------------------------------------ masked-row compaction (masked-LM head)
// Only the rows whose label != ignore_index contribute to the masked-LM cross-entropy (15 % of the tokens, vilbert.py:1578-1583),
// so when only the loss is wanted the 30522-way tied decoder runs on those rows alone: idx[r] = r-th selected row (ascending),
// -1 beyond the count; *count = number of selected rows (may exceed cap: the caller checks).
__global__ void __launch_bounds__(1024) compact_rows_kernel(const long long* __restrict__ labels, long long ignore_index, int rows, int cap,
                                                             int* __restrict__ idx, int* __restrict__ count, long long* __restrict__ labels_c) {
  pdl_entry();
  __shared__ int wsum[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  for (int i = threadIdx.x; i < cap; i += 1024) { idx[i] = -1; labels_c[i] = ignore_index; }
  __syncthreads();
  for (int base = 0; base < rows; base += 1024) {
    const int r = base + threadIdx.x;
    const int sel = (r < rows && labels[r] != ignore_index) ? 1 : 0;
    int v = sel;                                   // inclusive warp scan
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, v, o); if ((threadIdx.x & 31) >= o) v += n; }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
      int w = wsum[threadIdx.x];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, w, o); if (threadIdx.x >= o) w += n; }
      wsum[threadIdx.x] = w;
    }
    __syncthreads();
    const int before = carry + (threadIdx.x >= 32 ? wsum[(threadIdx.x >> 5) - 1] : 0) + v - sel;
    if (sel && before < cap) { idx[before] = r; labels_c[before] = labels[r]; }
    __syncthreads();
    if (threadIdx.x == 0) carry += wsum[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = carry;
}

// dst[r, :] = idx[r] >= 0 ? src[idx[r], :] : 0 (16-bit rows of `cols` elements, cols % 8 == 0), for up to two sources at once
__global__ void gather_rows16_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, const uint4* __restrict__ src2, uint4* __restrict__ dst2,
                                     const int* __restrict__ idx, int cap, int c8) {
  pdl_entry();
  const long long total = (long long)cap * c8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / c8), c = (int)(i % c8);
    const int s = idx[r];
    dst[i] = s >= 0 ? src[(long long)s * c8 + c] : make_uint4(0, 0, 0, 0);
    if (src2) dst2[i] = s >= 0 ? src2[(long long)s * c8 + c] : make_uint4(0, 0, 0, 0);
  }
}

// dst[idx[r], :] = src[r, :] for idx[r] >= 0 (fp32 rows, cols % 4 == 0); dst is zeroed by the caller. If more rows were selected
// than the capacity holds (*count > cap) the result would silently miss rows: the loss scalar is poisoned with NaN instead.
__global__ void scatter_rows_f32_kernel(const float4* __restrict__ src, float4* __restrict__ dst, const int* __restrict__ idx, int cap, int c4,
                                        const int* __restrict__ count, float* __restrict__ poison) {
  pdl_entry();
  if (count && poison && blockIdx.x == 0 && threadIdx.x == 0 && *count > cap) *poison = CUDART_NAN_F;
  const long long total = (long long)cap * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / c4), c = (int)(i % c4);
    const int d = idx[r];
    if (d >= 0) dst[(long long)d * c4 + c] = src[i];
  }
}

static inline int loss_grid(int rows) {
  int cap = sm_count() * 8;
  if (cap <= 0) cap = 132 * 8;
  return rows < cap ? (rows > 0 ? rows : 1) : cap;
}

}  // namespace vb

using namespace vb;

extern "C" vb_status vb_ce_loss(const float* logits, int64_t ld_logits, const int64_t* labels, int64_t ignore_index, float* loss,
                                float* dlogits_f32, int64_t ld_d32, void* dlogits_bf16, int64_t ld_d16, int32_t rows, int32_t cols,
                                float grad_scale, int32_t accumulate_loss, void* stream) {
  if (rows <= 0 || cols <= 0 || !logits || !labels || !loss) return set_error(VB_ERR_INVALID, "vb_ce_loss: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!accumulate_loss) {
    cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), st);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_ce_loss: memset: %s", cudaGetErrorString(e));
  }
  launch_pdl(ce_loss_kernel, dim3(loss_grid(rows)), dim3(LOSS_THREADS), (size_t)0, st, logits, (long long)ld_logits,
             reinterpret_cast<const long long*>(labels), (long long)ignore_index, loss, dlogits_f32, (long long)ld_d32,
             static_cast<__nv_bfloat16*>(dlogits_bf16), (long long)ld_d16, (int)rows, (int)cols, grad_scale);
  return check_launch("vb_ce_loss");
}

extern "C" vb_status vb_kl_masked_loss(const float* scores, const float* target, const int64_t* label, float* loss, float* dscores_f32,
                                       void* dscores_bf16, int64_t ld_d16, int32_t B, int32_t Nv, int32_t C, float grad_scale,
                                       int32_t accumulate_loss, void* stream) {
  if (B <= 0 || Nv <= 1 || C <= 0 || !scores || !target || !label || !loss) return set_error(VB_ERR_INVALID, "vb_kl_masked_loss: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!accumulate_loss) {
    cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), st);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_kl_masked_loss: memset: %s", cudaGetErrorString(e));
  }
  launch_pdl(kl_masked_loss_kernel, dim3(loss_grid(B * Nv)), dim3(LOSS_THREADS), (size_t)0, st, scores, target,
             reinterpret_cast<const long long*>(label), loss, dscores_f32, static_cast<__nv_bfloat16*>(dscores_bf16), (long long)ld_d16,
             (int)B, (int)Nv, (int)C, grad_scale);
  return check_launch("vb_kl_masked_loss");
}

extern "C" vb_status vb_compact_rows(const int64_t* labels, int64_t ignore_index, int32_t rows, int32_t cap, int32_t* idx, int32_t* count,
                                     int64_t* labels_compact, void* stream) {
  if (rows <= 0 || cap <= 0 || !labels || !idx || !count || !labels_compact) return set_error(VB_ERR_INVALID, "vb_compact_rows: bad arguments");
  launch_pdl(compact_rows_kernel, dim3(1), dim3(1024), (size_t)0, static_cast<cudaStream_t>(stream), reinterpret_cast<const long long*>(labels),
             (long long)ignore_index, (int)rows, (int)cap, idx, count, reinterpret_cast<long long*>(labels_compact));
  return check_launch("vb_compact_rows");
}

extern "C" vb_status vb_gather_rows16(const void* src, void* dst, const void* src2, void* dst2, const int32_t* idx, int32_t cap, int32_t cols,
                                      void* stream) {
  if (cap <= 0 || cols <= 0 || (cols & 7) || !src || !dst || !idx) return set_error(VB_ERR_INVALID, "vb_gather_rows16: bad arguments (cols % 8 == 0)");
  int grid = sm_count() * 8; if (grid <= 0) grid = 132 * 8;
  launch_pdl(gather_rows16_kernel, dim3(grid), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream), static_cast<const uint4*>(src),
             static_cast<uint4*>(dst), static_cast<const uint4*>(src2), static_cast<uint4*>(dst2), idx, (int)cap, (int)(cols / 8));
  return check_launch("vb_gather_rows16");
}

extern "C" vb_status vb_scatter_rows_f32(const float* src, float* dst, const int32_t* idx, int32_t cap, int32_t cols, const int32_t* count,
                                         float* poison, void* stream) {
  if (cap <= 0 || cols <= 0 || (cols & 3) || !src || !dst || !idx) return set_error(VB_ERR_INVALID, "vb_scatter_rows_f32: bad arguments (cols % 4 == 0)");
  int grid = sm_count() * 8; if (grid <= 0) grid = 132 * 8;
  launch_pdl(scatter_rows_f32_kernel, dim3(grid), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream), reinterpret_cast<const float4*>(src),
             reinterpret_cast<float4*>(dst), idx, (int)cap, (int)(cols / 4), count, poison);
  return check_launch("vb_scatter_rows_f32");
}
