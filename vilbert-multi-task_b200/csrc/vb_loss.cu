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
// A label outside [0, cols) (and != ignore_index) reads nothing: its row's gradient is 0 and the loss is NaN, as in bce_gather_rows.
// PARTIALS (deterministic plans): CTA b stores its share, with the NaN of "no valid row" in CTA 0's, into part[b] instead of adding
// it to *loss; vb_ce_loss_det sums the shares in CTA order.
template <bool PARTIALS>
__device__ __forceinline__ void
ce_loss_body(const float* __restrict__ z, long long ldz, const long long* __restrict__ labels, long long ignore_index,
             float* __restrict__ loss, float* __restrict__ d32, long long ldd32, __nv_bfloat16* __restrict__ d16, long long ldd16,
             int rows, int cols, float grad_scale, float* __restrict__ part) {
  pdl_entry();
  __shared__ float red[LOSS_THREADS / 32];
  const float n_valid = block_count(labels, rows, red, [&](long long l) { return l != ignore_index; });
  const float inv = n_valid > 0.f ? 1.f / n_valid : 0.f;
  float local = 0.f;
  for (int r = blockIdx.x; r < rows; r += gridDim.x) {
    const long long lab = labels[r];
    const float* zr = z + (long long)r * ldz;
    const bool live = lab != ignore_index;
    const bool in_range = lab >= 0 && lab < cols;
    if (!live || !in_range) {   // ignored row: zero gradient; a label outside [0, cols) reads nothing and makes the loss NaN
      for (int c = threadIdx.x; c < cols; c += LOSS_THREADS) {
        if (d32) d32[(long long)r * ldd32 + c] = 0.f;
        if (d16) d16[(long long)r * ldd16 + c] = __float2bfloat16(0.f);
      }
      if (live && threadIdx.x == 0) local += CUDART_NAN_F;
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
  if (PARTIALS) {
    if (threadIdx.x == 0) part[blockIdx.x] = (blockIdx.x == 0 && n_valid == 0.f) ? local + CUDART_NAN_F : local;
    return;
  }
  if (threadIdx.x == 0 && local != 0.f) atomicAdd(loss, local);
  if (threadIdx.x == 0 && blockIdx.x == 0 && n_valid == 0.f) atomicAdd(loss, CUDART_NAN_F);   // torch: mean over no rows = nan
}
__global__ void __launch_bounds__(LOSS_THREADS)
ce_loss_kernel(const float* __restrict__ z, long long ldz, const long long* __restrict__ labels, long long ignore_index,
               float* __restrict__ loss, float* __restrict__ d32, long long ldd32, __nv_bfloat16* __restrict__ d16, long long ldd16,
               int rows, int cols, float grad_scale) {
  ce_loss_body<false>(z, ldz, labels, ignore_index, loss, d32, ldd32, d16, ldd16, rows, cols, grad_scale, nullptr);
}
__global__ void __launch_bounds__(LOSS_THREADS)
ce_loss_det_kernel(const float* __restrict__ z, long long ldz, const long long* __restrict__ labels, long long ignore_index,
                   float* __restrict__ d32, long long ldd32, __nv_bfloat16* __restrict__ d16, long long ldd16, int rows, int cols,
                   float grad_scale, float* __restrict__ part) {
  ce_loss_body<true>(z, ldz, labels, ignore_index, nullptr, d32, ldd32, d16, ldd16, rows, cols, grad_scale, part);
}

// Masked-region objective (vilbert.py:1506-1525, visual_target == 0):
//   scores = prediction_scores_v[:, 1:]            (the global region 0 is dropped)
//   loss   = sum_{b,r: label[b,r] == 1} sum_c t * (log t - log_softmax(scores)_c)  /  max(#(label == 1), 0)
// scores: f32 [B, Nv, C] (ld = C between regions), target f32 [B, Nv-1, C], label int64 [B, Nv-1]. One CTA per (b, r) row.
// d scores_c = ((sum_c t) * softmax_c - t_c) * gs / n_pos on masked rows, 0 elsewhere (incl. region 0).
// PARTIALS: as ce_loss_body
template <bool PARTIALS>
__device__ __forceinline__ void
kl_masked_loss_body(const float* __restrict__ scores, const float* __restrict__ target, const long long* __restrict__ label,
                    float* __restrict__ loss, float* __restrict__ d32, __nv_bfloat16* __restrict__ d16, long long ldd16, int B, int Nv,
                    int C, float grad_scale, float* __restrict__ part) {
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
  if (PARTIALS) {
    if (threadIdx.x == 0) part[blockIdx.x] = (blockIdx.x == 0 && n_pos == 0.f) ? local + CUDART_NAN_F : local;
    return;
  }
  if (threadIdx.x == 0 && local != 0.f) atomicAdd(loss, local);
  if (threadIdx.x == 0 && blockIdx.x == 0 && n_pos == 0.f) atomicAdd(loss, CUDART_NAN_F);   // 0 / max(0, 0) in the reference
}
__global__ void __launch_bounds__(LOSS_THREADS)
kl_masked_loss_kernel(const float* __restrict__ scores, const float* __restrict__ target, const long long* __restrict__ label,
                      float* __restrict__ loss, float* __restrict__ d32, __nv_bfloat16* __restrict__ d16, long long ldd16, int B, int Nv,
                      int C, float grad_scale) {
  kl_masked_loss_body<false>(scores, target, label, loss, d32, d16, ldd16, B, Nv, C, grad_scale, nullptr);
}
__global__ void __launch_bounds__(LOSS_THREADS)
kl_masked_loss_det_kernel(const float* __restrict__ scores, const float* __restrict__ target, const long long* __restrict__ label,
                          float* __restrict__ d32, __nv_bfloat16* __restrict__ d16, long long ldd16, int B, int Nv, int C, float grad_scale,
                          float* __restrict__ part) {
  kl_masked_loss_body<true>(scores, target, label, nullptr, d32, d16, ldd16, B, Nv, C, grad_scale, part);
}

// ------------------------------------------------------------------------------------------ masked-row compaction (masked-LM head)
// Only the rows whose label != ignore_index contribute to the masked-LM cross-entropy (15 % of the tokens, vilbert.py:1578-1583),
// so when only the loss is wanted the 30522-way tied decoder runs on those rows alone: idx[r] = r-th selected row (ascending),
// -1 beyond the count; *count = number of selected rows (may exceed cap: the caller checks). With a row map (a packed stream,
// vb_pack.cu) row r stands for padded row map[r] and is selected when map[r] >= 0 and labels[map[r]] != ignore_index; idx then
// holds packed rows, in the order of their padded rows.
__global__ void __launch_bounds__(1024) compact_rows_kernel(const long long* __restrict__ labels, long long ignore_index, const int* __restrict__ map,
                                                             int rows, int cap, int* __restrict__ idx, int* __restrict__ count,
                                                             long long* __restrict__ labels_c) {
  pdl_entry();
  __shared__ int wsum[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  for (int i = threadIdx.x; i < cap; i += 1024) { idx[i] = -1; labels_c[i] = ignore_index; }
  __syncthreads();
  for (int base = 0; base < rows; base += 1024) {
    const int r = base + threadIdx.x;
    const int src = r < rows ? (map ? map[r] : r) : -1;
    const int sel = (src >= 0 && labels[src] != ignore_index) ? 1 : 0;
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
    if (sel && before < cap) { idx[before] = r; labels_c[before] = labels[src]; }
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

// ------------------------------------------------------------------------------------------ task objectives and scores (12-in-1)
// BCE-with-logits over gathered columns (task_utils.py:352-374): for row r and choice c, x = logits[r, off + ids[r, c]] (ids NULL:
// c), loss_rc = max(x,0) - x t + log1p(exp(-|x|)). One CTA per row; the logits row and the per-choice gradients live in shared
// memory. d logits[r, j] = sum over the choices c that gathered column j of (sigmoid(x) - t) * gs, summed in choice order by the
// thread owning column j (no atomics: the result does not depend on scheduling); columns nobody gathered get 0. An id outside
// [0, width - off) reads nothing and makes the row's loss NaN. row_loss[r] = sum_c loss_rc * loss_scale.
__global__ void __launch_bounds__(LOSS_THREADS)
bce_gather_rows_kernel(const float* __restrict__ logits, long long ld, int off, int width, const long long* __restrict__ ids,
                       const float* __restrict__ target, int C, float loss_scale, float* __restrict__ row_loss,
                       float* __restrict__ d32, long long ldd32, __nv_bfloat16* __restrict__ d16, long long ldd16) {
  pdl_entry();
  extern __shared__ float smem[];
  float* xs = smem;                                          // [width] the logits row
  float* gs = xs + width;                                    // [C] gradient of each choice
  int* col = reinterpret_cast<int*>(gs + C);                 // [C] column it gathered (-1: out of range)
  __shared__ float red[LOSS_THREADS / 32];
  const int r = blockIdx.x;
  const float* zr = logits + (long long)r * ld;
  for (int j = threadIdx.x; j < width; j += LOSS_THREADS) xs[j] = zr[j];
  __syncthreads();
  float acc = 0.f;
  for (int c = threadIdx.x; c < C; c += LOSS_THREADS) {
    const long long id = ids ? ids[(long long)r * C + c] : (long long)c;
    const bool ok = id >= 0 && id < (long long)(width - off);
    const float t = target[(long long)r * C + c];
    if (ok) {
      const int j = off + (int)id;
      const float x = xs[j];
      const float e = __expf(-fabsf(x));
      acc += fmaxf(x, 0.f) - x * t + log1pf(e);
      const float s = x >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
      gs[c] = (s - t) * loss_scale;
      col[c] = j;
    } else {
      acc += CUDART_NAN_F;
      gs[c] = 0.f;
      col[c] = -1;
    }
  }
  acc = block_reduce(acc, red, false);       // ends with a barrier: gs / col are visible
  if (threadIdx.x == 0) row_loss[r] = acc * loss_scale;
  for (int j = threadIdx.x; j < width; j += LOSS_THREADS) {
    float g = 0.f;
    if (ids) {
      for (int c = 0; c < C; ++c) g += col[c] == j ? gs[c] : 0.f;
    } else if (j >= off && j - off < C) {
      g = gs[j - off];
    }
    if (d32) d32[(long long)r * ldd32 + j] = g;
    if (d16) d16[(long long)r * ldd16 + j] = __float2bfloat16(g);
  }
}

// *loss (+)= sum of row_loss[0..rows) in a fixed order (one CTA)
__global__ void __launch_bounds__(LOSS_THREADS) sum_rows_kernel(const float* __restrict__ row_loss, int rows, float* __restrict__ loss, int accumulate) {
  pdl_entry();
  __shared__ float red[LOSS_THREADS / 32];
  float s = 0.f;
  for (int i = threadIdx.x; i < rows; i += LOSS_THREADS) s += row_loss[i];
  s = block_reduce(s, red, false);
  if (threadIdx.x == 0) *loss = accumulate ? *loss + s : s;
}

// torch.max(dim) rules: a NaN is the maximum, the first index wins among equals (and among NaNs)
__device__ __forceinline__ bool arg_better(float a, int ia, float b, int ib) {
  const bool na = a != a, nb = b != b;
  if (na || nb) return na && (!nb || ia < ib);
  return a > b || (a == b && ia < ib);
}

__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    const int k = __shfl_xor_sync(0xffffffffu, i, o);
    if (arg_better(w, k, v, i)) { v = w; i = k; }
  }
}

// one warp per row (grid-stride over the rows of one CTA): argmax, then the per-row score of `mode`; the CTA sums in fixed order
__global__ void __launch_bounds__(LOSS_THREADS)
task_score_kernel(int mode, const float* __restrict__ logits, long long ld, int off, int cols, const long long* __restrict__ ids,
                  int width, const float* __restrict__ target, long long ldt, const long long* __restrict__ labels, int rows,
                  float* __restrict__ score, int accumulate, long long* __restrict__ preds) {
  pdl_entry();
  __shared__ double part[LOSS_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double s = 0.0;
  for (int r = warp; r < rows; r += LOSS_THREADS / 32) {
    const float* zr = logits + (long long)r * ld;
    float v = -CUDART_INF_F;
    int a = 0x7fffffff;
    for (int c = lane; c < cols; c += 32) {
      float x;
      if (ids) {
        const long long id = ids[(long long)r * cols + c];
        x = (id >= 0 && id < (long long)(width - off)) ? zr[off + id] : CUDART_NAN_F;
      } else {
        x = zr[off + c];
      }
      if (arg_better(x, c, v, a)) { v = x; a = c; }
    }
    warp_argmax(v, a);
    const float* tr = target ? target + (long long)r * ldt : nullptr;
    float hit = 0.f;
    if (mode == VB_SCORE_SOFT) {
      hit = tr[a];
    } else if (mode == VB_SCORE_LABEL) {
      hit = (long long)a == labels[r] ? 1.f : 0.f;
    } else if (mode == VB_SCORE_THRESHOLD) {
      hit = tr[a] > 0.5f ? 1.f : 0.f;
    } else {   // VB_SCORE_CHOICE: argmax of the target row
      float tv = -CUDART_INF_F;
      int ta = 0x7fffffff;
      for (int c = lane; c < cols; c += 32)
        if (arg_better(tr[c], c, tv, ta)) { tv = tr[c]; ta = c; }
      warp_argmax(tv, ta);
      hit = a == ta ? 1.f : 0.f;
    }
    if (lane == 0) {
      s += (double)hit;
      if (preds) preds[r] = a;
    }
  }
  if (lane == 0) part[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < LOSS_THREADS / 32; ++w) t += part[w];
    *score = (float)((accumulate ? (double)*score : 0.0) + t);
  }
}

// per-row evaluation results (vb_task_results): one warp per row, RESULTS_ROWS rows per CTA, every row written by its own warp
constexpr int RESULTS_ROWS = LOSS_THREADS / 32;

__device__ __forceinline__ float result_logit(const float* zr, int off, const long long* idr, int width, int c) {
  if (!idr) return zr[off + c];
  const long long id = idr[c];
  return (id >= 0 && id < (long long)(width - off)) ? zr[off + id] : CUDART_NAN_F;
}

__global__ void __launch_bounds__(LOSS_THREADS)
task_results_kernel(int mode, const float* __restrict__ logits, long long ld, int off, int cols, const long long* __restrict__ ids,
                    int width, const float* __restrict__ target, long long ldt, int rows, long long* __restrict__ argmax,
                    float* __restrict__ values, long long ldv) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * RESULTS_ROWS + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* zr = logits + (long long)r * ld;
  const long long* idr = ids ? ids + (long long)r * cols : nullptr;
  float v = -CUDART_INF_F;
  int a = 0x7fffffff;
  for (int c = lane; c < cols; c += 32) {
    const float x = result_logit(zr, off, idr, width, c);
    if (arg_better(x, c, v, a)) { v = x; a = c; }
  }
  warp_argmax(v, a);
  if (lane == 0) {
    argmax[r] = a;
    if (mode == VB_RESULT_GATHER) values[r] = target[(long long)r * ldt + a];
  }
  if (mode != VB_RESULT_SOFTMAX) return;
  // softmax(row) = exp(x - max) / sum: the exponentials in double (exact to the float result, whatever --use_fast_math does to
  // expf) and summed in double; a NaN maximum (a NaN in the row) or an infinite one makes every probability NaN, as in torch
  double s = 0.0;
  for (int c = lane; c < cols; c += 32) s += exp((double)(result_logit(zr, off, idr, width, c) - v));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const double inv = 1.0 / s;
  float* out = values + (long long)r * ldv;
  for (int c = lane; c < cols; c += 32) out[c] = (float)(exp((double)(result_logit(zr, off, idr, width, c) - v)) * inv);
}

// ------------------------------------------------------------------------------------------ retrieval ranks (vb_retrieval_rank[_sets])
// Stable descending order of a score row as one 64-bit key per column, higher = earlier: the high word maps the float to an
// unsigned integer that orders like the number (-0.0 folded onto +0.0, every NaN to 0, below -inf), the low word is ~column, so
// equal scores keep the column order. Integer keys only: no float comparison, so --use_fast_math's flush-to-zero does not tie
// subnormal scores with 0.
constexpr int RANK_THREADS = 512;
constexpr int RANK_MAX_COLS = 50000;
constexpr int RANK_MAX_K = 64;

__device__ __forceinline__ uint32_t rank_key_hi(float x) {
  uint32_t u = __float_as_uint(x);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0u;          // NaN: after every number
  if (u == 0x80000000u) u = 0u;                              // -0.0 ties with +0.0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ unsigned long long rank_key(const uint32_t* hi, int j) {
  return ((unsigned long long)hi[j] << 32) | (uint32_t)~(uint32_t)j;
}

// block-wide max of a 64-bit key (red: RANK_THREADS / 32 entries); every thread gets the result
__device__ __forceinline__ unsigned long long block_max_u64(unsigned long long v, unsigned long long* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long r = red[0];
  for (int w = 1; w < RANK_THREADS / 32; ++w) r = red[w] > r ? red[w] : r;
  return r;
}

// one CTA per row: the row's keys are staged in dynamic shared memory (4 bytes per column). Row r's targets are
// idx[off[r] .. off[r+1]), or idx[r] alone when off is NULL (vb_retrieval_rank). The best-placed target is the largest of their
// keys, found with one block-wide max; the rank is one block-wide count of the keys above it, the top-k k block-wide arg-max
// rounds, each bounded by the previous pick. No atomics.
__global__ void __launch_bounds__(RANK_THREADS)
retrieval_rank_kernel(const float* __restrict__ scores, long long ld, int N, const long long* __restrict__ off,
                      const long long* __restrict__ idx, int k, int* __restrict__ rank_out, int* __restrict__ topk_out) {
  pdl_entry();
  extern __shared__ uint32_t keys[];
  __shared__ unsigned long long red64[RANK_THREADS / 32];
  __shared__ int red32[RANK_THREADS / 32];
  const int r = blockIdx.x;
  const float* row = scores + (long long)r * ld;
  for (int j = threadIdx.x; j < N; j += RANK_THREADS) keys[j] = rank_key_hi(row[j]);
  __syncthreads();
  // 0 stands for "no target in [0, N)": every key is at least 2^31, its low word being ~column. A negative or decreasing range
  // is empty, so it reads nothing before idx.
  const long long lo = off ? off[r] : r, hi = off ? off[r + 1] : r + 1;
  unsigned long long kt = 0ull;
  for (long long i = (lo >= 0 ? lo : hi) + threadIdx.x; i < hi; i += RANK_THREADS) {
    const long long t = idx[i];
    if (t >= 0 && t < N) {
      const unsigned long long x = rank_key(keys, (int)t);
      kt = x > kt ? x : kt;
    }
  }
  kt = block_max_u64(kt, red64);
  int above = 0;
  if (kt)
    for (int j = threadIdx.x; j < N; j += RANK_THREADS) above += rank_key(keys, j) > kt ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) above += __shfl_xor_sync(0xffffffffu, above, o);
  if ((threadIdx.x & 31) == 0) red32[threadIdx.x >> 5] = above;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < RANK_THREADS / 32; ++w) s += red32[w];
    rank_out[r] = kt ? s : -1;
  }
  if (!topk_out) return;
  int* out = topk_out + (long long)r * k;
  unsigned long long bound = ~0ull;                          // no key reaches it: the low word of a key is ~column, column < 2^31
  const int kk = k < N ? k : N;
  for (int i = 0; i < kk; ++i) {
    unsigned long long best = 0ull;
    for (int j = threadIdx.x; j < N; j += RANK_THREADS) {
      const unsigned long long x = rank_key(keys, j);
      if (x < bound && x > best) best = x;
    }
    best = block_max_u64(best, red64);
    if (threadIdx.x == 0) out[i] = (int)~(uint32_t)best;
    bound = best;
  }
  for (int i = kk + threadIdx.x; i < k; i += RANK_THREADS) out[i] = -1;
}

// ------------------------------------------------------------------------------------------ masked-region regression and NCE
// Both objectives score rows [b, r+1] of prediction_scores_v (region 0, the global feature, is dropped) against target[b, r] and
// label[b, r] == 1, R = Nv - 1. One CTA per row of scores (region 0 and unmasked rows write a zero gradient and a zero row loss);
// row_loss[B * Nv] is summed afterwards in a fixed order by sum_rows_kernel, so loss and gradient are bitwise reproducible.

// visual_target == 1 (vilbert.py:1507-1513): loss = sum over masked rows of sum_d (s - t)^2 / max(n_masked * D, 1)
__global__ void __launch_bounds__(LOSS_THREADS)
mse_masked_rows_kernel(const float* __restrict__ scores, const float* __restrict__ target, const long long* __restrict__ label, int B,
                       int Nv, int D, float grad_scale, float* __restrict__ row_loss, float* __restrict__ d32) {
  pdl_entry();
  __shared__ float red[LOSS_THREADS / 32];
  const int R = Nv - 1, rr = blockIdx.x, b = rr / Nv, reg = rr % Nv;
  const float n_pos = block_count(label, B * R, red, [](long long l) { return l == 1; });
  const float inv = 1.f / fmaxf(n_pos * (float)D, 1.f);
  const bool live = reg > 0 && label[(long long)b * R + reg - 1] == 1;
  const float* sr = scores + (long long)rr * D;
  const float* tr = target + ((long long)b * R + (reg > 0 ? reg - 1 : 0)) * D;
  float acc = 0.f;
  for (int j = threadIdx.x; j < D; j += LOSS_THREADS) {
    float g = 0.f;
    if (live) {
      const float e = sr[j] - tr[j];
      acc += e * e;
      g = 2.f * e * grad_scale * inv;
    }
    if (d32) d32[(long long)rr * D + j] = g;
  }
  acc = block_reduce(acc, red, false);
  if (threadIdx.x == 0) row_loss[rr] = acc * inv;
}

// visual_target == 2 (vilbert.py:1523-1575): for a masked row, candidate 0 is target[b, r] and candidate k >= 1 is row
// neg[b, r, k-1] of target viewed as [B * R, D]; score_k = <candidate_k, s>; loss = CE(score, 0) averaged over the masked rows.
// d s = sum_k (softmax_k - [k == 0]) candidate_k * gs / n_masked, summed in candidate order by the thread owning the columns.
// The prediction row lives in shared memory; candidates are read with 128-bit loads, once for the scores and once for the
// gradient. An index outside [0, B * R) is not read: it makes the row's loss NaN and adds nothing to the gradient.
__global__ void __launch_bounds__(LOSS_THREADS)
nce_region_rows_kernel(const float* __restrict__ scores, const float* __restrict__ target, const long long* __restrict__ label,
                       const long long* __restrict__ neg, int B, int Nv, int D, int n, float grad_scale, float* __restrict__ row_loss,
                       float* __restrict__ d32) {
  pdl_entry();
  extern __shared__ __align__(16) float smem[];
  float* s = smem;                          // [D] the prediction row
  float* sc = smem + D;                     // [n + 1] candidate scores (NaN: index out of range)
  __shared__ float red[LOSS_THREADS / 32];
  const int R = Nv - 1, rr = blockIdx.x, b = rr / Nv, reg = rr % Nv, D4 = D / 4;
  const long long rows_t = (long long)B * R;
  const float n_pos = block_count(label, (int)rows_t, red, [](long long l) { return l == 1; });
  const bool live = reg > 0 && label[(long long)b * R + reg - 1] == 1;
  float4* g4 = d32 ? reinterpret_cast<float4*>(d32 + (long long)rr * D) : nullptr;
  if (!live) {
    for (int j = threadIdx.x; j < D4; j += LOSS_THREADS)
      if (g4) g4[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (threadIdx.x == 0) row_loss[rr] = (rr == 0 && n_pos == 0.f) ? CUDART_NAN_F : 0.f;   // CE over no rows is NaN
    return;
  }
  const float4* s_src = reinterpret_cast<const float4*>(scores + (long long)rr * D);
  float4* s4 = reinterpret_cast<float4*>(s);
  for (int j = threadIdx.x; j < D4; j += LOSS_THREADS) s4[j] = s_src[j];
  __syncthreads();
  const long long own = (long long)b * R + reg - 1;
  const long long* nr = neg + own * n;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = warp; k <= n; k += LOSS_THREADS / 32) {     // one warp per candidate
    const long long row = k == 0 ? own : nr[k - 1];
    float dot = CUDART_NAN_F;
    if (row >= 0 && row < rows_t) {
      const float4* c4 = reinterpret_cast<const float4*>(target + row * D);
      float a = 0.f;
      for (int j = lane; j < D4; j += 32) {
        const float4 c = c4[j], p = s4[j];
        a += c.x * p.x + c.y * p.y + c.z * p.z + c.w * p.w;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      dot = a;
    }
    if (lane == 0) sc[k] = dot;
  }
  __syncthreads();
  float mx = -CUDART_INF_F;
  for (int k = threadIdx.x; k <= n; k += LOSS_THREADS) mx = fmaxf(mx, sc[k]);      // fmaxf drops NaN
  mx = block_reduce(mx, red, true);
  float se = 0.f, bad = 0.f;
  for (int k = threadIdx.x; k <= n; k += LOSS_THREADS) {
    if (sc[k] != sc[k]) bad = 1.f; else se += __expf(sc[k] - mx);
  }
  se = block_reduce(se, red, false);
  bad = block_reduce(bad, red, true);
  const float lse = mx + __logf(se);
  if (threadIdx.x == 0) row_loss[rr] = bad > 0.f ? CUDART_NAN_F : (lse - sc[0]) / n_pos;
  if (!g4) return;
  const float gs = grad_scale / n_pos;
  for (int j = threadIdx.x; j < D4; j += LOSS_THREADS) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = 0; k <= n; ++k) {
      const float z = sc[k];
      if (z != z) continue;
      const float w = (__expf(z - lse) - (k == 0 ? 1.f : 0.f)) * gs;
      const float4 c = reinterpret_cast<const float4*>(target + (k == 0 ? own : nr[k - 1]) * D)[j];
      acc.x += w * c.x; acc.y += w * c.y; acc.z += w * c.z; acc.w += w * c.w;
    }
    g4[j] = acc;
  }
}

// dst = src * (*scale): the head gradient of a forward-placed objective times the d(total)/d(loss) the caller holds on the device
__global__ void scale_by_device_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n, const float* __restrict__ scale) {
  pdl_entry();
  const float s = *scale;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i] * s;
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

extern "C" vb_status vb_ce_loss_det(const float* logits, int64_t ld_logits, const int64_t* labels, int64_t ignore_index, float* loss,
                                    float* dlogits_f32, int64_t ld_d32, void* dlogits_bf16, int64_t ld_d16, int32_t rows, int32_t cols,
                                    float grad_scale, int32_t accumulate_loss, float* ws, void* stream) {
  if (rows <= 0 || cols <= 0 || !logits || !labels || !loss || !ws) return set_error(VB_ERR_INVALID, "vb_ce_loss_det: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!accumulate_loss) {
    cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), st);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_ce_loss_det: memset: %s", cudaGetErrorString(e));
  }
  const int grid = loss_grid(rows) < VB_DET_LOSS_SLICES ? loss_grid(rows) : VB_DET_LOSS_SLICES;
  launch_pdl(ce_loss_det_kernel, dim3(grid), dim3(LOSS_THREADS), (size_t)0, st, logits, (long long)ld_logits,
             reinterpret_cast<const long long*>(labels), (long long)ignore_index, dlogits_f32, (long long)ld_d32,
             static_cast<__nv_bfloat16*>(dlogits_bf16), (long long)ld_d16, (int)rows, (int)cols, grad_scale, ws);
  if (int s = check_launch("vb_ce_loss_det")) return s;
  return launch_reduce_slices(ws, 1, grid, 1, loss, st);
}

extern "C" vb_status vb_bce_gather_loss(const float* logits, int64_t ld_logits, int32_t col_off, int32_t width, const int64_t* ids,
                                        const float* target, int32_t rows, int32_t C, float loss_mul, float* row_loss, float* loss,
                                        int32_t accumulate_loss, float* dlogits_f32, int64_t ld_d32, void* dlogits_bf16, int64_t ld_d16,
                                        void* stream) {
  if (rows <= 0 || C <= 0 || col_off < 0 || width <= col_off || (!ids && C > width - col_off) || !logits || !target || !row_loss || !loss)
    return set_error(VB_ERR_INVALID, "vb_bce_gather_loss: bad arguments");
  const size_t smem = (size_t)width * sizeof(float) + (size_t)C * (sizeof(float) + sizeof(int));
  if (smem > 48 * 1024) return set_error(VB_ERR_INVALID, "vb_bce_gather_loss: row of %d logits and %d choices exceeds 48 KiB of shared memory", width, C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const float scale = loss_mul / ((float)rows * (float)C);
  launch_pdl(bce_gather_rows_kernel, dim3(rows), dim3(LOSS_THREADS), smem, st, logits, (long long)ld_logits, (int)col_off, (int)width,
             reinterpret_cast<const long long*>(ids), target, (int)C, scale, row_loss, dlogits_f32, (long long)ld_d32,
             static_cast<__nv_bfloat16*>(dlogits_bf16), (long long)ld_d16);
  vb_status s = check_launch("vb_bce_gather_loss");
  if (s != VB_OK) return s;
  launch_pdl(sum_rows_kernel, dim3(1), dim3(LOSS_THREADS), (size_t)0, st, (const float*)row_loss, (int)rows, loss, (int)(accumulate_loss ? 1 : 0));
  return check_launch("vb_bce_gather_loss");
}

extern "C" vb_status vb_task_score(int32_t mode, const float* logits, int64_t ld_logits, int32_t col_off, int32_t cols, const int64_t* ids,
                                   int32_t width, const float* target, int64_t ld_target, const int64_t* labels, int32_t rows, float* score,
                                   int32_t accumulate, int64_t* preds, void* stream) {
  const bool need_target = mode == VB_SCORE_SOFT || mode == VB_SCORE_THRESHOLD || mode == VB_SCORE_CHOICE;
  if (mode < VB_SCORE_SOFT || mode > VB_SCORE_CHOICE || rows <= 0 || cols <= 0 || col_off < 0 || !logits || !score ||
      (need_target && !target) || (mode == VB_SCORE_LABEL && !labels) || (mode == VB_SCORE_CHOICE) != (ids != nullptr) ||
      (ids && width <= col_off))
    return set_error(VB_ERR_INVALID, "vb_task_score: bad arguments");
  launch_pdl(task_score_kernel, dim3(1), dim3(LOSS_THREADS), (size_t)0, static_cast<cudaStream_t>(stream), (int)mode, logits,
             (long long)ld_logits, (int)col_off, (int)cols, reinterpret_cast<const long long*>(ids), (int)width, target, (long long)ld_target,
             reinterpret_cast<const long long*>(labels), (int)rows, score, (int)(accumulate ? 1 : 0), reinterpret_cast<long long*>(preds));
  return check_launch("vb_task_score");
}

extern "C" vb_status vb_task_results(int32_t mode, const float* logits, int64_t ld_logits, int32_t col_off, int32_t cols, const int64_t* ids,
                                     int32_t width, const float* target, int64_t ld_target, int32_t rows, int64_t* argmax, float* values,
                                     int64_t ld_values, void* stream) {
  if (mode < VB_RESULT_ARGMAX || mode > VB_RESULT_GATHER || rows <= 0 || cols <= 0 || col_off < 0 || !logits || !argmax ||
      (ids && width <= col_off) || (mode == VB_RESULT_GATHER && (!target || !values)) ||
      (mode == VB_RESULT_SOFTMAX && (!values || ld_values < cols)))
    return set_error(VB_ERR_INVALID, "vb_task_results: bad arguments (mode %d, rows %d, cols %d, col_off %d)", (int)mode, (int)rows,
                     (int)cols, (int)col_off);
  const int grid = (int)(((long long)rows + RESULTS_ROWS - 1) / RESULTS_ROWS);
  launch_pdl(task_results_kernel, dim3(grid), dim3(LOSS_THREADS), (size_t)0, static_cast<cudaStream_t>(stream), (int)mode, logits,
             (long long)ld_logits, (int)col_off, (int)cols, reinterpret_cast<const long long*>(ids), (int)width, target, (long long)ld_target,
             (int)rows, reinterpret_cast<long long*>(argmax), values, (long long)ld_values);
  return check_launch("vb_task_results");
}

// both retrieval entry points: every refusal comes before the launch, so a refused call writes nothing
static vb_status retrieval_rank_launch(const char* name, const float* scores, int64_t ld_scores, int32_t rows, int32_t cols,
                                       const int64_t* off, const int64_t* idx, int32_t k, int32_t* rank_out, int32_t* topk_out,
                                       void* stream) {
  if (rows <= 0 || cols <= 0 || ld_scores < cols || !scores || !idx || !rank_out || (topk_out && (k <= 0 || k > RANK_MAX_K)))
    return set_error(VB_ERR_INVALID, "%s: bad arguments (rows %d, cols %d, ld %lld, k %d; 1 <= k <= %d)", name, (int)rows,
                     (int)cols, (long long)ld_scores, (int)k, RANK_MAX_K);
  if (cols > RANK_MAX_COLS)
    return set_error(VB_ERR_INVALID, "%s: %d columns exceed the %d a row of shared memory holds", name, (int)cols, RANK_MAX_COLS);
  const size_t smem = (size_t)cols * sizeof(uint32_t);
  if (smem > 48 * 1024) {      // set per call, as the attention kernels do: it holds for the current device only
    cudaError_t e = cudaFuncSetAttribute(retrieval_rank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "%s: cudaFuncSetAttribute: %s", name, cudaGetErrorString(e));
  }
  launch_pdl(retrieval_rank_kernel, dim3(rows), dim3(RANK_THREADS), smem, static_cast<cudaStream_t>(stream), scores, (long long)ld_scores,
             (int)cols, reinterpret_cast<const long long*>(off), reinterpret_cast<const long long*>(idx), (int)(topk_out ? k : 0),
             reinterpret_cast<int*>(rank_out), reinterpret_cast<int*>(topk_out));
  return check_launch(name);
}

extern "C" vb_status vb_retrieval_rank(const float* scores, int64_t ld_scores, int32_t rows, int32_t cols, const int64_t* target, int32_t k,
                                       int32_t* rank_out, int32_t* topk_out, void* stream) {
  return retrieval_rank_launch("vb_retrieval_rank", scores, ld_scores, rows, cols, nullptr, target, k, rank_out, topk_out, stream);
}

extern "C" vb_status vb_retrieval_rank_sets(const float* scores, int64_t ld_scores, int32_t rows, int32_t cols, const int64_t* set_off,
                                            const int64_t* set_idx, int32_t k, int32_t* rank_out, int32_t* topk_out, void* stream) {
  if (!set_off) return set_error(VB_ERR_INVALID, "vb_retrieval_rank_sets: set_off is NULL");
  return retrieval_rank_launch("vb_retrieval_rank_sets", scores, ld_scores, rows, cols, set_off, set_idx, k, rank_out, topk_out, stream);
}

extern "C" vb_status vb_scale_by_device(const float* src, float* dst, int64_t n, const float* scale, void* stream) {
  if (n <= 0 || !src || !dst || !scale) return set_error(VB_ERR_INVALID, "vb_scale_by_device: bad arguments");
  const int grid = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
  launch_pdl(scale_by_device_kernel, dim3(grid), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream), src, dst, (long long)n, scale);
  return check_launch("vb_scale_by_device");
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

extern "C" vb_status vb_kl_masked_loss_det(const float* scores, const float* target, const int64_t* label, float* loss, float* dscores_f32,
                                           void* dscores_bf16, int64_t ld_d16, int32_t B, int32_t Nv, int32_t C, float grad_scale,
                                           int32_t accumulate_loss, float* ws, void* stream) {
  if (B <= 0 || Nv <= 1 || C <= 0 || !scores || !target || !label || !loss || !ws)
    return set_error(VB_ERR_INVALID, "vb_kl_masked_loss_det: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!accumulate_loss) {
    cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), st);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_kl_masked_loss_det: memset: %s", cudaGetErrorString(e));
  }
  const int grid = loss_grid(B * Nv) < VB_DET_LOSS_SLICES ? loss_grid(B * Nv) : VB_DET_LOSS_SLICES;
  launch_pdl(kl_masked_loss_det_kernel, dim3(grid), dim3(LOSS_THREADS), (size_t)0, st, scores, target,
             reinterpret_cast<const long long*>(label), dscores_f32, static_cast<__nv_bfloat16*>(dscores_bf16), (long long)ld_d16,
             (int)B, (int)Nv, (int)C, grad_scale, ws);
  if (int s = check_launch("vb_kl_masked_loss_det")) return s;
  return launch_reduce_slices(ws, 1, grid, 1, loss, st);
}

extern "C" vb_status vb_mse_masked_loss(const float* scores, const float* target, const int64_t* label, int32_t B, int32_t Nv, int32_t D,
                                        float grad_scale, float* row_loss, float* loss, int32_t accumulate_loss, float* dscores_f32,
                                        void* stream) {
  if (B <= 0 || Nv <= 1 || D <= 0 || !scores || !target || !label || !row_loss || !loss)
    return set_error(VB_ERR_INVALID, "vb_mse_masked_loss: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rows = B * Nv;
  launch_pdl(mse_masked_rows_kernel, dim3(rows), dim3(LOSS_THREADS), (size_t)0, st, scores, target, reinterpret_cast<const long long*>(label),
             (int)B, (int)Nv, (int)D, grad_scale, row_loss, dscores_f32);
  vb_status s = check_launch("vb_mse_masked_loss");
  if (s != VB_OK) return s;
  launch_pdl(sum_rows_kernel, dim3(1), dim3(LOSS_THREADS), (size_t)0, st, (const float*)row_loss, rows, loss, (int)(accumulate_loss ? 1 : 0));
  return check_launch("vb_mse_masked_loss");
}

extern "C" vb_status vb_nce_region_loss(const float* scores, const float* target, const int64_t* label, const int64_t* neg_index, int32_t B,
                                        int32_t Nv, int32_t D, int32_t n_neg, float grad_scale, float* row_loss, float* loss,
                                        int32_t accumulate_loss, float* dscores_f32, void* stream) {
  if (B <= 0 || Nv <= 1 || D <= 0 || (D & 3) || n_neg < 0 || !scores || !target || !label || (n_neg > 0 && !neg_index) || !row_loss || !loss ||
      (reinterpret_cast<uintptr_t>(scores) & 15) || (reinterpret_cast<uintptr_t>(target) & 15) || (reinterpret_cast<uintptr_t>(dscores_f32) & 15))
    return set_error(VB_ERR_INVALID, "vb_nce_region_loss: bad arguments (D % 4 == 0, 16-byte aligned rows)");
  const size_t smem = ((size_t)D + (size_t)n_neg + 1) * sizeof(float);
  if (smem > 48 * 1024) return set_error(VB_ERR_INVALID, "vb_nce_region_loss: row of %d features and %d negatives exceeds 48 KiB of shared memory", D, n_neg);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rows = B * Nv;
  launch_pdl(nce_region_rows_kernel, dim3(rows), dim3(LOSS_THREADS), smem, st, scores, target, reinterpret_cast<const long long*>(label),
             reinterpret_cast<const long long*>(neg_index), (int)B, (int)Nv, (int)D, (int)n_neg, grad_scale, row_loss, dscores_f32);
  vb_status s = check_launch("vb_nce_region_loss");
  if (s != VB_OK) return s;
  launch_pdl(sum_rows_kernel, dim3(1), dim3(LOSS_THREADS), (size_t)0, st, (const float*)row_loss, rows, loss, (int)(accumulate_loss ? 1 : 0));
  return check_launch("vb_nce_region_loss");
}

static vb_status compact_rows(const char* name, const int64_t* labels, int64_t ignore_index, const int32_t* map, int32_t rows, int32_t cap,
                              int32_t* idx, int32_t* count, int64_t* labels_compact, void* stream) {
  if (rows <= 0 || cap <= 0 || !labels || !idx || !count || !labels_compact) return set_error(VB_ERR_INVALID, "%s: bad arguments", name);
  launch_pdl(compact_rows_kernel, dim3(1), dim3(1024), (size_t)0, static_cast<cudaStream_t>(stream), reinterpret_cast<const long long*>(labels),
             (long long)ignore_index, map, (int)rows, (int)cap, idx, count, reinterpret_cast<long long*>(labels_compact));
  return check_launch(name);
}

extern "C" vb_status vb_compact_rows(const int64_t* labels, int64_t ignore_index, int32_t rows, int32_t cap, int32_t* idx, int32_t* count,
                                     int64_t* labels_compact, void* stream) {
  return compact_rows("vb_compact_rows", labels, ignore_index, nullptr, rows, cap, idx, count, labels_compact, stream);
}

extern "C" vb_status vb_compact_rows_mapped(const int64_t* labels, int64_t ignore_index, const int32_t* map, int32_t rows, int32_t cap,
                                            int32_t* idx, int32_t* count, int64_t* labels_compact, void* stream) {
  if (!map) return set_error(VB_ERR_INVALID, "vb_compact_rows_mapped: no row map");
  return compact_rows("vb_compact_rows_mapped", labels, ignore_index, map, rows, cap, idx, count, labels_compact, stream);
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
