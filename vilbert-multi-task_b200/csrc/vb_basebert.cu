// vb_basebert.cu — kernels of the single-stream baseline (BaseBertForVLTasks, vilbert/basebert.py:893-978) that the two-stream
// model never needed: the LayerNorm of the concatenated text | image embeddings, the text-embedding scatter with padding rows in
// every table, weight norm with dim=None (SimpleClassifier), the tanh pooler and the concatenated additive mask.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "vb_internal.h"
#include "vb_ptx.cuh"

namespace vb {

constexpr int BB_WARPS = 8;
constexpr int BB_THREADS = BB_WARPS * 32;
constexpr int WN_BLOCKS = 64;      // fixed partial-sum grid of the weight-norm reductions: the sums do not depend on the device

__device__ __forceinline__ float bb_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void store16(void* hi, void* lo, __nv_bfloat16* b16, long long i, float v, int fp16) {
  if (hi) {
    const uint16_t h = cvt16(v, fp16);
    reinterpret_cast<uint16_t*>(hi)[i] = h;
    if (lo) reinterpret_cast<uint16_t*>(lo)[i] = cvt16(v - cvt16_to_f32(h, fp16), fp16);
  }
  if (b16) b16[i] = __float2bfloat16(v);
}

// Row r of the [B, Nt+Nv] stream: its pre-LayerNorm source row, and whether it is a text row. Image rows add the token-type row
// of type 1 (BertImageEmbeddings: every region has token type 1, basebert.py:351-355, 734-736).
struct StreamRow {
  const float* x;
  long long src;   // row index within its modality (dropout element index = src * H + col)
  bool text;
};
__device__ __forceinline__ StreamRow stream_row(long long r, const float* xt, const float* xv, int Nt, int Nv, int H) {
  const int N = Nt + Nv;
  const long long b = r / N;
  const int p = (int)(r % N);
  StreamRow s;
  s.text = p < Nt;
  s.src = s.text ? b * Nt + p : b * Nv + (p - Nt);
  s.x = (s.text ? xt : xv) + s.src * H;
  return s;
}

// LayerNorm of each modality with its own parameters, then its own dropout, written straight into the interleaved stream
// (basebert.py:316-321, 357-359, 738-747: LN -> dropout -> torch.cat(dim=1)). One warp per stream row, three passes over the row.
__global__ void __launch_bounds__(BB_THREADS)
concat_ln_fwd_kernel(const float* __restrict__ xt, const float* __restrict__ xv, const float* __restrict__ trow,
                     const float* __restrict__ gt, const float* __restrict__ bt, const float* __restrict__ gv, const float* __restrict__ bv,
                     float* __restrict__ y32, void* y16, void* ylo, __nv_bfloat16* yb16, int fp16, float* __restrict__ mean_out,
                     float* __restrict__ rstd_out, int B, int Nt, int Nv, int H, const DropCfg dt, const DropCfg dv) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const long long rows = (long long)B * (Nt + Nv);
  const uint32_t seed_t = dt.ctr ? drop_seed(dt) : 0u, seed_v = dv.ctr ? drop_seed(dv) : 0u;
  const float inv_h = 1.f / (float)H;
  for (long long r = (long long)blockIdx.x * BB_WARPS + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * BB_WARPS) {
    const StreamRow s = stream_row(r, xt, xv, Nt, Nv, H);
    const float* add = s.text ? nullptr : trow;
    float sum = 0.f;
    for (int c = lane; c < H; c += 32) sum += s.x[c] + (add ? add[c] : 0.f);
    const float mean = bb_warp_sum(sum) * inv_h;
    float q = 0.f;
    for (int c = lane; c < H; c += 32) {
      const float d = s.x[c] + (add ? add[c] : 0.f) - mean;
      q += d * d;
    }
    const float rstd = rsqrtf(bb_warp_sum(q) * inv_h + 1e-12f);
    if (lane == 0) { mean_out[r] = mean; rstd_out[r] = rstd; }
    const float* g = s.text ? gt : gv;
    const float* be = s.text ? bt : bv;
    const DropCfg& d = s.text ? dt : dv;
    const uint32_t seed = s.text ? seed_t : seed_v;
    for (int c = lane; c < H; c += 32) {
      float o = (s.x[c] + (add ? add[c] : 0.f) - mean) * rstd * g[c] + be[c];
      if (d.ctr) o = drop_apply(o, seed, (uint32_t)(s.src * H + c), d);
      const long long i = r * H + c;
      if (y32) y32[i] = o;
      store16(y16, ylo, yb16, i, o, fp16);
    }
  }
}

// Autograd of the above. Per row: dy masked by the row's dropout, dx = rstd (dy g - mean(dy g) - xhat mean(dy g xhat)). Text rows
// go to dxt (the text scatter-add reads it), image rows to dxv (f32: box projection backward) and dxv16 (bf16: the region-feature
// GEMM's weight gradient). Column sums per CTA in shared memory, then one atomic per column and CTA: dgamma / dbeta of both
// LayerNorms, and the image column sum of dx, which is the gradient of the image GEMM's bias and of the image token-type row 1.
__global__ void __launch_bounds__(BB_THREADS)
concat_ln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ xt, const float* __restrict__ xv, const float* __restrict__ trow,
                     const float* __restrict__ gt, const float* __restrict__ gv, const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                     float* __restrict__ dxt, float* __restrict__ dxv, __nv_bfloat16* __restrict__ dxv16, float* dgt, float* dbt, float* dgv, float* dbv,
                     float* dcol, float* dcol2, int B, int Nt, int Nv, int H, const DropCfg dt, const DropCfg dv) {
  pdl_entry();
  extern __shared__ float acc[];     // [5][H]: dgamma_t, dbeta_t, dgamma_v, dbeta_v, image column sum of dx
  for (int i = threadIdx.x; i < 5 * H; i += blockDim.x) acc[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long rows = (long long)B * (Nt + Nv);
  const uint32_t seed_t = dt.ctr ? drop_seed(dt) : 0u, seed_v = dv.ctr ? drop_seed(dv) : 0u;
  const float inv_h = 1.f / (float)H;
  for (long long r = (long long)blockIdx.x * BB_WARPS + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * BB_WARPS) {
    const StreamRow s = stream_row(r, xt, xv, Nt, Nv, H);
    const float* add = s.text ? nullptr : trow;
    const float* g = s.text ? gt : gv;
    const DropCfg& d = s.text ? dt : dv;
    const uint32_t seed = s.text ? seed_t : seed_v;
    const float mean = mean_in[r], rstd = rstd_in[r];
    const float* dyr = dy + r * H;
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < H; c += 32) {
      float u = dyr[c];
      if (d.ctr) u = drop_apply(u, seed, (uint32_t)(s.src * H + c), d);
      const float xh = (s.x[c] + (add ? add[c] : 0.f) - mean) * rstd;
      const float gu = u * g[c];
      s1 += gu;
      s2 += gu * xh;
      float* a = acc + (s.text ? 0 : 2 * H);
      atomicAdd(a + c, u * xh);
      atomicAdd(a + H + c, u);
    }
    s1 = bb_warp_sum(s1) * inv_h;
    s2 = bb_warp_sum(s2) * inv_h;
    for (int c = lane; c < H; c += 32) {
      float u = dyr[c];
      if (d.ctr) u = drop_apply(u, seed, (uint32_t)(s.src * H + c), d);
      const float xh = (s.x[c] + (add ? add[c] : 0.f) - mean) * rstd;
      const float dx = rstd * (u * g[c] - s1 - xh * s2);
      const long long o = s.src * H + c;
      if (s.text) {
        if (dxt) dxt[o] = dx;
      } else {
        if (dxv) dxv[o] = dx;
        if (dxv16) dxv16[o] = __float2bfloat16(dx);
        atomicAdd(acc + 4 * H + c, dx);
      }
    }
  }
  __syncthreads();
  float* outs[6] = {dgt, dbt, dgv, dbv, dcol, dcol2};
  for (int i = threadIdx.x; i < 6 * H; i += blockDim.x) {
    const int k = i / H, c = i % H;
    if (outs[k]) atomicAdd(outs[k] + c, acc[(k < 5 ? k : 4) * H + c]);
  }
}

// Text-embedding scatter-add where every table has padding_idx=0 (basebert.py:290-298): row 0 of the word, position and token-type
// tables receives no gradient. A NULL table (frozen) receives nothing.
__global__ void __launch_bounds__(BB_THREADS)
embed_text_bwd_padded_kernel(const float* __restrict__ dout, const long long* __restrict__ ids, const long long* __restrict__ tts,
                             float* __restrict__ dword, float* __restrict__ dpos, float* __restrict__ dtype, int B, int Nt, int H) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const long long rows = (long long)B * Nt;
  for (long long row = (long long)blockIdx.x * BB_WARPS + (threadIdx.x >> 5); row < rows; row += (long long)gridDim.x * BB_WARPS) {
    const int t = (int)(row % Nt);
    const long long id = ids[row], tt = tts[row];
    float* dw = (dword && id != 0) ? dword + id * H : nullptr;
    float* dp = (dpos && t != 0) ? dpos + (long long)t * H : nullptr;
    float* dty = (dtype && tt != 0) ? dtype + tt * H : nullptr;
    if (!dw && !dp && !dty) continue;
    const float* d = dout + row * H;
    for (int c = lane; c < H; c += 32) {
      const float v = d[c];
      if (dw) atomicAdd(dw + c, v);
      if (dp) atomicAdd(dp + c, v);
      if (dty) atomicAdd(dty + c, v);
    }
  }
}

// ---------------------------------------------------------------------------------------------- weight norm, dim=None
// torch._weight_norm(v, g, 0 -> dim=None): w = v * (g / ||v||_F). The reductions run on a fixed grid of WN_BLOCKS partial sums
// (fixed element-to-thread assignment, fixed-order tree per CTA) that the consumer adds in index order in double: bitwise
// reproducible, no float atomics.
template <bool BWD>
__global__ void __launch_bounds__(BB_THREADS)
wn_partials_kernel(const float* __restrict__ v, const float* __restrict__ dw, long long n, double* __restrict__ part) {
  pdl_entry();
  __shared__ float red[2][BB_WARPS];
  float vv = 0.f, dv = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float x = v[i];
    vv = fmaf(x, x, vv);
    if (BWD) dv = fmaf(dw[i], x, dv);
  }
  vv = bb_warp_sum(vv);
  if (BWD) dv = bb_warp_sum(dv);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[0][w] = vv; red[1][w] = dv; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < BB_WARPS; ++k) { a += red[0][k]; b += red[1][k]; }
    part[blockIdx.x] = a;
    part[WN_BLOCKS + blockIdx.x] = b;
  }
}

__device__ __forceinline__ void wn_totals(const double* part, bool bwd, float& norm, float& dot) {
  __shared__ float s[2];
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < WN_BLOCKS; ++k) { a += part[k]; if (bwd) b += part[WN_BLOCKS + k]; }
    s[0] = (float)sqrt(a);
    s[1] = (float)b;
  }
  __syncthreads();
  norm = s[0];
  dot = s[1];
}

__global__ void __launch_bounds__(BB_THREADS)
wn_fwd_kernel(const float* __restrict__ v, const float* __restrict__ g, long long n, const double* __restrict__ part, float* __restrict__ w32,
              void* w16, void* wlo, __nv_bfloat16* wb16, int fp16) {
  pdl_entry();
  float norm, dot;
  wn_totals(part, false, norm, dot);
  const float scale = g[0] / norm;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float w = v[i] * scale;
    if (w32) w32[i] = w;
    store16(w16, wlo, wb16, i, w, fp16);
  }
}

// dg = <dw, v> / ||v||;  dv = (g / ||v||) (dw - (dg / ||v||) v). Both ACCUMULATED (the flat gradient buffer); either may be NULL.
__global__ void __launch_bounds__(BB_THREADS)
wn_bwd_kernel(const float* __restrict__ dw, const float* __restrict__ v, const float* __restrict__ g, long long n, const double* __restrict__ part,
              float* __restrict__ dg, float* __restrict__ dv) {
  pdl_entry();
  float norm, dot;
  wn_totals(part, true, norm, dot);
  const float gd = dot / norm;
  if (dg && blockIdx.x == 0 && threadIdx.x == 0) dg[0] += gd;
  if (!dv) return;
  const float a = g[0] / norm, b = gd / norm;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dv[i] += a * (dw[i] - b * v[i]);
}

// ---------------------------------------------------------------------------------------------- tanh pooler, masks
// BertPooler's activation (basebert.py:507-519): y = tanh(x) as f32 and as the forward operand copies.
__global__ void tanh_fwd_kernel(const float* __restrict__ x, float* __restrict__ y32, void* y16, void* ylo, __nv_bfloat16* yb16, int fp16, long long n) {
  pdl_entry();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float y = tanhf(x[i]);
    if (y32) y32[i] = y;
    store16(y16, ylo, yb16, i, y, fp16);
  }
}

// dx = dy (1 - y^2) as the bf16 gradient operand; dbias[c] += sum over the M rows of dx (one thread per column, rows in order).
__global__ void tanh_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, __nv_bfloat16* __restrict__ dx16, float* __restrict__ dbias,
                                int M, int N) {
  pdl_entry();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  float s = 0.f;
  for (int m = 0; m < M; ++m) {
    const long long i = (long long)m * N + c;
    const float t = y[i];
    const float d = dy[i] * (1.f - t * t);
    if (dx16) dx16[i] = __float2bfloat16(d);
    s += d;
  }
  if (dbias) dbias[c] += s;
}

// torch.cat([(1 - mask_t) * -10000, (1 - mask_v) * -10000], dim=-1) (basebert.py:723-750)
__global__ void mask_concat_kernel(const long long* __restrict__ mt, const long long* __restrict__ mv, float* __restrict__ out, int B, int Nt, int Nv) {
  pdl_entry();
  const int N = Nt + Nv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)B * N; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / N;
    const int j = (int)(i % N);
    const long long m = j < Nt ? mt[b * Nt + j] : mv[b * Nv + (j - Nt)];
    out[i] = (1.0f - (float)m) * -10000.0f;
  }
}

static DropCfg bb_drop(const vb_dropout* d) {
  DropCfg c;
  const bool on = d && d->step && d->p > 0.f;
  c.ctr = on ? d->step : nullptr;
  c.site = d ? d->site : 0u;
  c.thresh = on ? (uint32_t)((double)d->p * 4294967296.0) : 0u;
  c.scale = on && d->p < 1.f ? 1.f / (1.f - d->p) : 1.f;
  return c;
}

static int bb_grid(long long work, int per_block) {
  long long blocks = (work + per_block - 1) / per_block;
  long long cap = (long long)sm_count() * 8;
  if (cap <= 0) cap = 132 * 8;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

}  // namespace vb

using namespace vb;
#define BB_ST(s) static_cast<cudaStream_t>(s)

extern "C" vb_status vb_concat_embed_ln_fwd(const float* xt, const float* xv, const float* v_type_row, const float* gamma_t, const float* beta_t,
                                            const float* gamma_v, const float* beta_v, float* y_f32, void* y16, void* y_lo, void* y_b16, int32_t y_fp16,
                                            float* mean, float* rstd, int32_t B, int32_t Nt, int32_t Nv, int32_t H, const vb_dropout* drop_t,
                                            const vb_dropout* drop_v, void* stream) {
  if (B <= 0 || Nt <= 0 || Nv <= 0 || H <= 0 || !xt || !xv || !v_type_row || !gamma_t || !beta_t || !gamma_v || !beta_v || !mean || !rstd ||
      (y_lo && !y16))
    return set_error(VB_ERR_INVALID, "vb_concat_embed_ln_fwd: bad arguments");
  launch_pdl(concat_ln_fwd_kernel, dim3(bb_grid((long long)B * (Nt + Nv), BB_WARPS)), dim3(BB_THREADS), (size_t)0, BB_ST(stream), xt, xv,
             v_type_row, gamma_t, beta_t, gamma_v, beta_v, y_f32, y16, y_lo, static_cast<__nv_bfloat16*>(y_b16), y_fp16 ? 1 : 0, mean, rstd,
             (int)B, (int)Nt, (int)Nv, (int)H, bb_drop(drop_t), bb_drop(drop_v));
  return check_launch("vb_concat_embed_ln_fwd");
}

extern "C" vb_status vb_concat_embed_ln_bwd(const float* dy, const float* xt, const float* xv, const float* v_type_row, const float* gamma_t,
                                            const float* gamma_v, const float* mean, const float* rstd, float* dxt, float* dxv, void* dxv_bf16,
                                            float* dgamma_t, float* dbeta_t, float* dgamma_v, float* dbeta_v, float* dcol_v, float* dcol_v2,
                                            int32_t B, int32_t Nt, int32_t Nv, int32_t H, const vb_dropout* drop_t, const vb_dropout* drop_v,
                                            void* stream) {
  if (B <= 0 || Nt <= 0 || Nv <= 0 || H <= 0 || H > 2048 || !dy || !xt || !xv || !v_type_row || !gamma_t || !gamma_v || !mean || !rstd)
    return set_error(VB_ERR_INVALID, "vb_concat_embed_ln_bwd: bad arguments (H <= 2048)");
  const size_t smem = (size_t)5 * H * sizeof(float);
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(concat_ln_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_concat_embed_ln_bwd: %s", cudaGetErrorString(e));
  }
  // fewer CTAs than the forward: every CTA ends with one atomic per column and parameter
  int grid = sm_count() * 2;
  const long long rows = (long long)B * (Nt + Nv);
  if (grid <= 0) grid = 264;
  if ((long long)grid * BB_WARPS > rows) grid = (int)((rows + BB_WARPS - 1) / BB_WARPS);
  launch_pdl(concat_ln_bwd_kernel, dim3(grid), dim3(BB_THREADS), smem, BB_ST(stream), dy, xt, xv, v_type_row, gamma_t, gamma_v, mean, rstd, dxt, dxv,
             static_cast<__nv_bfloat16*>(dxv_bf16), dgamma_t, dbeta_t, dgamma_v, dbeta_v, dcol_v, dcol_v2, (int)B, (int)Nt, (int)Nv, (int)H,
             bb_drop(drop_t), bb_drop(drop_v));
  return check_launch("vb_concat_embed_ln_bwd");
}

extern "C" vb_status vb_embed_text_bwd_padded(const float* dout, const int64_t* ids, const int64_t* token_type_ids, float* dword, float* dpos,
                                              float* dtype, int32_t B, int32_t Nt, int32_t H, void* stream) {
  if (B <= 0 || Nt <= 0 || H <= 0 || !dout || !ids || !token_type_ids) return set_error(VB_ERR_INVALID, "vb_embed_text_bwd_padded: bad arguments");
  launch_pdl(embed_text_bwd_padded_kernel, dim3(bb_grid((long long)B * Nt, BB_WARPS)), dim3(BB_THREADS), (size_t)0, BB_ST(stream), dout,
             reinterpret_cast<const long long*>(ids), reinterpret_cast<const long long*>(token_type_ids), dword, dpos, dtype, (int)B, (int)Nt, (int)H);
  return check_launch("vb_embed_text_bwd_padded");
}

extern "C" vb_status vb_weight_norm_fwd(const float* v, const float* g, int64_t n, float* w_f32, void* w16, void* w_lo, void* w_b16, int32_t w_fp16,
                                        double* scratch, void* stream) {
  if (n <= 0 || !v || !g || !scratch || (w_lo && !w16)) return set_error(VB_ERR_INVALID, "vb_weight_norm_fwd: bad arguments");
  launch_pdl(wn_partials_kernel<false>, dim3(WN_BLOCKS), dim3(BB_THREADS), (size_t)0, BB_ST(stream), v, (const float*)nullptr, (long long)n, scratch);
  launch_pdl(wn_fwd_kernel, dim3(bb_grid(n, BB_THREADS)), dim3(BB_THREADS), (size_t)0, BB_ST(stream), v, g, (long long)n, (const double*)scratch,
             w_f32, w16, w_lo, static_cast<__nv_bfloat16*>(w_b16), w_fp16 ? 1 : 0);
  return check_launch("vb_weight_norm_fwd");
}

extern "C" vb_status vb_weight_norm_bwd(const float* dw, const float* v, const float* g, int64_t n, float* dg, float* dv, double* scratch,
                                        void* stream) {
  if (n <= 0 || !dw || !v || !g || !scratch) return set_error(VB_ERR_INVALID, "vb_weight_norm_bwd: bad arguments");
  launch_pdl(wn_partials_kernel<true>, dim3(WN_BLOCKS), dim3(BB_THREADS), (size_t)0, BB_ST(stream), v, dw, (long long)n, scratch);
  launch_pdl(wn_bwd_kernel, dim3(dv ? bb_grid(n, BB_THREADS) : 1), dim3(BB_THREADS), (size_t)0, BB_ST(stream), dw, v, g, (long long)n,
             (const double*)scratch, dg, dv);
  return check_launch("vb_weight_norm_bwd");
}

extern "C" vb_status vb_tanh_fwd(const float* x, float* y_f32, void* y16, void* y_lo, void* y_b16, int32_t y_fp16, int64_t n, void* stream) {
  if (n <= 0 || !x || (y_lo && !y16)) return set_error(VB_ERR_INVALID, "vb_tanh_fwd: bad arguments");
  launch_pdl(tanh_fwd_kernel, dim3(bb_grid(n, 256)), dim3(256), (size_t)0, BB_ST(stream), x, y_f32, y16, y_lo, static_cast<__nv_bfloat16*>(y_b16),
             y_fp16 ? 1 : 0, (long long)n);
  return check_launch("vb_tanh_fwd");
}

extern "C" vb_status vb_tanh_bwd(const float* dy, const float* y, void* dx_bf16, float* dbias, int32_t M, int32_t N, void* stream) {
  if (M <= 0 || N <= 0 || !dy || !y) return set_error(VB_ERR_INVALID, "vb_tanh_bwd: bad arguments");
  launch_pdl(tanh_bwd_kernel, dim3((N + 127) / 128), dim3(128), (size_t)0, BB_ST(stream), dy, y, static_cast<__nv_bfloat16*>(dx_bf16), dbias,
             (int)M, (int)N);
  return check_launch("vb_tanh_bwd");
}

extern "C" vb_status vb_mask_concat_additive(const int64_t* mask_t, const int64_t* mask_v, float* out, int32_t B, int32_t Nt, int32_t Nv, void* stream) {
  if (B <= 0 || Nt <= 0 || Nv <= 0 || !mask_t || !mask_v || !out) return set_error(VB_ERR_INVALID, "vb_mask_concat_additive: bad arguments");
  launch_pdl(mask_concat_kernel, dim3(bb_grid((long long)B * (Nt + Nv), 256)), dim3(256), (size_t)0, BB_ST(stream),
             reinterpret_cast<const long long*>(mask_t), reinterpret_cast<const long long*>(mask_v), out, (int)B, (int)Nt, (int)Nv);
  return check_launch("vb_mask_concat_additive");
}
