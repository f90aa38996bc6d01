// vb_rowops.cu — the HBM-bound row-wise kernels around the tensor-core contractions: LayerNorm
// forward/backward (vilbert.py:304-317), text / image embedding assembly (:346-367, :1421-1432),
// bias-gradient column sums, tiny-N linears (1-3 logits), pooled fusion, casts, VQA BCE loss.
// All are 128-bit vectorised, one warp per row, sized in multiples of the SM count.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "vb_internal.h"
#include "vb_ptx.cuh"

namespace vb {

constexpr int ROW_WARPS = 8;                 // warps per CTA for warp-per-row kernels
constexpr int ROW_THREADS = ROW_WARPS * 32;
constexpr int MAX_V4 = 16;                   // float4 chunks per lane -> H <= 2048

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

static inline int row_grid(long long rows) {
  long long blocks = (rows + ROW_WARPS - 1) / ROW_WARPS;
  long long cap = (long long)sm_count() * 8;
  if (cap <= 0) cap = 132 * 8;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

// ------------------------------------------------------------------------------------------ LayerNorm fwd
// ADD: the LayerNorm of a residual stream, LN(dropout(d) + r) (BertSelfOutput / BertOutput / BertBiOutput): x = drop_in(d) + r is
// formed here, in the order the GEMM epilogue would form it (mask index row*H + col, then one fp32 add), and written over d when
// x_out is set (the backward reads it). The dense GEMM before it then stores d and reads nothing: its epilogue has no DRAM round
// trip on the tensor cores' critical path, while this kernel has many warps per SM to hide the extra read.
template <int NV4, bool ADD>
__global__ void __launch_bounds__(ROW_THREADS)
ln_fwd_kernel(const float* x, long long ldx, const float* __restrict__ gamma, const float* __restrict__ beta,
              float eps, float* __restrict__ y32, __nv_bfloat16* __restrict__ y16, long long ldy, float* __restrict__ mean_out,
              float* __restrict__ rstd_out, int M, int H, const DropCfg drop, int y_fp16, __nv_bfloat16* __restrict__ y_lo,
              __nv_bfloat16* __restrict__ y_b16, const float* __restrict__ r, long long ldr, const DropCfg drop_in, float* x_out) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int n4 = H >> 2;
  const float inv_h = 1.f / (float)H;
  const uint32_t dseed = drop.ctr ? drop_seed(drop) : 0u;
  const uint32_t seed_in = (ADD && drop_in.ctr) ? drop_seed(drop_in) : 0u;
  for (long long row = (long long)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); row < M; row += (long long)gridDim.x * ROW_WARPS) {
    const float4* xr = reinterpret_cast<const float4*>(x + row * ldx);
    float4 v[NV4];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV4; ++i) {
      const int c = lane + i * 32;
      v[i] = (c < n4) ? xr[c] : make_float4(0.f, 0.f, 0.f, 0.f);
      if (ADD && c < n4) {
        const float4 rv = reinterpret_cast<const float4*>(r + row * ldr)[c];
        if (drop_in.ctr) {
          const uint32_t e0 = drop_index(drop_in, row, H, c * 4);
          v[i].x = drop_apply(v[i].x, seed_in, e0, drop_in); v[i].y = drop_apply(v[i].y, seed_in, e0 + 1, drop_in);
          v[i].z = drop_apply(v[i].z, seed_in, e0 + 2, drop_in); v[i].w = drop_apply(v[i].w, seed_in, e0 + 3, drop_in);
        }
        v[i].x += rv.x; v[i].y += rv.y; v[i].z += rv.z; v[i].w += rv.w;
        if (x_out) reinterpret_cast<float4*>(x_out + row * ldx)[c] = v[i];
      }
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
    const float mean = warp_sum(s) * inv_h;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV4; ++i) {
      const int c = lane + i * 32;
      if (c < n4) {
        const float a = v[i].x - mean, b = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
        q += a * a + b * b + cc * cc + d * d;
      }
    }
    const float rstd = rsqrtf(warp_sum(q) * inv_h + eps);
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
#pragma unroll
    for (int i = 0; i < NV4; ++i) {
      const int c = lane + i * 32;
      if (c < n4) {
        const float4 g = reinterpret_cast<const float4*>(gamma)[c];
        const float4 b = reinterpret_cast<const float4*>(beta)[c];
        float4 o;
        o.x = (v[i].x - mean) * rstd * g.x + b.x;
        o.y = (v[i].y - mean) * rstd * g.y + b.y;
        o.z = (v[i].z - mean) * rstd * g.z + b.z;
        o.w = (v[i].w - mean) * rstd * g.w + b.w;
        if (drop.ctr) {   // dropout(LayerNorm(x)) of the embeddings (vilbert.py:365, 1430); element index row*H + col
          const uint32_t e0 = drop_index(drop, row, H, c * 4);
          o.x = drop_apply(o.x, dseed, e0, drop); o.y = drop_apply(o.y, dseed, e0 + 1, drop);
          o.z = drop_apply(o.z, dseed, e0 + 2, drop); o.w = drop_apply(o.w, dseed, e0 + 3, drop);
        }
        if (y32) reinterpret_cast<float4*>(y32 + row * ldy)[c] = o;
        if (y16) {
          if (y_lo) {   // split precision: operand copy as hi + lo
            uint32_t l01, l23;
            const uint32_t h01 = pack16_split(o.x, o.y, y_fp16, l01), h23 = pack16_split(o.z, o.w, y_fp16, l23);
            reinterpret_cast<uint2*>(y16 + row * ldy)[c] = make_uint2(h01, h23);
            reinterpret_cast<uint2*>(y_lo + row * ldy)[c] = make_uint2(l01, l23);
          } else {
            reinterpret_cast<uint2*>(y16 + row * ldy)[c] = make_uint2(pack16(o.x, o.y, y_fp16), pack16(o.z, o.w, y_fp16));
          }
        }
        if (y_b16) reinterpret_cast<uint2*>(y_b16 + row * ldy)[c] = make_uint2(pack_bf16(o.x, o.y), pack_bf16(o.z, o.w));
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ LayerNorm bwd
// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * gamma; dgamma += sum dy * xhat; dbeta += sum dy;
// dbias += sum dx (bias gradient of the Linear that produced the LayerNorm input).
// Optional: dx16 (and dbias) additionally multiplied by the saved GELU derivative `pre` (head transforms:
// Linear -> GELU -> LayerNorm).
//
// A row is handled by a TEAM of two warps (64 lanes x NV float4 chunks) so that the three per-column accumulators fit in
// ~110 registers and two 256-thread CTAs (16 warps) stay resident per SM; the two row sums cross the warps through a
// double-buffered smem slot and one 64-thread named barrier per row.
//
// dy2 (optional): a second fp32 gradient of the LayerNorm output, added to dy as it is read (dy + dy2: the residual-path gradient
// that a dgrad GEMM epilogue would otherwise have added into dy, in the same fp32 addition).
//
// PARTIALS (ln_bwd_det_kernel, deterministic plans): instead of one atomic per column and CTA, CTA b stores its column sums of pass
// k (dgamma, dbeta, dbias) into part[(k * gridDim.x + b) * H + col]; vb_reduce_slices adds them up in CTA order.
template <int NV, bool PARTIALS>
__device__ __forceinline__ void
ln_bwd_body(const float* __restrict__ dy, const float* __restrict__ dy2, long long lddy, const float* __restrict__ x, long long ldx,
            const float* __restrict__ gamma, const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
            float* __restrict__ dx32, __nv_bfloat16* __restrict__ dx16, long long lddx,
            const __nv_bfloat16* __restrict__ pre, long long ldpre, float* __restrict__ dgamma, float* __restrict__ dbeta,
            float* __restrict__ dbias, int M, int H, const DropCfg drop_out, const DropCfg drop_in, float* __restrict__ part) {
  pdl_entry();
  constexpr int TEAMS = ROW_THREADS / 64;
  const uint32_t seed_out = drop_out.ctr ? drop_seed(drop_out) : 0u;   // mask applied to this LayerNorm's output in forward
  const uint32_t seed_in = drop_in.ctr ? drop_seed(drop_in) : 0u;      // mask applied to the dense output feeding this LayerNorm
  __shared__ float xch[TEAMS][2][2][2];
  __shared__ float red[TEAMS][64 * 4 + 4];
  const int team = threadIdx.x >> 6, tl = threadIdx.x & 63, wih = (threadIdx.x >> 5) & 1, lane = threadIdx.x & 31;
  const int n4 = H >> 2;
  const float inv_h = 1.f / (float)H;
  float4 ag[NV], ab[NV], ad[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) ag[i] = ab[i] = ad[i] = make_float4(0.f, 0.f, 0.f, 0.f);

  int it = 0;
  for (long long row = (long long)blockIdx.x * TEAMS + team; row < M; row += (long long)gridDim.x * TEAMS, ++it) {
    const float4* dyr = reinterpret_cast<const float4*>(dy + row * lddy);
    const float4* xr = reinterpret_cast<const float4*>(x + row * ldx);
    const float mean = mean_in[row], rstd = rstd_in[row];
    float4 g[NV], xh[NV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = tl + i * 64;
      if (c < n4) {
        float4 d = dyr[c];
        if (dy2) {
          const float4 e = reinterpret_cast<const float4*>(dy2 + row * lddy)[c];
          d.x += e.x; d.y += e.y; d.z += e.z; d.w += e.w;
        }
        const float4 xv = xr[c], gm = reinterpret_cast<const float4*>(gamma)[c];
        if (drop_out.ctr) {
          const uint32_t e0 = drop_index(drop_out, row, H, c * 4);
          d.x = drop_apply(d.x, seed_out, e0, drop_out); d.y = drop_apply(d.y, seed_out, e0 + 1, drop_out);
          d.z = drop_apply(d.z, seed_out, e0 + 2, drop_out); d.w = drop_apply(d.w, seed_out, e0 + 3, drop_out);
        }
        xh[i] = make_float4((xv.x - mean) * rstd, (xv.y - mean) * rstd, (xv.z - mean) * rstd, (xv.w - mean) * rstd);
        g[i] = make_float4(d.x * gm.x, d.y * gm.y, d.z * gm.z, d.w * gm.w);
        s1 += g[i].x + g[i].y + g[i].z + g[i].w;
        s2 += g[i].x * xh[i].x + g[i].y * xh[i].y + g[i].z * xh[i].z + g[i].w * xh[i].w;
        ag[i].x += d.x * xh[i].x; ag[i].y += d.y * xh[i].y; ag[i].z += d.z * xh[i].z; ag[i].w += d.w * xh[i].w;
        ab[i].x += d.x; ab[i].y += d.y; ab[i].z += d.z; ab[i].w += d.w;
      } else {
        g[i] = xh[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    s1 = warp_sum(s1); s2 = warp_sum(s2);
    if (lane == 0) { xch[team][it & 1][wih][0] = s1; xch[team][it & 1][wih][1] = s2; }
    asm volatile("bar.sync %0, 64;" ::"r"(1 + team) : "memory");
    const float c1 = (xch[team][it & 1][0][0] + xch[team][it & 1][1][0]) * inv_h;
    const float c2 = (xch[team][it & 1][0][1] + xch[team][it & 1][1][1]) * inv_h;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = tl + i * 64;
      if (c < n4) {
        float4 o;
        o.x = (g[i].x - c1 - xh[i].x * c2) * rstd;
        o.y = (g[i].y - c1 - xh[i].y * c2) * rstd;
        o.z = (g[i].z - c1 - xh[i].z * c2) * rstd;
        o.w = (g[i].w - c1 - xh[i].w * c2) * rstd;
        if (dx32) reinterpret_cast<float4*>(dx32 + row * lddx)[c] = o;
        if (dx16 || dbias) {
          if (pre) {
            const uint2 pk = reinterpret_cast<const uint2*>(pre + row * ldpre)[c];
            const float2 p01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&pk.x));
            const float2 p23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&pk.y));
            o.x *= p01.x; o.y *= p01.y; o.z *= p23.x; o.w *= p23.y;   // pre = gelu'(pre-activation) saved by the forward GEMM
          }
          if (drop_in.ctr) {   // gradient of dropout(dense(x)): same mask as the forward GEMM epilogue (index row*H + col)
            const uint32_t e0 = drop_index(drop_in, row, H, c * 4);
            o.x = drop_apply(o.x, seed_in, e0, drop_in); o.y = drop_apply(o.y, seed_in, e0 + 1, drop_in);
            o.z = drop_apply(o.z, seed_in, e0 + 2, drop_in); o.w = drop_apply(o.w, seed_in, e0 + 3, drop_in);
          }
          if (dx16) reinterpret_cast<uint2*>(dx16 + row * lddx)[c] = make_uint2(pack_bf16(o.x, o.y), pack_bf16(o.z, o.w));
          ad[i].x += o.x; ad[i].y += o.y; ad[i].z += o.z; ad[i].w += o.w;
        }
      }
    }
  }
  if (!dgamma && !dbeta && !dbias) return;
  // CTA reduction of the per-team column partials, then one atomic per column per CTA
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (i * 64 >= n4) break;  // uniform
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {
      const float4 v = pass == 0 ? ag[i] : (pass == 1 ? ab[i] : ad[i]);
      float* dst = pass == 0 ? dgamma : (pass == 1 ? dbeta : dbias);
      __syncthreads();
      red[team][tl * 4 + 0] = v.x; red[team][tl * 4 + 1] = v.y; red[team][tl * 4 + 2] = v.z; red[team][tl * 4 + 3] = v.w;
      __syncthreads();
      if (dst) {
        float sacc = 0.f;
#pragma unroll
        for (int w = 0; w < TEAMS; ++w) sacc += red[w][threadIdx.x];
        const int col = (i * 64 + (threadIdx.x >> 2)) * 4 + (threadIdx.x & 3);
        if (PARTIALS) {
          if (col < H) part[((long long)pass * gridDim.x + blockIdx.x) * H + col] = sacc;
        } else {
          if (col < H) atomicAdd(dst + col, sacc);
        }
      }
    }
  }
}

#define VB_LN_BWD_PARAMS                                                                                                                   \
  const float* __restrict__ dy, const float* __restrict__ dy2, long long lddy, const float* __restrict__ x, long long ldx,                  \
      const float* __restrict__ gamma, const float* __restrict__ mean_in, const float* __restrict__ rstd_in, float* __restrict__ dx32,     \
      __nv_bfloat16* __restrict__ dx16, long long lddx, const __nv_bfloat16* __restrict__ pre, long long ldpre,                           \
      float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias, int M, int H, const DropCfg drop_out,             \
      const DropCfg drop_in
template <int NV>
__global__ void __launch_bounds__(ROW_THREADS, 2) ln_bwd_kernel(VB_LN_BWD_PARAMS) {
  ln_bwd_body<NV, false>(dy, dy2, lddy, x, ldx, gamma, mean_in, rstd_in, dx32, dx16, lddx, pre, ldpre, dgamma, dbeta, dbias, M, H, drop_out,
                         drop_in, nullptr);
}
template <int NV>
__global__ void __launch_bounds__(ROW_THREADS, 2) ln_bwd_det_kernel(VB_LN_BWD_PARAMS, float* __restrict__ part) {
  ln_bwd_body<NV, true>(dy, dy2, lddy, x, ldx, gamma, mean_in, rstd_in, dx32, dx16, lddx, pre, ldpre, dgamma, dbeta, dbias, M, H, drop_out,
                        drop_in, part);
}
#undef VB_LN_BWD_PARAMS

// ------------------------------------------------------------------------------------------ casts
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n4, long long n, int fp16,
                                     __nv_bfloat16* __restrict__ dst_lo, __nv_bfloat16* __restrict__ dst_b) {
  pdl_entry();
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    if (dst_lo) {
      uint32_t l01, l23;
      const uint32_t h01 = pack16_split(v.x, v.y, fp16, l01), h23 = pack16_split(v.z, v.w, fp16, l23);
      reinterpret_cast<uint2*>(dst)[i] = make_uint2(h01, h23);
      reinterpret_cast<uint2*>(dst_lo)[i] = make_uint2(l01, l23);
    } else {
      reinterpret_cast<uint2*>(dst)[i] = make_uint2(pack16(v.x, v.y, fp16), pack16(v.z, v.w, fp16));
    }
    if (dst_b) reinterpret_cast<uint2*>(dst_b)[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    const uint16_t hi = cvt16(src[i], fp16);
    reinterpret_cast<uint16_t*>(dst)[i] = hi;
    if (dst_lo) reinterpret_cast<uint16_t*>(dst_lo)[i] = cvt16(src[i] - cvt16_to_f32(hi, fp16), fp16);
    if (dst_b) dst_b[i] = __float2bfloat16(src[i]);
  }
}

// rows x cols with independent leading dims (pads bf16 operands whose row size is not a multiple of 8)
__global__ void cast2d_f32_bf16_kernel(const float* __restrict__ src, long long lds, __nv_bfloat16* __restrict__ dst, long long ldd,
                                       int rows, int cols, float scale) {
  pdl_entry();
  for (long long r = blockIdx.y; r < rows; r += gridDim.y)
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < cols; c += gridDim.x * blockDim.x)
      dst[r * ldd + c] = __float2bfloat16(src[r * lds + c] * scale);
}

// ------------------------------------------------------------------------------------------ text embeddings
// out[b, p, :] = word[ids[b, t]] + pos[t] + type[tt[b, t]]  for the original token t; with task tokens the
// task embedding row is inserted at output position 1 and carries no pos/type term (vilbert.py:358-362).
__global__ void __launch_bounds__(ROW_THREADS)
embed_text_fwd_kernel(const long long* __restrict__ ids, const long long* __restrict__ tts, const long long* __restrict__ task_ids,
                      const float* __restrict__ word, const float* __restrict__ pos, const float* __restrict__ type,
                      const float* __restrict__ task, float* __restrict__ out, int B, int Nt, int H, int has_task) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int No = Nt + (has_task ? 1 : 0);
  const long long rows = (long long)B * No;
  const int n4 = H >> 2;
  for (long long row = (long long)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); row < rows; row += (long long)gridDim.x * ROW_WARPS) {
    const int b = (int)(row / No), p = (int)(row % No);
    float4* o = reinterpret_cast<float4*>(out + row * H);
    if (has_task && p == 1) {
      const float4* te = reinterpret_cast<const float4*>(task + task_ids[b] * H);
      for (int c = lane; c < n4; c += 32) o[c] = te[c];
      continue;
    }
    const int t = (has_task && p > 1) ? p - 1 : p;
    const float4* w = reinterpret_cast<const float4*>(word + ids[(long long)b * Nt + t] * H);
    const float4* pe = reinterpret_cast<const float4*>(pos + (long long)t * H);
    const float4* ty = reinterpret_cast<const float4*>(type + tts[(long long)b * Nt + t] * H);
    for (int c = lane; c < n4; c += 32) {
      const float4 a = w[c], bb = pe[c], cc = ty[c];
      o[c] = make_float4(a.x + bb.x + cc.x, a.y + bb.y + cc.y, a.z + bb.z + cc.z, a.w + bb.w + cc.w);
    }
  }
}

// scatter-add of d(out) into the embedding tables; word row 0 is padding_idx (no gradient, vilbert.py:328-330). A NULL table
// (a frozen embedding) receives nothing.
__global__ void __launch_bounds__(ROW_THREADS)
embed_text_bwd_kernel(const float* __restrict__ dout, const long long* __restrict__ ids, const long long* __restrict__ tts,
                      const long long* __restrict__ task_ids, float* __restrict__ dword, float* __restrict__ dpos,
                      float* __restrict__ dtype, float* __restrict__ dtask, int B, int Nt, int H, int has_task) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int No = Nt + (has_task ? 1 : 0);
  const long long rows = (long long)B * No;
  for (long long row = (long long)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); row < rows; row += (long long)gridDim.x * ROW_WARPS) {
    const int b = (int)(row / No), p = (int)(row % No);
    const float* d = dout + row * H;
    if (has_task && p == 1) {
      if (dtask) {
        float* dt = dtask + task_ids[b] * H;
        for (int c = lane; c < H; c += 32) atomicAdd(dt + c, d[c]);
      }
      continue;
    }
    const int t = (has_task && p > 1) ? p - 1 : p;
    const long long id = ids[(long long)b * Nt + t];
    float* dw = (dword && id != 0) ? dword + id * H : nullptr;
    float* dp = dpos ? dpos + (long long)t * H : nullptr;
    float* dty = dtype ? dtype + tts[(long long)b * Nt + t] * H : nullptr;
    for (int c = lane; c < H; c += 32) {
      const float v = d[c];
      if (dw) atomicAdd(dw + c, v);
      if (dp) atomicAdd(dp + c, v);
      if (dty) atomicAdd(dty + c, v);
    }
  }
}

// ------------------------------------------------------------------------------------------ image location projection
// out[m, h] = sum_j loc[m, j] * W[h, j] + b[h],  j < 5  (BertImageEmbeddings.image_location_embeddings, vilbert.py:1416,1424)
__global__ void loc_proj_fwd_kernel(const float* __restrict__ loc, const float* __restrict__ W, const float* __restrict__ b,
                                    float* __restrict__ out, int M, int H) {
  pdl_entry();
  extern __shared__ float sw[];  // [H][5] + [H]
  for (int i = threadIdx.x; i < H * 5; i += blockDim.x) sw[i] = W[i];
  for (int i = threadIdx.x; i < H; i += blockDim.x) sw[H * 5 + i] = b[i];
  __syncthreads();
  for (long long m = blockIdx.x; m < M; m += gridDim.x) {
    float l[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) l[j] = loc[m * 5 + j];
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      float acc = sw[H * 5 + h];
#pragma unroll
      for (int j = 0; j < 5; ++j) acc += l[j] * sw[h * 5 + j];
      out[m * H + h] = acc;
    }
  }
}

// dW[h, j] += sum_m dy[m, h] * loc[m, j];  db[h] += sum_m dy[m, h]  (either may be NULL: not accumulated)
__global__ void loc_proj_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ loc, float* __restrict__ dW,
                                    float* __restrict__ db, int M, int H, int rows_per_block) {
  pdl_entry();
  const long long m0 = (long long)blockIdx.y * rows_per_block;
  const long long m1 = min((long long)M, m0 + rows_per_block);
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H) return;
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (long long m = m0; m < m1; ++m) {
    const float d = dy[m * H + h];
#pragma unroll
    for (int j = 0; j < 5; ++j) acc[j] += d * __ldg(loc + m * 5 + j);
    acc[5] += d;
  }
  if (dW) {
#pragma unroll
    for (int j = 0; j < 5; ++j) atomicAdd(dW + (long long)h * 5 + j, acc[j]);
  }
  if (db) atomicAdd(db + h, acc[5]);
}

// dx[m, j] = sum_h dy[m, h] * W[h, j]  (j < 5): the input gradient of loc_proj_fwd (d image_loc). One warp per row. W is staged
// transposed ([5][H]) in shared memory, so each 128-bit read of dy meets one 128-bit shared read per box coordinate. The five
// lane sums go through the same xor-shuffle tree in every launch and lane 0 stores them: no atomics, replays are bitwise equal.
template <bool VEC>
__global__ void __launch_bounds__(ROW_THREADS) loc_proj_dx_kernel(const float* __restrict__ dy, const float* __restrict__ W,
                                                                  float* __restrict__ dx, int M, int H) {
  pdl_entry();
  extern __shared__ __align__(16) float swt[];  // [5][H]
  for (int i = threadIdx.x; i < H * 5; i += blockDim.x) swt[(i % 5) * H + i / 5] = W[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (long long m = (long long)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); m < M; m += (long long)gridDim.x * ROW_WARPS) {
    const float* d = dy + m * H;
    float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (VEC) {
      for (int h = lane * 4; h < H; h += 128) {
        const float4 v = *reinterpret_cast<const float4*>(d + h);
#pragma unroll
        for (int j = 0; j < 5; ++j) {
          const float4 w = *reinterpret_cast<const float4*>(swt + j * H + h);
          acc[j] += v.x * w.x + v.y * w.y + v.z * w.z + v.w * w.w;
        }
      }
    } else {
      for (int h = lane; h < H; h += 32) {
        const float v = d[h];
#pragma unroll
        for (int j = 0; j < 5; ++j) acc[j] += v * swt[j * H + h];
      }
    }
#pragma unroll
    for (int j = 0; j < 5; ++j) acc[j] = warp_sum(acc[j]);
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < 5; ++j) dx[m * 5 + j] = acc[j];
    }
  }
}

// ------------------------------------------------------------------------------------------ column sums (bias grads)
template <typename T>
__device__ __forceinline__ float to_f(T v);
template <>
__device__ __forceinline__ float to_f<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

// out[n] += sum_m X[m, n]; block = 32 x 8 threads: 32 consecutive columns, 8 row lanes.
template <typename T>
__global__ void colsum_kernel(const T* __restrict__ X, long long ld, float* __restrict__ out, int M, int N, int rows_per_block) {
  pdl_entry();
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const long long m0 = (long long)blockIdx.y * rows_per_block;
  const long long m1 = min((long long)M, m0 + rows_per_block);
  float acc = 0.f;
  if (col < N)
    for (long long m = m0 + threadIdx.y; m < m1; m += 8) acc += to_f<T>(X[m * ld + col]);
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i][threadIdx.x];
    atomicAdd(out + col, s);
  }
}

// ------------------------------------------------------------------------------------------ tiny-N linear (N <= 8)
// y[m, j] = x[m, :] . W[j, :] + b[j] (+ addend[m]) — vil_logit / vil_tri_prediction / vision_logit /
// linguisic_logit / bi_seq_relationship / the 2-way output of vil_binary_prediction (vilbert.py:1620-1628,1684-1695).
__global__ void __launch_bounds__(ROW_THREADS)
small_linear_fwd_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ W, const float* __restrict__ b,
                        const float* __restrict__ addend, float* __restrict__ y, int M, int K, int N, const DropCfg drop) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const uint32_t dseed = drop.ctr ? drop_seed(drop) : 0u;   // dropout on the input x (vilbert.py:1692, 1695), index m*K + k
  for (long long row = (long long)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); row < M; row += (long long)gridDim.x * ROW_WARPS) {
    const float* xr = x + row * ldx;
    for (int j = 0; j < N; ++j) {
      float acc = 0.f;
      for (int k = lane; k < K; k += 32) {
        float xv = xr[k];
        if (drop.ctr) xv = drop_apply(xv, dseed, drop_index(drop, row, K, k), drop);
        acc += xv * __ldg(W + (long long)j * K + k);
      }
      acc = warp_sum(acc);
      if (lane == 0) y[row * N + j] = acc + (b ? b[j] : 0.f) + (addend ? addend[row] : 0.f);
    }
  }
}

// dx[m, :] (+)= sum_j dy[m, j] W[j, :];  dW[j, :] += sum_m dy[m, j] x[m, :];  db[j] += sum_m dy[m, j]  (NULL dx / dW / db: skipped)
__global__ void __launch_bounds__(ROW_THREADS)
small_linear_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, long long ldx, const float* __restrict__ W,
                        float* __restrict__ dx, long long lddx, int accumulate_dx, float* __restrict__ dW, float* __restrict__ db,
                        int M, int K, int N, const DropCfg drop) {
  pdl_entry();
  const uint32_t dseed = drop.ctr ? drop_seed(drop) : 0u;
  // one CTA handles a strided set of rows; per-thread partial dW over columns k = threadIdx.x + i*ROW_THREADS
  for (int j = 0; j < N; ++j) {
    float dbp = 0.f;
    if (dW) {
      for (int k = threadIdx.x; k < K; k += ROW_THREADS) {
        float acc = 0.f;
        for (long long m = blockIdx.x; m < M; m += gridDim.x) {
          float xv = x[m * ldx + k];
          if (drop.ctr) xv = drop_apply(xv, dseed, drop_index(drop, m, K, k), drop);
          acc += dy[m * N + j] * xv;
        }
        atomicAdd(dW + (long long)j * K + k, acc);
      }
    }
    if (db && threadIdx.x == 0) {
      for (long long m = blockIdx.x; m < M; m += gridDim.x) dbp += dy[m * N + j];
      atomicAdd(db + j, dbp);
    }
  }
  if (dx) {
    for (long long m = blockIdx.x; m < M; m += gridDim.x) {
      for (int k = threadIdx.x; k < K; k += ROW_THREADS) {
        float acc = 0.f;
        for (int j = 0; j < N; ++j) acc += dy[m * N + j] * __ldg(W + (long long)j * K + k);
        if (drop.ctr) acc = drop_apply(acc, dseed, drop_index(drop, m, K, k), drop);
        float* d = dx + m * lddx + k;
        *d = accumulate_dx ? (*d + acc) : acc;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ elementwise helpers
// out = a * b (fusion_method "mul") or a + b ("sum"), f32 + bf16 copies (vilbert.py:1677-1682, 1236-1241)
__global__ void fuse_pooled_fwd_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ o32,
                                       __nv_bfloat16* __restrict__ o16, long long n, int mul, const DropCfg drop, int fp16,
                                       __nv_bfloat16* __restrict__ o_lo, __nv_bfloat16* __restrict__ o_b) {
  pdl_entry();
  const uint32_t dseed = drop.ctr ? drop_seed(drop) : 0u;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = mul ? a[i] * b[i] : a[i] + b[i];
    if (drop.ctr) v = drop_apply(v, dseed, (uint32_t)i, drop);
    if (o32) o32[i] = v;
    if (o16) {
      const uint16_t hi = cvt16(v, fp16);
      reinterpret_cast<uint16_t*>(o16)[i] = hi;
      if (o_lo) reinterpret_cast<uint16_t*>(o_lo)[i] = cvt16(v - cvt16_to_f32(hi, fp16), fp16);
    }
    if (o_b) o_b[i] = __float2bfloat16(v);
  }
}
// da += d * b, db += d * a (mul) or da += d, db += d (sum)
__global__ void fuse_pooled_bwd_kernel(const float* __restrict__ d, const float* __restrict__ a, const float* __restrict__ b,
                                       float* __restrict__ da, float* __restrict__ db, long long n, int mul, const DropCfg drop) {
  pdl_entry();
  const uint32_t dseed = drop.ctr ? drop_seed(drop) : 0u;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float g = d[i];
    if (drop.ctr) g = drop_apply(g, dseed, (uint32_t)i, drop);
    if (da) da[i] += mul ? g * b[i] : g;     // a NULL side needs no gradient
    if (db) db[i] += mul ? g * a[i] : g;
  }
}
// dx = dy * (y > 0) -> bf16 (pooler ReLU, vilbert.py:1121,1136)
__global__ void relu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, __nv_bfloat16* __restrict__ dx16,
                                float* __restrict__ dx32, long long n) {
  pdl_entry();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = y[i] > 0.f ? dy[i] : 0.f;
    if (dx16) dx16[i] = __float2bfloat16(v);
    if (dx32) dx32[i] = v;
  }
}
// y (+)= x  (f32), used to merge gradient contributions
__global__ void axpy_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float alpha) {
  pdl_entry();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) y[i] += alpha * x[i];
}

// ------------------------------------------------------------------------------------------ VQA loss
// loss = mean(BCEWithLogits(z, t)) * n_cols  (task_utils.py:325-327); dz = (sigmoid(z) - t) / n_rows * grad_scale
// PARTIALS: CTA b stores its share into part[b] instead of adding it to *loss (deterministic plans; vb_reduce_slices sums them).
template <bool PARTIALS>
__device__ __forceinline__ void bce_logits_body(const float* __restrict__ z, const float* __restrict__ t, float* __restrict__ loss,
                                                float* __restrict__ dz32, __nv_bfloat16* __restrict__ dz16, long long lddz16, int rows,
                                                int cols, float grad_scale, float* __restrict__ part) {
  pdl_entry();
  __shared__ float red[32];
  const long long n = (long long)rows * cols;
  float acc = 0.f;
  const float inv_rows = 1.f / (float)rows;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float x = z[i], y = t[i];
    acc += fmaxf(x, 0.f) - x * y + log1pf(__expf(-fabsf(x)));
    const float g = (1.f / (1.f + __expf(-x)) - y) * inv_rows * grad_scale;
    if (dz32) dz32[i] = g;
    if (dz16) dz16[(i / cols) * lddz16 + (i % cols)] = __float2bfloat16(g);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) {
      if (PARTIALS) part[blockIdx.x] = v * inv_rows;
      else atomicAdd(loss, v * inv_rows);
    }
  }
}
__global__ void bce_logits_kernel(const float* __restrict__ z, const float* __restrict__ t, float* __restrict__ loss,
                                  float* __restrict__ dz32, __nv_bfloat16* __restrict__ dz16, long long lddz16, int rows, int cols,
                                  float grad_scale) {
  bce_logits_body<false>(z, t, loss, dz32, dz16, lddz16, rows, cols, grad_scale, nullptr);
}
__global__ void bce_logits_det_kernel(const float* __restrict__ z, const float* __restrict__ t, float* __restrict__ dz32,
                                      __nv_bfloat16* __restrict__ dz16, long long lddz16, int rows, int cols, float grad_scale,
                                      float* __restrict__ part) {
  bce_logits_body<true>(z, t, nullptr, dz32, dz16, lddz16, rows, cols, grad_scale, part);
}

// additive attention mask (vilbert.py:1341-1362): out[b, j] = (1 - m[b, j]) * -10000; with prepend_one the
// output row has N+1 entries and a leading 0 (task-token mask extension, :1331-1334)
__global__ void mask_to_additive_kernel(const long long* __restrict__ m, float* __restrict__ out, int B, int N, int prepend) {
  pdl_entry();
  const int No = N + prepend;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)B * No; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / No), j = (int)(i % No);
    float v = 0.f;
    if (!(prepend && j == 0)) v = (1.0f - (float)m[(long long)b * N + (j - prepend)]) * -10000.0f;
    out[i] = v;
  }
}

// ------------------------------------------------------------------------------------------ dynamic_attention (vilbert.py:577-586)
// BertImageSelfAttention with config.dynamic_attention: pool = masked mean of the current text states over the tokens,
// gate = 1 + sigmoid(dyLinear(pool)) per (sample, channel), queries and keys of the image self-attention are multiplied by it.
// (1 - m) * -10000 -> m, exactly: a correctly rounded division (not the approximate one of --use_fast_math, which leaves a masked
// token a weight of about 6e-8 in the mean and a non-zero gradient)
__device__ __forceinline__ float mask_weight(float add) { return 1.f + __fdiv_rn(add, 10000.f); }
__device__ __forceinline__ float sigmoidf_(float z) { return 1.f / (1.f + expf(-z)); }

// pool[b, c] = sum_n w[b, n] x[b, n, c] / sum_n w[b, n]   (x fp32 [B, N, H]; also the 16-bit GEMM operand copies of pool)
__global__ void __launch_bounds__(256)
masked_mean_fwd_kernel(const float* __restrict__ x, const float* __restrict__ addmask, float* __restrict__ pool, uint16_t* __restrict__ p16,
                       uint16_t* __restrict__ p16_lo, __nv_bfloat16* __restrict__ p16_b, int fp16, int N, int H) {
  pdl_entry();
  const int b = blockIdx.y, c = blockIdx.x * 256 + threadIdx.x;
  if (c >= H) return;
  float acc = 0.f, ws = 0.f;
  for (int n = 0; n < N; ++n) {
    const float w = mask_weight(addmask[(long long)b * N + n]);
    acc += w * x[((long long)b * N + n) * H + c];
    ws += w;
  }
  const float v = acc / ws;
  const long long o = (long long)b * H + c;
  pool[o] = v;
  const uint16_t hi = cvt16(v, fp16);
  p16[o] = hi;
  if (p16_lo) p16_lo[o] = cvt16(v - cvt16_to_f32(hi, fp16), fp16);
  if (p16_b) p16_b[o] = __float2bfloat16(v);
}

// dx[b, n, c] (+)= w[b, n] / sum_n w[b, n] * dpool[b, c]
__global__ void __launch_bounds__(256)
masked_mean_bwd_kernel(const float* __restrict__ dpool, const float* __restrict__ addmask, float* __restrict__ dx, int accumulate, int N, int H) {
  pdl_entry();
  const int b = blockIdx.y, c = blockIdx.x * 256 + threadIdx.x;
  if (c >= H) return;
  float ws = 0.f;
  for (int n = 0; n < N; ++n) ws += mask_weight(addmask[(long long)b * N + n]);
  const float d = dpool[(long long)b * H + c] / ws;
  for (int n = 0; n < N; ++n) {
    const float g = mask_weight(addmask[(long long)b * N + n]) * d;
    float* o = dx + ((long long)b * N + n) * H + c;
    *o = accumulate ? *o + g : g;
  }
}

// qk[b * N + n, c] *= 1 + sigmoid(z[b, c]) for c < cols (the Q | K sections of a [B * N, ld] 16-bit projection buffer; hi (+ lo)
// parts in the operand format). Two columns per thread.
__global__ void gate_scale_fwd_kernel(uint32_t* __restrict__ qk, uint32_t* __restrict__ qk_lo, long long ld2, const float* __restrict__ z, int N,
                                      int cols, long long total2, int fp16) {
  pdl_entry();
  const int c2n = cols >> 1;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total2; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / c2n;
    const int c2 = (int)(i % c2n);
    const float2 zz = *reinterpret_cast<const float2*>(z + (row / N) * cols + 2 * c2);
    const float g0 = 1.f + sigmoidf_(zz.x), g1 = 1.f + sigmoidf_(zz.y);
    float2 v = unpack16(qk[row * ld2 + c2], fp16);
    if (qk_lo) {
      const float2 l = unpack16(qk_lo[row * ld2 + c2], fp16);
      uint32_t lo;
      qk[row * ld2 + c2] = pack16_split((v.x + l.x) * g0, (v.y + l.y) * g1, fp16, lo);
      qk_lo[row * ld2 + c2] = lo;
    } else {
      qk[row * ld2 + c2] = pack16(v.x * g0, v.y * g1, fp16);
    }
  }
}

// Backward of the gate: with q = gate * q_pre,   d q_pre = gate * dq (in place, bf16)   and
// d z[b, c] = s (1 - s) * sum_n dq[b, n, c] q_pre[b, n, c],   s = sigmoid(z) = gate - 1,   q_pre = q / gate  (gate in (1, 2)).
// dz and dz16 may each be NULL (a frozen gate Linear over text states that need no gradient): with both NULL only dq is scaled.
__global__ void __launch_bounds__(256)
gate_scale_bwd_kernel(__nv_bfloat16* __restrict__ dqk, long long ldd, const uint16_t* __restrict__ qk, const uint16_t* __restrict__ qk_lo, long long ld,
                      const float* __restrict__ z, float* __restrict__ dz, __nv_bfloat16* __restrict__ dz16, int N, int cols, int fp16) {
  pdl_entry();
  const int b = blockIdx.y, c = blockIdx.x * 256 + threadIdx.x;
  if (c >= cols) return;
  const float s = sigmoidf_(z[(long long)b * cols + c]), g = 1.f + s;
  const bool want_dz = dz || dz16;
  float acc = 0.f;
  for (int n = 0; n < N; ++n) {
    const long long r = (long long)b * N + n;
    const float d = __bfloat162float(dqk[r * ldd + c]);
    if (want_dz) {
      float q = cvt16_to_f32(qk[r * ld + c], fp16);
      if (qk_lo) q += cvt16_to_f32(qk_lo[r * ld + c], fp16);
      acc += d * q;
    }
    dqk[r * ldd + c] = __float2bfloat16(d * g);
  }
  if (!want_dz) return;
  const float v = acc / g * s * (1.f - s);
  if (dz) dz[(long long)b * cols + c] = v;
  if (dz16) dz16[(long long)b * cols + c] = __float2bfloat16(v);
}

// dst[r][i] = src[i] for r < repeats (16-byte words): FAST_MODE broadcast of the batch-1 text stream to the image batch
__global__ void broadcast_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, long long n16, int repeats) {
  pdl_entry();
  const long long total = n16 * repeats;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i % n16];
}

// dst[i * repeats + r] = src[i] (items of n16 16-byte words): the on-device form of x.unsqueeze(1).expand(B, R, ...).contiguous()
__global__ void repeat_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, long long n16, long long items, int repeats) {
  pdl_entry();
  const long long total = n16 * items * repeats;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long w = i % n16, row = i / n16;
    dst[i] = src[(row / repeats) * n16 + w];
  }
}

// dst[k][e] (+)= sum_r src[k * stride_k + r * stride_r + e], e < n (fp32, n % 4 == 0): the backward of the in_batch_pairs expansion
// (the gradient of an item broadcast to B pairs is the sum over its B copies)
__global__ void sum_strided_kernel(const float4* __restrict__ src, float4* __restrict__ dst, long long n4, int count_k, long long stride_k4,
                                   int count_r, long long stride_r4, int accumulate) {
  pdl_entry();
  const long long total = n4 * count_k;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long k = i / n4, e = i % n4;
    float4 acc = accumulate ? dst[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4* s = src + k * stride_k4 + e;
    for (int r = 0; r < count_r; ++r) {
      const float4 v = s[(long long)r * stride_r4];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    dst[i] = acc;
  }
}

__global__ void step_bump_kernel(uint32_t* ctr) {
  pdl_entry();
  if (threadIdx.x == 0 && blockIdx.x == 0) *ctr += 1u;
}

static inline DropCfg make_drop(const vb_dropout* d) {
  DropCfg c;
  const bool on = d && d->step && d->p > 0.f;
  c.ctr = on ? d->step : nullptr;
  c.site = d ? d->site : 0u;
  c.thresh = on ? (uint32_t)((double)d->p * 4294967296.0) : 0u;
  c.scale = on && d->p < 1.f ? 1.f / (1.f - d->p) : 1.f;
  c.rows = on ? d->row_map : nullptr;
  return c;
}

// ------------------------------------------------------------------------------------------ deterministic reductions
// The kernels of deterministic plans (DESIGN.md §4h) replace "per-block partial, then a float atomic" by "per-block partial into a
// workspace slice, then one ordered sum": dst[i] += part[0 * stride + i] + part[1 * stride + i] + ... in slice order. The slice
// count is a function of the problem shape only, so the sum has the same order in every run.
__global__ void reduce_slices_kernel(const float* __restrict__ part, long long stride, int slices, long long n, float* __restrict__ dst) {
  pdl_entry();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < slices; ++k) s += part[k * stride + i];
    dst[i] += s;
  }
}

// colsum_kernel with the CTA's column sums stored into part[blockIdx.y * N + col]
template <typename T>
__global__ void colsum_partial_kernel(const T* __restrict__ X, long long ld, float* __restrict__ part, int M, int N, int rows_per_block) {
  pdl_entry();
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const long long m0 = (long long)blockIdx.y * rows_per_block;
  const long long m1 = min((long long)M, m0 + rows_per_block);
  float acc = 0.f;
  if (col < N)
    for (long long m = m0 + threadIdx.y; m < m1; m += 8) acc += to_f<T>(X[m * ld + col]);
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i][threadIdx.x];
    part[(long long)blockIdx.y * N + col] = s;
  }
}

// loc_proj_bwd_kernel with the row block's sums stored into part[blockIdx.y * 6H + ...]: dW (h * 5 + j) then db (5H + h)
__global__ void loc_proj_bwd_partial_kernel(const float* __restrict__ dy, const float* __restrict__ loc, float* __restrict__ part, int M,
                                            int H, int rows_per_block) {
  pdl_entry();
  const long long m0 = (long long)blockIdx.y * rows_per_block;
  const long long m1 = min((long long)M, m0 + rows_per_block);
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H) return;
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (long long m = m0; m < m1; ++m) {
    const float d = dy[m * H + h];
#pragma unroll
    for (int j = 0; j < 5; ++j) acc[j] += d * __ldg(loc + m * 5 + j);
    acc[5] += d;
  }
  float* o = part + (long long)blockIdx.y * 6 * H;
#pragma unroll
  for (int j = 0; j < 5; ++j) o[(long long)h * 5 + j] = acc[j];
  o[5LL * H + h] = acc[5];
}

// the dW / db sums of small_linear_bwd_kernel with CTA b's share stored into part[b * (N K + N) + ...]: dW (j * K + k) then db (N K + j)
__global__ void __launch_bounds__(ROW_THREADS)
small_linear_wgrad_partial_kernel(const float* __restrict__ dy, const float* __restrict__ x, long long ldx, float* __restrict__ part,
                                  int M, int K, int N, const DropCfg drop) {
  pdl_entry();
  const uint32_t dseed = drop.ctr ? drop_seed(drop) : 0u;
  float* o = part + (long long)blockIdx.x * ((long long)N * K + N);
  for (int j = 0; j < N; ++j) {
    for (int k = threadIdx.x; k < K; k += ROW_THREADS) {
      float acc = 0.f;
      for (long long m = blockIdx.x; m < M; m += gridDim.x) {
        float xv = x[m * ldx + k];
        if (drop.ctr) xv = drop_apply(xv, dseed, drop_index(drop, m, K, k), drop);
        acc += dy[m * N + j] * xv;
      }
      o[(long long)j * K + k] = acc;
    }
    if (threadIdx.x == 0) {
      float dbp = 0.f;
      for (long long m = blockIdx.x; m < M; m += gridDim.x) dbp += dy[m * N + j];
      o[(long long)N * K + j] = dbp;
    }
  }
}

// Embedding-table gradients without atomics. Output row r of the text embedding selects one row of each table (embed_key: the word
// id, the token type, the task id of the task-token row, the position); -1 = none (word id 0 is padding_idx, vilbert.py:328-330).
// One warp per (table, output row): the warp of the FIRST output row that selects a table row (found by a ballot scan over the
// earlier rows) owns that table row, adds d(out) of every output row that selects it in row order, and adds the sum to the table
// row with a plain store. Each table row has one writer, each sum one order. The scans cost rows^2 / 32 key reads per table (2.4k
// rows at B = 64 x 37 tokens: ~0.2M), which is small next to the step; H <= 1024 (8 float4 columns per lane).
constexpr int EMBED_DET_V4 = 8;
__device__ __forceinline__ long long embed_key(int table, long long row, const long long* __restrict__ ids, const long long* __restrict__ tts,
                                               const long long* __restrict__ task_ids, int Nt, int has_task) {
  const int No = Nt + has_task;
  const int b = (int)(row / No), p = (int)(row % No);
  if (has_task && p == 1) return table == 2 ? task_ids[b] : -1;
  const int t = (has_task && p > 1) ? p - 1 : p;
  if (table == 0) { const long long id = ids[(long long)b * Nt + t]; return id != 0 ? id : -1; }
  if (table == 1) return tts[(long long)b * Nt + t];
  if (table == 3) return t;
  return -1;
}
__global__ void __launch_bounds__(ROW_THREADS)
embed_text_bwd_det_kernel(const float* __restrict__ dout, const long long* __restrict__ ids, const long long* __restrict__ tts,
                          const long long* __restrict__ task_ids, float* __restrict__ dword, float* __restrict__ dpos,
                          float* __restrict__ dtype, float* __restrict__ dtask, int B, int Nt, int H, int has_task) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const long long rows = (long long)B * (Nt + has_task);
  const int n4 = H >> 2;
  for (long long item = (long long)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); item < 4 * rows; item += (long long)gridDim.x * ROW_WARPS) {
    const int table = (int)(item / rows);
    const long long row = item % rows;
    float* dst = table == 0 ? dword : (table == 1 ? dtype : (table == 2 ? dtask : dpos));
    if (!dst) continue;
    const long long key = embed_key(table, row, ids, tts, task_ids, Nt, has_task);
    if (key < 0) continue;
    bool first = true;
    for (long long base = 0; base < row && first; base += 32) {
      const long long r = base + lane;
      first = !__any_sync(0xffffffffu, r < row && embed_key(table, r, ids, tts, task_ids, Nt, has_task) == key);
    }
    if (!first) continue;
    float4 acc[EMBED_DET_V4];
#pragma unroll
    for (int i = 0; i < EMBED_DET_V4; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long base = row; base < rows; base += 32) {
      const long long r = base + lane;
      unsigned hit = __ballot_sync(0xffffffffu, r < rows && embed_key(table, r, ids, tts, task_ids, Nt, has_task) == key);
      while (hit) {
        const int j = __ffs(hit) - 1;
        hit &= hit - 1;
        const float4* d = reinterpret_cast<const float4*>(dout + (base + j) * H);
#pragma unroll
        for (int i = 0; i < EMBED_DET_V4; ++i) {
          const int c = lane + 32 * i;
          if (c < n4) {
            const float4 v = d[c];
            acc[i].x += v.x; acc[i].y += v.y; acc[i].z += v.z; acc[i].w += v.w;
          }
        }
      }
    }
    float4* o = reinterpret_cast<float4*>(dst + key * H);
#pragma unroll
    for (int i = 0; i < EMBED_DET_V4; ++i) {
      const int c = lane + 32 * i;
      if (c < n4) {
        float4 v = o[c];
        v.x += acc[i].x; v.y += acc[i].y; v.z += acc[i].z; v.w += acc[i].w;
        o[c] = v;
      }
    }
  }
}

static inline int ew_grid(long long n, int threads = 256) {
  long long blocks = (n + threads - 1) / threads;
  long long cap = (long long)sm_count() * 8;
  if (cap <= 0) cap = 132 * 8;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}
static inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace vb

using namespace vb;
#define ST(s) static_cast<cudaStream_t>(s)

// r == NULL: plain LayerNorm of x; otherwise of dropout(x) + r (ln_fwd_kernel<., true>)
static vb_status layernorm_fwd(const char* name, const float* x, int64_t ldx, const float* r, int64_t ldr, const vb_dropout* in_dropout,
                               float* x_out, const float* gamma, const float* beta, float eps, float* y_f32, void* y_bf16, int64_t ldy, float* mean,
                               float* rstd, int32_t M, int32_t H, const vb_dropout* out_dropout, int32_t y_fp16, void* y_lo, void* y_b16, void* stream) {
  if (M <= 0 || H <= 0) return set_error(VB_ERR_INVALID, "%s: empty problem", name);
  if ((H & 3) || H > MAX_V4 * 128 || (ldx & 3) || (ldy & 3) || !al16(x) || !al16(gamma) || !al16(beta) || (y_f32 && !al16(y_f32)) ||
      (y_bf16 && (reinterpret_cast<uintptr_t>(y_bf16) & 7)) || (y_lo && ((reinterpret_cast<uintptr_t>(y_lo) & 7) || !y_bf16)) ||
      (reinterpret_cast<uintptr_t>(y_b16) & 7) || (r && ((ldr & 3) || !al16(r))) || (x_out && !al16(x_out)))
    return set_error(VB_ERR_INVALID, "%s: need H %% 4 == 0, H <= %d, ld %% 4 == 0, 16-byte aligned rows", name, MAX_V4 * 128);
  const DropCfg dc = make_drop(out_dropout), dc_in = make_drop(in_dropout);
  if (dc_in.ctr && ldx != H) return set_error(VB_ERR_INVALID, "%s: the dropout mask is indexed row*H + col and needs dense rows", name);
  const int nv4 = (H / 4 + 31) / 32;
  const int grid = row_grid(M);
  __nv_bfloat16* y16 = static_cast<__nv_bfloat16*>(y_bf16);
#define LN_F(NV) (r ? launch_pdl(ln_fwd_kernel<NV, true>, dim3(grid), dim3(ROW_THREADS), (size_t)(0), ST(stream), x, ldx, gamma, beta, eps, y_f32, y16, ldy, mean, rstd, M, H, dc, (int)(y_fp16 ? 1 : 0), static_cast<__nv_bfloat16*>(y_lo), static_cast<__nv_bfloat16*>(y_b16), r, (long long)ldr, dc_in, x_out) \
                    : launch_pdl(ln_fwd_kernel<NV, false>, dim3(grid), dim3(ROW_THREADS), (size_t)(0), ST(stream), x, ldx, gamma, beta, eps, y_f32, y16, ldy, mean, rstd, M, H, dc, (int)(y_fp16 ? 1 : 0), static_cast<__nv_bfloat16*>(y_lo), static_cast<__nv_bfloat16*>(y_b16), r, (long long)ldr, dc_in, x_out))
  if (nv4 <= 1) LN_F(1); else if (nv4 <= 2) LN_F(2); else if (nv4 <= 4) LN_F(4); else if (nv4 <= 6) LN_F(6);
  else if (nv4 <= 8) LN_F(8); else LN_F(16);
#undef LN_F
  return check_launch(name);
}

extern "C" vb_status vb_layernorm_fwd(const float* x, int64_t ldx, const float* gamma, const float* beta, float eps, float* y_f32,
                                      void* y_bf16, int64_t ldy, float* mean, float* rstd, int32_t M, int32_t H, const vb_dropout* out_dropout,
                                      int32_t y_fp16, void* y_lo, void* y_b16, void* stream) {
  return layernorm_fwd("vb_layernorm_fwd", x, ldx, nullptr, 0, nullptr, nullptr, gamma, beta, eps, y_f32, y_bf16, ldy, mean, rstd, M, H,
                       out_dropout, y_fp16, y_lo, y_b16, stream);
}

extern "C" vb_status vb_add_layernorm_fwd(const float* d, const float* residual, int64_t ld, const vb_dropout* dropout, float* x_out,
                                          const float* gamma, const float* beta, float eps, float* y_f32, void* y_bf16, int64_t ldy, float* mean,
                                          float* rstd, int32_t M, int32_t H, int32_t y_fp16, void* y_lo, void* y_b16, void* stream) {
  if (!d || !residual) return set_error(VB_ERR_INVALID, "vb_add_layernorm_fwd: d and residual are required");
  if (x_out && x_out != d) return set_error(VB_ERR_INVALID, "vb_add_layernorm_fwd: x_out must be NULL or d (the sum is written in place)");
  return layernorm_fwd("vb_add_layernorm_fwd", d, ld, residual, ld, dropout, x_out, gamma, beta, eps, y_f32, y_bf16, ldy, mean, rstd, M, H,
                       nullptr, y_fp16, y_lo, y_b16, stream);
}

static vb_status layernorm_bwd(const char* name, const float* dy, const float* dy2, int64_t lddy, const float* x, int64_t ldx, const float* gamma,
                               const float* mean, const float* rstd, float* dx_f32, void* dx_bf16, int64_t lddx, const void* gelu_pre,
                               int64_t ld_pre, float* dgamma, float* dbeta, float* dbias, int32_t M, int32_t H,
                               const vb_dropout* out_dropout, const vb_dropout* in_dropout, void* stream) {
  if (M <= 0 || H <= 0) return set_error(VB_ERR_INVALID, "%s: empty problem", name);
  if ((H & 3) || H > MAX_V4 * 128 || (ldx & 3) || (lddy & 3) || (lddx & 3) || (gelu_pre && (ld_pre & 3)) || !al16(dy) || !al16(x) || !al16(gamma) ||
      (dy2 && !al16(dy2)))
    return set_error(VB_ERR_INVALID, "%s: need H %% 4 == 0, H <= %d, ld %% 4 == 0, 16-byte aligned rows", name, MAX_V4 * 128);
  const DropCfg dc_out = make_drop(out_dropout), dc_in = make_drop(in_dropout);
  if ((dc_out.ctr || dc_in.ctr) && (ldx != H || lddy != H || lddx != H))
    return set_error(VB_ERR_INVALID, "%s: dropout masks are indexed row*H + col and need dense rows", name);
  const int nv = (H / 4 + 63) / 64;   // float4 chunks per lane of a 64-lane row team
  long long blocks = ((long long)M + 3) / 4;
  const int cap = sm_count() * 2;     // two resident CTAs per SM; fewer CTAs -> fewer dgamma/dbeta atomics
  int grid = (int)(blocks < cap || cap <= 0 ? (blocks > 0 ? blocks : 1) : cap);
  __nv_bfloat16* dx16 = static_cast<__nv_bfloat16*>(dx_bf16);
  const __nv_bfloat16* pre = static_cast<const __nv_bfloat16*>(gelu_pre);
#define LN_B(NV) launch_pdl(ln_bwd_kernel<NV>, dim3(grid), dim3(ROW_THREADS), (size_t)(0), ST(stream), dy, dy2, lddy, x, ldx, gamma, mean, rstd, dx_f32, dx16, lddx, pre, ld_pre, dgamma, dbeta, dbias, M, H, dc_out, dc_in)
  if (nv <= 1) LN_B(1); else if (nv <= 2) LN_B(2); else if (nv <= 3) LN_B(3); else if (nv <= 4) LN_B(4); else LN_B(8);
#undef LN_B
  return check_launch(name);
}

namespace vb {
int launch_reduce_slices(const float* part, long long stride, int slices, long long n, float* dst, cudaStream_t stream) {
  if (n <= 0 || slices <= 0 || !dst) return VB_OK;
  launch_pdl(reduce_slices_kernel, dim3(ew_grid(n)), dim3(256), (size_t)0, stream, part, stride, slices, n, dst);
  return check_launch("vb_reduce_slices");
}
}  // namespace vb

extern "C" vb_status vb_reduce_slices(const float* part, int64_t stride, int32_t slices, int64_t n, float* dst, void* stream) {
  if (slices < 0 || n < 0 || stride < n || (slices > 0 && n > 0 && (!part || !dst)))
    return set_error(VB_ERR_INVALID, "vb_reduce_slices: bad arguments (slices %d, n %lld, stride %lld)", (int)slices, (long long)n, (long long)stride);
  return launch_reduce_slices(part, stride, slices, n, dst, ST(stream));
}

// vb_layernorm_bwd / vb_add_layernorm_bwd (dy2 may be NULL) of deterministic plans: the column sums go through `ws`
extern "C" vb_status vb_layernorm_bwd_det(const float* dy, const float* dy2, int64_t lddy, const float* x, int64_t ldx, const float* gamma,
                                          const float* mean, const float* rstd, float* dx_f32, void* dx_bf16, int64_t lddx, const void* gelu_pre,
                                          int64_t ld_pre, float* dgamma, float* dbeta, float* dbias, int32_t M, int32_t H,
                                          const vb_dropout* out_dropout, const vb_dropout* in_dropout, float* ws, void* stream) {
  const char* name = "vb_layernorm_bwd_det";
  if (M <= 0 || H <= 0) return set_error(VB_ERR_INVALID, "%s: empty problem", name);
  if ((H & 3) || H > MAX_V4 * 128 || (ldx & 3) || (lddy & 3) || (lddx & 3) || (gelu_pre && (ld_pre & 3)) || !al16(dy) || !al16(x) || !al16(gamma) ||
      (dy2 && !al16(dy2)))
    return set_error(VB_ERR_INVALID, "%s: need H %% 4 == 0, H <= %d, ld %% 4 == 0, 16-byte aligned rows", name, MAX_V4 * 128);
  const bool sums = dgamma || dbeta || dbias;
  if (sums && !ws) return set_error(VB_ERR_INVALID, "%s: the column sums need a workspace", name);
  const DropCfg dc_out = make_drop(out_dropout), dc_in = make_drop(in_dropout);
  if ((dc_out.ctr || dc_in.ctr) && (ldx != H || lddy != H || lddx != H))
    return set_error(VB_ERR_INVALID, "%s: dropout masks are indexed row*H + col and need dense rows", name);
  const int nv = (H / 4 + 63) / 64;
  const long long blocks = ((long long)M + 3) / 4;
  const int grid = (int)(blocks < VB_DET_LN_SLICES ? blocks : VB_DET_LN_SLICES);   // a function of M only: the sums keep their order
  __nv_bfloat16* dx16 = static_cast<__nv_bfloat16*>(dx_bf16);
  const __nv_bfloat16* pre = static_cast<const __nv_bfloat16*>(gelu_pre);
#define LN_BD(NV) launch_pdl(ln_bwd_det_kernel<NV>, dim3(grid), dim3(ROW_THREADS), (size_t)(0), ST(stream), dy, dy2, lddy, x, ldx, gamma, mean, rstd, dx_f32, dx16, lddx, pre, ld_pre, dgamma, dbeta, dbias, M, H, dc_out, dc_in, ws)
  if (nv <= 1) LN_BD(1); else if (nv <= 2) LN_BD(2); else if (nv <= 3) LN_BD(3); else if (nv <= 4) LN_BD(4); else LN_BD(8);
#undef LN_BD
  if (int st = check_launch(name)) return st;
  float* dst[3] = {dgamma, dbeta, dbias};
  for (int k = 0; k < 3; ++k)
    if (dst[k])
      if (int st = launch_reduce_slices(ws + (long long)k * grid * H, H, grid, H, dst[k], ST(stream))) return st;
  return VB_OK;
}

extern "C" vb_status vb_layernorm_bwd(const float* dy, int64_t lddy, const float* x, int64_t ldx, const float* gamma, const float* mean,
                                      const float* rstd, float* dx_f32, void* dx_bf16, int64_t lddx, const void* gelu_pre,
                                      int64_t ld_pre, float* dgamma, float* dbeta, float* dbias, int32_t M, int32_t H,
                                      const vb_dropout* out_dropout, const vb_dropout* in_dropout, void* stream) {
  return layernorm_bwd("vb_layernorm_bwd", dy, nullptr, lddy, x, ldx, gamma, mean, rstd, dx_f32, dx_bf16, lddx, gelu_pre, ld_pre, dgamma, dbeta,
                       dbias, M, H, out_dropout, in_dropout, stream);
}

extern "C" vb_status vb_add_layernorm_bwd(const float* dy, const float* dy2, int64_t lddy, const float* x, int64_t ldx, const float* gamma,
                                          const float* mean, const float* rstd, float* dx_f32, void* dx_bf16, int64_t lddx, const void* gelu_pre,
                                          int64_t ld_pre, float* dgamma, float* dbeta, float* dbias, int32_t M, int32_t H,
                                          const vb_dropout* out_dropout, const vb_dropout* in_dropout, void* stream) {
  if (!dy2) return set_error(VB_ERR_INVALID, "vb_add_layernorm_bwd: dy2 is required");
  return layernorm_bwd("vb_add_layernorm_bwd", dy, dy2, lddy, x, ldx, gamma, mean, rstd, dx_f32, dx_bf16, lddx, gelu_pre, ld_pre, dgamma, dbeta,
                       dbias, M, H, out_dropout, in_dropout, stream);
}

extern "C" vb_status vb_cast_f32_to_bf16(const float* src, void* dst, int64_t n, int32_t fp16, void* dst_lo, void* dst_b16, void* stream) {
  if (n <= 0) return VB_OK;
  if (!al16(src) || (reinterpret_cast<uintptr_t>(dst) & 7) || (reinterpret_cast<uintptr_t>(dst_lo) & 7) || (reinterpret_cast<uintptr_t>(dst_b16) & 7))
    return set_error(VB_ERR_INVALID, "vb_cast_f32_to_bf16: misaligned buffers");
  launch_pdl(cast_f32_bf16_kernel, dim3(ew_grid(n / 4 + 1)), dim3(256), (size_t)(0), ST(stream), src, static_cast<__nv_bfloat16*>(dst), n / 4, n,
             (int)(fp16 ? 1 : 0), static_cast<__nv_bfloat16*>(dst_lo), static_cast<__nv_bfloat16*>(dst_b16));
  return check_launch("vb_cast_f32_to_bf16");
}

extern "C" vb_status vb_cast2d_f32_to_bf16(const float* src, int64_t lds, void* dst, int64_t ldd, int32_t rows, int32_t cols, float scale,
                                           void* stream) {
  if (rows <= 0 || cols <= 0) return VB_OK;
  dim3 grid((cols + 255) / 256 > 64 ? 64 : (cols + 255) / 256, rows > 4096 ? 4096 : rows);
  launch_pdl(cast2d_f32_bf16_kernel, dim3(grid), dim3(256), (size_t)(0), ST(stream), src, lds, static_cast<__nv_bfloat16*>(dst), ldd, rows, cols, scale);
  return check_launch("vb_cast2d_f32_to_bf16");
}

extern "C" vb_status vb_embed_text_fwd(const int64_t* ids, const int64_t* token_type_ids, const int64_t* task_ids, const float* word,
                                       const float* pos, const float* type, const float* task, float* out, int32_t B, int32_t Nt,
                                       int32_t H, void* stream) {
  if (B <= 0 || Nt <= 0 || (H & 3)) return set_error(VB_ERR_INVALID, "vb_embed_text_fwd: bad shape");
  const int has_task = task_ids != nullptr;
  if (has_task && !task) return set_error(VB_ERR_INVALID, "vb_embed_text_fwd: task ids without a task table");
  const long long rows = (long long)B * (Nt + has_task);
  launch_pdl(embed_text_fwd_kernel, dim3(row_grid(rows)), dim3(ROW_THREADS), (size_t)(0), ST(stream), 
      reinterpret_cast<const long long*>(ids), reinterpret_cast<const long long*>(token_type_ids),
      reinterpret_cast<const long long*>(task_ids), word, pos, type, task, out, B, Nt, H, has_task);
  return check_launch("vb_embed_text_fwd");
}

extern "C" vb_status vb_embed_text_bwd(const float* dout, const int64_t* ids, const int64_t* token_type_ids, const int64_t* task_ids,
                                       float* dword, float* dpos, float* dtype, float* dtask, int32_t B, int32_t Nt, int32_t H,
                                       void* stream) {
  if (B <= 0 || Nt <= 0) return set_error(VB_ERR_INVALID, "vb_embed_text_bwd: bad shape");
  const int has_task = task_ids != nullptr;
  if (!dword && !dpos && !dtype && !(has_task && dtask)) return VB_OK;     // every table frozen
  const long long rows = (long long)B * (Nt + has_task);
  launch_pdl(embed_text_bwd_kernel, dim3(row_grid(rows)), dim3(ROW_THREADS), (size_t)(0), ST(stream), 
      dout, reinterpret_cast<const long long*>(ids), reinterpret_cast<const long long*>(token_type_ids),
      reinterpret_cast<const long long*>(task_ids), dword, dpos, dtype, dtask, B, Nt, H, has_task);
  return check_launch("vb_embed_text_bwd");
}

extern "C" vb_status vb_embed_text_bwd_det(const float* dout, const int64_t* ids, const int64_t* token_type_ids, const int64_t* task_ids,
                                           float* dword, float* dpos, float* dtype, float* dtask, int32_t B, int32_t Nt, int32_t H,
                                           void* stream) {
  if (B <= 0 || Nt <= 0 || (H & 3) || H > EMBED_DET_V4 * 128 || !al16(dout))
    return set_error(VB_ERR_INVALID, "vb_embed_text_bwd_det: bad shape (H %% 4 == 0, H <= %d, 16-byte aligned rows)", EMBED_DET_V4 * 128);
  const int has_task = task_ids != nullptr;
  if (!dword && !dpos && !dtype && !(has_task && dtask)) return VB_OK;
  const long long rows = (long long)B * (Nt + has_task);
  launch_pdl(embed_text_bwd_det_kernel, dim3(row_grid(4 * rows)), dim3(ROW_THREADS), (size_t)(0), ST(stream),
      dout, reinterpret_cast<const long long*>(ids), reinterpret_cast<const long long*>(token_type_ids),
      reinterpret_cast<const long long*>(task_ids), dword, dpos, dtype, has_task ? dtask : nullptr, B, Nt, H, has_task);
  return check_launch("vb_embed_text_bwd_det");
}

extern "C" vb_status vb_loc_proj_fwd(const float* loc, const float* W, const float* b, float* out, int32_t M, int32_t H, void* stream) {
  if (M <= 0 || H <= 0) return set_error(VB_ERR_INVALID, "vb_loc_proj_fwd: bad shape");
  const size_t smem = (size_t)H * 6 * sizeof(float);
  if (smem > 48 * 1024) return set_error(VB_ERR_UNSUPPORTED, "vb_loc_proj_fwd: H too large");
  int grid = sm_count() * 4; if (grid > M) grid = M; if (grid <= 0) grid = 1;
  launch_pdl(loc_proj_fwd_kernel, dim3(grid), dim3(256), (size_t)(smem), ST(stream), loc, W, b, out, M, H);
  return check_launch("vb_loc_proj_fwd");
}

extern "C" vb_status vb_loc_proj_bwd(const float* dy, const float* loc, float* dW, float* db, int32_t M, int32_t H, void* stream) {
  if (M <= 0 || H <= 0) return set_error(VB_ERR_INVALID, "vb_loc_proj_bwd: bad shape");
  if (!dW && !db) return VB_OK;
  const int rpb = 64;
  dim3 grid((H + 127) / 128, (M + rpb - 1) / rpb);
  launch_pdl(loc_proj_bwd_kernel, dim3(grid), dim3(128), (size_t)(0), ST(stream), dy, loc, dW, db, M, H, rpb);
  return check_launch("vb_loc_proj_bwd");
}

extern "C" vb_status vb_loc_proj_bwd_det(const float* dy, const float* loc, float* dW, float* db, int32_t M, int32_t H, float* ws, void* stream) {
  if (M <= 0 || H <= 0) return set_error(VB_ERR_INVALID, "vb_loc_proj_bwd_det: bad shape");
  if (!dW && !db) return VB_OK;
  if (!ws) return set_error(VB_ERR_INVALID, "vb_loc_proj_bwd_det: no workspace");
  int rpb = (M + VB_DET_SLICES - 1) / VB_DET_SLICES; if (rpb < 64) rpb = 64;
  const int slices = (M + rpb - 1) / rpb;
  launch_pdl(loc_proj_bwd_partial_kernel, dim3((H + 127) / 128, slices), dim3(128), (size_t)(0), ST(stream), dy, loc, ws, M, H, rpb);
  if (int st = check_launch("vb_loc_proj_bwd_det")) return st;
  if (dW) if (int st = launch_reduce_slices(ws, 6LL * H, slices, 5LL * H, dW, ST(stream))) return st;
  if (db) if (int st = launch_reduce_slices(ws + 5LL * H, 6LL * H, slices, H, db, ST(stream))) return st;
  return VB_OK;
}

extern "C" vb_status vb_loc_proj_dx(const float* dy, const float* W, float* dx, int32_t M, int32_t H, void* stream) {
  if (M <= 0 || H <= 0) return set_error(VB_ERR_INVALID, "vb_loc_proj_dx: bad shape");
  const size_t smem = (size_t)H * 5 * sizeof(float);
  if (smem > 48 * 1024) return set_error(VB_ERR_UNSUPPORTED, "vb_loc_proj_dx: H too large");
  const bool vec = H % 4 == 0 && (reinterpret_cast<uintptr_t>(dy) & 15) == 0;
  if (vec) launch_pdl(loc_proj_dx_kernel<true>, dim3(row_grid(M)), dim3(ROW_THREADS), smem, ST(stream), dy, W, dx, M, H);
  else launch_pdl(loc_proj_dx_kernel<false>, dim3(row_grid(M)), dim3(ROW_THREADS), smem, ST(stream), dy, W, dx, M, H);
  return check_launch("vb_loc_proj_dx");
}

extern "C" vb_status vb_colsum(const void* X, int32_t is_bf16, int64_t ld, float* out, int32_t M, int32_t N, void* stream) {
  if (M <= 0 || N <= 0) return set_error(VB_ERR_INVALID, "vb_colsum: bad shape");
  int rpb = (M + 31) / 32; if (rpb < 64) rpb = 64;
  dim3 grid((N + 31) / 32, (M + rpb - 1) / rpb), block(32, 8);
  if (is_bf16) launch_pdl(colsum_kernel<__nv_bfloat16>, dim3(grid), dim3(block), (size_t)(0), ST(stream), static_cast<const __nv_bfloat16*>(X), ld, out, M, N, rpb);
  else launch_pdl(colsum_kernel<float>, dim3(grid), dim3(block), (size_t)(0), ST(stream), static_cast<const float*>(X), ld, out, M, N, rpb);
  return check_launch("vb_colsum");
}

extern "C" vb_status vb_colsum_det(const void* X, int32_t is_bf16, int64_t ld, float* out, int32_t M, int32_t N, float* ws, void* stream) {
  if (M <= 0 || N <= 0 || !ws) return set_error(VB_ERR_INVALID, "vb_colsum_det: bad shape or no workspace");
  int rpb = (M + VB_DET_SLICES - 1) / VB_DET_SLICES; if (rpb < 64) rpb = 64;
  const int slices = (M + rpb - 1) / rpb;
  dim3 grid((N + 31) / 32, slices), block(32, 8);
  if (is_bf16) launch_pdl(colsum_partial_kernel<__nv_bfloat16>, dim3(grid), dim3(block), (size_t)(0), ST(stream), static_cast<const __nv_bfloat16*>(X), ld, ws, M, N, rpb);
  else launch_pdl(colsum_partial_kernel<float>, dim3(grid), dim3(block), (size_t)(0), ST(stream), static_cast<const float*>(X), ld, ws, M, N, rpb);
  if (int st = check_launch("vb_colsum_det")) return st;
  return launch_reduce_slices(ws, N, slices, N, out, ST(stream));
}

extern "C" vb_status vb_small_linear_fwd(const float* x, int64_t ldx, const float* W, const float* b, const float* row_addend, float* y,
                                         int32_t M, int32_t K, int32_t N, const vb_dropout* in_dropout, void* stream) {
  if (M <= 0 || K <= 0 || N <= 0 || N > 8) return set_error(VB_ERR_INVALID, "vb_small_linear_fwd: bad shape (N <= 8)");
  launch_pdl(small_linear_fwd_kernel, dim3(row_grid(M)), dim3(ROW_THREADS), (size_t)(0), ST(stream), x, ldx, W, b, row_addend, y, M, K, N, make_drop(in_dropout));
  return check_launch("vb_small_linear_fwd");
}

extern "C" vb_status vb_small_linear_bwd(const float* dy, const float* x, int64_t ldx, const float* W, float* dx, int64_t lddx,
                                         int32_t accumulate_dx, float* dW, float* db, int32_t M, int32_t K, int32_t N,
                                         const vb_dropout* in_dropout, void* stream) {
  if (M <= 0 || K <= 0 || N <= 0 || N > 8) return set_error(VB_ERR_INVALID, "vb_small_linear_bwd: bad shape (N <= 8)");
  if (!dx && !dW && !db) return VB_OK;
  int grid = sm_count(); if (grid > M) grid = M; if (grid <= 0) grid = 1;
  launch_pdl(small_linear_bwd_kernel, dim3(grid), dim3(ROW_THREADS), (size_t)(0), ST(stream), dy, x, ldx, W, dx, lddx, accumulate_dx, dW, db, M, K, N, make_drop(in_dropout));
  return check_launch("vb_small_linear_bwd");
}

extern "C" vb_status vb_small_linear_bwd_det(const float* dy, const float* x, int64_t ldx, const float* W, float* dx, int64_t lddx,
                                             int32_t accumulate_dx, float* dW, float* db, int32_t M, int32_t K, int32_t N,
                                             const vb_dropout* in_dropout, float* ws, void* stream) {
  if (M <= 0 || K <= 0 || N <= 0 || N > 8) return set_error(VB_ERR_INVALID, "vb_small_linear_bwd_det: bad shape (N <= 8)");
  if ((dW || db) && !ws) return set_error(VB_ERR_INVALID, "vb_small_linear_bwd_det: no workspace");
  const DropCfg dc = make_drop(in_dropout);
  if (dx) {   // the input gradient has no atomics: the default kernel without its dW / db sums
    int grid = sm_count(); if (grid > M) grid = M; if (grid <= 0) grid = 1;
    launch_pdl(small_linear_bwd_kernel, dim3(grid), dim3(ROW_THREADS), (size_t)(0), ST(stream), dy, x, ldx, W, dx, lddx, accumulate_dx,
               (float*)nullptr, (float*)nullptr, M, K, N, dc);
    if (int st = check_launch("vb_small_linear_bwd_det")) return st;
  }
  if (!dW && !db) return VB_OK;
  const int slices = M < VB_DET_SLICES ? M : VB_DET_SLICES;
  const long long stride = (long long)N * K + N;
  launch_pdl(small_linear_wgrad_partial_kernel, dim3(slices), dim3(ROW_THREADS), (size_t)(0), ST(stream), dy, x, ldx, ws, M, K, N, dc);
  if (int st = check_launch("vb_small_linear_bwd_det")) return st;
  if (dW) if (int st = launch_reduce_slices(ws, stride, slices, (long long)N * K, dW, ST(stream))) return st;
  if (db) if (int st = launch_reduce_slices(ws + (long long)N * K, stride, slices, N, db, ST(stream))) return st;
  return VB_OK;
}

extern "C" vb_status vb_fuse_pooled_fwd(const float* a, const float* b, float* out_f32, void* out_bf16, int64_t n, int32_t mul,
                                        const vb_dropout* dropout, int32_t out_fp16, void* out_lo, void* out_b16, void* stream) {
  if (n <= 0) return VB_OK;
  launch_pdl(fuse_pooled_fwd_kernel, dim3(ew_grid(n)), dim3(256), (size_t)(0), ST(stream), a, b, out_f32, static_cast<__nv_bfloat16*>(out_bf16), n, mul, make_drop(dropout),
             (int)(out_fp16 ? 1 : 0), static_cast<__nv_bfloat16*>(out_lo), static_cast<__nv_bfloat16*>(out_b16));
  return check_launch("vb_fuse_pooled_fwd");
}
extern "C" vb_status vb_fuse_pooled_bwd(const float* d, const float* a, const float* b, float* da, float* db, int64_t n, int32_t mul,
                                        const vb_dropout* dropout, void* stream) {
  if (n <= 0) return VB_OK;
  launch_pdl(fuse_pooled_bwd_kernel, dim3(ew_grid(n)), dim3(256), (size_t)(0), ST(stream), d, a, b, da, db, n, mul, make_drop(dropout));
  return check_launch("vb_fuse_pooled_bwd");
}
extern "C" vb_status vb_relu_bwd(const float* dy, const float* y, void* dx_bf16, float* dx_f32, int64_t n, void* stream) {
  if (n <= 0) return VB_OK;
  launch_pdl(relu_bwd_kernel, dim3(ew_grid(n)), dim3(256), (size_t)(0), ST(stream), dy, y, static_cast<__nv_bfloat16*>(dx_bf16), dx_f32, n);
  return check_launch("vb_relu_bwd");
}
extern "C" vb_status vb_axpy_f32(const float* x, float* y, int64_t n, float alpha, void* stream) {
  if (n <= 0) return VB_OK;
  launch_pdl(axpy_kernel, dim3(ew_grid(n)), dim3(256), (size_t)(0), ST(stream), x, y, n, alpha);
  return check_launch("vb_axpy_f32");
}
extern "C" vb_status vb_bce_logits_loss(const float* logits, const float* target, float* loss, float* dlogits_f32, void* dlogits_bf16,
                                        int64_t ld_dlogits_bf16, int32_t rows, int32_t cols, float grad_scale, void* stream) {
  if (rows <= 0 || cols <= 0) return set_error(VB_ERR_INVALID, "vb_bce_logits_loss: bad shape");
  cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), ST(stream));
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_bce_logits_loss: memset: %s", cudaGetErrorString(e));
  launch_pdl(bce_logits_kernel, dim3(ew_grid((long long)rows * cols)), dim3(256), (size_t)(0), ST(stream), logits, target, loss, dlogits_f32,
                                                                              static_cast<__nv_bfloat16*>(dlogits_bf16), ld_dlogits_bf16, rows,
                                                                              cols, grad_scale);
  return check_launch("vb_bce_logits_loss");
}
extern "C" vb_status vb_bce_logits_loss_det(const float* logits, const float* target, float* loss, float* dlogits_f32, void* dlogits_bf16,
                                            int64_t ld_dlogits_bf16, int32_t rows, int32_t cols, float grad_scale, float* ws, void* stream) {
  if (rows <= 0 || cols <= 0 || !ws) return set_error(VB_ERR_INVALID, "vb_bce_logits_loss_det: bad shape or no workspace");
  cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), ST(stream));
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_bce_logits_loss_det: memset: %s", cudaGetErrorString(e));
  int grid = ew_grid((long long)rows * cols);
  if (grid > VB_DET_LOSS_SLICES) grid = VB_DET_LOSS_SLICES;
  launch_pdl(bce_logits_det_kernel, dim3(grid), dim3(256), (size_t)(0), ST(stream), logits, target, dlogits_f32,
             static_cast<__nv_bfloat16*>(dlogits_bf16), ld_dlogits_bf16, rows, cols, grad_scale, ws);
  if (int st = check_launch("vb_bce_logits_loss_det")) return st;
  return launch_reduce_slices(ws, 1, grid, 1, loss, ST(stream));
}
extern "C" vb_status vb_mask_to_additive(const int64_t* mask, float* out, int32_t B, int32_t N, int32_t prepend_one, void* stream) {
  if (B <= 0 || N <= 0) return set_error(VB_ERR_INVALID, "vb_mask_to_additive: bad shape");
  launch_pdl(mask_to_additive_kernel, dim3(ew_grid((long long)B * (N + 1))), dim3(256), (size_t)(0), ST(stream), reinterpret_cast<const long long*>(mask), out, B, N, prepend_one ? 1 : 0);
  return check_launch("vb_mask_to_additive");
}
extern "C" vb_status vb_broadcast_rows(const void* src, void* dst, int64_t bytes, int32_t repeats, void* stream) {
  if (bytes <= 0 || repeats <= 0) return VB_OK;
  if ((bytes & 15) || !al16(src) || !al16(dst)) return set_error(VB_ERR_INVALID, "vb_broadcast_rows: needs 16-byte aligned buffers and size");
  launch_pdl(broadcast_rows_kernel, dim3(ew_grid(bytes / 16 * repeats)), dim3(256), (size_t)0, ST(stream), static_cast<const uint4*>(src), static_cast<uint4*>(dst),
             (long long)(bytes / 16), (int)repeats);
  return check_launch("vb_broadcast_rows");
}

extern "C" vb_status vb_repeat_rows(const void* src, void* dst, int64_t bytes, int64_t items, int32_t repeats, void* stream) {
  if (bytes <= 0 || items <= 0 || repeats <= 0) return VB_OK;
  if ((bytes & 15) || !al16(src) || !al16(dst)) return set_error(VB_ERR_INVALID, "vb_repeat_rows: needs 16-byte aligned buffers and item size");
  launch_pdl(repeat_rows_kernel, dim3(ew_grid(bytes / 16 * items * repeats)), dim3(256), (size_t)0, ST(stream), static_cast<const uint4*>(src),
             static_cast<uint4*>(dst), (long long)(bytes / 16), (long long)items, (int)repeats);
  return check_launch("vb_repeat_rows");
}

extern "C" vb_status vb_sum_strided(const float* src, float* dst, int64_t n, int32_t count_k, int64_t stride_k, int32_t count_r, int64_t stride_r,
                                    int32_t accumulate, void* stream) {
  if (n <= 0 || count_k <= 0 || count_r <= 0) return VB_OK;
  if ((n & 3) || (stride_k & 3) || (stride_r & 3) || !al16(src) || !al16(dst)) return set_error(VB_ERR_INVALID, "vb_sum_strided: sizes / strides must be multiples of 4 floats, buffers 16-byte aligned");
  launch_pdl(sum_strided_kernel, dim3(ew_grid(n / 4 * count_k)), dim3(256), (size_t)0, ST(stream), reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(dst),
             (long long)(n / 4), (int)count_k, (long long)(stride_k / 4), (int)count_r, (long long)(stride_r / 4), (int)(accumulate ? 1 : 0));
  return check_launch("vb_sum_strided");
}

extern "C" vb_status vb_masked_mean_fwd(const float* x, const float* add_mask, float* pool, void* pool16, void* pool16_lo, void* pool16_b,
                                        int32_t out_fp16, int32_t B, int32_t N, int32_t H, void* stream) {
  if (B <= 0 || N <= 0 || H <= 0 || !x || !add_mask || !pool || !pool16) return set_error(VB_ERR_INVALID, "vb_masked_mean_fwd: bad arguments");
  launch_pdl(masked_mean_fwd_kernel, dim3((H + 255) / 256, B), dim3(256), (size_t)0, ST(stream), x, add_mask, pool, static_cast<uint16_t*>(pool16),
             static_cast<uint16_t*>(pool16_lo), static_cast<__nv_bfloat16*>(pool16_b), (int)(out_fp16 ? 1 : 0), (int)N, (int)H);
  return check_launch("vb_masked_mean_fwd");
}

extern "C" vb_status vb_masked_mean_bwd(const float* dpool, const float* add_mask, float* dx, int32_t accumulate, int32_t B, int32_t N, int32_t H,
                                        void* stream) {
  if (B <= 0 || N <= 0 || H <= 0 || !dpool || !add_mask || !dx) return set_error(VB_ERR_INVALID, "vb_masked_mean_bwd: bad arguments");
  launch_pdl(masked_mean_bwd_kernel, dim3((H + 255) / 256, B), dim3(256), (size_t)0, ST(stream), dpool, add_mask, dx, (int)(accumulate ? 1 : 0), (int)N, (int)H);
  return check_launch("vb_masked_mean_bwd");
}

extern "C" vb_status vb_gate_scale_fwd(void* qk, void* qk_lo, int64_t ld, const float* z, int32_t B, int32_t N, int32_t cols, int32_t fp16,
                                       void* stream) {
  if (B <= 0 || N <= 0 || cols <= 0 || (cols & 1) || (ld & 1) || !qk || !z || (reinterpret_cast<uintptr_t>(qk) & 3) ||
      (reinterpret_cast<uintptr_t>(qk_lo) & 3) || (reinterpret_cast<uintptr_t>(z) & 7))
    return set_error(VB_ERR_INVALID, "vb_gate_scale_fwd: bad arguments (even cols / ld, 4-byte aligned rows)");
  const long long total2 = (long long)B * N * (cols / 2);
  launch_pdl(gate_scale_fwd_kernel, dim3(ew_grid(total2)), dim3(256), (size_t)0, ST(stream), static_cast<uint32_t*>(qk), static_cast<uint32_t*>(qk_lo),
             (long long)(ld / 2), z, (int)N, (int)cols, total2, (int)(fp16 ? 1 : 0));
  return check_launch("vb_gate_scale_fwd");
}

extern "C" vb_status vb_gate_scale_bwd(void* dqk, int64_t ldd, const void* qk, const void* qk_lo, int64_t ld, const float* z, float* dz, void* dz16,
                                       int32_t B, int32_t N, int32_t cols, int32_t fp16, void* stream) {
  if (B <= 0 || N <= 0 || cols <= 0 || !dqk || !qk || !z) return set_error(VB_ERR_INVALID, "vb_gate_scale_bwd: bad arguments");
  launch_pdl(gate_scale_bwd_kernel, dim3((cols + 255) / 256, B), dim3(256), (size_t)0, ST(stream), static_cast<__nv_bfloat16*>(dqk), (long long)ldd,
             static_cast<const uint16_t*>(qk), static_cast<const uint16_t*>(qk_lo), (long long)ld, z, dz, static_cast<__nv_bfloat16*>(dz16), (int)N,
             (int)cols, (int)(fp16 ? 1 : 0));
  return check_launch("vb_gate_scale_bwd");
}

extern "C" vb_status vb_step_counter_bump(uint32_t* step, void* stream) {
  if (!step) return set_error(VB_ERR_INVALID, "vb_step_counter_bump: null counter");
  cudaError_t e = launch_pdl(step_bump_kernel, dim3(1), dim3(32), (size_t)0, ST(stream), step);
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_step_counter_bump: %s", cudaGetErrorString(e));
  return VB_OK;
}
extern "C" vb_status vb_memset_zero(void* ptr, int64_t bytes, void* stream) {
  if (bytes <= 0) return VB_OK;
  cudaError_t e = cudaMemsetAsync(ptr, 0, (size_t)bytes, ST(stream));
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_memset_zero: %s", cudaGetErrorString(e));
  return VB_OK;
}
