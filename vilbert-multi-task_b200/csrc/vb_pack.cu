// vb_pack.cu — packed task steps: the text tokens and image regions of a batch that its masks mark valid, laid out as
// contiguous per-sample row ranges so that every GEMM and LayerNorm of the encoder runs on valid rows only.
//
// A packed stream holds `rows` rows (the batch's valid-row count rounded up to a capacity bucket by the host). Sample b owns
// rows off[b] .. off[b] + len[b] - 1; rows off[B] .. rows - 1 belong to no sample. map[r] is the padded row (b * N + i) of packed
// row r, -1 for a row of no sample. The masks must be prefix-valid (the host checks that before it builds a packed plan).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "vb_internal.h"
#include "vb_ptx.cuh"

namespace vb {

constexpr int PACK_THREADS = 1024;

// One CTA: lengths from the 0/1 masks (+1 for the task token inserted at text position 1), exclusive prefix sums (off has B + 1
// entries: off[B] = rows used), then the row maps. A batch with more valid rows than the capacity is clamped to it (memory safety;
// the host sizes the capacity from the same masks).
__global__ void __launch_bounds__(PACK_THREADS) pack_build_kernel(const long long* __restrict__ mt, int Nt_in, int has_task,
                                                                  const long long* __restrict__ mv, int Nv, int B, int rows_t, int rows_v,
                                                                  int* __restrict__ off_t, int* __restrict__ len_t, int* __restrict__ map_t,
                                                                  int* __restrict__ off_v, int* __restrict__ len_v, int* __restrict__ map_v) {
  pdl_entry();
  const int Nt = Nt_in + has_task;
  for (int b = threadIdx.x; b < B; b += PACK_THREADS) {
    int n = 0;
    for (int j = 0; j < Nt_in; ++j) n += mt[(long long)b * Nt_in + j] != 0;
    len_t[b] = n + has_task;   // the task token's row is always valid (the mask gets a leading 1)
    n = 0;
    for (int j = 0; j < Nv; ++j) n += mv[(long long)b * Nv + j] != 0;
    len_v[b] = n;
  }
  for (int r = threadIdx.x; r < rows_t; r += PACK_THREADS) map_t[r] = -1;
  for (int r = threadIdx.x; r < rows_v; r += PACK_THREADS) map_v[r] = -1;
  __syncthreads();
  if (threadIdx.x == 0) {
    int ot = 0, ov = 0;
    for (int b = 0; b < B; ++b) {
      len_t[b] = min(len_t[b], rows_t - ot); off_t[b] = ot; ot += len_t[b];
      len_v[b] = min(len_v[b], rows_v - ov); off_v[b] = ov; ov += len_v[b];
    }
    off_t[B] = ot; off_v[B] = ov;
  }
  __syncthreads();
  for (int b = 0; b < B; ++b) {
    for (int i = threadIdx.x; i < len_t[b]; i += PACK_THREADS) map_t[off_t[b] + i] = b * Nt + i;
    for (int i = threadIdx.x; i < len_v[b]; i += PACK_THREADS) map_v[off_v[b] + i] = b * Nv + i;
  }
}

// pack_build_kernel for one stream: the image stream of a retrieval chunk (built once per chunk, in the image prefix) or the text
// stream of a caption (built per caption from its loaded mask). Same layout, same clamp.
__global__ void __launch_bounds__(PACK_THREADS) pack_segments_kernel(const long long* __restrict__ mask, int N_in, int has_task, int B,
                                                                     int rows, int* __restrict__ off, int* __restrict__ len,
                                                                     int* __restrict__ map) {
  pdl_entry();
  const int N = N_in + has_task;
  for (int b = threadIdx.x; b < B; b += PACK_THREADS) {
    int n = 0;
    for (int j = 0; j < N_in; ++j) n += mask[(long long)b * N_in + j] != 0;
    len[b] = n + has_task;
  }
  for (int r = threadIdx.x; r < rows; r += PACK_THREADS) map[r] = -1;
  __syncthreads();
  if (threadIdx.x == 0) {
    int o = 0;
    for (int b = 0; b < B; ++b) {
      len[b] = min(len[b], rows - o); off[b] = o; o += len[b];
    }
    off[B] = o;
  }
  __syncthreads();
  for (int b = 0; b < B; ++b)
    for (int i = threadIdx.x; i < len[b]; i += PACK_THREADS) map[off[b] + i] = b * N + i;
}

// A one-sample packed stream of L = *len valid rows repeated as `repeats` contiguous segments: dst row r = b * L + i (b < repeats)
// is src row i, every other row of the `rows` is zero. 16-byte units (c16 per row); L is read on the device, so the launch stays
// graph-capturable while the caption length changes.
__global__ void broadcast_segment_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int c16, const int* __restrict__ len,
                                              int repeats, int rows) {
  pdl_entry();
  const int L = max(*len, 1);
  const long long n = (long long)rows * c16, stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
    const int r = (int)(e / c16), c = (int)(e % c16), b = r / L;
    dst[e] = b < repeats ? __ldg(src + (long long)(r - b * L) * c16 + c) : make_uint4(0u, 0u, 0u, 0u);
  }
}

// dst[r, :] = src[map[r], :] (0 where map[r] < 0), f32 rows of `cols`
__global__ void pack_rows_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ map, int rows, int cols) {
  pdl_entry();
  const long long n = (long long)rows * cols, stride = (long long)gridDim.x * blockDim.x;
  if ((cols & 3) == 0) {
    const int c4 = cols >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n / 4; i += stride) {
      const int r = (int)(i / c4), c = (int)(i % c4);
      const int m = map[r];
      reinterpret_cast<float4*>(dst)[i] = m >= 0 ? reinterpret_cast<const float4*>(src)[(long long)m * c4 + c] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
      const int r = (int)(i / cols), c = (int)(i % cols);
      const int m = map[r];
      dst[i] = m >= 0 ? src[(long long)m * cols + c] : 0.f;
    }
  }
}

// The region features of the packed rows as a tensor-core operand: hi (+ split-precision lo, + bf16 copy), bitwise what
// vb_cast_f32_to_bf16 writes for the same element of the padded tensor. 8 columns per thread: two 128-bit loads, one 128-bit store
// per output.
__global__ void pack_regions_kernel(const float* __restrict__ src, const int* __restrict__ map, int rows, int cols, int fp16,
                                    __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, __nv_bfloat16* __restrict__ bw) {
  pdl_entry();
  const int c8 = cols >> 3;
  const long long n = (long long)rows * c8, stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int r = (int)(i / c8), c = (int)(i % c8);
    const int m = map[r];
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (m >= 0) {
      const float4* s = reinterpret_cast<const float4*>(src + (long long)m * cols) + 2 * c;
      a = __ldg(s); b = __ldg(s + 1);
    }
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t h[4], l[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) h[k] = lo ? pack16_split(v[2 * k], v[2 * k + 1], fp16, l[k]) : pack16(v[2 * k], v[2 * k + 1], fp16);
    reinterpret_cast<uint4*>(hi)[i] = make_uint4(h[0], h[1], h[2], h[3]);
    if (lo) reinterpret_cast<uint4*>(lo)[i] = make_uint4(l[0], l[1], l[2], l[3]);
    if (bw) {
#pragma unroll
      for (int k = 0; k < 4; ++k) h[k] = pack_bf16(v[2 * k], v[2 * k + 1]);
      reinterpret_cast<uint4*>(bw)[i] = make_uint4(h[0], h[1], h[2], h[3]);
    }
  }
}

// dst[b * N + i, :] = i < len[b] ? src[off[b] + i, :] : fill (f32 rows of `cols`)
__global__ void unpack_rows_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ off,
                                       const int* __restrict__ len, int B, int N, int cols, float fill) {
  pdl_entry();
  const long long n = (long long)B * N * cols, stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
    const long long row = e / cols;
    const int c = (int)(e % cols), b = (int)(row / N), i = (int)(row % N);
    dst[e] = i < len[b] ? src[(long long)(off[b] + i) * cols + c] : fill;
  }
}

// dst[idx[r], :] += src[r, :] for r < rows (distinct indices: no atomics)
__global__ void scatter_add_rows_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ idx, int rows, int cols) {
  pdl_entry();
  const long long n = (long long)rows * cols, stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
    const int r = (int)(e / cols), c = (int)(e % cols);
    dst[(long long)idx[r] * cols + c] += src[e];
  }
}

// Rows [*first, rows) of up to three 16-bit or f32 tensors (row pitch ld bytes, `bytes` per row, multiples of 16) set to zero
__global__ void zero_tail_rows_kernel(uint8_t* __restrict__ a, uint8_t* __restrict__ b, uint8_t* __restrict__ c, long long ld, int bytes,
                                      const int* __restrict__ first, int rows) {
  pdl_entry();
  const int r0 = *first, c16 = bytes >> 4;
  const long long n = (long long)(rows - r0) * c16, stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
    const long long o = (long long)(r0 + e / c16) * ld + (e % c16) * 16;
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    *reinterpret_cast<uint4*>(a + o) = z;
    if (b) *reinterpret_cast<uint4*>(b + o) = z;
    if (c) *reinterpret_cast<uint4*>(c + o) = z;
  }
}

// Whether a pre-training batch can be packed, in one small buffer read back with one copy (layout: vb_pack_summary in
// include/vilbert_b200.h). One CTA, a
// thread per sample. A sample's mask is prefix-valid and non-empty when it has n >= 1 valid entries and the last one sits at n - 1.
// A NULL mask is all valid; NULL labels count nothing.
constexpr int SUMMARY_THREADS = 256;

__global__ void __launch_bounds__(SUMMARY_THREADS) pack_summary_kernel(const long long* __restrict__ mt, const long long* __restrict__ mv, int B,
                                                                       int Nt, int Nv, const long long* __restrict__ lm,
                                                                       const long long* __restrict__ il, int* __restrict__ out) {
  pdl_entry();
  __shared__ int total[5];
  if (threadIdx.x < 5) total[threadIdx.x] = 0;
  __syncthreads();
  int bad_t = 0, bad_v = 0, lab_t = 0, lab_v = 0, n_lab = 0;
  for (int b = threadIdx.x; b < B; b += SUMMARY_THREADS) {
    int n = 0, last = -1;
    for (int j = 0; j < Nt; ++j) {
      const long long e = (long long)b * Nt + j;
      const bool on = !mt || mt[e] != 0;
      if (on) { ++n; last = j; }
      if (lm && lm[e] != -1) { ++n_lab; lab_t += !on; }
    }
    out[b] = n;
    bad_t += n == 0 || last != n - 1;
    n = 0; last = -1;
    for (int j = 0; j < Nv; ++j) {
      const bool on = !mv || mv[(long long)b * Nv + j] != 0;
      if (on) { ++n; last = j; }
      if (il && j > 0 && il[(long long)b * (Nv - 1) + j - 1] == 1) lab_v += !on;    // image_label covers regions 1 .. Nv - 1
    }
    out[B + b] = n;
    bad_v += n == 0 || last != n - 1;
  }
  if (bad_t) atomicAdd(&total[0], bad_t);
  if (bad_v) atomicAdd(&total[1], bad_v);
  if (lab_t) atomicAdd(&total[2], lab_t);
  if (lab_v) atomicAdd(&total[3], lab_v);
  if (n_lab) atomicAdd(&total[4], n_lab);
  __syncthreads();
  if (threadIdx.x < 5) out[2 * B + threadIdx.x] = total[threadIdx.x];
}

static inline int grid_for(long long n) {
  long long blocks = (n + 255) / 256, cap = (long long)sm_count() * 8;
  if (cap <= 0) cap = 132 * 8;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}
static inline bool a16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace vb

using namespace vb;

extern "C" vb_status vb_pack_build(const int64_t* text_mask, int32_t Nt_in, int32_t has_task, const int64_t* image_mask, int32_t Nv, int32_t B,
                                   int32_t rows_t, int32_t rows_v, int32_t* off_t, int32_t* len_t, int32_t* map_t, int32_t* off_v, int32_t* len_v,
                                   int32_t* map_v, void* stream) {
  if (B <= 0 || Nt_in <= 0 || Nv <= 0 || rows_t <= 0 || rows_v <= 0 || !text_mask || !image_mask || !off_t || !len_t || !map_t || !off_v ||
      !len_v || !map_v)
    return set_error(VB_ERR_INVALID, "vb_pack_build: bad arguments");
  launch_pdl(pack_build_kernel, dim3(1), dim3(PACK_THREADS), (size_t)0, static_cast<cudaStream_t>(stream),
             reinterpret_cast<const long long*>(text_mask), (int)Nt_in, (int)(has_task ? 1 : 0), reinterpret_cast<const long long*>(image_mask),
             (int)Nv, (int)B, (int)rows_t, (int)rows_v, off_t, len_t, map_t, off_v, len_v, map_v);
  return check_launch("vb_pack_build");
}

extern "C" vb_status vb_pack_segments(const int64_t* mask, int32_t N_in, int32_t has_task, int32_t B, int32_t rows, int32_t* off, int32_t* len,
                                      int32_t* map, void* stream) {
  if (B <= 0 || N_in <= 0 || rows <= 0 || !mask || !off || !len || !map) return set_error(VB_ERR_INVALID, "vb_pack_segments: bad arguments");
  launch_pdl(pack_segments_kernel, dim3(1), dim3(PACK_THREADS), (size_t)0, static_cast<cudaStream_t>(stream),
             reinterpret_cast<const long long*>(mask), (int)N_in, (int)(has_task ? 1 : 0), (int)B, (int)rows, off, len, map);
  return check_launch("vb_pack_segments");
}

extern "C" vb_status vb_broadcast_segment_rows(const void* src, void* dst, int32_t row_bytes, const int32_t* len, int32_t repeats, int32_t rows,
                                               void* stream) {
  if (row_bytes <= 0 || (row_bytes & 15) || repeats <= 0 || rows <= 0 || !src || !dst || !len || !a16(src) || !a16(dst))
    return set_error(VB_ERR_INVALID, "vb_broadcast_segment_rows: bad arguments (16-byte rows and bases)");
  launch_pdl(broadcast_segment_rows_kernel, dim3(grid_for((long long)rows * (row_bytes / 16))), dim3(256), (size_t)0,
             static_cast<cudaStream_t>(stream), static_cast<const uint4*>(src), static_cast<uint4*>(dst), (int)(row_bytes / 16), len,
             (int)repeats, (int)rows);
  return check_launch("vb_broadcast_segment_rows");
}

extern "C" vb_status vb_pack_rows_f32(const float* src, float* dst, const int32_t* map, int32_t rows, int32_t cols, void* stream) {
  if (rows <= 0 || cols <= 0 || !src || !dst || !map) return set_error(VB_ERR_INVALID, "vb_pack_rows_f32: bad arguments");
  if ((cols & 3) == 0 && (!a16(src) || !a16(dst))) return set_error(VB_ERR_INVALID, "vb_pack_rows_f32: misaligned rows");
  launch_pdl(pack_rows_f32_kernel, dim3(grid_for((long long)rows * cols / ((cols & 3) ? 1 : 4))), dim3(256), (size_t)0,
             static_cast<cudaStream_t>(stream), src, dst, map, (int)rows, (int)cols);
  return check_launch("vb_pack_rows_f32");
}

extern "C" vb_status vb_pack_regions(const float* features, const int32_t* map, int32_t rows, int32_t cols, int32_t fp16, void* dst, void* dst_lo,
                                     void* dst_b16, void* stream) {
  if (rows <= 0 || cols <= 0 || (cols & 7) || !features || !map || !dst) return set_error(VB_ERR_INVALID, "vb_pack_regions: bad arguments (cols % 8 == 0)");
  if (!a16(features) || !a16(dst) || (dst_lo && !a16(dst_lo)) || (dst_b16 && !a16(dst_b16)))
    return set_error(VB_ERR_INVALID, "vb_pack_regions: misaligned buffers");
  launch_pdl(pack_regions_kernel, dim3(grid_for((long long)rows * (cols / 8))), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream), features,
             map, (int)rows, (int)cols, (int)(fp16 ? 1 : 0), static_cast<__nv_bfloat16*>(dst), static_cast<__nv_bfloat16*>(dst_lo),
             static_cast<__nv_bfloat16*>(dst_b16));
  return check_launch("vb_pack_regions");
}

extern "C" vb_status vb_unpack_rows_f32(const float* src, float* dst, const int32_t* off, const int32_t* len, int32_t B, int32_t N, int32_t cols,
                                        float fill, void* stream) {
  if (B <= 0 || N <= 0 || cols <= 0 || !src || !dst || !off || !len) return set_error(VB_ERR_INVALID, "vb_unpack_rows_f32: bad arguments");
  launch_pdl(unpack_rows_f32_kernel, dim3(grid_for((long long)B * N * cols)), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream), src, dst, off,
             len, (int)B, (int)N, (int)cols, fill);
  return check_launch("vb_unpack_rows_f32");
}

extern "C" vb_status vb_scatter_add_rows_f32(const float* src, float* dst, const int32_t* idx, int32_t rows, int32_t cols, void* stream) {
  if (rows <= 0 || cols <= 0 || !src || !dst || !idx) return set_error(VB_ERR_INVALID, "vb_scatter_add_rows_f32: bad arguments");
  launch_pdl(scatter_add_rows_f32_kernel, dim3(grid_for((long long)rows * cols)), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream), src, dst,
             idx, (int)rows, (int)cols);
  return check_launch("vb_scatter_add_rows_f32");
}

extern "C" vb_status vb_zero_tail_rows(void* a, void* b, void* c, int64_t ld_bytes, int32_t row_bytes, const int32_t* first, int32_t rows,
                                       void* stream) {
  if (rows <= 0 || row_bytes <= 0 || (row_bytes & 15) || (ld_bytes & 15) || !a || !first || !a16(a) || (b && !a16(b)) || (c && !a16(c)))
    return set_error(VB_ERR_INVALID, "vb_zero_tail_rows: bad arguments (16-byte rows and bases)");
  launch_pdl(zero_tail_rows_kernel, dim3(grid_for((long long)rows * (row_bytes / 16))), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream),
             static_cast<uint8_t*>(a), static_cast<uint8_t*>(b), static_cast<uint8_t*>(c), (long long)ld_bytes, (int)row_bytes, first, (int)rows);
  return check_launch("vb_zero_tail_rows");
}

extern "C" vb_status vb_pack_summary(const int64_t* text_mask, const int64_t* image_mask, int32_t B, int32_t Nt, int32_t Nv,
                                     const int64_t* lm_labels, const int64_t* image_label, int32_t* out, void* stream) {
  if (B <= 0 || Nt <= 0 || Nv <= 1 || !out) return set_error(VB_ERR_INVALID, "vb_pack_summary: bad arguments");
  launch_pdl(pack_summary_kernel, dim3(1), dim3(SUMMARY_THREADS), (size_t)0, static_cast<cudaStream_t>(stream),
             reinterpret_cast<const long long*>(text_mask), reinterpret_cast<const long long*>(image_mask), (int)B, (int)Nt, (int)Nv,
             reinterpret_cast<const long long*>(lm_labels), reinterpret_cast<const long long*>(image_label), out);
  return check_launch("vb_pack_summary");
}
