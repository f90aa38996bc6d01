// vb_nan_check: the NaN scan behind torch.autograd.set_detect_anomaly(True) for the plan-backed backward (engine.Plan(anomaly=True)).
// A launch scans a device table of regions (logical rows x cols extents with a row pitch) and atomicMin's the id of every region
// holding a NaN into a device flag, so after the backward the flag names the first region, in the plan's op-list order, that held
// one. The test is on the bit pattern: the library builds with --use_fast_math, under which isnan() may be folded away.
#include <climits>

#include "vb_internal.h"
#include "vb_ptx.cuh"

namespace vb {
namespace {

__device__ __forceinline__ bool nan16(uint32_t h, uint32_t inf) { return (h & 0x7fffu) > inf; }

// one 32-bit word: one fp32 value or two 16-bit values (inf = 0x7c00 for fp16, 0x7f80 for bf16)
__device__ __forceinline__ bool nan_word(uint32_t w, bool f32, uint32_t inf) {
  return f32 ? (w & 0x7fffffffu) > 0x7f800000u : (nan16(w & 0xffffu, inf) | nan16(w >> 16, inf));
}

__device__ __forceinline__ bool nan_vec(uint4 v, bool f32, uint32_t inf) {
  return nan_word(v.x, f32, inf) | nan_word(v.y, f32, inf) | nan_word(v.z, f32, inf) | nan_word(v.w, f32, inf);
}

__device__ __forceinline__ bool nan_elem(const char* p, bool f32, uint32_t inf) {
  return f32 ? nan_word(__ldg(reinterpret_cast<const uint32_t*>(p)), true, inf) : nan16(__ldg(reinterpret_cast<const unsigned short*>(p)), inf);
}

// n elements from p, thread `tid` of `nthr`: scalar loads up to the first 16-byte boundary, 128-bit loads (four in flight per
// thread) over the aligned body, scalar loads over the tail. Nothing outside [p, p + n elements) is read.
__device__ bool scan_run(const char* p, long long n, bool f32, uint32_t inf, long long tid, long long nthr) {
  const int es = f32 ? 4 : 2;
  bool bad = false;
  long long head = (long long)((16u - (uint32_t)(reinterpret_cast<uintptr_t>(p) & 15u)) & 15u) / es;
  if (head > n) head = n;
  for (long long i = tid; i < head; i += nthr) bad |= nan_elem(p + i * es, f32, inf);
  const uint4* v = reinterpret_cast<const uint4*>(p + head * es);
  const long long nv = (n - head) * es / 16;
  long long i = tid;
  for (; i + 3 * nthr < nv; i += 4 * nthr) {
    const uint4 a = __ldg(v + i), b = __ldg(v + i + nthr), c = __ldg(v + i + 2 * nthr), d = __ldg(v + i + 3 * nthr);
    bad |= nan_vec(a, f32, inf) | nan_vec(b, f32, inf) | nan_vec(c, f32, inf) | nan_vec(d, f32, inf);
  }
  for (; i < nv; i += nthr) bad |= nan_vec(__ldg(v + i), f32, inf);
  for (long long j = head + nv * 16 / es + tid; j < n; j += nthr) bad |= nan_elem(p + j * es, f32, inf);
  return bad;
}

__global__ void __launch_bounds__(256) nan_check_kernel(const vb_nan_region* __restrict__ regions, int n, int* flag) {
  pdl_entry();
  const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x, gthr = (long long)gridDim.x * blockDim.x;
  for (int r = 0; r < n; ++r) {
    const vb_nan_region g = regions[r];
    const bool f32 = g.dtype == VB_NAN_F32;
    const uint32_t inf = g.dtype == VB_NAN_F16 ? 0x7c00u : 0x7f80u;
    const char* p = static_cast<const char*>(g.ptr);
    bool bad = false;
    if (g.rows == 1 || g.ld == g.cols) {        // one contiguous run: every thread of the grid strides over it
      bad = scan_run(p, g.rows * g.cols, f32, inf, gtid, gthr);
    } else {                                    // pitched rows: a CTA per row, the pitch padding is never read
      const long long pitch = g.ld * (f32 ? 4 : 2);
      for (long long row = blockIdx.x; row < g.rows; row += gridDim.x)
        bad |= scan_run(p + row * pitch, g.cols, f32, inf, threadIdx.x, blockDim.x);
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicMin(flag, g.id);
  }
}

__global__ void nan_flag_reset_kernel(int* flag) {
  pdl_entry();
  if (threadIdx.x == 0 && blockIdx.x == 0) *flag = INT_MAX;
}

}  // namespace
}  // namespace vb

extern "C" vb_status vb_nan_check(const vb_nan_region* regions, int32_t n_regions, int32_t* flag, int32_t reset, void* stream) {
  using namespace vb;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!flag || n_regions < 0 || (n_regions > 0 && !regions) || (reset && n_regions))
    return set_error(VB_ERR_INVALID, "vb_nan_check: null flag, null table, negative count, or a reset with regions");
  cudaError_t e = cudaSuccess;
  if (reset) {
    e = launch_pdl(nan_flag_reset_kernel, dim3(1), dim3(32), (size_t)0, st, flag);
  } else if (n_regions) {
    int sms = sm_count();
    e = launch_pdl(nan_check_kernel, dim3((sms > 0 ? sms : 132) * 4), dim3(256), (size_t)0, st, regions, (int)n_regions, flag);
  }
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "vb_nan_check: %s", cudaGetErrorString(e));
  return VB_OK;
}
