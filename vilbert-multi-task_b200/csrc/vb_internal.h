// Internal helpers shared by the translation units of libvilbert_b200.so.
#pragma once
#include <cuda_runtime.h>

#include "../../include/vilbert_b200.h"

namespace vb {
// Records a printf-style message for vb_last_error() and returns `code`.
int set_error(int code, const char* fmt, ...);
inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(VB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return VB_OK;
}
int sm_count();
// dst[i] += part[0 * stride + i] + part[1 * stride + i] + ... (slices terms, in slice order): the ordered sum of deterministic plans
int launch_reduce_slices(const float* part, long long stride, int slices, long long n, float* dst, cudaStream_t stream);

// Programmatic dependent launch (PDL): every kernel of the library starts with `griddepcontrol.wait` (all global
// traffic happens after it) followed by `griddepcontrol.launch_dependents`, and is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization so that launch processing, CTA scheduling and per-CTA setup
// (barrier init, tensor-map prefetch) of kernel N+1 overlap the tail of kernel N — also inside
// captured CUDA graphs. VB_PDL=0 in the environment restores plain stream serialization.
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
}  // namespace vb
