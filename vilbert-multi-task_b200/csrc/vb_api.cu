// vb_api.cu — error reporting, version and device queries of the C ABI (include/vilbert_b200.h).
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include "vb_internal.h"

namespace vb {
static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("VB_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
  if (!cached[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    cached[dev] = n;
  }
  return cached[dev];
}
}  // namespace vb

extern "C" int vb_version(void) { return 4; }

extern "C" const char* vb_last_error(void) { return vb::g_err; }

extern "C" vb_status vb_device_info(int* sm_count_out, int* cc_out) {
  static int cc_cached[64] = {0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return vb::set_error(VB_ERR_CUDA, "cudaGetDevice: %s", cudaGetErrorString(e));
  if (dev < 0 || dev >= 64) return vb::set_error(VB_ERR_INVALID, "device index %d out of range", dev);
  if (!cc_cached[dev]) {
    int major = 0, minor = 0;
    e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
    if (e != cudaSuccess) return vb::set_error(VB_ERR_CUDA, "cudaDeviceGetAttribute: %s", cudaGetErrorString(e));
    cc_cached[dev] = major * 10 + minor;
  }
  const int n = vb::sm_count();
  if (n <= 0) return vb::set_error(VB_ERR_CUDA, "could not query the SM count");
  if (sm_count_out) *sm_count_out = n;
  if (cc_out) *cc_out = cc_cached[dev];
  return VB_OK;
}
