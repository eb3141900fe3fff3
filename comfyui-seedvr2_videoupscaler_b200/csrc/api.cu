// C-ABI housekeeping: error channel, version, device check.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include "svr2_internal.h"

namespace svr2 {
static thread_local char g_err[512] = "";
int set_error(int code, const char* msg) {
  snprintf(g_err, sizeof g_err, "%s", msg ? msg : "");
  return code;
}
}  // namespace svr2

extern "C" const char* svr2_last_error(void) { return svr2::g_err; }
extern "C" int svr2_version(void) { return 100; }

extern "C" int svr2_device_check(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return svr2::set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) return svr2::set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  if (prop.major != 9) return svr2::set_error(SVR2_ERR_ARCH, "libsvr2 requires an sm_90 (H100) device");
  return SVR2_OK;
}
