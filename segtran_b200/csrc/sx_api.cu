// C-ABI glue: version, thread-local error string, device info.
#include <stdarg.h>
#include <string.h>

#include "sx_common.cuh"

static thread_local char g_err[1024] = "";

void sx_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" int sx_version(void) { return SX_VERSION; }

extern "C" const char* sx_last_error(void) { return g_err; }

extern "C" int sx_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  SX_CHECK_CUDA(cudaGetDevice(&dev));
  int n = 0, ma = 0, mi = 0;
  SX_CHECK_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  SX_CHECK_CUDA(cudaDeviceGetAttribute(&ma, cudaDevAttrComputeCapabilityMajor, dev));
  SX_CHECK_CUDA(cudaDeviceGetAttribute(&mi, cudaDevAttrComputeCapabilityMinor, dev));
  if (sm_count) *sm_count = n;
  if (cc_major) *cc_major = ma;
  if (cc_minor) *cc_minor = mi;
  SX_REQUIRE(ma == 9 && mi == 0, "segtran_b200 needs an sm_90 (H100) device, found sm_%d%d", ma, mi);
  return 0;
}
