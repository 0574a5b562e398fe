// Error reporting, version and device queries of the C ABI (include/nsr_b200.h).
#include "common.cuh"
#include <stdarg.h>

static thread_local char g_err[512] = "";

void nsr_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// launch-shape fallback when the device query fails: the SM count of an H100 SXM (the launch itself then reports the error)
constexpr int kFallbackSms = 132;

int nsr_sm_count() {
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return kFallbackSms;
  if (dev != cached_dev) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kFallbackSms;
    cached = n;
    cached_dev = dev;
  }
  return cached;
}

extern "C" const char* nsr_last_error(void) { return g_err; }
extern "C" int nsr_version(void) { return NSR_VERSION; }
extern "C" int nsr_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    nsr_set_error("nsr_device_info: %s", cudaGetErrorString(e));
    return 2;
  }
  cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev);
  return 0;
}
