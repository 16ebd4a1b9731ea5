// C-ABI plumbing shared by all translation units: error string, version, device queries.
#include <stdarg.h>

#include "common.cuh"

static thread_local char g_err[512] = "";

void coda_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int coda_sm_count() {
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev != cached_dev) {
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 132;
    cached = p.multiProcessorCount;
    cached_dev = dev;
  }
  return cached;
}

extern "C" const char* coda_b200_last_error(void) { return g_err; }
extern "C" int coda_b200_version(void) { return CODA_B200_VERSION; }
extern "C" int coda_b200_sm_count(void) { return coda_sm_count(); }

extern "C" int coda_b200_device_check(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    coda_set_error("no CUDA device: %s", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    return CODA_B200_ECUDA;
  }
  int dev = 0;
  CODA_CUDA_OK(cudaGetDevice(&dev));
  cudaDeviceProp p;
  CODA_CUDA_OK(cudaGetDeviceProperties(&p, dev));
  if (p.major != 9 || p.minor != 0) {
    coda_set_error("device %d is sm_%d%d; this library is built for sm_90a only", dev, p.major, p.minor);
    return CODA_B200_ECUDA;
  }
  return CODA_B200_OK;
}

extern "C" int coda_b200_set_l2_fetch_granularity(int bytes) {
  CODA_CHECK_ARG(bytes == 32 || bytes == 64 || bytes == 128, "l2 fetch granularity must be 32, 64 or 128");
  CODA_CUDA_OK(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)bytes));
  return CODA_B200_OK;
}
