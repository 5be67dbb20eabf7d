// Library-wide state: error string, device properties, ABI version.
#include "common.cuh"
#include "gspb200.h"

namespace gsp {

char* error_buffer() {
  static thread_local char buf[512] = {0};
  return buf;
}

static unsigned long long g_launches = 0;
void note_launch(int n) { __atomic_fetch_add(&g_launches, (unsigned long long)n, __ATOMIC_RELAXED); }
unsigned long long launches() { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0)
      v = 132;
    cached[dev] = v;
  }
  return cached[dev];
}

}  // namespace gsp

extern "C" {

int gsp_abi_version(void) { return GSPB200_ABI_VERSION; }

const char* gsp_last_error(void) { return gsp::error_buffer(); }

uint64_t gsp_launch_count(void) { return gsp::launches(); }

int gsp_device_info(int* sm_count, int* cc_major, int* cc_minor, int64_t* l2_bytes) {
  int dev = 0;
  GSP_CUDA(cudaGetDevice(&dev));
  int v = 0;
  GSP_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
  if (sm_count) *sm_count = v;
  GSP_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev));
  if (cc_major) *cc_major = v;
  GSP_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev));
  if (cc_minor) *cc_minor = v;
  GSP_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, dev));
  if (l2_bytes) *l2_bytes = v;
  return GSP_OK;
}

}  // extern "C"
