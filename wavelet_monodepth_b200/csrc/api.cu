// Library-level entry points and shared host state of libwmd.
#include "common.cuh"

namespace wmd {
thread_local int g_last_cuda_error = 0;
thread_local long long g_launches = 0;

int sm_count() {
  static int cached[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}
}  // namespace wmd

extern "C" int wmd_version(void) { return WMD_VERSION; }

extern "C" const char* wmd_status_string(int status) {
  switch (status) {
    case WMD_OK: return "ok";
    case WMD_ERR_ARG: return "invalid argument (null pointer or bad enum)";
    case WMD_ERR_SHAPE: return "unsupported shape or alignment";
    case WMD_ERR_CUDA: return "CUDA error (see wmd_last_cuda_error)";
    case WMD_ERR_WORKSPACE: return "workspace too small";
    case WMD_ERR_UNSUPPORTED: return "unsupported configuration";
    default: return "unknown status";
  }
}

extern "C" int wmd_last_cuda_error(void) { return wmd::g_last_cuda_error; }
extern "C" long long wmd_launch_count(void) { return wmd::g_launches; }
