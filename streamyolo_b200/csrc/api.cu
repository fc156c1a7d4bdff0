// Runtime entry points: error text, version, device check.
#include <stdarg.h>

#include "common.cuh"

namespace sy {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace sy

extern "C" const char* sy_last_error_string(void) { return sy::g_err; }
extern "C" int sy_version(void) { return 101; }

extern "C" int sy_check_device(void) {
  int dev = 0;
  SY_CUDA(cudaGetDevice(&dev));
  int major = 0, minor = 0;
  SY_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  SY_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  SY_REQUIRE(major == 9 && minor == 0, SY_EARCH, "device %d is sm_%d%d; libstreamyolo needs sm_90 (H100)", dev, major,
             minor);
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  SY_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres));
  SY_REQUIRE(qres == cudaDriverEntryPointSuccess && ptr != nullptr, SY_EARCH, "driver lacks cuTensorMapEncodeTiled");
  return SY_OK;
}
