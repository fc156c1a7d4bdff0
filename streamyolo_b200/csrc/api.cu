// Runtime entry points: error text, version, device check.
#include <stdarg.h>
#include <stdlib.h>

#include "common.cuh"

namespace sy {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
// read on every launch (a getenv is ~100 ns) so that a process can switch it between two measurements
bool pdl_enabled() {
  const char* e = getenv("SY_PDL");
  return !(e != nullptr && e[0] == '0');
}
}  // namespace sy

extern "C" const char* sy_last_error_string(void) { return sy::g_err; }
extern "C" int sy_version(void) { return 100; }

// L2 residency of the conv -> normalise hand-off: the raw conv output of a train-mode BaseConv is written by one kernel and
// read back by the next (the BatchNorm statistics sit in between).  All layers whose raw tensor fits draw it from ONE arena;
// marking that address window "persisting" on the launching stream keeps those lines in the set-aside part of the 50 MB L2,
// so the normalise pass reads them from L2 and the next layer overwrites them before they are ever written back to HBM.
// The set-aside is taken from every other kernel's share of L2: on an H100 (at most 32.8 MB of 50 MB persisting) the step is
// faster without it, and the engine only asks for a window when SY_RAW_ARENA_MB is set (model/engine.py).
// Returns the usable window size in *granted (0: the device grants no persisting L2).  bytes = 0 clears the window.
extern "C" int sy_l2_persist_window(void* ptr, size_t bytes, float hit_ratio, size_t* granted, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int dev = 0, max_persist = 0, max_window = 0;
  SY_CUDA(cudaGetDevice(&dev));
  SY_CUDA(cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev));
  SY_CUDA(cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev));
  size_t want = bytes;
  if (want > (size_t)max_persist) want = (size_t)max_persist;
  if (want > (size_t)max_window) want = (size_t)max_window;
  if (granted) *granted = want;
  cudaStreamAttrValue v = {};
  if (bytes == 0 || want == 0) {
    v.accessPolicyWindow.base_ptr = nullptr;
    v.accessPolicyWindow.num_bytes = 0;
    v.accessPolicyWindow.hitRatio = 0.f;
    v.accessPolicyWindow.hitProp = cudaAccessPropertyNormal;
    v.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
    SY_CUDA(cudaStreamSetAttribute(stream, cudaStreamAttributeAccessPolicyWindow, &v));
    return SY_OK;
  }
  SY_CUDA(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want));
  v.accessPolicyWindow.base_ptr = ptr;
  v.accessPolicyWindow.num_bytes = want;
  v.accessPolicyWindow.hitRatio = hit_ratio;
  v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
  v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
  SY_CUDA(cudaStreamSetAttribute(stream, cudaStreamAttributeAccessPolicyWindow, &v));
  return SY_OK;
}

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
