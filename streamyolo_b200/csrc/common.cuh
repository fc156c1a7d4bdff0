// Shared helpers for libstreamyolo_sm100.so (built for sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/streamyolo_sm100.h"

namespace sy {

// thread-local last error text (sy_last_error_string)
void set_error(const char* fmt, ...);

#define SY_REQUIRE(cond, code, ...)      \
  do {                                   \
    if (!(cond)) {                       \
      ::sy::set_error(__VA_ARGS__);      \
      return (code);                     \
    }                                    \
  } while (0)

#define SY_CUDA(expr)                                                                   \
  do {                                                                                  \
    cudaError_t e__ = (expr);                                                           \
    if (e__ != cudaSuccess) {                                                           \
      ::sy::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, \
                      __LINE__);                                                        \
      return SY_ELAUNCH;                                                                \
    }                                                                                   \
  } while (0)

inline int launch_status(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("launch of %s failed: %s", what, cudaGetErrorString(e));
    return SY_ELAUNCH;
  }
  return SY_OK;
}

inline bool view_ok(const SyTensor& t) {
  return t.ptr != nullptr && t.n > 0 && t.h > 0 && t.w > 0 && t.c > 0 && t.pitch >= t.c &&
         (t.c % 8) == 0 && (t.pitch % 8) == 0 && ((uintptr_t)t.ptr % 16) == 0;
}

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// SM count of the current device (cached; 132 = an H100 SXM when there is no device, for host-only queries).  Grid-stride
// kernels cap their grids at a few waves of it.
inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      n = 132;
    }
  }
  return n;
}

// ---- programmatic dependent launch (PDL) -------------------------------------------------
// Kernels launched through launch_pdl() may be scheduled while their predecessor on the stream is still
// draining: they call pdl_launch_dependents() first thing (lets the *next* kernel do the same) and pdl_wait()
// before their first access to global memory (returns once every prerequisite grid has completed and its
// writes are visible).  Both are no-ops for a normally launched grid.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---- bf16 pack helpers -------------------------------------------------------
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 p = __floats2bfloat162_rn(a, b);  // .x = a (low half), .y = b
  return *reinterpret_cast<uint32_t*>(&p);
}

// ---- fp16 pack helpers (SY_STORAGE_F16: the eval / streaming forwards with IEEE half activations) ----------------
__device__ __forceinline__ float f16_lo(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v & 0xffffu))); }
__device__ __forceinline__ float f16_hi(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v >> 16))); }
__device__ __forceinline__ uint32_t pack_f16(float a, float b) {
  __half2 p = __floats2half2_rn(a, b);             // .x = a (low half), .y = b
  return *reinterpret_cast<uint32_t*>(&p);
}
// the 16-bit activation storage type as a template flag: F16 = IEEE half, otherwise bf16
template <bool F16>
__device__ __forceinline__ float st_lo(uint32_t v) {
  if constexpr (F16) return f16_lo(v); else return bf16_lo(v);
}
template <bool F16>
__device__ __forceinline__ float st_hi(uint32_t v) {
  if constexpr (F16) return f16_hi(v); else return bf16_hi(v);
}
template <bool F16>
__device__ __forceinline__ uint32_t st_pack(float a, float b) {
  if constexpr (F16) return pack_f16(a, b); else return pack_bf16(a, b);
}
// eight 16-bit values of one 16-byte chunk as floats
template <bool F16>
__device__ __forceinline__ void st_unpack8(const uint4& u, float (&v)[8]) {
  v[0] = st_lo<F16>(u.x); v[1] = st_hi<F16>(u.x); v[2] = st_lo<F16>(u.y); v[3] = st_hi<F16>(u.y);
  v[4] = st_lo<F16>(u.z); v[5] = st_hi<F16>(u.z); v[6] = st_lo<F16>(u.w); v[7] = st_hi<F16>(u.w);
}

// SiLU = v * rcp(1 + 2^(-v * log2 e)) on the two approximate SFU ops (ex2.approx, rcp.approx: ~2 ulp fp32, far below
// the bf16 output rounding) = 5 instructions per value; the normalise pass is issue-bound otherwise (a correctly
// rounded divide costs ~10 instructions, div.approx adds range fix-ups).  v << 0: 2^x overflows to +inf, rcp(inf) = 0,
// the product is -0, the correct limit.
__device__ __forceinline__ float silu_f(float v) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return v * r;
}
// silu'(z) = s (1 + z (1 - s)), s = sigmoid(z) on the approximate SFU ops (ex2 / rcp, ~2 ulp fp32; the result is stored as bf16)
__device__ __forceinline__ float dsilu(float z) {
  float e, s;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(z * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(s) : "f"(1.0f + e));
  return s * (1.0f + z * (1.0f - s));
}

constexpr float kLreluSlope = 0.1f;     // nn.LeakyReLU(0.1), what [yolox] get_activation("lrelu") builds

// act(v) for an SY_ACT_* code.  ReLU / LeakyReLU are PyTorch's expressions (v > 0 ? v : 0 / v * 0.1f): -0 and NaN map like
// theirs.  A compile-time code folds to one branch; a run-time one (the FUSED epilogues) is a short select chain in front
// of the unchanged SiLU.
__device__ __forceinline__ float act_f(int code, float v) {
  if (code == SY_ACT_SILU) return silu_f(v);
  if (code == SY_ACT_RELU) return v > 0.f ? v : 0.f;
  if (code == SY_ACT_LRELU) return v > 0.f ? v : v * kLreluSlope;
  return v;
}
// d act / dz at the pre-activation z, autograd's convention at z = 0: 0 for ReLU, 0.1 for LeakyReLU
__device__ __forceinline__ float dact_f(int code, float z) {
  if (code == SY_ACT_SILU) return dsilu(z);
  if (code == SY_ACT_RELU) return z > 0.f ? 1.f : 0.f;
  if (code == SY_ACT_LRELU) return z > 0.f ? 1.f : kLreluSlope;
  return 1.f;
}
inline bool act_ok(int code) { return code >= SY_ACT_NONE && code <= SY_ACT_LRELU; }

}  // namespace sy
