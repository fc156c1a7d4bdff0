// Shared pieces of the tensor-core kernels (conv_tc.cu, conv_wgrad.cu): PTX wrappers, fast division, tensor-map encoders.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace sy {
namespace tc {

constexpr uint64_t kSpinLimit = 6000000000ull;  // ~3 s of SM clocks, then trap instead of hanging

// division by a runtime constant without the ~40-cycle integer divide (libdivide's branch-free u32 scheme);
// the per-tile coordinate decode sits on the critical path of every warp role
struct FastDiv {
  uint32_t mul, shr, d;
};
static inline FastDiv make_fastdiv(uint32_t d) {
  FastDiv f{0u, 0u, d};
  if (d > 1) {
    uint32_t s = 0;
    while ((1ull << s) < d) ++s;
    f.mul = (uint32_t)((((1ull << 32) * ((1ull << s) - d)) / d) + 1);
    f.shr = s - 1;
  }
  return f;
}
__device__ __forceinline__ int fdiv(int n, const FastDiv& f) {
  if (f.d == 1) return n;
  const uint32_t t = __umulhi((uint32_t)n, f.mul);
  return (int)((t + (((uint32_t)n - t) >> 1)) >> f.shr);
}

// ----------------------------------------------------------------------------- PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  long long t0 = 0;
  uint32_t spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) break;
    if ((++spins & 1023u) == 0) {
      long long now = clock64();
      if (t0 == 0) t0 = now;
      else if ((unsigned long long)(now - t0) > kSpinLimit) __trap();
    }
  }
}
// (Tried and rejected, round 2: polling with ONE lane per warp + __syncwarp instead of all 32 lanes -- 31.4 -> 36.0 us on the
// 3x3 256->256 layer: the wake-up after the phase flip gets slower, and nothing else gets faster.)
// one lane of a fully converged warp; keeps the surrounding control flow warp-uniform so that the
// compiler holds descriptors / addresses in uniform registers (no per-lane serialisation loops)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col-mode load: 128 consecutive output pixels' worth of input pixels (base pixel (w, h, n) in INPUT coordinates =
// -pad + out * stride, walked along w, then h, then n inside the tensor map's bounding box) shifted by the filter tap
__device__ __forceinline__ void tma_load_im2col_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int w,
                                                   int h, int n, uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// ---- wgmma (sm_90a warpgroup MMA): four consecutive warps (a warpgroup) issue together, the accumulators live in registers.
// Accumulator fragment of m64nNk16, thread t of the warpgroup: rows 16 (t / 32) + (t % 32) / 4 (+ 8), columns
// 8 j + 2 (t % 4) (+ 1) for j < N / 8 -> registers d[4 j + 0, 1] (row) and d[4 j + 2, 3] (row + 8).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// per-warpgroup register budget (the whole warpgroup executes it): producers hand registers to the MMA warpgroups
template <int R>
__device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// shared-memory matrix descriptor, 128B swizzle: start address, leading / stride byte offsets, swizzle phase of the start
__device__ __forceinline__ uint64_t make_gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t base_offset = 0) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);          // bits [0,14)
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16; // bits [16,30)
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32; // bits [32,46)
  d |= (uint64_t)(base_offset & 7u) << 49;           // bits [49,52)
  d |= (uint64_t)1 << 62;                            // SWIZZLE_128B
  return d;
}
// D[64 x N] (+)= A[64 x 16] * B[16 x N] from shared-memory descriptors, 16-bit inputs (bf16, or fp16 with F16), fp32
// accumulators in registers (sm_90a).  Both input types take the same descriptors and fragment layouts.
// TA / TB = 1: the operand is MN-major (transposed) in shared memory.
// SY_WGMMA_ASM(N, R, TY): the instruction for N columns (R accumulator registers) and input type TY; SY_WGMMA_ACC_R: the
// accumulator operand list
#define SY_WGMMA_ACC_32 \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
    "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
    "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
    "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define SY_WGMMA_ACC_64 \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
    "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
    "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
    "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
    "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
    "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
    "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
    "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define SY_WGMMA_ACC_128 \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
    "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
    "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
    "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
    "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
    "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
    "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
    "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), \
    "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
    "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
    "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
    "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), \
    "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
    "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
    "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
    "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
#define SY_WGMMA_ASM_64(TY) \
    "{\n\t.reg .pred p;\n\t" \
    "setp.ne.b32 p, %34, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " " \
    "{" \
    "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
    "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31" \
    "}, %32, %33, p, 1, 1, %35, %36;\n\t}"
#define SY_WGMMA_ASM_128(TY) \
    "{\n\t.reg .pred p;\n\t" \
    "setp.ne.b32 p, %66, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " " \
    "{" \
    "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
    "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
    "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
    "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63" \
    "}, %64, %65, p, 1, 1, %67, %68;\n\t}"
#define SY_WGMMA_ASM_256(TY) \
    "{\n\t.reg .pred p;\n\t" \
    "setp.ne.b32 p, %130, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " " \
    "{" \
    "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
    "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
    "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
    "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, " \
    "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
    "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, " \
    "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, " \
    "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127" \
    "}, %128, %129, p, 1, 1, %131, %132;\n\t}"
template <int N, int TA, int TB, bool F16 = false> struct Wgmma;
template <int TA, int TB, bool F16> struct Wgmma<64, TA, TB, F16> {
  __device__ __forceinline__ static void mma(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (F16)
      asm volatile(SY_WGMMA_ASM_64("f16") : SY_WGMMA_ACC_32 : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
    else
      asm volatile(SY_WGMMA_ASM_64("bf16") : SY_WGMMA_ACC_32 : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB, bool F16> struct Wgmma<128, TA, TB, F16> {
  __device__ __forceinline__ static void mma(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (F16)
      asm volatile(SY_WGMMA_ASM_128("f16") : SY_WGMMA_ACC_64 : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
    else
      asm volatile(SY_WGMMA_ASM_128("bf16") : SY_WGMMA_ACC_64 : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB, bool F16> struct Wgmma<256, TA, TB, F16> {
  __device__ __forceinline__ static void mma(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (F16)
      asm volatile(SY_WGMMA_ASM_256("f16") : SY_WGMMA_ACC_128 : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
    else
      asm volatile(SY_WGMMA_ASM_256("bf16") : SY_WGMMA_ACC_128 : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

static EncodeIm2colFn get_encode_im2col() {
  static EncodeIm2colFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeIm2colFn>(ptr);
  }
  return fn;
}

// ---- tensor maps of 16-bit tensors (bf16 by default, or `dt` = CU_TENSOR_MAP_DATA_TYPE_FLOAT16): 128B swizzle, 256-byte
// L2 promotion, out-of-bounds elements read as zero.  Both encoders need their driver entry point (get_encode /
// get_encode_im2col), which the caller checks first.

// an NHWC view as the 4-D tensor (C, W, H, N): dimension sizes and the byte strides of W, H, N
static void nhwc_dims(const SyTensor& t, cuuint64_t (&dims)[4], cuuint64_t (&strides)[3]) {
  dims[0] = (cuuint64_t)t.c; dims[1] = (cuuint64_t)t.w; dims[2] = (cuuint64_t)t.h; dims[3] = (cuuint64_t)t.n;
  strides[0] = (cuuint64_t)t.pitch * 2;
  strides[1] = (cuuint64_t)t.pitch * 2 * t.w;
  strides[2] = (cuuint64_t)t.pitch * 2 * t.w * t.h;
}

// tiled map of a rank-`rank` tensor (innermost dimension first), box `box`, unit element strides
static CUresult encode_tiled(CUtensorMap* map, cuuint32_t rank, const void* ptr, const cuuint64_t* dims,
                                  const cuuint64_t* strides, const cuuint32_t* box,
                                  CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return get_encode()(map, dt, rank, const_cast<void*>(ptr), dims, strides, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// im2col map of the input view x of a kh x kw convolution (padding (k - 1) / 2, stride `stride`): the bounding box of
// base pixels is [-pad, dim + pad - (k - 1)) per spatial dim, walked with the stride; one load brings `pixels`
// consecutive base pixels x 64 channels (one 128-byte swizzle row), shifted by the filter tap
static CUresult encode_im2col_nhwc(CUtensorMap* map, const SyTensor& x, int kh, int kw, int stride, int pixels,
                                   CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
  cuuint64_t dims[4], strides[3];
  nhwc_dims(x, dims, strides);
  const int ph = (kh - 1) / 2, pw = (kw - 1) / 2;
  int lower[2] = {-pw, -ph};                                   // {W, H}
  int upper[2] = {pw - (kw - 1), ph - (kh - 1)};
  const cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  return get_encode_im2col()(map, dt, 4, x.ptr, dims, strides, lower, upper, 64,
                             (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

static int num_sms() { return sm_count(); }

}  // namespace tc
}  // namespace sy
