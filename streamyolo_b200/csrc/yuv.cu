// sy_yuv_to_bgr_sized: raw camera frames (NV12, NV21, I420, YV12, YUYV, UYVY) -> uint8 BGR slots, bit-identical to
// cv2.cvtColor(frame, COLOR_YUV2BGR_*) (OpenCV's BT.601 fixed-point formula, chroma replicated over its 2x2 or 2x1 group).
// One thread converts a run of 16 columns: the two rows of eight 2x2 groups (4:2:0) or one row of eight 2x1 groups (4:2:2).
// A run that is whole and 16-byte aligned is read with 16-byte loads (8-byte ones for I420's half-width chroma rows) and
// written with 16-byte stores; the last run of a row narrower than 16, or a misaligned one, goes byte by byte and reads
// nothing past the row's end, so nothing past the frame's own bytes is read.
#include "common.cuh"

namespace sy {

constexpr int kRun = 16;   // columns per thread

// ITUR_BT_601_* of OpenCV's color_yuv: 20-bit fixed point
constexpr int kCY = 1220542, kCUB = 2116026, kCUG = -409993, kCVG = -852492, kCVR = 1673527, kShift = 20;

__device__ __forceinline__ uint32_t byte_at(const uint32_t* w, int k) { return (w[k >> 2] >> (8 * (k & 3))) & 255u; }

// N bytes (N = 16 or 8) from p into words w; only the first n are read (the rest are zero)
template <int N>
__device__ __forceinline__ void load_run(uint32_t (&w)[N / 4], const uint8_t* __restrict__ p, int n) {
  if (n == N && (reinterpret_cast<uintptr_t>(p) & (N - 1)) == 0) {
    if constexpr (N == 16) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
      w[0] = v.x, w[1] = v.y, w[2] = v.z, w[3] = v.w;
    } else {
      const uint2 v = __ldg(reinterpret_cast<const uint2*>(p));
      w[0] = v.x, w[1] = v.y;
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < N / 4; ++i) w[i] = 0;
#pragma unroll
  for (int k = 0; k < N; ++k)
    if (k < n) w[k >> 2] |= (uint32_t)__ldg(p + k) << (8 * (k & 3));
}

// the first 3 * n bytes of words o to q
__device__ __forceinline__ void store_run(uint8_t* __restrict__ q, const uint32_t (&o)[12], int n) {
  if (n == kRun && (reinterpret_cast<uintptr_t>(q) & 15) == 0) {
    uint4* d = reinterpret_cast<uint4*>(q);
    d[0] = make_uint4(o[0], o[1], o[2], o[3]);
    d[1] = make_uint4(o[4], o[5], o[6], o[7]);
    d[2] = make_uint4(o[8], o[9], o[10], o[11]);
    return;
  }
#pragma unroll
  for (int k = 0; k < 3 * kRun; ++k)
    if (k < 3 * n) q[k] = (uint8_t)byte_at(o, k);
}

__device__ __forceinline__ uint32_t clip_shift(int x) { return (uint32_t)min(max(x >> kShift, 0), 255); }

// one row of a run: luma bytes y[0..15], chroma of group g = (u[g], v[g]) -> BGR bytes o[0..47]
__device__ __forceinline__ void convert_row(const uint32_t (&y)[4], const uint32_t (&u)[2], const uint32_t (&v)[2],
                                            uint32_t (&o)[12]) {
#pragma unroll
  for (int i = 0; i < 12; ++i) o[i] = 0;
#pragma unroll
  for (int g = 0; g < kRun / 2; ++g) {
    const int cu = (int)byte_at(u, g) - 128, cv = (int)byte_at(v, g) - 128;
    const int ruv = (1 << (kShift - 1)) + kCVR * cv;
    const int guv = (1 << (kShift - 1)) + kCVG * cv + kCUG * cu;
    const int buv = (1 << (kShift - 1)) + kCUB * cu;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = 2 * g + j;
      const int yy = max((int)byte_at(y, k) - 16, 0) * kCY;
      const uint32_t px[3] = {clip_shift(yy + buv), clip_shift(yy + guv), clip_shift(yy + ruv)};
#pragma unroll
      for (int c = 0; c < 3; ++c) o[(3 * k + c) >> 2] |= px[c] << (8 * ((3 * k + c) & 3));
    }
  }
}

// blockIdx.z = frame, (x, y) = (16-column run, row pair or row) of the slot grid; frames smaller than the slot exit early
template <int FMT>
__global__ void __launch_bounds__(128) yuv_to_bgr_sized_kernel(const uint8_t* __restrict__ src, long long max_bytes,
                                                               const int32_t* __restrict__ sizes, int slot_h, int slot_w,
                                                               uint8_t* __restrict__ out) {
  constexpr bool k420 = FMT <= SY_YUV_YV12;
  const int k = blockIdx.z;
  const int h = sizes[2 * k], w = sizes[2 * k + 1];
  const long long bytes = k420 ? (long long)h * w * 3 / 2 : (long long)h * w * 2;
  if (h < 1 || w < 1 || h > slot_h || w > slot_w || (w & 1) || (k420 && (h & 1)) || bytes > max_bytes) return;
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * kRun, r = blockIdx.y * blockDim.y + threadIdx.y;
  if (x0 >= w || r >= (k420 ? h / 2 : h)) return;
  const int n = min(kRun, w - x0);
  const uint8_t* f = src + max_bytes * k;
  uint8_t* o_img = out + (long long)slot_h * slot_w * 3 * k;
  uint32_t y[4], u[2], v[2], o[12];
  if constexpr (k420) {
    const long long plane = (long long)h * w;
    if constexpr (FMT == SY_YUV_NV12 || FMT == SY_YUV_NV21) {
      uint32_t c[4];                                   // n bytes of interleaved chroma: n / 2 pairs
      load_run<16>(c, f + plane + (long long)r * w + x0, n);
      u[0] = u[1] = v[0] = v[1] = 0;
#pragma unroll
      for (int g = 0; g < kRun / 2; ++g) {
        const uint32_t a = byte_at(c, 2 * g), b = byte_at(c, 2 * g + 1);
        u[g >> 2] |= (FMT == SY_YUV_NV12 ? a : b) << (8 * (g & 3));
        v[g >> 2] |= (FMT == SY_YUV_NV12 ? b : a) << (8 * (g & 3));
      }
    } else {
      const long long quarter = (long long)(h / 2) * (w / 2), off = (long long)r * (w / 2) + x0 / 2;
      const uint8_t* pu = f + plane + (FMT == SY_YUV_I420 ? 0 : quarter) + off;
      const uint8_t* pv = f + plane + (FMT == SY_YUV_I420 ? quarter : 0) + off;
      load_run<8>(u, pu, n / 2);
      load_run<8>(v, pv, n / 2);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int row = 2 * r + j;
      load_run<16>(y, f + (long long)row * w + x0, n);
      convert_row(y, u, v, o);
      store_run(o_img + ((long long)row * slot_w + x0) * 3, o, n);
    }
  } else {
    uint32_t p0[4], p1[4];                             // 2n bytes: n / 2 groups of four, 16 in each half
    const uint8_t* q = f + (long long)r * w * 2 + 2 * x0;
    load_run<16>(p0, q, min(2 * n, 16));
    load_run<16>(p1, q + 16, max(2 * n - 16, 0));
    y[0] = y[1] = y[2] = y[3] = u[0] = u[1] = v[0] = v[1] = 0;
    constexpr int oy = FMT == SY_YUV_YUY2 ? 0 : 1, ou = FMT == SY_YUV_YUY2 ? 1 : 0;
#pragma unroll
    for (int g = 0; g < kRun / 2; ++g) {
      const uint32_t* p = g < 4 ? p0 : p1;
      const int b = 4 * (g & 3);
      y[(2 * g) >> 2] |= byte_at(p, b + oy) << (8 * ((2 * g) & 3));
      y[(2 * g + 1) >> 2] |= byte_at(p, b + oy + 2) << (8 * ((2 * g + 1) & 3));
      u[g >> 2] |= byte_at(p, b + ou) << (8 * (g & 3));
      v[g >> 2] |= byte_at(p, b + ou + 2) << (8 * (g & 3));
    }
    convert_row(y, u, v, o);
    store_run(o_img + ((long long)r * slot_w + x0) * 3, o, n);
  }
}

}  // namespace sy

using namespace sy;

extern "C" int sy_yuv_to_bgr_sized(const SyYuvToBgrSizedDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->src != nullptr && d->sizes != nullptr && d->out != nullptr, SY_EINVAL,
             "yuv_to_bgr_sized: null pointer");
  SY_REQUIRE(d->format >= SY_YUV_NV12 && d->format <= SY_YUV_UYVY, SY_EINVAL, "yuv_to_bgr_sized: unknown format %d",
             d->format);
  SY_REQUIRE(d->n > 0 && d->n <= 65535 && d->max_bytes > 0 && d->slot_h > 0 && d->slot_h <= 65535 && d->slot_w > 0,
             SY_EINVAL, "yuv_to_bgr_sized: bad sizes (n %d, max_bytes %lld, slot %dx%d)", d->n, (long long)d->max_bytes,
             d->slot_h, d->slot_w);
  const dim3 block(32, 4);
  const int rows = d->format <= SY_YUV_YV12 ? d->slot_h / 2 : d->slot_h;
  if (rows == 0) return SY_OK;                       // a one-row slot holds no 4:2:0 frame
  const dim3 grid(cdiv(cdiv(d->slot_w, kRun), 32), cdiv(rows, 4), d->n);
  decltype(&yuv_to_bgr_sized_kernel<0>) k = nullptr;
  switch (d->format) {
    case SY_YUV_NV12: k = yuv_to_bgr_sized_kernel<SY_YUV_NV12>; break;
    case SY_YUV_NV21: k = yuv_to_bgr_sized_kernel<SY_YUV_NV21>; break;
    case SY_YUV_I420: k = yuv_to_bgr_sized_kernel<SY_YUV_I420>; break;
    case SY_YUV_YV12: k = yuv_to_bgr_sized_kernel<SY_YUV_YV12>; break;
    case SY_YUV_YUY2: k = yuv_to_bgr_sized_kernel<SY_YUV_YUY2>; break;
    default: k = yuv_to_bgr_sized_kernel<SY_YUV_UYVY>; break;
  }
  k<<<grid, block, 0, stream>>>(d->src, d->max_bytes, d->sizes, d->slot_h, d->slot_w, d->out);
  return launch_status("yuv_to_bgr_sized_kernel");
}
