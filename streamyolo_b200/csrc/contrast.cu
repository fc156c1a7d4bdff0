// sy_splice_frames: the split screen of the sAP toolkit's vis_contrast.py (sAP/vis/vis_contrast.py:148-165) on pairs
// of frames in slots: frame B past a split line over frame A, written into A in place, with a coloured band at the split.
#include "common.cuh"

namespace sy {

// One thread per run of 16 pixels (48 bytes) of a row of A.  Each pixel is the band colour where its coordinate along
// the split axis lies in [band_start, band_end), B's pixel where it is >= split, and A's otherwise.  A whole, 16-byte
// aligned run of B's pixels or of the band is three 16-byte stores (after three 16-byte loads of B); a run of A's pixels
// is not touched; a run that straddles a boundary or the frame's right edge, or a misaligned one, goes pixel by pixel.
constexpr int kSpliceRun = 16, kSpliceX = 32, kSpliceY = 4;

__device__ __forceinline__ int splice_kind(int c, int split, int band_start, int band_end) {
  return c >= band_start && c < band_end ? 2 : (c >= split ? 1 : 0);    // 2 band, 1 B, 0 A
}

__global__ void __launch_bounds__(kSpliceX * kSpliceY) splice_frames_kernel(
    uint8_t* __restrict__ a, const uint8_t* __restrict__ b, const int32_t* __restrict__ sizes,
    const int32_t* __restrict__ splits, int max_h, int max_w, int horizontal, uint32_t c0, uint32_t c1, uint32_t c2) {
  const int img = blockIdx.z;
  const int y = blockIdx.y * kSpliceY + threadIdx.y;
  const int x0 = (blockIdx.x * kSpliceX + threadIdx.x) * kSpliceRun;
  const int h = sizes[2 * img], w = sizes[2 * img + 1];
  if (h < 1 || w < 1 || h > max_h || w > max_w || y >= h || x0 >= w) return;
  const int split = splits[3 * img], band_start = splits[3 * img + 1], band_end = splits[3 * img + 2];
  const int np = min(kSpliceRun, w - x0);
  int first = splice_kind(horizontal ? y : x0, split, band_start, band_end);
  bool uniform = true;
  if (!horizontal)
    for (int p = 1; p < np; ++p) uniform &= splice_kind(x0 + p, split, band_start, band_end) == first;
  if (uniform && first == 0) return;                      // A's pixels stay
  const long long at = (((long long)img * max_h + y) * max_w + x0) * 3;
  uint8_t* q = a + at;
  const uint8_t* r = b + at;
  // the band colour over 12 bytes (4 pixels): B G R B | G R B G | R B G R, as little-endian words
  const uint32_t band[3] = {c0 | c1 << 8 | c2 << 16 | c0 << 24, c1 | c2 << 8 | c0 << 16 | c1 << 24,
                            c2 | c0 << 8 | c1 << 16 | c2 << 24};
  // B's run is at the same offset as A's, but B need not start where A does modulo 16 (a view into a larger buffer)
  const uintptr_t align = reinterpret_cast<uintptr_t>(q) | (first == 1 ? reinterpret_cast<uintptr_t>(r) : 0);
  if (uniform && np == kSpliceRun && (align & 15) == 0) {
    uint4* d = reinterpret_cast<uint4*>(q);
    if (first == 1) {
      const uint4* s = reinterpret_cast<const uint4*>(r);
#pragma unroll
      for (int k = 0; k < 3; ++k) d[k] = __ldg(s + k);
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) d[k] = make_uint4(band[k % 3], band[(k + 1) % 3], band[(k + 2) % 3], band[k % 3]);
    }
    return;
  }
  const uint8_t col[3] = {(uint8_t)c0, (uint8_t)c1, (uint8_t)c2};
  for (int p = 0; p < np; ++p) {
    const int kind = horizontal ? first : splice_kind(x0 + p, split, band_start, band_end);
    if (kind == 0) continue;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) q[3 * p + ch] = kind == 2 ? col[ch] : __ldg(r + 3 * p + ch);
  }
}

}  // namespace sy

using namespace sy;

extern "C" int sy_splice_frames(const SySpliceFramesDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->a != nullptr && d->b != nullptr && d->sizes != nullptr && d->splits != nullptr,
             SY_EINVAL, "splice_frames: null pointer");
  SY_REQUIRE(d->a != d->b, SY_EINVAL, "splice_frames: a and b must be different buffers");
  SY_REQUIRE(d->n >= 1 && d->n <= 65535 && d->max_h >= 1 && d->max_h <= 65535 && d->max_w >= 1 && d->max_w <= 65535,
             SY_EINVAL, "splice_frames: bad slots (n %d, slot %dx%d)", d->n, d->max_h, d->max_w);
  SY_REQUIRE(d->horizontal == 0 || d->horizontal == 1, SY_EINVAL, "splice_frames: horizontal = %d, not 0 or 1",
             d->horizontal);
  const dim3 block(kSpliceX, kSpliceY);
  const dim3 grid(cdiv(cdiv(d->max_w, kSpliceRun), kSpliceX), cdiv(d->max_h, kSpliceY), d->n);
  splice_frames_kernel<<<grid, block, 0, stream>>>(d->a, d->b, d->sizes, d->splits, d->max_h, d->max_w, d->horizontal,
                                                   d->color[0], d->color[1], d->color[2]);
  return launch_status("splice_frames_kernel");
}
