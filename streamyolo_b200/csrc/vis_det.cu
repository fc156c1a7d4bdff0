// sy_draw_outlines: the drawing of the sAP toolkit's vis_det (sAP/det/__init__.py:152-174, masks None): 1-pixel
// rectangles (cv2.rectangle thickness 1) and a list of pixels (the label strokes the host rasterised with cv2.putText), all
// in one colour, in place.  One warp per box walks its four clipped edges; one thread per listed pixel.  Every write stores
// the same colour, so overlapping writes need no ordering and the result does not depend on scheduling.
#include "common.cuh"

namespace sy {

constexpr int kThreads = 256;
constexpr int kBoxesPerCta = kThreads / 32;

__device__ __forceinline__ void put_px(uint8_t* img, int max_w, int y, int x, uchar3 c) {
  uint8_t* p = img + ((long long)y * max_w + x) * 3;
  p[0] = c.x, p[1] = c.y, p[2] = c.z;
}

// blockIdx.y = image.  Blocks [0, box_ctas) take kBoxesPerCta boxes each, a warp per box; the rest take kThreads listed
// pixels each.
__global__ void __launch_bounds__(kThreads) draw_outlines_kernel(
    uint8_t* img, const int32_t* __restrict__ sizes, int max_h, int max_w, const int4* __restrict__ boxes,
    const int32_t* __restrict__ counts, int K, const int32_t* __restrict__ points, const int32_t* __restrict__ n_points,
    int M, int box_ctas, uchar3 c) {
  const int i = blockIdx.y;
  const int h = sizes[2 * i], w = sizes[2 * i + 1];
  if (h < 1 || w < 1 || h > max_h || w > max_w) return;
  uint8_t* im = img + (long long)i * max_h * max_w * 3;
  if ((int)blockIdx.x < box_ctas) {
    const int j = blockIdx.x * kBoxesPerCta + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (j >= min(max(counts[i], 0), K)) return;
    const int4 v = boxes[(long long)i * K + j];
    const int x1 = min(v.x, v.z), x2 = max(v.x, v.z), y1 = min(v.y, v.w), y2 = max(v.y, v.w);
    // clipped spans; a line of cv2's LINE_8 between two points on a row or column is every pixel between them
    const int cx1 = max(x1, 0), cx2 = min(x2, w - 1), cy1 = max(y1, 0), cy2 = min(y2, h - 1);
    for (int x = cx1 + lane; x <= cx2; x += 32) {
      if (y1 >= 0 && y1 < h) put_px(im, max_w, y1, x, c);
      if (y2 >= 0 && y2 < h) put_px(im, max_w, y2, x, c);
    }
    for (int y = cy1 + lane; y <= cy2; y += 32) {
      if (x1 >= 0 && x1 < w) put_px(im, max_w, y, x1, c);
      if (x2 >= 0 && x2 < w) put_px(im, max_w, y, x2, c);
    }
    return;
  }
  const int j = (blockIdx.x - box_ctas) * kThreads + threadIdx.x;
  if (j >= min(max(n_points[i], 0), M)) return;
  const int q = points[(long long)i * M + j];
  if (q < 0 || (long long)q >= (long long)h * w) return;
  put_px(im, max_w, q / w, q % w, c);
}

}  // namespace sy

using namespace sy;

extern "C" int sy_draw_outlines(const SyDrawOutlinesDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->img != nullptr && d->sizes != nullptr && d->boxes != nullptr && d->counts != nullptr &&
                 d->points != nullptr && d->n_points != nullptr,
             SY_EINVAL, "draw_outlines: null pointer");
  SY_REQUIRE(d->n >= 1 && d->n <= 65535 && d->max_h >= 1 && d->max_h <= 65535 && d->max_w >= 1 && d->max_w <= 65535 &&
                 (long long)d->max_h * d->max_w < (1ll << 31),
             SY_EINVAL, "draw_outlines: bad slots (n %d, slot %dx%d)", d->n, d->max_h, d->max_w);
  SY_REQUIRE(d->K >= 1 && d->K <= (1 << 24) && d->M >= 1 && d->M <= (1 << 24), SY_EINVAL,
             "draw_outlines: K = %d or M = %d outside 1..2^24", d->K, d->M);
  SY_REQUIRE((reinterpret_cast<uintptr_t>(d->boxes) & 15) == 0, SY_EINVAL, "draw_outlines: boxes must be 16-byte aligned");
  const int box_ctas = cdiv(d->K, kBoxesPerCta);
  const dim3 grid(box_ctas + cdiv(d->M, kThreads), d->n);
  draw_outlines_kernel<<<grid, kThreads, 0, stream>>>(d->img, d->sizes, d->max_h, d->max_w,
                                                      reinterpret_cast<const int4*>(d->boxes), d->counts, d->K,
                                                      d->points, d->n_points, d->M, box_ctas,
                                                      make_uchar3(d->color[0], d->color[1], d->color[2]));
  return launch_status("draw_outlines_kernel");
}
