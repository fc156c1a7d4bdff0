// sy_draw_boxes: the box branch of the sAP toolkit's vis_obj_fancy (sAP/vis/vis_det_th.py:99-120) on uint8 images in
// slots: filled rectangles blended at 0.8 / 0.2 (cv2.rectangle thickness -1, cv2.addWeighted), then thickness-2 outlines
// (cv2.rectangle thickness 2), the last box in list order deciding each pixel.  One CTA per 64 x 32 tile of an image: it
// compacts, in list order and 256 boxes at a time, the boxes whose outline bounds touch the tile into shared memory, and
// each thread walks that list for its eight pixels, so no pixel's value depends on scheduling.
// sy_vis_det_boxes: a streaming tick's NMS rows -> those boxes, as the host path from the driver's output computes them.
#include <climits>

#include "common.cuh"

namespace sy {

constexpr int kTileW = 64, kTileH = 32, kThreads = 256, kRows = kTileH * kTileW / kThreads;   // 8 pixels per thread
constexpr uint32_t kSet = 1u << 24;                       // a colour word: bytes 0..2 the colour, bit 24 "set"

// the CTA's ordered compaction: the rank of this thread's kept item among the block's, and the number kept
__device__ __forceinline__ int block_rank(bool keep, int* warp_base, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) warp_base[warp] = __popc(m);
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int i = 0; i < kThreads / 32; ++i) {
      const int c = warp_base[i];
      warp_base[i] = s;
      s += c;
    }
    warp_base[kThreads / 32] = s;
  }
  __syncthreads();
  total = warp_base[kThreads / 32];
  return warp_base[warp] + __popc(m & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(kThreads) draw_boxes_kernel(
    const uint8_t* src, const int32_t* __restrict__ sizes, int max_h, int max_w, const int4* __restrict__ boxes,
    const int32_t* __restrict__ labels, const int32_t* __restrict__ counts, int K, const uint8_t* __restrict__ palette,
    int P, uint8_t* dst) {
  __shared__ int4 s_box[kThreads];                        // normalised: x1 <= x2, y1 <= y2
  __shared__ uint32_t s_col[kThreads];
  __shared__ int s_warp[kThreads / 32 + 1];
  const int img = blockIdx.z;
  const int h = sizes[2 * img], w = sizes[2 * img + 1];
  const int tx0 = blockIdx.x * kTileW, ty0 = blockIdx.y * kTileH;
  if (h < 1 || w < 1 || h > max_h || w > max_w || tx0 >= w || ty0 >= h) return;    // uniform over the CTA
  const int tx1 = min(tx0 + kTileW, w) - 1, ty1 = min(ty0 + kTileH, h) - 1;       // the tile's last pixel in the image
  const int count = min(max(counts[img], 0), K);
  const int x = tx0 + (threadIdx.x % kTileW), yb = ty0 + threadIdx.x / kTileW;     // rows yb, yb + 4, ...
  uint32_t fill[kRows], line[kRows];
#pragma unroll
  for (int r = 0; r < kRows; ++r) fill[r] = line[r] = 0;
  const int4* bx = boxes + (long long)img * K;
  const int32_t* lb = labels + (long long)img * K;
  for (int base = 0; base < count; base += kThreads) {
    const int i = base + threadIdx.x;
    int4 b = make_int4(0, 0, 0, 0);
    uint32_t col = 0;
    bool keep = false;
    if (i < count) {
      const int4 v = bx[i];
      const int l = lb[i];
      b = make_int4(min(v.x, v.z), min(v.y, v.w), max(v.x, v.z), max(v.y, v.w));
      // the outline reaches one pixel past the box on every side: [x1 - 1, x2 + 1] x [y1 - 1, y2 + 1], compared without
      // forming x1 - 1 (boxes may hold any int32)
      keep = l >= 0 && l < P && b.x <= tx1 + 1 && b.z >= tx0 - 1 && b.y <= ty1 + 1 && b.w >= ty0 - 1;
      if (keep)
        col = kSet | palette[3 * l] | ((uint32_t)palette[3 * l + 1] << 8) | ((uint32_t)palette[3 * l + 2] << 16);
    }
    int total;
    const int rank = block_rank(keep, s_warp, total);
    if (keep) {
      s_box[rank] = b;
      s_col[rank] = col;
    }
    __syncthreads();
    for (int j = 0; j < total; ++j) {
      const int4 q = s_box[j];
      const uint32_t c = s_col[j];
      // column classes, pixel coordinates in [0, 65535] so x +- 2 cannot overflow
      const bool fx = x >= q.x && x <= q.z;                               // inside the filled box's columns
      const bool ox = x + 1 >= q.x && x - 1 <= q.z;                       // inside the outline's columns
      const bool ix = x - 2 >= q.x && x + 2 <= q.z;                       // strictly inside the outline's hole
      const bool cx = x + 1 == q.x || x - 1 == q.z;                       // the columns just outside the box
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        const int y = yb + r * (kThreads / kTileW);
        const bool fy = y >= q.y && y <= q.w;
        const bool oy = y + 1 >= q.y && y - 1 <= q.w;
        const bool iy = y - 2 >= q.y && y + 2 <= q.w;
        const bool cy = y + 1 == q.y || y - 1 == q.w;
        if (fx && fy) fill[r] = c;
        if (ox && oy && !(ix && iy) && !(cx && cy)) line[r] = c;
      }
    }
    __syncthreads();                                      // the list is rewritten by the next chunk
  }
  if (x > tx1) return;
  uint8_t* out = dst + ((long long)img * max_h * max_w + x) * 3;
  const uint8_t* in = src + ((long long)img * max_h * max_w + x) * 3;
#pragma unroll
  for (int r = 0; r < kRows; ++r) {
    const int y = yb + r * (kThreads / kTileW);
    if (y > ty1) break;
    const long long at = (long long)y * max_w * 3;
    if (line[r]) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) out[at + ch] = (uint8_t)(line[r] >> (8 * ch));
    } else if (fill[r]) {
      // cv2.addWeighted(orig, 0.8, filled, 0.2, 0) on uint8: saturate_cast<uchar>(v * 0.8f + p * 0.2f), fp32, each
      // product rounded, rounded to nearest even
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float v = (float)in[at + ch], p = (float)((fill[r] >> (8 * ch)) & 255u);
        const int o = __float2int_rn(__fadd_rn(__fmul_rn(v, 0.8f), __fmul_rn(p, 0.2f)));
        out[at + ch] = (uint8_t)min(max(o, 0), 255);
      }
    }
  }
}

// numpy's .round().astype(np.int32) of an fp32 value: half to even, and INT_MIN (x86's "integer indefinite", what the
// cast gives) for NaN, infinities and values outside int32 -- a random-weight head can emit non-finite boxes
__device__ __forceinline__ int np_round_i32(float v) {
  const float r = rintf(v);
  return r >= -2147483648.f && r < 2147483648.f ? (int)r : INT_MIN;
}

// one CTA per stream: rows kept in order through the same ordered compaction
__global__ void __launch_bounds__(kThreads) vis_det_boxes_kernel(const float* __restrict__ det,
                                                                 const int32_t* __restrict__ count, int A, float th,
                                                                 int4* __restrict__ boxes, int32_t* __restrict__ labels,
                                                                 int32_t* __restrict__ counts) {
  __shared__ int s_warp[kThreads / 32 + 1];
  const int s = blockIdx.x;
  const int n = min(max(count[s], 0), A);
  const float* rows = det + (long long)s * A * 7;
  int kept = 0;
  for (int base = 0; base < n; base += kThreads) {
    const int i = base + threadIdx.x;
    bool keep = false;
    float r[7];
    if (i < n) {
#pragma unroll
      for (int k = 0; k < 7; ++k) r[k] = rows[(long long)i * 7 + k];
      keep = __fmul_rn(r[4], r[5]) >= th;
    }
    int total;
    const int rank = kept + block_rank(keep, s_warp, total);
    if (keep) {
      // ltrb -> ltwh -> ltrb in fp32, then numpy's round half to even
      const float x2 = __fadd_rn(r[0], __fsub_rn(r[2], r[0])), y2 = __fadd_rn(r[1], __fsub_rn(r[3], r[1]));
      boxes[(long long)s * A + rank] = make_int4(np_round_i32(r[0]), np_round_i32(r[1]), np_round_i32(x2),
                                                 np_round_i32(y2));
      labels[(long long)s * A + rank] = (int32_t)r[6];
    }
    kept += total;
    __syncthreads();                                      // s_warp is rewritten by the next chunk
  }
  if (threadIdx.x == 0) counts[s] = kept;
}

}  // namespace sy

using namespace sy;

extern "C" int sy_draw_boxes(const SyDrawBoxesDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->src != nullptr && d->sizes != nullptr && d->boxes != nullptr && d->labels != nullptr &&
                 d->counts != nullptr && d->palette != nullptr && d->dst != nullptr,
             SY_EINVAL, "draw_boxes: null pointer");
  SY_REQUIRE(d->n >= 1 && d->n <= 65535 && d->max_h >= 1 && d->max_h <= 65535 && d->max_w >= 1 && d->max_w <= 65535,
             SY_EINVAL, "draw_boxes: bad slots (n %d, slot %dx%d)", d->n, d->max_h, d->max_w);
  SY_REQUIRE(d->K >= 1 && d->K <= (1 << 24), SY_EINVAL, "draw_boxes: K = %d outside 1..2^24", d->K);
  SY_REQUIRE(d->P >= 1 && d->P <= 65536, SY_EINVAL, "draw_boxes: P = %d outside 1..65536", d->P);
  SY_REQUIRE(d->dst_h == d->max_h && d->dst_w == d->max_w, SY_EINVAL,
             "draw_boxes: dst slots of %dx%d for src slots of %dx%d", d->dst_h, d->dst_w, d->max_h, d->max_w);
  SY_REQUIRE((reinterpret_cast<uintptr_t>(d->boxes) & 15) == 0, SY_EINVAL, "draw_boxes: boxes must be 16-byte aligned");
  const dim3 grid(cdiv(d->max_w, kTileW), cdiv(d->max_h, kTileH), d->n);
  draw_boxes_kernel<<<grid, kThreads, 0, stream>>>(d->src, d->sizes, d->max_h, d->max_w,
                                                   reinterpret_cast<const int4*>(d->boxes), d->labels, d->counts, d->K,
                                                   d->palette, d->P, d->dst);
  return launch_status("draw_boxes_kernel");
}

extern "C" int sy_vis_det_boxes(const SyVisDetBoxesDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->det != nullptr && d->count != nullptr && d->boxes != nullptr && d->labels != nullptr &&
                 d->counts != nullptr,
             SY_EINVAL, "vis_det_boxes: null pointer");
  SY_REQUIRE(d->S >= 1 && d->S <= 65535 && d->A >= 1 && d->A <= (1 << 24), SY_EINVAL,
             "vis_det_boxes: bad sizes (S %d, A %d)", d->S, d->A);
  SY_REQUIRE((reinterpret_cast<uintptr_t>(d->boxes) & 15) == 0, SY_EINVAL, "vis_det_boxes: boxes must be 16-byte aligned");
  vis_det_boxes_kernel<<<d->S, kThreads, 0, stream>>>(d->det, d->count, d->A, d->score_th,
                                                      reinterpret_cast<int4*>(d->boxes), d->labels, d->counts);
  return launch_status("vis_det_boxes_kernel");
}
