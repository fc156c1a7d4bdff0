// The input transforms of the training and streaming paths, from uint8 BGR frames to the model's fp32 input:
//   * sy_pair_labels   the label half of DoubleTrainTransform (/root/reference/exps/data/data_augment_flip.py:176-234):
//                      mirror, xyxy -> cxcywh, * r, the min(w, h) > 1 filter and its all-filtered fallback, padding to
//                      max_labels; also the per-frame mirror bit the image kernel applies
//   * sy_frame_labels  the same per frame for single frames: the label half of TrainTransform (data_augment_flip.py:170-234)
//   * sy_letterbox     the image half: cv2.resize(INTER_LINEAR) on uint8 (OpenCV's 11-bit fixed-point bilinear), the
//                      mirror, the 114 pad and HWC uint8 -> CHW fp32; optionally preceded by load_resized_img's resize
//                      (tal_flip_one_future_argoversedataset.py:179-187).  With no pad and no flags it is the streaming
//                      driver's preproc (sAP/streamyolo/streamyolo_det.py:57-60).
//   * sy_letterbox_sized  the same resize with a source size and a resized extent per frame, the frames in slots of one
//                      size: the evaluation preproc (data_augment_flip.py:151-167) of camera streams of different sizes.
//   * sy_resize_sized  that resize into uint8 slots, no pad: mmcv.imrescale(bilinear) of the sAP toolkit's vis_det.
// Built with -fmad=false: the tap positions (x + 0.5) * scale - 0.5 and the fp64 label arithmetic must round every
// operation separately, as OpenCV and numpy do.  The output is then bit-identical to cv2 / numpy.
#include <math.h>

#include "common.cuh"

namespace sy {

constexpr int kPadValue = 114;

struct ResizeStage {
  int src_h, src_w, dst_h, dst_w;
  double scale_y, scale_x;             // 1 / (dst / src), computed on the host like OpenCV's
};

// One axis of cv2's INTER_LINEAR on 8-bit data: source taps s0, s1 and their weights in units of 1/2048.  Columns clamp the
// tap and zero the fraction at both borders; rows keep the fraction and only the fetched rows are clamped.
__device__ __forceinline__ void linear_axis(int d, double scale, int src, bool clamp, int& s0, int& s1, int& w0, int& w1) {
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f -= (float)s;
  if (clamp) {
    if (s < 0) s = 0, f = 0.f;
    if (s >= src - 1) s = src - 1, f = 0.f;
  }
  w0 = __float2int_rn((1.f - f) * 2048.f);
  w1 = __float2int_rn(f * 2048.f);
  s0 = min(max(s, 0), src - 1);
  s1 = min(max(s + 1, 0), src - 1);
}

// vertical pass of OpenCV's VResizeLinear (8-bit, SIMD form) over two horizontal sums
__device__ __forceinline__ int vmix(int S0, int S1, int b0, int b1) {
  return min(max((((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2, 0), 255);
}

__device__ __forceinline__ void load_px(const uint8_t* __restrict__ img, int w, int r, int c, int p[3]) {
  const uint8_t* q = img + (r * w + c) * 3;
  p[0] = q[0], p[1] = q[1], p[2] = q[2];
}

// pixel (r, c) of the first-stage image: the raw frame resized by stage `a` when FIRST, else the raw frame itself
template <bool FIRST>
__device__ __forceinline__ void stage1_px(const uint8_t* __restrict__ img, const ResizeStage& a, int r, int c, int p[3]) {
  if constexpr (!FIRST) {
    load_px(img, a.src_w, r, c, p);
  } else {
    int y0, y1, b0, b1, x0, x1, a0, a1;
    linear_axis(r, a.scale_y, a.src_h, false, y0, y1, b0, b1);
    linear_axis(c, a.scale_x, a.src_w, true, x0, x1, a0, a1);
    int p00[3], p01[3], p10[3], p11[3];
    load_px(img, a.src_w, y0, x0, p00);
    load_px(img, a.src_w, y0, x1, p01);
    load_px(img, a.src_w, y1, x0, p10);
    load_px(img, a.src_w, y1, x1, p11);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) p[ch] = vmix(p00[ch] * a0 + p01[ch] * a1, p10[ch] * a0 + p11[ch] * a1, b0, b1);
  }
}

// Value at (y, x) of the dst region of one frame: stage b applied to the (mirrored) first-stage image, or, without a
// second stage, the first-stage image at the mirrored column.  Shared by letterbox_kernel and letterbox_sized_kernel.
template <bool FIRST, bool SECOND>
__device__ __forceinline__ void letterbox_px(const uint8_t* __restrict__ img, const ResizeStage& a, const ResizeStage& b,
                                             bool mir, int y, int x, int p[3]) {
  const int mid_w = b.src_w;                       // width of the first-stage image (the mirror axis)
  if constexpr (!SECOND) {
    stage1_px<FIRST>(img, a, y, mir ? mid_w - 1 - x : x, p);
  } else {
    int y0, y1, b0, b1, x0, x1, a0, a1;
    linear_axis(y, b.scale_y, b.src_h, false, y0, y1, b0, b1);
    linear_axis(x, b.scale_x, b.src_w, true, x0, x1, a0, a1);
    if (mir) x0 = mid_w - 1 - x0, x1 = mid_w - 1 - x1;
    int p00[3], p01[3], p10[3], p11[3];
    stage1_px<FIRST>(img, a, y0, x0, p00);
    stage1_px<FIRST>(img, a, y0, x1, p01);
    stage1_px<FIRST>(img, a, y1, x0, p10);
    stage1_px<FIRST>(img, a, y1, x1, p11);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) p[ch] = vmix(p00[ch] * a0 + p01[ch] * a1, p10[ch] * a0 + p11[ch] * a1, b0, b1);
  }
}

// One thread per output pixel (three planes): blockIdx.z = frame, blockIdx.y = output row, x along the row (coalesced fp32
// stores, no index divisions).  Inside the dst_h x dst_w region: letterbox_px.  Outside: 114.
template <bool FIRST, bool SECOND>
__global__ void __launch_bounds__(128) letterbox_kernel(const uint8_t* __restrict__ src, ResizeStage a, ResizeStage b,
                                                        int out_h, int out_w, const int32_t* __restrict__ flags,
                                                        float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, k = blockIdx.z;
  if (x >= out_w) return;
  const long long plane = (long long)out_h * out_w;
  float* o = out + 3 * plane * k + (long long)y * out_w + x;
  if (y >= b.dst_h || x >= b.dst_w) {
    o[0] = o[plane] = o[2 * plane] = (float)kPadValue;
    return;
  }
  const uint8_t* img = src + (long long)a.src_h * a.src_w * 3 * k;
  const bool mir = flags != nullptr && flags[k] != 0;
  int p[3];
  letterbox_px<FIRST, SECOND>(img, a, b, mir, y, x, p);
  o[0] = (float)p[0];
  o[plane] = (float)p[1];
  o[2 * plane] = (float)p[2];
}

// The same per frame k of slots of slot_h x slot_w: sizes[k] = (h, w, dst_h, dst_w), the frame at the slot's top-left, its
// resize to dst_h x dst_w (none when equal) and the 114 pad.  The tap scales are OpenCV's 1 / (dst / src), in fp64 as the
// host computes them for sy_letterbox.  A row that does not fit the slot or the canvas leaves image k untouched.
__global__ void __launch_bounds__(128) letterbox_sized_kernel(const uint8_t* __restrict__ src, int slot_h, int slot_w,
                                                              const int32_t* __restrict__ sizes, int out_h, int out_w,
                                                              float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, k = blockIdx.z;
  if (x >= out_w) return;
  const int h = sizes[4 * k], w = sizes[4 * k + 1], dh = sizes[4 * k + 2], dw = sizes[4 * k + 3];
  if (h < 1 || w < 1 || h > slot_h || w > slot_w || dh < 1 || dw < 1 || dh > out_h || dw > out_w) return;
  const long long plane = (long long)out_h * out_w;
  float* o = out + 3 * plane * k + (long long)y * out_w + x;
  if (y >= dh || x >= dw) {
    o[0] = o[plane] = o[2 * plane] = (float)kPadValue;
    return;
  }
  const ResizeStage a{h, slot_w, h, w, 1.0, 1.0};  // no first stage: only the row pitch (slot_w pixels) is read
  const ResizeStage b{h, w, dh, dw, 1.0 / ((double)dh / h), 1.0 / ((double)dw / w)};
  const uint8_t* img = src + (long long)slot_h * slot_w * 3 * k;
  int p[3];
  if (dh != h || dw != w) letterbox_px<false, true>(img, a, b, false, y, x, p);
  else letterbox_px<false, false>(img, a, b, false, y, x, p);
  o[0] = (float)p[0];
  o[plane] = (float)p[1];
  o[2 * plane] = (float)p[2];
}

// The same resize into uint8 slots (mmcv.imrescale of the sAP toolkit's vis_det): frame k resized to dst_h x dst_w at the
// top-left of out slot k, channel order kept, the rest of the slot not written.
__global__ void __launch_bounds__(128) resize_sized_kernel(const uint8_t* __restrict__ src, int slot_h, int slot_w,
                                                           const int32_t* __restrict__ sizes, int out_h, int out_w,
                                                           uint8_t* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, k = blockIdx.z;
  const int h = sizes[4 * k], w = sizes[4 * k + 1], dh = sizes[4 * k + 2], dw = sizes[4 * k + 3];
  if (h < 1 || w < 1 || h > slot_h || w > slot_w || dh < 1 || dw < 1 || dh > out_h || dw > out_w) return;
  if (y >= dh || x >= dw) return;
  const ResizeStage a{h, slot_w, h, w, 1.0, 1.0};  // no first stage: only the row pitch (slot_w pixels) is read
  const ResizeStage b{h, w, dh, dw, 1.0 / ((double)dh / h), 1.0 / ((double)dw / w)};
  const uint8_t* img = src + (long long)slot_h * slot_w * 3 * k;
  int p[3];
  if (dh != h || dw != w) letterbox_px<false, true>(img, a, b, false, y, x, p);
  else letterbox_px<false, false>(img, a, b, false, y, x, p);
  uint8_t* o = out + (((long long)k * out_h + y) * out_w + x) * 3;
  o[0] = (uint8_t)p[0];
  o[1] = (uint8_t)p[1];
  o[2] = (uint8_t)p[2];
}

// One warp per (pair, frame).  Rows are x1, y1, x2, y2, cls in fp64; output rows cls, cx, cy, w, h in fp32.
__device__ __forceinline__ void frame_box(const double* row, bool mirror, double width, double r, double v[4]) {
  double x1 = row[0], x2 = row[2];
  if (mirror) {
    const double m1 = width - x2, m2 = width - x1;
    x1 = m1, x2 = m2;
  }
  const double w = x2 - x1, h = row[3] - row[1];
  v[0] = (x1 + w * 0.5) * r;
  v[1] = (row[1] + h * 0.5) * r;
  v[2] = w * r;
  v[3] = h * r;
}

// The label transform of one frame, run by one warp (every lane takes part in the ballots): ``ann`` [n][5] rows, ``want`` =
// the frame's mirror was drawn and flip is on; writes [max_labels][5] ``out`` and the effective mirror bit.
__device__ __forceinline__ void frame_labels_warp(const double* __restrict__ ann, int n, bool want, double width, double r,
                                                  int max_labels, float* __restrict__ out, int32_t* flag_out) {
  const int lane = threadIdx.x & 31;
  const bool a = want && n > 0;
  int kept = 0;                                    // rows that survive the min(w, h) > 1 filter
  for (int i0 = 0; i0 < n; i0 += 32) {
    bool keep = false;
    if (i0 + lane < n) {
      double v[4];
      frame_box(ann + (i0 + lane) * 5, a, width, r, v);
      keep = fmin(v[2], v[3]) > 1.0;
    }
    kept += __popc(__ballot_sync(0xffffffffu, keep));
  }
  const bool fallback = kept == 0;                 // nothing left: the unmirrored frame and all rows, unfiltered
  const bool mirror = a && !fallback;
  int written = 0;
  for (int i0 = 0; i0 < n && written < max_labels; i0 += 32) {
    const int i = i0 + lane;
    double v[4];
    bool keep = false;
    if (i < n) {
      frame_box(ann + i * 5, mirror, width, r, v);
      keep = fallback || fmin(v[2], v[3]) > 1.0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    const int slot = written + __popc(m & ((1u << lane) - 1u));
    if (keep && slot < max_labels) {
      float* q = out + slot * 5;
      q[0] = (float)ann[i * 5 + 4];
      q[1] = (float)v[0], q[2] = (float)v[1], q[3] = (float)v[2], q[4] = (float)v[3];
    }
    written += __popc(m);
  }
  for (int e = min(written, max_labels) * 5 + lane; e < max_labels * 5; e += 32) out[e] = 0.f;
  if (lane == 0) *flag_out = mirror ? 1 : 0;
}

__global__ void __launch_bounds__(128) pair_labels_kernel(SyPairLabelsDesc d) {
  const int fi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;     // (item, frame) = (fi >> 1, fi & 1)
  if (fi >= 2 * d.n_items) return;
  const int item = fi >> 1, frame = fi & 1;
  const int n = min(max(d.counts[fi], 0), d.max_rows);
  const bool want = d.flip != 0 && d.mirror != nullptr && d.mirror[item] != 0;
  float* out = (frame == 0 ? d.labels_fut : d.labels_cur) + (long long)item * d.max_labels * 5;
  frame_labels_warp(d.ann + (long long)fi * d.max_rows * 5, n, want, (double)d.width, d.r, d.max_labels, out,
                    d.flags_out + fi);
}

// One warp per frame of a single-frame batch (TrainTransform).
__global__ void __launch_bounds__(128) frame_labels_kernel(SyFrameLabelsDesc d) {
  const int fi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (fi >= d.n) return;
  const int n = min(max(d.counts[fi], 0), d.max_rows);
  const bool want = d.flip != 0 && d.mirror != nullptr && d.mirror[fi] != 0;
  frame_labels_warp(d.ann + (long long)fi * d.max_rows * 5, n, want, (double)d.width, d.r, d.max_labels,
                    d.labels + (long long)fi * d.max_labels * 5, d.flags_out + fi);
}

}  // namespace sy

using namespace sy;

extern "C" int sy_pair_labels(const SyPairLabelsDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->ann != nullptr && d->counts != nullptr && d->labels_fut != nullptr &&
                 d->labels_cur != nullptr && d->flags_out != nullptr, SY_EINVAL, "pair_labels: null pointer");
  SY_REQUIRE(d->n_items > 0 && d->max_rows > 0 && d->max_labels > 0 && d->width > 0 && d->r > 0.0, SY_EINVAL,
             "pair_labels: bad sizes (items %d, rows %d, max_labels %d, width %d)", d->n_items, d->max_rows, d->max_labels,
             d->width);
  SY_REQUIRE(d->flip == 0 || d->mirror != nullptr, SY_EINVAL, "pair_labels: flip without mirror bits");
  const int warps = 2 * d->n_items;
  pair_labels_kernel<<<cdiv(warps, 4), 128, 0, stream>>>(*d);
  return launch_status("pair_labels_kernel");
}

extern "C" int sy_frame_labels(const SyFrameLabelsDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->ann != nullptr && d->counts != nullptr && d->labels != nullptr && d->flags_out != nullptr,
             SY_EINVAL, "frame_labels: null pointer");
  SY_REQUIRE(d->n > 0 && d->max_rows > 0 && d->max_labels > 0 && d->width > 0 && d->r > 0.0, SY_EINVAL,
             "frame_labels: bad sizes (frames %d, rows %d, max_labels %d, width %d)", d->n, d->max_rows, d->max_labels,
             d->width);
  SY_REQUIRE(d->flip == 0 || d->mirror != nullptr, SY_EINVAL, "frame_labels: flip without mirror bits");
  frame_labels_kernel<<<cdiv(d->n, 4), 128, 0, stream>>>(*d);
  return launch_status("frame_labels_kernel");
}

extern "C" int sy_letterbox(const SyLetterboxDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->src != nullptr && d->out != nullptr, SY_EINVAL, "letterbox: null pointer");
  SY_REQUIRE(d->n > 0 && d->n <= 65535 && d->h > 0 && d->w > 0 && d->mid_h > 0 && d->mid_w > 0 && d->dst_h > 0 &&
                 d->dst_w > 0, SY_EINVAL, "letterbox: bad sizes");
  SY_REQUIRE(d->dst_h <= d->out_h && d->dst_w <= d->out_w && d->out_h <= 65535, SY_EINVAL,
             "letterbox: %dx%d does not fit the %dx%d canvas", d->dst_h, d->dst_w, d->out_h, d->out_w);
  SY_REQUIRE((long long)d->h * d->w * 3 < (1ll << 31), SY_EINVAL, "letterbox: frame too large");
  ResizeStage a{d->h, d->w, d->mid_h, d->mid_w, 1.0 / ((double)d->mid_h / d->h), 1.0 / ((double)d->mid_w / d->w)};
  ResizeStage b{d->mid_h, d->mid_w, d->dst_h, d->dst_w, 1.0 / ((double)d->dst_h / d->mid_h),
                1.0 / ((double)d->dst_w / d->mid_w)};
  const bool first = d->mid_h != d->h || d->mid_w != d->w, second = d->dst_h != d->mid_h || d->dst_w != d->mid_w;
  const dim3 grid(cdiv(d->out_w, 128), d->out_h, d->n);
  auto k = first ? (second ? letterbox_kernel<true, true> : letterbox_kernel<true, false>)
                 : (second ? letterbox_kernel<false, true> : letterbox_kernel<false, false>);
  k<<<grid, 128, 0, stream>>>(d->src, a, b, d->out_h, d->out_w, d->flags, d->out);
  return launch_status("letterbox_kernel");
}

extern "C" int sy_letterbox_sized(const SyLetterboxSizedDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->src != nullptr && d->sizes != nullptr && d->out != nullptr, SY_EINVAL,
             "letterbox_sized: null pointer");
  SY_REQUIRE(d->n > 0 && d->n <= 65535 && d->slot_h > 0 && d->slot_w > 0 && d->out_h > 0 && d->out_w > 0 &&
                 d->out_h <= 65535, SY_EINVAL, "letterbox_sized: bad sizes");
  SY_REQUIRE((long long)d->slot_h * d->slot_w * 3 < (1ll << 31), SY_EINVAL, "letterbox_sized: slot too large");
  const dim3 grid(cdiv(d->out_w, 128), d->out_h, d->n);
  letterbox_sized_kernel<<<grid, 128, 0, stream>>>(d->src, d->slot_h, d->slot_w, d->sizes, d->out_h, d->out_w, d->out);
  return launch_status("letterbox_sized_kernel");
}

extern "C" int sy_resize_sized(const SyResizeSizedDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->src != nullptr && d->sizes != nullptr && d->out != nullptr, SY_EINVAL,
             "resize_sized: null pointer");
  SY_REQUIRE(d->src != d->out, SY_EINVAL, "resize_sized: src and out must be different buffers");
  SY_REQUIRE(d->n > 0 && d->n <= 65535 && d->slot_h > 0 && d->slot_w > 0 && d->slot_h <= 65535 && d->slot_w <= 65535 &&
                 d->out_h > 0 && d->out_w > 0 && d->out_h <= 65535 && d->out_w <= 65535,
             SY_EINVAL, "resize_sized: bad sizes");
  SY_REQUIRE((long long)d->slot_h * d->slot_w * 3 < (1ll << 31) && (long long)d->out_h * d->out_w * 3 < (1ll << 31),
             SY_EINVAL, "resize_sized: slot too large");
  const dim3 grid(cdiv(d->out_w, 128), d->out_h, d->n);
  resize_sized_kernel<<<grid, 128, 0, stream>>>(d->src, d->slot_h, d->slot_w, d->sizes, d->out_h, d->out_w, d->out);
  return launch_status("resize_sized_kernel");
}
