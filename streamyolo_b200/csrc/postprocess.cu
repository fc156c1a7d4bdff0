// Detection post-processing on the device: confidence threshold + greedy NMS; the streaming tick's gating and box
// division; the evaluators' COCO detection rows (coco_rows_kernel).
//
// Replaces [yolox 0.3.0] yolox.utils.postprocess (called at /root/reference/exps/evaluators/onex_stream_evaluator.py:148,
// sAP/streamyolo/streamyolo_det.py:62-83): cxcywh -> xyxy, class_conf / class_pred = max over the class scores,
// keep obj * class_conf >= conf_thre, torchvision.ops.batched_nms(boxes, obj * class_conf, class, nms_thre) (class-
// agnostic: torchvision.ops.nms), rows [x1, y1, x2, y2, obj, class_conf, class_pred] in decreasing score order.  The
// reference runs it per image on CUDA tensors, where torchvision 0.26's batched_nms takes _batched_nms_coordinate_trick
// (up to 100 000 box coordinates; this kernel takes at most 16 384 anchors): every candidate box is shifted by
// class * (max candidate coordinate + 1) in fp32 (a NaN coordinate makes every offset NaN), then one class-agnostic nms
// runs on the shifted boxes, so boxes of different classes can suppress each other when their shifted boxes overlap.
// Here one CTA per image: composite-key bitonic sort in shared memory (score descending, anchor index ascending on ties,
// as torchvision's stable sort), the same offsets, greedy suppression with the IoU arithmetic of torchvision's CUDA
// kernel (devIoU as compiled for sm_90: inter / (fma(w_b, h_b, w_a * h_a) - inter) > float(thr), a the earlier box, b
// the later one, no +1), compaction of the unshifted boxes.  Compiled with -fmad=false and explicit _rn intrinsics:
// every decision is bit-exact against the fp32 restatement in oracle/postprocess_oracle.py (nms_reference).
#include "common.cuh"

namespace sy {

constexpr int kNmsThreads = 1024;

struct NmsArgs {
  const float* pred;       // [B][A][5 + NC]
  int A, NC, Apad, max_det;
  float conf_thre, nms_thre;
  int class_agnostic;
  float* boxes;            // workspace [B][A][4] sorted xyxy
  int* cls;                // workspace [B][A]
  float* det;              // [B][max_det][7]
  int* count;              // [B]
};

// xyxy of one prediction row, as yolox: cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2, one rounding each (w * 0.5 is
// w / 2 exactly)
__device__ __forceinline__ void box_corners(const float* r, float c[4]) {
  const float hw = __fmul_rn(r[2], 0.5f), hh = __fmul_rn(r[3], 0.5f);
  c[0] = __fsub_rn(r[0], hw); c[1] = __fsub_rn(r[1], hh); c[2] = __fadd_rn(r[0], hw); c[3] = __fadd_rn(r[1], hh);
}

// max that propagates NaN, like torch.max (fmaxf ignores it)
__device__ __forceinline__ float max_nan(float a, float b) { return (b > a || b != b) ? b : a; }

// torchvision's devIoU(a, b) > thr as compiled for sm_90 (nms_kernel_impl<float>): a is the earlier box (cur_box), its
// area a plain product; the later box's area is fused into the sum; fmaxf / fminf for the intersection.  inter == 0
// makes the ratio +-0 or NaN, which is never > a threshold >= 0: the division is skipped then.
__device__ __forceinline__ bool iou_above(float ax1, float ay1, float ax2, float ay2, float a_area, float bx1, float by1,
                                          float bx2, float by2, float thr) {
  const float w = fmaxf(__fsub_rn(fminf(ax2, bx2), fmaxf(ax1, bx1)), 0.f);
  const float h = fmaxf(__fsub_rn(fminf(ay2, by2), fmaxf(ay1, by1)), 0.f);
  const float inter = __fmul_rn(w, h);
  if (!(inter > 0.f) && thr >= 0.f) return false;
  const float den = __fsub_rn(__fmaf_rn(__fsub_rn(bx2, bx1), __fsub_rn(by2, by1), a_area), inter);
  return __fdiv_rn(inter, den) > thr;
}

__global__ void __launch_bounds__(kNmsThreads) nms_kernel(const NmsArgs q) {
  extern __shared__ unsigned long long keys[];                 // [Apad], then removed flags [Apad] bytes, then scan scratch
  unsigned char* removed = reinterpret_cast<unsigned char*>(keys + q.Apad);
  __shared__ int s_scan[kNmsThreads / 32];
  __shared__ int s_n;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int no = 5 + q.NC;
  const float* P = q.pred + (size_t)b * q.A * no;
  // ---- 1. scores -> composite keys (0 = rejected)
  for (int a = tid; a < q.Apad; a += kNmsThreads) {
    unsigned long long key = 0ull;
    if (a < q.A) {
      const float* r = P + (size_t)a * no;
      float best = r[5];
      for (int k = 1; k < q.NC; ++k) best = r[5 + k] > best ? r[5 + k] : best;      // first maximum, like torch.max
      const float score = r[4] * best;
      if (score >= q.conf_thre)
        key = ((unsigned long long)__float_as_uint(score) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)a);
    }
    keys[a] = key;
  }
  __syncthreads();
  // ---- 2. bitonic sort, descending
  for (int k = 2; k <= q.Apad; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < q.Apad; i += kNmsThreads) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long x = keys[i], y = keys[l];
          const bool desc = (i & k) == 0;
          if (desc ? (x < y) : (x > y)) { keys[i] = y; keys[l] = x; }
        }
      }
      __syncthreads();
    }
  }
  // ---- 3. number of candidates (keys are sorted: first zero key), sorted boxes / classes, the max candidate coordinate
  if (tid == 0) s_n = 0;
  __syncthreads();
  for (int i = tid; i < q.Apad; i += kNmsThreads)
    if (keys[i] != 0ull && (i + 1 == q.Apad || keys[i + 1] == 0ull)) s_n = i + 1;
  __syncthreads();
  const int n = s_n;
  float* BX = q.boxes + (size_t)b * q.A * 4;
  int* CL = q.cls + (size_t)b * q.A;
  float mx = -INFINITY;
  for (int j = tid; j < n; j += kNmsThreads) {
    const int a = (int)(0xFFFFFFFFu - (unsigned)(keys[j] & 0xFFFFFFFFull));
    const float* r = P + (size_t)a * no;
    float c[4];
    box_corners(r, c);
    for (int e = 0; e < 4; ++e) {
      BX[j * 4 + e] = c[e];
      mx = max_nan(mx, c[e]);
    }
    int best = 0;
    float bv = r[5];
    for (int k = 1; k < q.NC; ++k)
      if (r[5 + k] > bv) { bv = r[5 + k]; best = k; }
    CL[j] = best;
    removed[j] = 0;
  }
  // batched_nms's offsets: boxes + class * (boxes.max() + 1), fp32, NaN propagating like torch.max.  Each thread shifts
  // the boxes it wrote.
  __shared__ float s_max[kNmsThreads / 32];
  for (int m = 16; m > 0; m >>= 1) mx = max_nan(mx, __shfl_xor_sync(0xffffffffu, mx, m));
  if ((tid & 31) == 0) s_max[tid >> 5] = mx;
  __syncthreads();
  if (!q.class_agnostic) {
    mx = s_max[0];
    for (int w = 1; w < kNmsThreads / 32; ++w) mx = max_nan(mx, s_max[w]);
    const float step = __fadd_rn(mx, 1.f);
    for (int j = tid; j < n; j += kNmsThreads) {
      const float off = __fmul_rn((float)CL[j], step);
      for (int e = 0; e < 4; ++e) BX[j * 4 + e] = __fadd_rn(BX[j * 4 + e], off);
    }
  }
  __syncthreads();
  // ---- 4. greedy suppression in score order, 32 candidates at a time.  (One block-wide barrier per candidate -- the first
  //         version -- cost ~0.25 ms for 2000 candidates; now two barriers per 32.)
  //   (a) warp 0 settles the chunk among its own members: lane l owns candidate c0 + l; for i = 0..31 in order, if candidate
  //       i is still alive, the later lanes test their box against it (the box of i comes by shuffle);
  //   (b) all threads apply the chunk's survivors to the candidates behind the chunk.
  //   Same decisions as the sequential loop: a candidate is removed iff a kept earlier candidate overlaps it, the earlier
  //   one in devIoU's first place.  No class test: the offsets keep classes apart exactly as far as the reference does.
  __shared__ float s_kbox[32][4];
  __shared__ float s_karea[32];
  __shared__ int s_nk;
  const float thr = q.nms_thre;
  for (int c0 = 0; c0 < n; c0 += 32) {
    if (tid < 32) {
      const int j = c0 + tid;
      const bool in = j < n;
      float x1 = 0.f, y1 = 0.f, x2 = 0.f, y2 = 0.f;
      bool alive = false;
      if (in) {
        x1 = BX[j * 4]; y1 = BX[j * 4 + 1]; x2 = BX[j * 4 + 2]; y2 = BX[j * 4 + 3];
        alive = removed[j] == 0;
      }
      const float area = __fmul_rn(__fsub_rn(x2, x1), __fsub_rn(y2, y1));
      for (int i = 0; i < 32; ++i) {
        const unsigned live = __ballot_sync(0xffffffffu, alive);
        if (!((live >> i) & 1u)) continue;                   // candidate i was removed (or lies past n): uniform
        const float ix1 = __shfl_sync(0xffffffffu, x1, i), iy1 = __shfl_sync(0xffffffffu, y1, i);
        const float ix2 = __shfl_sync(0xffffffffu, x2, i), iy2 = __shfl_sync(0xffffffffu, y2, i);
        const float iarea = __shfl_sync(0xffffffffu, area, i);
        if (alive && tid > i && iou_above(ix1, iy1, ix2, iy2, iarea, x1, y1, x2, y2, thr)) alive = false;
      }
      if (in && !alive) removed[j] = 1;
      // survivors of the chunk, compacted (order irrelevant for step (b))
      const unsigned live = __ballot_sync(0xffffffffu, alive);
      if (alive) {
        const int k = __popc(live & ((1u << tid) - 1u));
        s_kbox[k][0] = x1; s_kbox[k][1] = y1; s_kbox[k][2] = x2; s_kbox[k][3] = y2;
        s_karea[k] = area;
      }
      if (tid == 0) s_nk = __popc(live);
    }
    __syncthreads();
    const int nk = s_nk;
    if (nk > 0) {
      for (int j = c0 + 32 + tid; j < n; j += kNmsThreads) {
        if (removed[j]) continue;
        const float x1 = BX[j * 4], y1 = BX[j * 4 + 1], x2 = BX[j * 4 + 2], y2 = BX[j * 4 + 3];
        for (int k = 0; k < nk; ++k) {
          if (iou_above(s_kbox[k][0], s_kbox[k][1], s_kbox[k][2], s_kbox[k][3], s_karea[k], x1, y1, x2, y2, thr)) {
            removed[j] = 1;
            break;
          }
        }
      }
    }
    __syncthreads();
  }
  // ---- 5. compaction in score order
  int base = 0;
  for (int j0 = 0; j0 < n; j0 += kNmsThreads) {
    const int j = j0 + tid;
    const int keep = (j < n && !removed[j]) ? 1 : 0;
    // block-wide exclusive scan of keep
    int v = keep;
    const int lane = tid & 31, warp = tid >> 5;
    for (int m = 1; m < 32; m <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, v, m);
      if (lane >= m) v += t;
    }
    if (lane == 31) s_scan[warp] = v;
    __syncthreads();
    if (warp == 0) {
      int w = lane < kNmsThreads / 32 ? s_scan[lane] : 0;
      for (int m = 1; m < 32; m <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, m);
        if (lane >= m) w += t;
      }
      if (lane < kNmsThreads / 32) s_scan[lane] = w;
    }
    __syncthreads();
    const int pos = base + (warp ? s_scan[warp - 1] : 0) + v - keep;
    if (keep && pos < q.max_det) {
      const int a = (int)(0xFFFFFFFFu - (unsigned)(keys[j] & 0xFFFFFFFFull));
      const float* r = P + (size_t)a * no;
      float bv = r[5];
      for (int k = 1; k < q.NC; ++k) bv = r[5 + k] > bv ? r[5 + k] : bv;
      float* o = q.det + ((size_t)b * q.max_det + pos) * 7;
      box_corners(r, o);                                       // the unshifted corners
      o[4] = r[4]; o[5] = bv; o[6] = (float)CL[j];
    }
    base += s_scan[kNmsThreads / 32 - 1];
    __syncthreads();
  }
  if (tid == 0) q.count[b] = base < q.max_det ? base : q.max_det;
}

// Per-stream gating of a streaming tick (see sy_stream_gate): a stream whose frame did not decode starts nothing and
// keeps its buffer.
__global__ void __launch_bounds__(128) stream_gate_kernel(const int32_t* __restrict__ status,
                                                          const int32_t* __restrict__ flags, int n,
                                                          int32_t* __restrict__ start, int32_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool ok = status == nullptr || status[i] == SY_JPEG_OK;
  start[i] = ok && flags[i] != 0;
  keep[i] = ok;
}

// One CTA per stream: the boxes of its count rows / ratio (IEEE fp32 division, as numpy divides the float32 rows by the
// ratio), or no rows when its frame did not decode.
__global__ void __launch_bounds__(128) stream_rescale_kernel(float* __restrict__ det, int max_det, int32_t* __restrict__ count,
                                                             const int32_t* __restrict__ status,
                                                             const float* __restrict__ ratio) {
  const int b = blockIdx.x;
  const int n = min(max(count[b], 0), max_det);
  __syncthreads();                                 // every thread has read count[b] before thread 0 may clear it
  if (status != nullptr && status[b] != SY_JPEG_OK) {
    if (threadIdx.x == 0) count[b] = 0;
    return;
  }
  const float r = ratio[b];
  float* rows = det + (size_t)b * max_det * 7;
  for (int e = threadIdx.x; e < 4 * n; e += blockDim.x) {
    float* v = rows + (e >> 2) * 7 + (e & 3);
    *v = __fdiv_rn(*v, r);
  }
}

// Device half of the evaluators' convert_to_coco_format (see sy_coco_rows).  One CTA per image: its first output row is
// the sum of the emitted counts of the images before it (image-major order; B is a batch, so the O(B) sum is short),
// then one thread per row.  Block 0 also writes the total.  Explicit _rn intrinsics: the reference's fp32 torch CPU ops,
// one rounding each.
__device__ __forceinline__ int coco_rows_n(const int32_t* count, const int32_t* image_id, const int32_t* status, int fpi,
                                           int max_det, int b) {
  if (image_id[b] < 0) return 0;
  if (status != nullptr)
    for (int f = 0; f < fpi; ++f)
      if (status[b * fpi + f] != SY_JPEG_OK) return 0;
  return min(max(count[b], 0), max_det);
}

__global__ void __launch_bounds__(256) coco_rows_kernel(const SyCocoRowsDesc q) {
  __shared__ int s_base, s_total;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    int base = 0, total = 0;
    for (int k = 0; k < q.b; ++k) {
      const int n = coco_rows_n(q.count, q.image_id, q.status, q.frames_per_image, q.max_det, k);
      if (k < b) base += n;
      total += n;
    }
    s_base = base;
    s_total = total;
  }
  __syncthreads();
  if (b == 0 && threadIdx.x == 0) *q.total_out = s_total;
  const int n = coco_rows_n(q.count, q.image_id, q.status, q.frames_per_image, q.max_det, b);
  const float r = q.ratio[b];
  const int id = q.image_id[b];
  const float* rows = q.det + (size_t)b * q.max_det * 7;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const float* d = rows + (size_t)j * 7;
    const int o = s_base + j;
    // bboxes /= scale (fp32 tensor / Python float: torch divides by the float-rounded scale), then xyxy2xywh in place
    const float x1 = __fdiv_rn(d[0], r), y1 = __fdiv_rn(d[1], r);
    const float x2 = __fdiv_rn(d[2], r), y2 = __fdiv_rn(d[3], r);
    q.bbox_out[(size_t)o * 4 + 0] = x1;
    q.bbox_out[(size_t)o * 4 + 1] = y1;
    q.bbox_out[(size_t)o * 4 + 2] = __fsub_rn(x2, x1);
    q.bbox_out[(size_t)o * 4 + 3] = __fsub_rn(y2, y1);
    q.score_out[o] = __fmul_rn(d[4], d[5]);                    // output[:, 4] * output[:, 5]
    const int c = (int)d[6];                                    // class_ids[int(cls)]
    q.category_out[o] = (c >= 0 && c < q.num_classes) ? q.class_ids[c] : -1;
    q.image_id_out[o] = id;
  }
}

static inline size_t nms_ws_bytes(int B, int A) { return ((size_t)B * A * 4 * sizeof(float) + 255) / 256 * 256 + (size_t)B * A * sizeof(int); }

}  // namespace sy

using namespace sy;

extern "C" size_t sy_postprocess_nms_workspace_bytes(int32_t b, int32_t a_total) {
  return b > 0 && a_total > 0 ? nms_ws_bytes(b, a_total) : 0;
}

extern "C" int sy_postprocess_nms(const SyNmsDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  SY_REQUIRE(d->b > 0 && d->a_total > 0 && d->num_classes >= 1 && d->max_det > 0, SY_EINVAL, "postprocess_nms: bad sizes");
  SY_REQUIRE(d->pred && d->det_out && d->count_out && d->workspace, SY_EINVAL, "postprocess_nms: null pointer");
  SY_REQUIRE(d->workspace_bytes >= nms_ws_bytes(d->b, d->a_total), SY_EWORKSPACE, "postprocess_nms: workspace %zu < %zu",
             d->workspace_bytes, nms_ws_bytes(d->b, d->a_total));
  SY_REQUIRE(((uintptr_t)d->workspace % 16) == 0, SY_EINVAL, "postprocess_nms: workspace must be 16B aligned");
  int apad = 32;
  while (apad < d->a_total) apad <<= 1;
  const size_t smem = (size_t)apad * 9;
  SY_REQUIRE(smem <= 200 * 1024, SY_EINVAL, "postprocess_nms: %d anchors exceed the shared-memory sort (max 16384)", d->a_total);
  if (smem > 48 * 1024) SY_CUDA(cudaFuncSetAttribute(nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  NmsArgs q{};
  q.pred = d->pred; q.A = d->a_total; q.NC = d->num_classes; q.Apad = apad; q.max_det = d->max_det;
  q.conf_thre = d->conf_thre; q.nms_thre = d->nms_thre; q.class_agnostic = d->class_agnostic;
  q.boxes = reinterpret_cast<float*>(d->workspace);
  q.cls = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(d->workspace) +
                                 ((size_t)d->b * d->a_total * 4 * sizeof(float) + 255) / 256 * 256);
  q.det = d->det_out; q.count = d->count_out;
  nms_kernel<<<d->b, kNmsThreads, smem, stream>>>(q);
  return launch_status("nms_kernel");
}

extern "C" int sy_stream_gate(const int32_t* status, const int32_t* flags, int32_t n, int32_t* start, int32_t* keep,
                              sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(flags != nullptr && start != nullptr && keep != nullptr, SY_EINVAL, "stream_gate: null pointer");
  SY_REQUIRE(n > 0, SY_EINVAL, "stream_gate: %d streams", n);
  stream_gate_kernel<<<cdiv(n, 128), 128, 0, stream>>>(status, flags, n, start, keep);
  return launch_status("stream_gate_kernel");
}

extern "C" int sy_stream_rescale(float* det, int32_t n, int32_t max_det, int32_t* count, const int32_t* status,
                                 const float* ratio, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(det != nullptr && count != nullptr && ratio != nullptr, SY_EINVAL, "stream_rescale: null pointer");
  SY_REQUIRE(n > 0 && n <= 65535 && max_det > 0, SY_EINVAL, "stream_rescale: bad sizes (%d streams, max_det %d)", n, max_det);
  stream_rescale_kernel<<<n, 128, 0, stream>>>(det, max_det, count, status, ratio);
  return launch_status("stream_rescale_kernel");
}

extern "C" int sy_coco_rows(const SyCocoRowsDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  SY_REQUIRE(d->det && d->count && d->ratio && d->image_id && d->class_ids && d->bbox_out && d->score_out &&
             d->image_id_out && d->category_out && d->total_out, SY_EINVAL, "coco_rows: null pointer");
  SY_REQUIRE(d->b > 0 && d->b <= 4096 && d->max_det > 0 && d->num_classes > 0, SY_EINVAL,
             "coco_rows: bad sizes (%d images, max_det %d, %d classes)", d->b, d->max_det, d->num_classes);
  SY_REQUIRE(d->status == nullptr || d->frames_per_image >= 1, SY_EINVAL, "coco_rows: frames_per_image %d",
             d->frames_per_image);
  coco_rows_kernel<<<d->b, 256, 0, stream>>>(*d);
  return launch_status("coco_rows_kernel");
}
