// Head prediction convs + box decode, batched SimOTA assignment and the Trend-Aware loss, all
// on device with no host synchronisation (the reference loops over images in Python with
// .item() syncs and torch.cuda.empty_cache() per image: /root/reference/exps/model/tal_head.py:305-415).
// fp32 throughout; this translation unit is compiled with -fmad=false so that the geometric
// predicates and IoUs are evaluated with exactly the roundings of the reference expressions.
#include <math.h>

#include "common.cuh"

namespace sy {

// ================================================================ prediction + decode
// Four threads per pixel: thread ks takes the 16-byte channel chunks ks, ks+4, ks+8, ... of both feature
// maps (the four threads read 64 contiguous bytes), keeps 5+ncls partial dot products, and two shuffles per
// output combine them.  Weights live in shared memory as fp32 (conflict-free: the four threads of a pixel
// read neighbouring 32-byte segments, the eight pixels of a warp broadcast).
// Output row layout [reg4, obj1, cls*] (tal_head.py:174,197-199); anchors row-major y then x (:236-239).
constexpr int kMaxPred = 5 + 32;

// PT pixels per thread (64 * PT pixels per block and pass): every weight chunk read from shared memory is used for PT
// pixels.  With one pixel per thread the kernel was bound by its shared-memory weight reads (26 LDS.128 per 104 FMAs: 51 us
// for the 73 MB of level-0 features = 1.4 TB/s); the per-pixel arithmetic (order of the products and sums) is unchanged, so
// the results are bit-identical for every PT.  F16: the tower features are fp16 (SyHeadPredDesc.storage).
template <int NO, int PT, bool F16>
__global__ void __launch_bounds__(256)
head_pred_kernel(const SyHeadPredDesc d, int B, int H, int W, int C) {
  extern __shared__ float wsm[];   // [NO][C] : reg(4), obj(1), cls(NO-5)
  for (int i = threadIdx.x; i < NO * C; i += blockDim.x) {
    const int o = i / C, c = i % C;
    wsm[i] = (o < 4) ? d.w_reg[o * C + c] : (o == 4 ? d.w_obj[c] : d.w_cls[(o - 5) * C + c]);
  }
  __syncthreads();
  const int ks = threadIdx.x & 3;
  const long long npix = (long long)B * H * W;
  const __nv_bfloat16* cf = reinterpret_cast<const __nv_bfloat16*>(d.cls_feat.ptr);
  const __nv_bfloat16* rf = reinterpret_cast<const __nv_bfloat16*>(d.reg_feat.ptr);
  const int chunks = C / 8;
  for (long long pix0 = (long long)blockIdx.x * (64 * PT); pix0 < npix; pix0 += (long long)gridDim.x * (64 * PT)) {
    long long pix[PT];
    bool live[PT];
#pragma unroll
    for (int j = 0; j < PT; ++j) {
      pix[j] = pix0 + 64 * j + (threadIdx.x >> 2);
      live[j] = pix[j] < npix;
    }
    float acc[PT][NO];
#pragma unroll
    for (int j = 0; j < PT; ++j)
#pragma unroll
      for (int o = 0; o < NO; ++o) acc[j][o] = 0.f;
    for (int ch = ks; ch < chunks; ch += 4) {
      uint4 rv[PT], cv[PT];
#pragma unroll
      for (int j = 0; j < PT; ++j) {             // all loads of the pass first: 2 * PT independent 16-byte requests in flight
        rv[j] = live[j] ? *reinterpret_cast<const uint4*>(rf + pix[j] * d.reg_feat.pitch + ch * 8) : make_uint4(0u, 0u, 0u, 0u);
        cv[j] = live[j] ? *reinterpret_cast<const uint4*>(cf + pix[j] * d.cls_feat.pitch + ch * 8) : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int part = 0; part < 2; ++part) {     // reg | obj outputs read the reg features, the class outputs the cls features
        float v[PT][8];
#pragma unroll
        for (int j = 0; j < PT; ++j) {
          st_unpack8<F16>(part == 0 ? rv[j] : cv[j], v[j]);
        }
#pragma unroll
        for (int o = (part == 0 ? 0 : 5); o < (part == 0 ? 5 : NO); ++o) {
          const float4 w0 = *reinterpret_cast<const float4*>(wsm + o * C + ch * 8);
          const float4 w1 = *reinterpret_cast<const float4*>(wsm + o * C + ch * 8 + 4);
#pragma unroll
          for (int j = 0; j < PT; ++j) {
            float s = v[j][0] * w0.x;     // explicit FMAs: this unit is compiled with -fmad=false for the loss
            s = __fmaf_rn(v[j][1], w0.y, s); s = __fmaf_rn(v[j][2], w0.z, s); s = __fmaf_rn(v[j][3], w0.w, s);
            s = __fmaf_rn(v[j][4], w1.x, s); s = __fmaf_rn(v[j][5], w1.y, s); s = __fmaf_rn(v[j][6], w1.z, s);
            s = __fmaf_rn(v[j][7], w1.w, s);
            acc[j][o] += s;
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < PT; ++j) {
#pragma unroll
      for (int o = 0; o < NO; ++o) {
        acc[j][o] += __shfl_xor_sync(0xffffffffu, acc[j][o], 1);
        acc[j][o] += __shfl_xor_sync(0xffffffffu, acc[j][o], 2);
      }
      if (live[j] && ks == 0) {
        const int x = (int)(pix[j] % W), y = (int)((pix[j] / W) % H);
        const int b = (int)(pix[j] / ((long long)W * H));
        const long long a = (long long)b * d.a_total + d.anchor_offset + (long long)y * W + x;
        float* out = d.out + a * NO;
        float reg[4];
#pragma unroll
        for (int o = 0; o < 4; ++o) reg[o] = acc[j][o] + d.b_reg[o];
        if (d.origin) {
          float* og = d.origin + a * 4;
          og[0] = reg[0]; og[1] = reg[1]; og[2] = reg[2]; og[3] = reg[3];
        }
        const float s = (float)d.stride;
        if (d.decode) {
          out[0] = (reg[0] + (float)x) * s;
          out[1] = (reg[1] + (float)y) * s;
          out[2] = expf(reg[2]) * s;
          out[3] = expf(reg[3]) * s;
        } else {
          out[0] = reg[0]; out[1] = reg[1]; out[2] = reg[2]; out[3] = reg[3];
        }
        const float obj = acc[j][4] + d.b_obj[0];
        out[4] = d.sigmoid ? 1.0f / (1.0f + expf(-obj)) : obj;
#pragma unroll
        for (int o = 5; o < NO; ++o) {
          const float v = acc[j][o] + d.b_cls[o - 5];
          out[o] = d.sigmoid ? 1.0f / (1.0f + expf(-v)) : v;
        }
      }
    }
  }
}

// Any class count (the reference head takes `num_classes` freely, tal_head.py:27): the outputs are walked in groups of eight
// compile-time accumulators, re-reading the pixel's features (L1 / L2) for every group.  Same per-output arithmetic as above.
template <bool F16>
__global__ void __launch_bounds__(256)
head_pred_generic_kernel(const SyHeadPredDesc d, int B, int H, int W, int C, int NO) {
  extern __shared__ float wsm[];   // [NO][C]
  for (int i = threadIdx.x; i < NO * C; i += blockDim.x) {
    const int o = i / C, c = i % C;
    wsm[i] = (o < 4) ? d.w_reg[o * C + c] : (o == 4 ? d.w_obj[c] : d.w_cls[(o - 5) * C + c]);
  }
  __syncthreads();
  const int ks = threadIdx.x & 3;
  const long long npix = (long long)B * H * W;
  const __nv_bfloat16* cf = reinterpret_cast<const __nv_bfloat16*>(d.cls_feat.ptr);
  const __nv_bfloat16* rf = reinterpret_cast<const __nv_bfloat16*>(d.reg_feat.ptr);
  const int chunks = C / 8;
  for (long long pix0 = (long long)blockIdx.x * 64; pix0 < npix; pix0 += (long long)gridDim.x * 64) {
    const long long pix = pix0 + (threadIdx.x >> 2);
    const bool live = pix < npix;
    const int x = live ? (int)(pix % W) : 0, y = live ? (int)((pix / W) % H) : 0;
    const int b = live ? (int)(pix / ((long long)W * H)) : 0;
    const long long a = (long long)b * d.a_total + d.anchor_offset + (long long)y * W + x;
    for (int o0 = 0; o0 < NO; o0 += 8) {       // group 0 = reg(4) + obj + 3 classes
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
      if (live) {
        for (int ch = ks; ch < chunks; ch += 4) {
          const uint4 rv = *reinterpret_cast<const uint4*>(rf + pix * d.reg_feat.pitch + ch * 8);
          const uint4 cv = *reinterpret_cast<const uint4*>(cf + pix * d.cls_feat.pitch + ch * 8);
          float r[8], c[8];
          st_unpack8<F16>(rv, r);
          st_unpack8<F16>(cv, c);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int o = o0 + i;
            if (o < NO) {
              const float4 w0 = *reinterpret_cast<const float4*>(wsm + o * C + ch * 8);
              const float4 w1 = *reinterpret_cast<const float4*>(wsm + o * C + ch * 8 + 4);
              const bool use_r = o < 5;
              float s = (use_r ? r[0] : c[0]) * w0.x;
              s = __fmaf_rn(use_r ? r[1] : c[1], w0.y, s); s = __fmaf_rn(use_r ? r[2] : c[2], w0.z, s);
              s = __fmaf_rn(use_r ? r[3] : c[3], w0.w, s); s = __fmaf_rn(use_r ? r[4] : c[4], w1.x, s);
              s = __fmaf_rn(use_r ? r[5] : c[5], w1.y, s); s = __fmaf_rn(use_r ? r[6] : c[6], w1.z, s);
              s = __fmaf_rn(use_r ? r[7] : c[7], w1.w, s);
              acc[i] += s;
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 1);
        acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 2);
      }
      if (live && ks == 0) {
        float* out = d.out + a * NO;
        const float s = (float)d.stride;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int o = o0 + i;
          if (o >= NO) continue;
          if (o < 4) {
            const float reg = acc[i] + d.b_reg[o];
            if (d.origin) d.origin[a * 4 + o] = reg;
            out[o] = !d.decode ? reg : (o == 0 ? (reg + (float)x) * s : (o == 1 ? (reg + (float)y) * s : expf(reg) * s));
          } else {
            const float v = acc[i] + (o == 4 ? d.b_obj[0] : d.b_cls[o - 5]);
            out[o] = d.sigmoid ? 1.0f / (1.0f + expf(-v)) : v;
          }
        }
      }
    }
  }
}

static int head_pixels_per_thread(long long npix) {
  return npix >= 32768 ? 2 : 1;                          // small levels: more blocks matter more than the weight reuse
}

template <int NO, int PT, bool F16>
static int launch_head_pred_pt(const SyHeadPredDesc* d, const SyTensor& f, cudaStream_t stream) {
  const size_t smem = sizeof(float) * NO * f.c;
  if (smem > 48 * 1024)
    SY_CUDA(cudaFuncSetAttribute(head_pred_kernel<NO, PT, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const long long npix = (long long)f.n * f.h * f.w;
  int blocks = (int)((npix + 64 * PT - 1) / (64 * PT));
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  head_pred_kernel<NO, PT, F16><<<blocks, 256, smem, stream>>>(*d, f.n, f.h, f.w, f.c);
  return launch_status("head_pred_kernel");
}

template <int NO, bool F16>
static int launch_head_pred(const SyHeadPredDesc* d, const SyTensor& f, cudaStream_t stream) {
  if (head_pixels_per_thread((long long)f.n * f.h * f.w) == 2) return launch_head_pred_pt<NO, 2, F16>(d, f, stream);
  return launch_head_pred_pt<NO, 1, F16>(d, f, stream);
}

template <bool F16>
static int launch_head_pred_generic(const SyHeadPredDesc* d, const SyTensor& f, cudaStream_t stream) {
  const int NO = 5 + d->num_classes;
  const size_t smem = sizeof(float) * NO * f.c;
  if (smem > 48 * 1024)
    SY_CUDA(cudaFuncSetAttribute(head_pred_generic_kernel<F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const long long npix = (long long)f.n * f.h * f.w;
  int blocks = (int)((npix + 63) / 64);
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  head_pred_generic_kernel<F16><<<blocks, 256, smem, stream>>>(*d, f.n, f.h, f.w, f.c, NO);
  return launch_status("head_pred_generic_kernel");
}

template <bool F16>
static int launch_head_pred_classes(const SyHeadPredDesc* d, const SyTensor& f, cudaStream_t stream) {
  switch (d->num_classes) {           // compile-time output counts for the class counts in use (Argoverse-HD: 8); any other: generic
    case 8: return launch_head_pred<13, F16>(d, f, stream);
    case 1: return launch_head_pred<6, F16>(d, f, stream);
    case 20: return launch_head_pred<25, F16>(d, f, stream);
    default: break;
  }
  return launch_head_pred_generic<F16>(d, f, stream);
}

// ======================================================================= loss
struct LossWs {
  int* ngt; int* nsup;          // [B]
  float* tal;                   // [B][L]
  int* cand;                    // [B][A]
  float* clsterm;               // [B][A][2*NC]
  float* iou; float* cost;      // [B][L][A]
  int* cnt; int* match;         // [B][A]
  double* part;                 // [nblk][8]
  int* mres; float* piou;       // [B][A] resolved match (-1: background) and matched IoU: kept for the backward pass
  double* tot;                  // [8] the seven sums of k_final: kept for the backward pass
  size_t bytes;
};

static inline size_t align256(size_t v) { return (v + 255) & ~size_t(255); }
constexpr int kLossThreads = 256;

static LossWs carve(void* base, int B, int A, int L, int NC) {
  LossWs w{};
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align256(off + bytes); return o; };
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  const size_t o_ngt = take(sizeof(int) * B), o_nsup = take(sizeof(int) * B);
  const size_t o_tal = take(sizeof(float) * B * L);
  const size_t o_cand = take(sizeof(int) * (size_t)B * A);
  const size_t o_cls = take(sizeof(float) * (size_t)B * A * 2 * NC);
  const size_t o_iou = take(sizeof(float) * (size_t)B * L * A);
  const size_t o_cost = take(sizeof(float) * (size_t)B * L * A);
  const size_t o_cnt = take(sizeof(int) * (size_t)B * A);
  const size_t o_match = take(sizeof(int) * (size_t)B * A);
  const int nblk = cdiv(A, kLossThreads) * B;
  const size_t o_part = take(sizeof(double) * (size_t)nblk * 8);
  const size_t o_mres = take(sizeof(int) * (size_t)B * A), o_piou = take(sizeof(float) * (size_t)B * A);
  const size_t o_tot = take(sizeof(double) * 8);
  w.bytes = off;
  if (p) {
    w.ngt = (int*)(p + o_ngt); w.nsup = (int*)(p + o_nsup); w.tal = (float*)(p + o_tal);
    w.cand = (int*)(p + o_cand); w.clsterm = (float*)(p + o_cls); w.iou = (float*)(p + o_iou);
    w.cost = (float*)(p + o_cost); w.cnt = (int*)(p + o_cnt); w.match = (int*)(p + o_match);
    w.part = (double*)(p + o_part);
    w.mres = (int*)(p + o_mres); w.piou = (float*)(p + o_piou); w.tot = (double*)(p + o_tot);
  }
  return w;
}

struct Box { float cx, cy, w, h; };

// yolox bboxes_iou(xyxy=False): no epsilon
__device__ __forceinline__ float pair_iou(const Box a, const Box b) {
  const float tlx = fmaxf(a.cx - a.w / 2.f, b.cx - b.w / 2.f), tly = fmaxf(a.cy - a.h / 2.f, b.cy - b.h / 2.f);
  const float brx = fminf(a.cx + a.w / 2.f, b.cx + b.w / 2.f), bry = fminf(a.cy + a.h / 2.f, b.cy + b.h / 2.f);
  const float en = (tlx < brx && tly < bry) ? 1.f : 0.f;
  const float ai = (brx - tlx) * (bry - tly) * en;
  return ai / (a.w * a.h + b.w * b.h - ai);
}
// yolox IOUloss: +1e-16 in the union
__device__ __forceinline__ float loss_iou(const Box p, const Box t) {
  const float tlx = fmaxf(p.cx - p.w / 2.f, t.cx - t.w / 2.f), tly = fmaxf(p.cy - p.h / 2.f, t.cy - t.h / 2.f);
  const float brx = fminf(p.cx + p.w / 2.f, t.cx + t.w / 2.f), bry = fminf(p.cy + p.h / 2.f, t.cy + t.h / 2.f);
  const float en = (tlx < brx && tly < bry) ? 1.f : 0.f;
  const float ai = (brx - tlx) * (bry - tly) * en;
  const float au = p.w * p.h + t.w * t.h - ai;
  const float iou = ai / (au + 1e-16f);
  return 1.f - iou * iou;
}
__device__ __forceinline__ float bce_logits(float x, float t) {
  return fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x)));
}

// torch.sum of n fp32 terms along a contiguous last dimension, added in the order of ATen's CUDA reduce kernel, measured
// on the H100 for n <= 127 at 16 to 100 000 rows: 32 accumulators (accumulator e takes terms e, e + 32, ... left to
// right), combined by halving (e += e + 16, then e + 8, 4, 2, 1).  Rows of 128 and more are loaded as vectors by ATen and
// are not in its order here.  The reference sums its top-10 IoUs (dynamic k) and its per-class BCE terms (class cost)
// this way when it trains on CUDA tensors.  W leaves suffice for n <= W (the missing accumulators are zeros); they are
// visited in bit-reversed order, so that neighbours merge like the halving pairs, with partial sums per level in
// registers.
__host__ __device__ constexpr int bit_reverse(int k, int bits) {
  return bits == 0 ? 0 : ((k & 1) << (bits - 1)) | bit_reverse(k >> 1, bits - 1);
}

template <int W, typename Term>
__device__ __forceinline__ float aten_sum_w(int n, Term term) {
  constexpr int bits = W == 8 ? 3 : (W == 16 ? 4 : 5);
  float lvl[5];
  float v = 0.f;
#pragma unroll
  for (int k = 0; k < W; ++k) {
    const int e = bit_reverse(k, bits);
    v = e < n ? term(e) : 0.f;
    for (int j = e + 32; j < n; j += 32) v += term(j);
#pragma unroll
    for (int b = 0; b < 5; ++b) {
      if (!((k >> b) & 1)) { lvl[b] = v; break; }
      v = lvl[b] + v;
    }
  }
  return v;
}

template <typename Term>
__device__ __forceinline__ float aten_sum(int n, Term term) {
  if (n <= 8) return aten_sum_w<8>(n, term);
  if (n <= 16) return aten_sum_w<16>(n, term);
  return aten_sum_w<32>(n, term);
}

struct Levels { int n; int h[4], w[4], s[4]; };
__device__ __forceinline__ void anchor_geom(const Levels& lv, int a, float* gx, float* gy, float* gs) {
  int off = 0;
  for (int l = 0; l < lv.n; ++l) {
    const int cnt = lv.h[l] * lv.w[l];
    if (a < off + cnt || l == lv.n - 1) {
      const int loc = a - off;
      *gx = (float)(loc % lv.w[l]); *gy = (float)(loc / lv.w[l]); *gs = (float)lv.s[l];
      return;
    }
    off += cnt;
  }
}
// get_in_boxes_info predicates (tal_head.py:603-669) for one (gt, anchor)
__device__ __forceinline__ void in_tests(const Box g, float xc, float yc, float s, bool* in_box, bool* in_ctr) {
  const float bl = xc - (g.cx - 0.5f * g.w), br = (g.cx + 0.5f * g.w) - xc;
  const float bt = yc - (g.cy - 0.5f * g.h), bb = (g.cy + 0.5f * g.h) - yc;
  *in_box = fminf(fminf(bl, bt), fminf(br, bb)) > 0.0f;
  const float r = 2.5f * s;
  const float cl = xc - (g.cx - r), cr = (g.cx + r) - xc, ct = yc - (g.cy - r), cb = (g.cy + r) - yc;
  *in_ctr = fminf(fminf(cl, ct), fminf(cr, cb)) > 0.0f;
}

// ---- 1. label counts + trend IoU per future GT (tal_head.py:285-286, 394-403)
__global__ void k_labels(const float* fut, const float* cur, int L, float thr, float ign, int* ngt, int* nsup, float* tal) {
  const int b = blockIdx.x;
  // counts of non-empty label rows, all threads in parallel (a single thread walking 2 x 120 rows took ~30 us)
  int c0 = 0, c1 = 0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const float* r0 = fut + ((size_t)b * L + i) * 5;
    const float* r1 = cur + ((size_t)b * L + i) * 5;
    if ((((r0[0] + r0[1]) + r0[2]) + r0[3]) + r0[4] > 0.f) ++c0;
    if ((((r1[0] + r1[1]) + r1[2]) + r1[3]) + r1[4] > 0.f) ++c1;
  }
  __shared__ int s_n[2];
  if (threadIdx.x == 0) { s_n[0] = 0; s_n[1] = 0; }
  __syncthreads();
  if (c0) atomicAdd(&s_n[0], c0);
  if (c1) atomicAdd(&s_n[1], c1);
  __syncthreads();
  const int G = s_n[0], GS = s_n[1];
  if (threadIdx.x == 0) { ngt[b] = G; nsup[b] = GS; }
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float v = 1.0f;
    if (GS > 0) {
      const float* r = fut + ((size_t)b * L + g) * 5;
      const Box a{r[1], r[2], r[3], r[4]};
      float m = -INFINITY;
      for (int j = 0; j < GS; ++j) {
        const float* q = cur + ((size_t)b * L + j) * 5;
        m = fmaxf(m, pair_iou(a, Box{q[1], q[2], q[3], q[4]}));
      }
      v = (m < thr) ? ign : m;
    }
    tal[(size_t)b * L + g] = v;
  }
}

// ---- 2. per anchor: candidate flag + class-cost terms (tal_head.py:539-546, 594-672)
__global__ void k_anchor_prep(const float* outputs, const float* fut, const int* ngt, Levels lv, int A, int L, int NC,
                              int* cand, float* clsterm) {
  const int b = blockIdx.y, a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= A) return;
  const int G = ngt[b];
  float gx, gy, gs;
  anchor_geom(lv, a, &gx, &gy, &gs);
  const float xc = gx * gs + 0.5f * gs, yc = gy * gs + 0.5f * gs;
  bool any = false;
  for (int g = 0; g < G; ++g) {
    const float* r = fut + ((size_t)b * L + g) * 5;
    bool ib, ic;
    in_tests(Box{r[1], r[2], r[3], r[4]}, xc, yc, gs, &ib, &ic);
    any = any || ib || ic;
  }
  cand[(size_t)b * A + a] = any ? 1 : 0;
  if (!any) return;
  const float* o = outputs + ((size_t)b * A + a) * (5 + NC);
  const float so = 1.0f / (1.0f + expf(-o[4]));
  float* ct = clsterm + ((size_t)b * A + a) * 2 * NC;
  for (int c = 0; c < NC; ++c) {
    const float sc = 1.0f / (1.0f + expf(-o[5 + c]));
    const float p = sqrtf(sc * so);
    ct[c] = -fmaxf(logf(p), -100.f);            // target 1
    ct[NC + c] = -fmaxf(log1pf(-p), -100.f);      // target 0 (ATen's CUDA binary_cross_entropy takes log1p(-p))
  }
}

// ---- 3. pairwise IoU + cost (tal_head.py:526-553)
__global__ void k_pair(const float* outputs, const float* fut, const int* ngt, const int* cand, const float* clsterm,
                       Levels lv, int A, int L, int NC, float* iou_m, float* cost_m) {
  const int b = blockIdx.z, g = blockIdx.y;
  if (g >= ngt[b]) return;
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= A) return;
  const size_t o_idx = ((size_t)b * L + g) * A + a;
  if (!cand[(size_t)b * A + a]) {
    iou_m[o_idx] = -INFINITY; cost_m[o_idx] = INFINITY;
    return;
  }
  const float* r = fut + ((size_t)b * L + g) * 5;
  const Box gt{r[1], r[2], r[3], r[4]};
  const int gcls = (int)r[0];
  const float* o = outputs + ((size_t)b * A + a) * (5 + NC);
  const float iou = pair_iou(gt, Box{o[0], o[1], o[2], o[3]});
  float gx, gy, gs;
  anchor_geom(lv, a, &gx, &gy, &gs);
  bool ib, ic;
  in_tests(gt, gx * gs + 0.5f * gs, gy * gs + 0.5f * gs, gs, &ib, &ic);
  const float* ct = clsterm + ((size_t)b * A + a) * 2 * NC;
  const float cls_cost = aten_sum(NC, [&](int c) { return (c == gcls) ? ct[c] : ct[NC + c]; });
  const float iou_cost = -logf(iou + 1e-8f);
  const float cost = (cls_cost + 3.0f * iou_cost) + 100000.0f * ((ib && ic) ? 0.f : 1.f);
  iou_m[o_idx] = iou; cost_m[o_idx] = cost;
}

// block-wide arg-extreme with lowest index on ties; result broadcast through smem
template <bool kMax>
__device__ __forceinline__ void block_arg(float v, int i, float* s_v, int* s_i, float* out_v, int* out_i) {
  for (int m = 16; m >= 1; m >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, m);
    const int oi = __shfl_xor_sync(0xffffffffu, i, m);
    const bool better = kMax ? (ov > v || (ov == v && oi < i)) : (ov < v || (ov == v && oi < i));
    if (better) { v = ov; i = oi; }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (lane == 0) { s_v[warp] = v; s_i[warp] = i; }
  __syncthreads();
  if (warp == 0) {
    v = lane < nw ? s_v[lane] : (kMax ? -INFINITY : INFINITY);
    i = lane < nw ? s_i[lane] : 0x7fffffff;
    for (int m = 16; m >= 1; m >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, m);
      const int oi = __shfl_xor_sync(0xffffffffu, i, m);
      const bool better = kMax ? (ov > v || (ov == v && oi < i)) : (ov < v || (ov == v && oi < i));
      if (better) { v = ov; i = oi; }
    }
    if (lane == 0) { s_v[32] = v; s_i[32] = i; }
  }
  __syncthreads();
  *out_v = s_v[32]; *out_i = s_i[32];
  __syncthreads();
}

// ---- 4. dynamic-k matching per (image, gt) (tal_head.py:679-692)
// Only the image's candidate anchors (in some box or centre region: a few hundred to a few thousand of the 11 850) can be
// selected -- every other entry of the row is -inf (IoU) / +inf (cost) -- so the block first compacts the candidates'
// (anchor, IoU) pairs into shared memory and runs the ten arg-max / dynamic-k arg-min rounds over that short list.
// Selection order is by (value, anchor index): independent of the order in which the list was filled.
__global__ void k_dynk(const int* ngt, const int* cand, const float* iou_m, const float* cost_m, int A, int L, int* cnt,
                       int* match) {
  extern __shared__ float row[];   // [A] values, then [A] anchor indices
  int* idx = reinterpret_cast<int*>(row + A);
  __shared__ float s_v[33];
  __shared__ int s_i[33];
  __shared__ int s_n;
  __shared__ float s_top[10];
  const int b = blockIdx.y, g = blockIdx.x;
  if (g >= ngt[b]) return;
  const float* ir = iou_m + ((size_t)b * L + g) * A;
  const float* cr = cost_m + ((size_t)b * L + g) * A;
  const int* cd = cand + (size_t)b * A;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  for (int a0 = 0; a0 < A; a0 += blockDim.x) {              // warp-aggregated compaction
    const int a = a0 + threadIdx.x;
    const bool is = a < A && cd[a] != 0;
    const unsigned m = __ballot_sync(0xffffffffu, is);
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == 0 && m) base = atomicAdd(&s_n, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (is) {
      const int pos = base + __popc(m & ((1u << lane) - 1u));
      idx[pos] = a;
      row[pos] = ir[a];
    }
  }
  __syncthreads();
  const int n = s_n;
  int ntop = 0;
  for (int k = 0; k < 10; ++k) {
    float bv = -INFINITY; int bi = 0x7fffffff, bp = -1;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
      const float v = row[j];
      const int a = idx[j];
      if (v > bv || (v == bv && a < bi)) { bv = v; bi = a; bp = j; }
    }
    float wv; int wi;
    block_arg<true>(bv, bi, s_v, s_i, &wv, &wi);
    if (!(wv > -INFINITY)) break;     // fewer than 10 candidates (uniform across the block)
    if (threadIdx.x == 0) s_top[k] = wv;
    ntop = k + 1;
    if (bp >= 0 && bi == wi) row[bp] = -INFINITY;   // the one thread that holds the winner retires it
    __syncthreads();
  }
  // topk_ious.sum(1): the descending top values summed in ATen's order
  const float acc = ntop > 0 ? aten_sum(ntop, [&](int j) { return s_top[j]; }) : 0.f;
  int dk = (int)acc;
  if (dk < 1) dk = 1;
  for (int j = threadIdx.x; j < n; j += blockDim.x) row[j] = cr[idx[j]];
  __syncthreads();
  for (int k = 0; k < dk; ++k) {
    float bv = INFINITY; int bi = 0x7fffffff, bp = -1;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
      const float v = row[j];
      const int a = idx[j];
      if (v < bv || (v == bv && a < bi)) { bv = v; bi = a; bp = j; }
    }
    float wv; int wi;
    block_arg<false>(bv, bi, s_v, s_i, &wv, &wi);
    if (!(wv < INFINITY)) break;      // ran out of candidates
    if (bp >= 0 && bi == wi) {
      row[bp] = INFINITY;
      atomicAdd(&cnt[(size_t)b * A + wi], 1);
      match[(size_t)b * A + wi] = g;
    }
    __syncthreads();
  }
}

// ---- 5. conflict resolution + loss terms (tal_head.py:696-711, 379-461)
struct LossArgs {
  const float* outputs; const float* origin; const float* fut;
  const int* ngt; const float* tal; const float* iou_m; const float* cost_m; const int* cnt; const int* match;
  Levels lv; int A, L, NC; float gamma; int use_l1;
  double* part; int* fg_out; int* matched_out; float* piou_out;
  int* mres; float* piou_ws;
};

__global__ void k_resolve_loss(const LossArgs q) {
  const int b = blockIdx.y, a = blockIdx.x * blockDim.x + threadIdx.x;
  float v[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // S_iou, S_wiou, S_l1, S_wl1, S_obj, S_cls, N_fg
  if (a < q.A) {
    const size_t ba = (size_t)b * q.A + a;
    const int G = q.ngt[b];
    const int c = G > 0 ? q.cnt[ba] : 0;
    const bool fg = c > 0;
    int mg = -1;
    float piou = 0.f;
    const float* o = q.outputs + ba * (5 + q.NC);
    v[4] = bce_logits(o[4], fg ? 1.f : 0.f);
    if (fg) {
      mg = q.match[ba];
      if (c > 1) {   // anchor claimed by several GTs: keep the lowest cost over ALL gts, first minimum
        float best = INFINITY;
        for (int g = 0; g < G; ++g) {
          const float cv = q.cost_m[((size_t)b * q.L + g) * q.A + a];
          if (cv < best) { best = cv; mg = g; }
        }
      }
      piou = q.iou_m[((size_t)b * q.L + mg) * q.A + a];
      const float* r = q.fut + ((size_t)b * q.L + mg) * 5;
      const Box gt{r[1], r[2], r[3], r[4]};
      const int gcls = (int)r[0];
      const float li = loss_iou(Box{o[0], o[1], o[2], o[3]}, gt);
      const float t = q.tal[(size_t)b * q.L + mg];
      const float tp = (q.gamma == 1.0f) ? t : powf(t, q.gamma);
      const float w = 1.0f / (tp + 1e-8f);
      float lc = 0.f;
      for (int k = 0; k < q.NC; ++k) lc += bce_logits(o[5 + k], k == gcls ? piou : 0.f);
      float l1 = 0.f;
      if (q.use_l1) {
        float gx, gy, gs;
        anchor_geom(q.lv, a, &gx, &gy, &gs);
        const float* og = q.origin + ba * 4;
        l1 = fabsf(og[0] - (gt.cx / gs - gx));
        l1 += fabsf(og[1] - (gt.cy / gs - gy));
        l1 += fabsf(og[2] - logf(gt.w / gs + 1e-8f));
        l1 += fabsf(og[3] - logf(gt.h / gs + 1e-8f));
      }
      v[0] = li; v[1] = w * li; v[2] = l1; v[3] = w * l1; v[5] = lc; v[6] = 1.f;
    }
    q.mres[ba] = mg;
    q.piou_ws[ba] = piou;
    if (q.fg_out) q.fg_out[ba] = fg ? 1 : 0;
    if (q.matched_out) q.matched_out[ba] = mg;
    if (q.piou_out) q.piou_out[ba] = piou;
  }
  __shared__ double red[kLossThreads / 32][7];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double dv[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    dv[i] = (double)v[i];
    for (int m = 16; m >= 1; m >>= 1) dv[i] += __shfl_xor_sync(0xffffffffu, dv[i], m);
    if (lane == 0) red[warp][i] = dv[i];
  }
  __syncthreads();
  if (threadIdx.x < 7) {
    double s = 0.0;
    for (int w2 = 0; w2 < kLossThreads / 32; ++w2) s += red[w2][threadIdx.x];
    q.part[((size_t)b * gridDim.x + blockIdx.x) * 8 + threadIdx.x] = s;
  }
}

// ---- 6. final scalars (tal_head.py:441-470)
__global__ void k_final(const double* part, int nblk, const int* ngt, int B, int use_l1, float* out, double* tot_out) {
  // 7 sums over nblk partial rows: warp w (of 8) owns sum w; its lanes take rows lane, lane+32, ... in order and a fixed
  // shuffle tree combines them (deterministic; one thread per sum walking ~380 rows cost ~25 us of serial L2 latency)
  __shared__ double tot[7];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp < 7) {
    double s = 0.0;
    for (int i = lane; i < nblk; i += 32) s += part[(size_t)i * 8 + warp];
    for (int m = 16; m >= 1; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    if (lane == 0) tot[warp] = s;
  }
  __syncthreads();
  if (threadIdx.x < 7) tot_out[threadIdx.x] = tot[threadIdx.x];
  if (threadIdx.x == 0) {
    int num_gts = 0;
    for (int b = 0; b < B; ++b) num_gts += ngt[b];
    const double nfg_raw = tot[6];
    const double num_fg = nfg_raw > 1.0 ? nfg_raw : 1.0;
    // sum_i ((w_i * S) / SW) * l_i  ==  (S / SW) * SW  (NaN like the reference when SW == 0 with fg > 0)
    double l_iou = 0.0, l_l1 = 0.0;
    if (nfg_raw > 0.0) {
      l_iou = (tot[0] / tot[1]) * tot[1] / num_fg;
      if (use_l1) l_l1 = (tot[2] / tot[3]) * tot[3] / num_fg;
    }
    const double l_obj = tot[4] / num_fg, l_cls = tot[5] / num_fg;
    out[0] = (float)(5.0 * l_iou + l_obj + l_cls + l_l1);
    out[1] = (float)(5.0 * l_iou);
    out[2] = (float)l_obj;
    out[3] = (float)l_cls;
    out[4] = (float)l_l1;
    out[5] = (float)(num_fg / (double)(num_gts > 1 ? num_gts : 1));
  }
}

// ---- 7. backward of the loss (autograd of tal_head.py:426-461 as run by double_trainer.py:114).
// The assignment, the matched IoUs (class targets) and the TAL weights are constants of the backward pass
// (tal_head.py:479 @no_grad, weights detached), so every anchor contributes independently:
//   d 5*L_iou / d box   = 5 * (w_i * S / SW) / N * d(1 - IoU^2)/d box          (fg anchors)
//   d L_obj  / d logit  = (sigmoid(x) - [fg]) / N                              (all anchors)
//   d L_cls  / d logit  = (sigmoid(x) - onehot * IoU_matched) / N              (fg anchors)
//   d L_l1   / d origin = (w_i * S1 / SW1) / N * sign(origin - target)         (fg anchors, use_l1)
// with N = max(N_fg, 1) and the sums S, SW, S1, SW1 left in the workspace by sy_tal_loss.
struct LossBwdArgs {
  const float* outputs; const float* origin; const float* fut; const float* tal;
  const int* mres; const float* piou; const double* tot;
  Levels lv; int A, L, NC; float gamma; int use_l1; float gscale;
  float* g_out; float* g_origin; float* g_raw;
};

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
// d max(a, b) / d a as torch.maximum differentiates it (ties split evenly)
__device__ __forceinline__ float dmax_a(float a, float b) { return a > b ? 1.f : (a == b ? 0.5f : 0.f); }
__device__ __forceinline__ float dmin_a(float a, float b) { return a < b ? 1.f : (a == b ? 0.5f : 0.f); }

__global__ void k_loss_backward(const LossBwdArgs q) {
  const int b = blockIdx.y, a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= q.A) return;
  const size_t ba = (size_t)b * q.A + a;
  const int no = 5 + q.NC;
  const float* o = q.outputs + ba * no;
  const double nfg_raw = q.tot[6];
  const float inv_n = (float)(1.0 / (nfg_raw > 1.0 ? nfg_raw : 1.0)) * q.gscale;
  const int mg = q.mres[ba];
  const bool fg = mg >= 0;
  float gbox[4] = {0.f, 0.f, 0.f, 0.f}, gorg[4] = {0.f, 0.f, 0.f, 0.f};
  const float gobj = (sigmoidf_(o[4]) - (fg ? 1.f : 0.f)) * inv_n;
  float gs = 1.f, gx = 0.f, gy = 0.f;
  anchor_geom(q.lv, a, &gx, &gy, &gs);
  if (fg) {
    const float* r = q.fut + ((size_t)b * q.L + mg) * 5;
    const Box t{r[1], r[2], r[3], r[4]}, p{o[0], o[1], o[2], o[3]};
    const float tt = q.tal[(size_t)b * q.L + mg];
    const float w = 1.0f / (((q.gamma == 1.0f) ? tt : powf(tt, q.gamma)) + 1e-8f);
    // IoU loss
    {
      const float wi = (float)((double)w * q.tot[0] / q.tot[1]);       // w * S / SW
      const float pl = p.cx - p.w / 2.f, tl_ = t.cx - t.w / 2.f, pr = p.cx + p.w / 2.f, tr = t.cx + t.w / 2.f;
      const float pt = p.cy - p.h / 2.f, tt_ = t.cy - t.h / 2.f, pb = p.cy + p.h / 2.f, tb = t.cy + t.h / 2.f;
      const float tlx = fmaxf(pl, tl_), brx = fminf(pr, tr), tly = fmaxf(pt, tt_), bry = fminf(pb, tb);
      const float en = (tlx < brx && tly < bry) ? 1.f : 0.f;
      const float iw = brx - tlx, ih = bry - tly;
      const float ai = iw * ih * en;
      const float au = p.w * p.h + t.w * t.h - ai;
      const float den = au + 1e-16f;
      const float iou = ai / den;
      const float dl_diou = -2.f * iou * 5.f * wi * inv_n;             // d(5 * wi * (1 - iou^2) / N) / d iou
      const float diou_dai = 1.f / den + ai / (den * den);             // union depends on the intersection too
      const float diou_dap = -ai / (den * den);                        // through the predicted box area
      const float g_ai = dl_diou * diou_dai, g_ap = dl_diou * diou_dap;
      const float g_tlx = -g_ai * ih * en, g_brx = g_ai * ih * en, g_tly = -g_ai * iw * en, g_bry = g_ai * iw * en;
      const float a_tlx = g_tlx * dmax_a(pl, tl_), a_brx = g_brx * dmin_a(pr, tr);
      const float a_tly = g_tly * dmax_a(pt, tt_), a_bry = g_bry * dmin_a(pb, tb);
      gbox[0] = a_tlx + a_brx;
      gbox[1] = a_tly + a_bry;
      gbox[2] = 0.5f * (a_brx - a_tlx) + g_ap * p.h;
      gbox[3] = 0.5f * (a_bry - a_tly) + g_ap * p.w;
    }
    if (q.use_l1) {
      const float w1 = (float)((double)w * q.tot[2] / q.tot[3]) * inv_n;
      const float* og = q.origin + ba * 4;
      const float tg[4] = {t.cx / gs - gx, t.cy / gs - gy, logf(t.w / gs + 1e-8f), logf(t.h / gs + 1e-8f)};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float dlt = og[i] - tg[i];
        gorg[i] = w1 * (dlt > 0.f ? 1.f : (dlt < 0.f ? -1.f : 0.f));
      }
    }
  }
  const int gcls = fg ? (int)q.fut[((size_t)b * q.L + mg) * 5] : -1;
  const float piou = fg ? q.piou[ba] : 0.f;
  if (q.g_out) {
    float* g = q.g_out + ba * no;
    g[0] = gbox[0]; g[1] = gbox[1]; g[2] = gbox[2]; g[3] = gbox[3]; g[4] = gobj;
    for (int k = 0; k < q.NC; ++k) g[5 + k] = fg ? (sigmoidf_(o[5 + k]) - (k == gcls ? piou : 0.f)) * inv_n : 0.f;
  }
  if (q.g_origin) {
    float* g = q.g_origin + ba * 4;
    g[0] = gorg[0]; g[1] = gorg[1]; g[2] = gorg[2]; g[3] = gorg[3];
  }
  if (q.g_raw) {
    // decode chain (tal_head.py:237-241): box_xy = (raw_xy + grid) * stride, box_wh = exp(raw_wh) * stride = o[2:4];
    // origin_preds is the raw regression output itself (tal_head.py:185-194)
    float* g = q.g_raw + ba * no;
    g[0] = gbox[0] * gs + gorg[0];
    g[1] = gbox[1] * gs + gorg[1];
    g[2] = gbox[2] * o[2] + gorg[2];
    g[3] = gbox[3] * o[3] + gorg[3];
    g[4] = gobj;
    for (int k = 0; k < q.NC; ++k) g[5 + k] = fg ? (sigmoidf_(o[5 + k]) - (k == gcls ? piou : 0.f)) * inv_n : 0.f;
  }
}

}  // namespace sy

using namespace sy;

extern "C" int sy_head_pred_decode(const SyHeadPredDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  SY_REQUIRE(view_ok(d->cls_feat) && view_ok(d->reg_feat), SY_EINVAL, "head_pred: bad feature views");
  const SyTensor& f = d->cls_feat;
  SY_REQUIRE(d->reg_feat.n == f.n && d->reg_feat.h == f.h && d->reg_feat.w == f.w && d->reg_feat.c == f.c, SY_EINVAL,
             "head_pred: cls/reg feature mismatch");
  SY_REQUIRE(d->num_classes >= 1 && d->num_classes <= 251 && d->out && d->w_reg && d->w_obj && d->w_cls && d->b_reg &&
                 d->b_obj && d->b_cls,
             SY_EINVAL, "head_pred: null weights or num_classes out of range");
  SY_REQUIRE(d->anchor_offset >= 0 && d->anchor_offset + f.h * f.w <= d->a_total, SY_EINVAL, "head_pred: anchor range");
  SY_REQUIRE((f.c % 8) == 0 && sizeof(float) * (5 + d->num_classes) * f.c <= 200 * 1024, SY_EINVAL,
             "head_pred: %d channels x %d outputs do not fit the shared-memory weight tile", f.c, 5 + d->num_classes);
  SY_REQUIRE(d->storage == SY_STORAGE_BF16 || d->storage == SY_STORAGE_F16, SY_EINVAL, "head_pred: storage %d unsupported",
             d->storage);
  return d->storage == SY_STORAGE_F16 ? launch_head_pred_classes<true>(d, f, stream) : launch_head_pred_classes<false>(d, f, stream);
}

extern "C" size_t sy_tal_loss_workspace_bytes(int32_t b, int32_t a_total, int32_t max_labels, int32_t num_classes) {
  return carve(nullptr, b, a_total, max_labels, num_classes).bytes;
}

extern "C" int sy_tal_loss(const SyTalLossDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  SY_REQUIRE(d->b > 0 && d->a_total > 0 && d->max_labels > 0 && d->num_classes > 0 && d->n_levels >= 1 && d->n_levels <= 4,
             SY_EINVAL, "tal_loss: bad sizes");
  SY_REQUIRE(d->outputs && d->labels_fut && d->labels_cur && d->loss_out && d->workspace, SY_EINVAL, "tal_loss: null pointer");
  SY_REQUIRE(!d->use_l1 || d->origin, SY_EINVAL, "tal_loss: use_l1 needs origin preds");
  Levels lv{};
  lv.n = d->n_levels;
  int asum = 0;
  for (int l = 0; l < d->n_levels; ++l) {
    lv.h[l] = d->level_h[l]; lv.w[l] = d->level_w[l]; lv.s[l] = d->level_stride[l];
    asum += lv.h[l] * lv.w[l];
  }
  SY_REQUIRE(asum == d->a_total, SY_EINVAL, "tal_loss: levels give %d anchors, a_total=%d", asum, d->a_total);
  const int B = d->b, A = d->a_total, L = d->max_labels, NC = d->num_classes;
  LossWs w = carve(d->workspace, B, A, L, NC);
  SY_REQUIRE(d->workspace_bytes >= w.bytes, SY_EWORKSPACE, "tal_loss: workspace %zu < %zu", d->workspace_bytes, w.bytes);
  SY_REQUIRE(((uintptr_t)d->workspace % 256) == 0, SY_EINVAL, "tal_loss: workspace must be 256B aligned");
  SY_CUDA(cudaMemsetAsync(w.cnt, 0, sizeof(int) * (size_t)B * A, stream));
  k_labels<<<B, 128, 0, stream>>>(d->labels_fut, d->labels_cur, L, d->ignore_thr, d->ignore_value, w.ngt, w.nsup, w.tal);
  const int ab = cdiv(A, kLossThreads);
  k_anchor_prep<<<dim3(ab, B), kLossThreads, 0, stream>>>(d->outputs, d->labels_fut, w.ngt, lv, A, L, NC, w.cand, w.clsterm);
  k_pair<<<dim3(ab, L, B), kLossThreads, 0, stream>>>(d->outputs, d->labels_fut, w.ngt, w.cand, w.clsterm, lv, A, L, NC,
                                                      w.iou, w.cost);
  const size_t row_bytes = 2 * sizeof(float) * (size_t)A;       // candidate values + anchor indices
  SY_REQUIRE(row_bytes <= 200 * 1024, SY_EINVAL, "tal_loss: %d anchors exceed the shared-memory row", A);
  if (row_bytes > 48 * 1024) SY_CUDA(cudaFuncSetAttribute(k_dynk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)row_bytes));
  k_dynk<<<dim3(L, B), 1024, row_bytes, stream>>>(w.ngt, w.cand, w.iou, w.cost, A, L, w.cnt, w.match);
  LossArgs q{};
  q.outputs = d->outputs; q.origin = d->origin; q.fut = d->labels_fut; q.ngt = w.ngt; q.tal = w.tal;
  q.iou_m = w.iou; q.cost_m = w.cost; q.cnt = w.cnt; q.match = w.match; q.lv = lv; q.A = A; q.L = L; q.NC = NC;
  q.gamma = d->gamma; q.use_l1 = d->use_l1; q.part = w.part;
  q.fg_out = d->fg_out; q.matched_out = d->matched_out; q.piou_out = d->pred_iou_out;
  q.mres = w.mres; q.piou_ws = w.piou;
  k_resolve_loss<<<dim3(ab, B), kLossThreads, 0, stream>>>(q);
  k_final<<<1, 256, 0, stream>>>(w.part, ab * B, w.ngt, B, d->use_l1, d->loss_out, w.tot);
  return launch_status("tal_loss kernels");
}

extern "C" int sy_tal_loss_backward(const SyTalLossBwdDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  SY_REQUIRE(d->b > 0 && d->a_total > 0 && d->max_labels > 0 && d->num_classes > 0 && d->n_levels >= 1 && d->n_levels <= 4,
             SY_EINVAL, "tal_loss_backward: bad sizes");
  SY_REQUIRE(d->outputs && d->labels_fut && d->workspace, SY_EINVAL, "tal_loss_backward: null pointer");
  SY_REQUIRE(!d->use_l1 || d->origin, SY_EINVAL, "tal_loss_backward: use_l1 needs origin preds");
  SY_REQUIRE(d->grad_outputs || d->grad_origin || d->grad_raw, SY_EINVAL, "tal_loss_backward: no gradient requested");
  Levels lv{};
  lv.n = d->n_levels;
  int asum = 0;
  for (int l = 0; l < d->n_levels; ++l) {
    lv.h[l] = d->level_h[l]; lv.w[l] = d->level_w[l]; lv.s[l] = d->level_stride[l];
    asum += lv.h[l] * lv.w[l];
  }
  SY_REQUIRE(asum == d->a_total, SY_EINVAL, "tal_loss_backward: levels give %d anchors, a_total=%d", asum, d->a_total);
  LossWs w = carve(d->workspace, d->b, d->a_total, d->max_labels, d->num_classes);
  SY_REQUIRE(d->workspace_bytes >= w.bytes, SY_EWORKSPACE, "tal_loss_backward: workspace %zu < %zu", d->workspace_bytes, w.bytes);
  LossBwdArgs q{};
  q.outputs = d->outputs; q.origin = d->origin; q.fut = d->labels_fut; q.tal = w.tal;
  q.mres = w.mres; q.piou = w.piou; q.tot = w.tot; q.lv = lv; q.A = d->a_total; q.L = d->max_labels; q.NC = d->num_classes;
  q.gamma = d->gamma; q.use_l1 = d->use_l1; q.gscale = d->grad_scale;
  q.g_out = d->grad_outputs; q.g_origin = d->grad_origin; q.g_raw = d->grad_raw;
  k_loss_backward<<<dim3(cdiv(d->a_total, kLossThreads), d->b), kLossThreads, 0, stream>>>(q);
  return launch_status("k_loss_backward");
}
