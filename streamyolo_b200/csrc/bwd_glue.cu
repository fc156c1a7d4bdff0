// Small backward kernels around the convolutions (autograd of the reference's graph under loss.backward(),
// /root/reference/exps/train_utils/double_trainer.py:114):
//   * sy_dilate2            zero-insertion of a stride-2 conv's output gradient, so that its data gradient is the stride-1
//                           forward kernel on the flipped filter (dark2..dark5 first convs, bu_conv1/2)
//   * sy_upsample_nearest_backward   F.interpolate(mode="nearest") backward (dfp_pafpn.py:126,131): each source pixel sums
//                           the destination pixels that read it (same fp32 index expression as the forward)
//   * sy_head_pred_backward the three 1x1 prediction convs of a head level (tal_head.py:101-131): data gradient into the
//                           cls / reg tower outputs, weight + bias gradients (two-stage, fixed-order reduction)
//   * sy_head_pred_backward_wide    the same for any class count the forward takes (COCO's 80 included): shared-memory
//                           weight tile, outputs tiled in groups of 32 so that no accumulator array grows with the class count
#include <math.h>

#include "common.cuh"

namespace sy {

__device__ __forceinline__ void unpack8g(const uint4& v, float* f) {
  f[0] = bf16_lo(v.x); f[1] = bf16_hi(v.x); f[2] = bf16_lo(v.y); f[3] = bf16_hi(v.y);
  f[4] = bf16_lo(v.z); f[5] = bf16_hi(v.z); f[6] = bf16_lo(v.w); f[7] = bf16_hi(v.w);
}

// D[n, 2i, 2j, :] = g[n, i, j, :], zero elsewhere; D is [n, H, W, c] with H in {2h-1, 2h}, W in {2w-1, 2w}
__global__ void dilate2_kernel(const __nv_bfloat16* g, long long gp, int N, int h, int w, __nv_bfloat16* D, long long dp, int H,
                               int W, int C) {
  // one block pass per output row (n, y); threads walk (x, chunk) with 32-bit index arithmetic
  const int G = C / 8;
  const int rows = N * H, per_row = W * G;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const int n = row / H, y = row - n * H;
    const bool yrow = ((y & 1) == 0) && ((y >> 1) < h);
    const __nv_bfloat16* src = g + ((long long)n * h + (y >> 1)) * w * gp;
    __nv_bfloat16* dst = D + (long long)row * W * dp;
    for (int e = threadIdx.x; e < per_row; e += blockDim.x) {
      const int x = e / G, cg = e - x * G;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (yrow && (x & 1) == 0 && (x >> 1) < w) v = *reinterpret_cast<const uint4*>(src + (long long)(x >> 1) * gp + cg * 8);
      *reinterpret_cast<uint4*>(dst + (long long)x * dp + cg * 8) = v;
    }
  }
}

// dx[n, iy, ix] = sum of dy[n, oy, ox] over the destination pixels with src(oy) == iy, src(ox) == ix
__global__ void upsample_nearest_bwd_kernel(const __nv_bfloat16* dy, long long dyp, int N, int Ho, int Wo, __nv_bfloat16* dx,
                                            long long dxp, int Hi, int Wi, int C) {
  const int G = C / 8;
  const float sh = (float)Hi / (float)Ho, sw = (float)Wi / (float)Wo;
  const long long total = (long long)N * Hi * Wi * G;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(idx % G);
    const long long pix = idx / G;
    const int ix = (int)(pix % Wi), iy = (int)((pix / Wi) % Hi);
    const int n = (int)(pix / ((long long)Wi * Hi));
    // candidate destination rows / columns: a window around iy / sh that certainly contains every match
    const int oy0 = max(0, (int)floorf((float)iy / sh) - 2), oy1 = min(Ho - 1, (int)ceilf((float)(iy + 1) / sh) + 2);
    const int ox0 = max(0, (int)floorf((float)ix / sw) - 2), ox1 = min(Wo - 1, (int)ceilf((float)(ix + 1) / sw) + 2);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int oy = oy0; oy <= oy1; ++oy) {
      if (min((int)floorf(__fmul_rn((float)oy, sh)), Hi - 1) != iy) continue;
      for (int ox = ox0; ox <= ox1; ++ox) {
        if (min((int)floorf(__fmul_rn((float)ox, sw)), Wi - 1) != ix) continue;
        float f[8];
        unpack8g(*reinterpret_cast<const uint4*>(dy + (((long long)n * Ho + oy) * Wo + ox) * dyp + cg * 8), f);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += f[i];
      }
    }
    *reinterpret_cast<uint4*>(dx + pix * dxp + cg * 8) =
        make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]), pack_bf16(acc[4], acc[5]), pack_bf16(acc[6], acc[7]));
  }
}

// ---- head prediction convs: out[a][o] = sum_c feat_o[a][c] * w[o][c] + b[o], o = reg(4) | obj(1) | cls(NC);
//      reg and obj read the reg tower output, cls reads the cls tower output
struct HeadBwdArgs {
  const float* g;          // [B][a_total][NO] gradient w.r.t. the raw outputs
  const __nv_bfloat16* cf; long long cfp;
  const __nv_bfloat16* rf; long long rfp;
  const float* w_reg; const float* w_obj; const float* w_cls;
  int B, H, W, C, NO, a_total, anchor_offset;
  __nv_bfloat16* dcf; long long dcfp;
  __nv_bfloat16* drf; long long drfp;
  float* partial;          // [nblk][NO][C + 1]  (last column: bias)
};

__global__ void head_pred_bwd_data_kernel(const HeadBwdArgs q) {
  // a thread keeps its 8-channel chunk (its 2 x NO x 8 weights stay in L1) and walks the pixels; 32-bit index arithmetic
  const int G = q.C / 8;
  const int HW = q.H * q.W;
  const int npix = q.B * HW;
  const int ppb = (int)blockDim.x / G;             // G <= 256 (C <= 2048, checked by the host)
  const int prow = (int)threadIdx.x / G, cg = (int)threadIdx.x - prow * G;
  if (prow >= ppb) return;
  for (int pix = blockIdx.x * ppb + prow; pix < npix; pix += gridDim.x * ppb) {
    const int b = pix / HW;
    const long long a = (long long)b * q.a_total + q.anchor_offset + (pix - b * HW);
    const float* g = q.g + a * q.NO;
    float dr[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, dc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int o = 0; o < q.NO; ++o) {
      const float gv = g[o];
      const float* wrow = (o < 4) ? q.w_reg + (size_t)o * q.C : (o == 4 ? q.w_obj : q.w_cls + (size_t)(o - 5) * q.C);
      float* dst = (o < 5) ? dr : dc;
#pragma unroll
      for (int i = 0; i < 8; ++i) dst[i] += gv * wrow[cg * 8 + i];
    }
    *reinterpret_cast<uint4*>(q.drf + (long long)pix * q.drfp + cg * 8) =
        make_uint4(pack_bf16(dr[0], dr[1]), pack_bf16(dr[2], dr[3]), pack_bf16(dr[4], dr[5]), pack_bf16(dr[6], dr[7]));
    *reinterpret_cast<uint4*>(q.dcf + (long long)pix * q.dcfp + cg * 8) =
        make_uint4(pack_bf16(dc[0], dc[1]), pack_bf16(dc[2], dc[3]), pack_bf16(dc[4], dc[5]), pack_bf16(dc[6], dc[7]));
  }
}

constexpr int kHeadBwdPix = 256;      // pixels per partial row
// block = one chunk of pixels; thread t owns channels t, t + 256, ...; partial[blk][o][c] = sum_p g[p][o] * feat_o[p][c]
// NO (5 + classes) is a template parameter so that the accumulators stay in registers (a runtime bound put them in local
// memory: 227 us per launch at 8 x 75 x 120 anchors); 0 = generic runtime bound for unusual class counts.
template <int TNO>
__global__ void __launch_bounds__(256) head_pred_bwd_weight_kernel(const HeadBwdArgs q) {
  extern __shared__ float gsm[];       // [kHeadBwdPix][NO]
  const int NO = TNO > 0 ? TNO : q.NO;
  const long long npix = (long long)q.B * q.H * q.W;
  const long long p0 = (long long)blockIdx.x * kHeadBwdPix;
  const int np = (int)min((long long)kHeadBwdPix, npix - p0);
  for (int i = threadIdx.x; i < np * q.NO; i += blockDim.x) {
    const long long pix = p0 + i / q.NO;
    const int b = (int)(pix / ((long long)q.H * q.W));
    const long long a = (long long)b * q.a_total + q.anchor_offset + (pix - (long long)b * q.H * q.W);
    gsm[i] = q.g[a * q.NO + i % q.NO];
  }
  __syncthreads();
  float* out = q.partial + (size_t)blockIdx.x * NO * (q.C + 1);
  for (int c = threadIdx.x; c < q.C; c += blockDim.x) {
    constexpr int kA = TNO > 0 ? TNO : 32;
    float acc[kA];
#pragma unroll
    for (int o = 0; o < kA; ++o) acc[o] = 0.f;
    // eight pixels per pass: their 16 feature loads are issued before the first FMA (one global-memory round trip per pass;
    // one pixel per iteration left the 256 iterations latency-bound: 141 us per launch); same order of the sums
    constexpr int kPB = 8;
    for (int pp = 0; pp < np; pp += kPB) {
      float r[kPB], cv[kPB];
#pragma unroll
      for (int j = 0; j < kPB; ++j) {
        const bool in = pp + j < np;
        r[j] = in ? __bfloat162float(q.rf[(p0 + pp + j) * q.rfp + c]) : 0.f;
        cv[j] = in ? __bfloat162float(q.cf[(p0 + pp + j) * q.cfp + c]) : 0.f;
      }
#pragma unroll
      for (int j = 0; j < kPB; ++j) {
        if (pp + j < np) {
          const float* g = gsm + (pp + j) * NO;
#pragma unroll
          for (int o = 0; o < kA; ++o)
            if (TNO > 0 || o < NO) acc[o] += g[o] * (o < 5 ? r[j] : cv[j]);
        }
      }
    }
#pragma unroll
    for (int o = 0; o < kA; ++o)
      if (TNO > 0 || o < NO) out[(size_t)o * (q.C + 1) + c] = acc[o];
  }
  if (threadIdx.x < NO) {              // bias gradient of this chunk
    float s = 0.f;
    for (int pp = 0; pp < np; ++pp) s += gsm[pp * NO + threadIdx.x];
    out[(size_t)threadIdx.x * (q.C + 1) + q.C] = s;
  }
}

// dW rows in the nn.Conv2d layouts: reg [4][C], obj [1][C], cls [NC][C]; biases [4], [1], [NC]
__global__ void head_pred_bwd_finalize_kernel(const float* __restrict__ partial, int nblk, int NO, int C, float* dw_reg, float* dw_obj,
                                              float* dw_cls, float* db_reg, float* db_obj, float* db_cls, int accumulate) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= NO * (C + 1)) return;
  const int o = idx / (C + 1), c = idx % (C + 1);
  float s = 0.f;
  for (int b = 0; b < nblk; ++b) s += partial[(size_t)b * NO * (C + 1) + idx];
  float* dst;
  if (c < C) dst = (o < 4) ? dw_reg + (size_t)o * C + c : (o == 4 ? dw_obj + c : dw_cls + (size_t)(o - 5) * C + c);
  else dst = (o < 4) ? db_reg + o : (o == 4 ? db_obj : db_cls + (o - 5));
  *dst = accumulate ? *dst + s : s;
}

// ---- the same backward for any class count the forward takes (sy_head_pred_backward_wide): nothing grows with NO except
// the grid.  The data gradient keeps the whole [NO][C] weight tile in shared memory (the forward's own limit,
// (5 + nc) * C * 4 <= 200 KiB, sy_head_pred_decode) and gives each thread kWidePT pixels of one 8-channel chunk, so one
// shared-memory read of eight weights serves kWidePT pixels; the sums run over o = 0 .. NO-1 in the order of
// head_pred_bwd_data_kernel.
constexpr int kWidePT = 2;            // pixels per thread of the data gradient
constexpr int kWideOG = 32;           // outputs per block of the weight gradient
__global__ void __launch_bounds__(256) head_pred_bwd_data_wide_kernel(const HeadBwdArgs q) {
  extern __shared__ float wsm[];       // [NO][C]: reg(4), obj(1), cls(NO - 5)
  const int NO = q.NO, C = q.C;
  for (int i = threadIdx.x; i < NO * C; i += blockDim.x) {
    const int o = i / C, c = i - o * C;
    wsm[i] = (o < 4) ? q.w_reg[(size_t)o * C + c] : (o == 4 ? q.w_obj[c] : q.w_cls[(size_t)(o - 5) * C + c]);
  }
  __syncthreads();
  const int G = C / 8;
  const int HW = q.H * q.W;
  const int npix = q.B * HW;
  const int ppb = (int)blockDim.x / G;             // G <= 256 (C <= 2048, checked by the host)
  const int prow = (int)threadIdx.x / G, cg = (int)threadIdx.x - prow * G;
  if (prow >= ppb) return;
  const int step = gridDim.x * ppb * kWidePT;
  for (int pix0 = (blockIdx.x * ppb + prow) * kWidePT; pix0 < npix; pix0 += step) {
    const float* g[kWidePT];
#pragma unroll
    for (int j = 0; j < kWidePT; ++j) {
      const int pix = min(pix0 + j, npix - 1);     // past the end: recompute the last pixel, not stored
      const int b = pix / HW;
      g[j] = q.g + ((long long)b * q.a_total + q.anchor_offset + (pix - b * HW)) * NO;
    }
    float dr[kWidePT][8], dc[kWidePT][8];
#pragma unroll
    for (int j = 0; j < kWidePT; ++j)
#pragma unroll
      for (int i = 0; i < 8; ++i) { dr[j][i] = 0.f; dc[j][i] = 0.f; }
#pragma unroll
    for (int o = 0; o < 5; ++o) {
      const float4 w0 = *reinterpret_cast<const float4*>(wsm + o * C + cg * 8);
      const float4 w1 = *reinterpret_cast<const float4*>(wsm + o * C + cg * 8 + 4);
      const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int j = 0; j < kWidePT; ++j) {
        const float gv = g[j][o];
#pragma unroll
        for (int i = 0; i < 8; ++i) dr[j][i] += gv * w[i];
      }
    }
    for (int o = 5; o < NO; ++o) {
      const float4 w0 = *reinterpret_cast<const float4*>(wsm + o * C + cg * 8);
      const float4 w1 = *reinterpret_cast<const float4*>(wsm + o * C + cg * 8 + 4);
      const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int j = 0; j < kWidePT; ++j) {
        const float gv = g[j][o];
#pragma unroll
        for (int i = 0; i < 8; ++i) dc[j][i] += gv * w[i];
      }
    }
#pragma unroll
    for (int j = 0; j < kWidePT; ++j) {
      if (pix0 + j >= npix) break;
      const long long pix = pix0 + j;
      *reinterpret_cast<uint4*>(q.drf + pix * q.drfp + cg * 8) =
          make_uint4(pack_bf16(dr[j][0], dr[j][1]), pack_bf16(dr[j][2], dr[j][3]), pack_bf16(dr[j][4], dr[j][5]),
                     pack_bf16(dr[j][6], dr[j][7]));
      *reinterpret_cast<uint4*>(q.dcf + pix * q.dcfp + cg * 8) =
          make_uint4(pack_bf16(dc[j][0], dc[j][1]), pack_bf16(dc[j][2], dc[j][3]), pack_bf16(dc[j][4], dc[j][5]),
                     pack_bf16(dc[j][6], dc[j][7]));
    }
  }
}

// Weight gradient: block (x, y) = 256-pixel row x, outputs y * kWideOG ...; thread t owns channels t, t + 256, ... and
// kWideOG accumulators whatever NO is.  partial[x][o][c] as head_pred_bwd_weight_kernel writes it: each sum runs over the
// row's pixels in order, so head_pred_bwd_finalize_kernel's fixed-order reduction makes the result deterministic.
__global__ void __launch_bounds__(256) head_pred_bwd_weight_wide_kernel(const HeadBwdArgs q) {
  __shared__ __align__(16) float gsm[kHeadBwdPix][kWideOG];
  const int NO = q.NO;
  const int o0 = blockIdx.y * kWideOG;
  const int no = min(kWideOG, NO - o0);
  const long long npix = (long long)q.B * q.H * q.W;
  const long long p0 = (long long)blockIdx.x * kHeadBwdPix;
  const int np = (int)min((long long)kHeadBwdPix, npix - p0);
  for (int i = threadIdx.x; i < np * kWideOG; i += blockDim.x) {
    const int pp = i / kWideOG, o = i - pp * kWideOG;
    const long long pix = p0 + pp;
    const int b = (int)(pix / ((long long)q.H * q.W));
    const long long a = (long long)b * q.a_total + q.anchor_offset + (pix - (long long)b * q.H * q.W);
    gsm[pp][o] = o < no ? q.g[a * NO + o0 + o] : 0.f;
  }
  __syncthreads();
  const int n_reg = max(0, min(5 - o0, kWideOG));  // outputs of this group that read the reg tower (group 0 only)
  float* out = q.partial + (size_t)blockIdx.x * NO * (q.C + 1);
  for (int c = threadIdx.x; c < q.C; c += blockDim.x) {
    float acc[kWideOG];
#pragma unroll
    for (int o = 0; o < kWideOG; ++o) acc[o] = 0.f;
    // eight pixels per pass, their feature loads issued before the first FMA (head_pred_bwd_weight_kernel)
    constexpr int kPB = 8;
    for (int pp = 0; pp < np; pp += kPB) {
      float r[kPB], cv[kPB];
#pragma unroll
      for (int j = 0; j < kPB; ++j) {
        const bool in = pp + j < np;
        r[j] = in && n_reg > 0 ? __bfloat162float(q.rf[(p0 + pp + j) * q.rfp + c]) : 0.f;
        cv[j] = in ? __bfloat162float(q.cf[(p0 + pp + j) * q.cfp + c]) : 0.f;
      }
#pragma unroll
      for (int j = 0; j < kPB; ++j) {
        if (pp + j < np) {
          const float4* g4 = reinterpret_cast<const float4*>(gsm[pp + j]);
#pragma unroll
          for (int o4 = 0; o4 < kWideOG / 4; ++o4) {
            const float4 gv = g4[o4];
            const float gg[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[4 * o4 + i] += gg[i] * (4 * o4 + i < n_reg ? r[j] : cv[j]);
          }
        }
      }
    }
#pragma unroll
    for (int o = 0; o < kWideOG; ++o)
      if (o < no) out[(size_t)(o0 + o) * (q.C + 1) + c] = acc[o];
  }
  if (threadIdx.x < no) {              // bias gradient of this row
    float s = 0.f;
    for (int pp = 0; pp < np; ++pp) s += gsm[pp][threadIdx.x];
    out[(size_t)(o0 + threadIdx.x) * (q.C + 1) + q.C] = s;
  }
}

// y += x (bf16, fp32 add, one rounding): gradient accumulation where a tensor feeds several consumers (residual
// shortcuts, FPN features read by two branches, the DFP fusion's "+ cur")
__global__ void add_kernel(const __nv_bfloat16* x, long long xp, __nv_bfloat16* y, long long yp, long long npix, int C) {
  // a thread keeps its 16-byte channel chunk and walks the pixels (no per-element index division), two pairs in flight
  const int G = C / 8;
  auto add8 = [](const uint4& xa, const uint4& ya) {
    float a[8], b[8];
    unpack8g(xa, a);
    unpack8g(ya, b);
    return make_uint4(pack_bf16(a[0] + b[0], a[1] + b[1]), pack_bf16(a[2] + b[2], a[3] + b[3]), pack_bf16(a[4] + b[4], a[5] + b[5]),
                      pack_bf16(a[6] + b[6], a[7] + b[7]));
  };
  if (G <= (int)blockDim.x) {
    const int ppb = (int)blockDim.x / G;
    const int prow = (int)threadIdx.x / G, g = (int)threadIdx.x - prow * G;
    if (prow >= ppb) return;
    const long long step = (long long)gridDim.x * ppb;
    for (long long pix0 = (long long)blockIdx.x * ppb + prow; pix0 < npix; pix0 += 2 * step) {
      uint4 xa[2], ya[2];
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (pix0 + j * step < npix) {
          xa[j] = *reinterpret_cast<const uint4*>(x + (pix0 + j * step) * xp + g * 8);
          ya[j] = *reinterpret_cast<const uint4*>(y + (pix0 + j * step) * yp + g * 8);
        }
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (pix0 + j * step < npix) *reinterpret_cast<uint4*>(y + (pix0 + j * step) * yp + g * 8) = add8(xa[j], ya[j]);
    }
  } else {
    for (long long pix = blockIdx.x; pix < npix; pix += gridDim.x)
      for (int g = threadIdx.x; g < G; g += blockDim.x)
        *reinterpret_cast<uint4*>(y + pix * yp + g * 8) =
            add8(*reinterpret_cast<const uint4*>(x + pix * xp + g * 8), *reinterpret_cast<const uint4*>(y + pix * yp + g * 8));
  }
}

// ---- SPP max pools backward ([yolox] SPPBottleneck: MaxPool2d(k, stride 1, padding k/2), k = 5, 9, 13, each applied to
// the same x).  PyTorch routes a window's gradient to its FIRST maximum in row-major scan order (strict >): pass 1 records
// that position per output element and pool, pass 2 lets every input element gather the outputs that point at it
// (deterministic, no atomics).
__device__ __forceinline__ void gt8(const uint4& v, const uint4& m, bool* g) {
  float a[8], b[8];
  unpack8g(v, a);
  unpack8g(m, b);
#pragma unroll
  for (int i = 0; i < 8; ++i) g[i] = a[i] > b[i];
}

// amax[k][n][y][x][c] = (window row * 16 + window col) of the first maximum, as uint8 (13 x 13 windows fit)
__global__ void spp_argmax_kernel(const __nv_bfloat16* x, long long xp, int N, int H, int W, int C, uint8_t* amax) {
  const int G = C / 8;
  const long long total = (long long)N * H * W * G;
  const int ks[3] = {5, 9, 13};
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(idx % G);
    const long long pix = idx / G;
    const int px = (int)(pix % W), py = (int)((pix / W) % H);
    const int n = (int)(pix / ((long long)W * H));
    for (int kk = 0; kk < 3; ++kk) {
      const int r = ks[kk] / 2;
      float best[8];
      uint8_t pos[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) { best[i] = -INFINITY; pos[i] = 0; }
      for (int dy = -r; dy <= r; ++dy) {
        const int yy = py + dy;
        if (yy < 0 || yy >= H) continue;
        for (int dx = -r; dx <= r; ++dx) {
          const int xx = px + dx;
          if (xx < 0 || xx >= W) continue;
          float v[8];
          unpack8g(*reinterpret_cast<const uint4*>(x + (((long long)n * H + yy) * W + xx) * xp + cg * 8), v);
          const uint8_t code = (uint8_t)((dy + r) * 16 + (dx + r));
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (v[i] > best[i]) { best[i] = v[i]; pos[i] = code; }
        }
      }
      uint8_t* dst = amax + (((size_t)kk * N * H * W + pix) * C) + cg * 8;
      *reinterpret_cast<uint2*>(dst) = make_uint2(pos[0] | (pos[1] << 8) | (pos[2] << 16) | ((uint32_t)pos[3] << 24),
                                                  pos[4] | (pos[5] << 8) | (pos[6] << 16) | ((uint32_t)pos[7] << 24));
    }
  }
}

// dx[p] = sum over pools k and outputs o whose window contains p and whose recorded maximum is p of dy_k[o]
__global__ void spp_bwd_gather_kernel(const uint8_t* amax, const __nv_bfloat16* d5, long long p5, const __nv_bfloat16* d9, long long p9,
                                      const __nv_bfloat16* d13, long long p13, int N, int H, int W, int C, __nv_bfloat16* dx,
                                      long long dxp) {
  const int G = C / 8;
  const long long total = (long long)N * H * W * G;
  const int ks[3] = {5, 9, 13};
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(idx % G);
    const long long pix = idx / G;
    const int px = (int)(pix % W), py = (int)((pix / W) % H);
    const int n = (int)(pix / ((long long)W * H));
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int kk = 0; kk < 3; ++kk) {
      const int r = ks[kk] / 2;
      const __nv_bfloat16* dk = kk == 0 ? d5 : (kk == 1 ? d9 : d13);
      const long long dp = kk == 0 ? p5 : (kk == 1 ? p9 : p13);
      for (int oy = max(0, py - r); oy <= min(H - 1, py + r); ++oy) {
        for (int ox = max(0, px - r); ox <= min(W - 1, px + r); ++ox) {
          const long long opix = ((long long)n * H + oy) * W + ox;
          const uint2 pk = *reinterpret_cast<const uint2*>(amax + (((size_t)kk * N * H * W + opix) * C) + cg * 8);
          const uint8_t want = (uint8_t)((py - oy + r) * 16 + (px - ox + r));    // p's position inside o's window
          uint32_t any = 0;
          uint8_t code[8];
#pragma unroll
          for (int i = 0; i < 4; ++i) { code[i] = (pk.x >> (8 * i)) & 0xff; code[4 + i] = (pk.y >> (8 * i)) & 0xff; }
#pragma unroll
          for (int i = 0; i < 8; ++i) any |= (code[i] == want);
          if (!any) continue;
          float g[8];
          unpack8g(*reinterpret_cast<const uint4*>(dk + opix * dp + cg * 8), g);
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (code[i] == want) acc[i] += g[i];
        }
      }
    }
    *reinterpret_cast<uint4*>(dx + pix * dxp + cg * 8) =
        make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]), pack_bf16(acc[4], acc[5]), pack_bf16(acc[6], acc[7]));
  }
}

static inline int grid_cap(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b < (long long)sm_count() * 16 ? b : (long long)sm_count() * 16));
}

}  // namespace sy

using namespace sy;

extern "C" int sy_dilate2(SyTensor g, SyTensor D, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(view_ok(g) && view_ok(D) && g.n == D.n && g.c == D.c, SY_EINVAL, "dilate2: bad views");
  SY_REQUIRE((D.h == 2 * g.h || D.h == 2 * g.h - 1) && (D.w == 2 * g.w || D.w == 2 * g.w - 1), SY_EINVAL,
             "dilate2: output %dx%d does not match input %dx%d", D.h, D.w, g.h, g.w);
  const long long total = (long long)D.n * D.h * D.w * (D.c / 8);
  dilate2_kernel<<<grid_cap(total, 256), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(g.ptr), g.pitch, g.n, g.h, g.w,
                                                           reinterpret_cast<__nv_bfloat16*>(D.ptr), D.pitch, D.h, D.w, D.c);
  return launch_status("dilate2_kernel");
}

extern "C" int sy_upsample_nearest_backward(SyTensor dy, SyTensor dx, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(view_ok(dy) && view_ok(dx) && dy.n == dx.n && dy.c == dx.c, SY_EINVAL, "upsample_backward: bad views");
  const long long total = (long long)dx.n * dx.h * dx.w * (dx.c / 8);
  upsample_nearest_bwd_kernel<<<grid_cap(total, 256), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(dy.ptr), dy.pitch,
                                                                        dy.n, dy.h, dy.w, reinterpret_cast<__nv_bfloat16*>(dx.ptr),
                                                                        dx.pitch, dx.h, dx.w, dx.c);
  return launch_status("upsample_nearest_bwd_kernel");
}

extern "C" int sy_head_pred_bwd_rows(int32_t b, int32_t h, int32_t w) { return cdiv(b * h * w, kHeadBwdPix); }

extern "C" int sy_head_pred_backward(const SyHeadPredBwdDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  const SyTensor& f = d->cls_feat;
  SY_REQUIRE(view_ok(f) && view_ok(d->reg_feat) && view_ok(d->d_cls_feat) && view_ok(d->d_reg_feat), SY_EINVAL,
             "head_pred_backward: bad views");
  SY_REQUIRE(d->reg_feat.n == f.n && d->reg_feat.h == f.h && d->reg_feat.w == f.w && d->reg_feat.c == f.c &&
                 d->d_cls_feat.c == f.c && d->d_reg_feat.c == f.c && d->d_cls_feat.h == f.h && d->d_reg_feat.w == f.w,
             SY_EINVAL, "head_pred_backward: shape mismatch");
  SY_REQUIRE(d->num_classes >= 1 && d->num_classes <= 27, SY_EINVAL, "head_pred_backward: num_classes out of range");
  SY_REQUIRE(d->grad_raw && d->w_reg && d->w_obj && d->w_cls && d->dw_reg && d->dw_obj && d->dw_cls && d->db_reg && d->db_obj &&
                 d->db_cls && d->partials,
             SY_EINVAL, "head_pred_backward: null pointer");
  SY_REQUIRE(d->anchor_offset >= 0 && d->anchor_offset + f.h * f.w <= d->a_total, SY_EINVAL, "head_pred_backward: anchor range");
  const int rows = sy_head_pred_bwd_rows(f.n, f.h, f.w);
  SY_REQUIRE(d->n_partials >= rows, SY_EWORKSPACE, "head_pred_backward: %d partial rows, need %d", d->n_partials, rows);
  HeadBwdArgs q{};
  q.g = d->grad_raw;
  q.cf = reinterpret_cast<const __nv_bfloat16*>(f.ptr); q.cfp = f.pitch;
  q.rf = reinterpret_cast<const __nv_bfloat16*>(d->reg_feat.ptr); q.rfp = d->reg_feat.pitch;
  q.w_reg = d->w_reg; q.w_obj = d->w_obj; q.w_cls = d->w_cls;
  q.B = f.n; q.H = f.h; q.W = f.w; q.C = f.c; q.NO = 5 + d->num_classes; q.a_total = d->a_total; q.anchor_offset = d->anchor_offset;
  q.dcf = reinterpret_cast<__nv_bfloat16*>(d->d_cls_feat.ptr); q.dcfp = d->d_cls_feat.pitch;
  q.drf = reinterpret_cast<__nv_bfloat16*>(d->d_reg_feat.ptr); q.drfp = d->d_reg_feat.pitch;
  q.partial = d->partials;
  SY_REQUIRE(f.c % 8 == 0 && f.c <= 2048 && (long long)f.n * f.h * f.w < (1ll << 31), SY_EINVAL,
             "head_pred_backward: %d channels / %d x %d x %d pixels unsupported", f.c, f.n, f.h, f.w);
  const long long total = (long long)f.n * f.h * f.w * (f.c / 8);
  head_pred_bwd_data_kernel<<<grid_cap(total, 256), 256, 0, stream>>>(q);
  const size_t wsm = sizeof(float) * kHeadBwdPix * q.NO;
  switch (q.NO) {
    case 13: head_pred_bwd_weight_kernel<13><<<rows, 256, wsm, stream>>>(q); break;
    case 6: head_pred_bwd_weight_kernel<6><<<rows, 256, wsm, stream>>>(q); break;
    case 25: head_pred_bwd_weight_kernel<25><<<rows, 256, wsm, stream>>>(q); break;
    default: head_pred_bwd_weight_kernel<0><<<rows, 256, wsm, stream>>>(q); break;
  }
  const int n_out = q.NO * (f.c + 1);
  head_pred_bwd_finalize_kernel<<<cdiv(n_out, 256), 256, 0, stream>>>(d->partials, rows, q.NO, f.c, d->dw_reg, d->dw_obj, d->dw_cls,
                                                                     d->db_reg, d->db_obj, d->db_cls, d->accumulate);
  return launch_status("head_pred_backward kernels");
}

extern "C" int sy_head_pred_backward_wide(const SyHeadPredBwdDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  const SyTensor& f = d->cls_feat;
  SY_REQUIRE(view_ok(f) && view_ok(d->reg_feat) && view_ok(d->d_cls_feat) && view_ok(d->d_reg_feat), SY_EINVAL,
             "head_pred_backward_wide: bad views");
  SY_REQUIRE(d->reg_feat.n == f.n && d->reg_feat.h == f.h && d->reg_feat.w == f.w && d->reg_feat.c == f.c &&
                 d->d_cls_feat.n == f.n && d->d_cls_feat.h == f.h && d->d_cls_feat.w == f.w && d->d_cls_feat.c == f.c &&
                 d->d_reg_feat.n == f.n && d->d_reg_feat.h == f.h && d->d_reg_feat.w == f.w && d->d_reg_feat.c == f.c,
             SY_EINVAL, "head_pred_backward_wide: shape mismatch");
  SY_REQUIRE(d->num_classes >= 1 && d->num_classes <= 251, SY_EINVAL, "head_pred_backward_wide: num_classes out of range");
  SY_REQUIRE(f.c % 8 == 0 && sizeof(float) * (5 + d->num_classes) * f.c <= 200 * 1024, SY_EINVAL,
             "head_pred_backward_wide: %d channels x %d outputs do not fit the shared-memory weight tile", f.c,
             5 + d->num_classes);
  SY_REQUIRE(f.c <= 2048 && (long long)f.n * f.h * f.w <= (1ll << 30), SY_EINVAL,
             "head_pred_backward_wide: %d channels / %d x %d x %d pixels unsupported", f.c, f.n, f.h, f.w);
  SY_REQUIRE(d->grad_raw && d->w_reg && d->w_obj && d->w_cls && d->dw_reg && d->dw_obj && d->dw_cls && d->db_reg && d->db_obj &&
                 d->db_cls && d->partials,
             SY_EINVAL, "head_pred_backward_wide: null pointer");
  SY_REQUIRE(d->anchor_offset >= 0 && d->anchor_offset + f.h * f.w <= d->a_total, SY_EINVAL,
             "head_pred_backward_wide: anchor range");
  const int rows = sy_head_pred_bwd_rows(f.n, f.h, f.w);
  SY_REQUIRE(d->n_partials >= rows, SY_EWORKSPACE, "head_pred_backward_wide: %d partial rows, need %d", d->n_partials, rows);
  HeadBwdArgs q{};
  q.g = d->grad_raw;
  q.cf = reinterpret_cast<const __nv_bfloat16*>(f.ptr); q.cfp = f.pitch;
  q.rf = reinterpret_cast<const __nv_bfloat16*>(d->reg_feat.ptr); q.rfp = d->reg_feat.pitch;
  q.w_reg = d->w_reg; q.w_obj = d->w_obj; q.w_cls = d->w_cls;
  q.B = f.n; q.H = f.h; q.W = f.w; q.C = f.c; q.NO = 5 + d->num_classes; q.a_total = d->a_total; q.anchor_offset = d->anchor_offset;
  q.dcf = reinterpret_cast<__nv_bfloat16*>(d->d_cls_feat.ptr); q.dcfp = d->d_cls_feat.pitch;
  q.drf = reinterpret_cast<__nv_bfloat16*>(d->d_reg_feat.ptr); q.drfp = d->d_reg_feat.pitch;
  q.partial = d->partials;
  // data gradient: a resident grid (the weight tile is loaded once per block) walking groups of kWidePT pixels
  const size_t smem = sizeof(float) * q.NO * f.c;
  if (smem > 48 * 1024)
    SY_CUDA(cudaFuncSetAttribute(head_pred_bwd_data_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int per_sm = (int)((227 * 1024) / (smem + 1024));
  const int groups = cdiv(f.n * f.h * f.w, kWidePT * (256 / (f.c / 8)));
  const int blocks = min(groups, sm_count() * max(1, min(per_sm, 8)));
  head_pred_bwd_data_wide_kernel<<<blocks, 256, smem, stream>>>(q);
  head_pred_bwd_weight_wide_kernel<<<dim3(rows, cdiv(q.NO, kWideOG)), 256, 0, stream>>>(q);
  const int n_out = q.NO * (f.c + 1);
  head_pred_bwd_finalize_kernel<<<cdiv(n_out, 256), 256, 0, stream>>>(d->partials, rows, q.NO, f.c, d->dw_reg, d->dw_obj, d->dw_cls,
                                                                     d->db_reg, d->db_obj, d->db_cls, d->accumulate);
  return launch_status("head_pred_backward_wide kernels");
}

extern "C" int sy_add(SyTensor x, SyTensor y, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(view_ok(x) && view_ok(y) && x.n == y.n && x.h == y.h && x.w == y.w && x.c == y.c, SY_EINVAL, "add: view mismatch");
  const long long npix = (long long)x.n * x.h * x.w;
  add_kernel<<<grid_cap(npix * (x.c / 8), 256), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x.ptr), x.pitch,
                                                                 reinterpret_cast<__nv_bfloat16*>(y.ptr), y.pitch, npix, x.c);
  return launch_status("add_kernel");
}

extern "C" size_t sy_spp_maxpool_backward_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t c) {
  return (size_t)3 * n * h * w * c;
}

extern "C" int sy_spp_maxpool_backward(SyTensor x, SyTensor d5, SyTensor d9, SyTensor d13, SyTensor dx, void* workspace,
                                       size_t workspace_bytes, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(view_ok(x) && view_ok(d5) && view_ok(d9) && view_ok(d13) && view_ok(dx), SY_EINVAL, "spp_backward: bad views");
  SY_REQUIRE(d5.c == x.c && d9.c == x.c && d13.c == x.c && dx.c == x.c && d5.h == x.h && d5.w == x.w && d5.n == x.n &&
                 dx.h == x.h && dx.w == x.w && dx.n == x.n,
             SY_EINVAL, "spp_backward: shape mismatch");
  SY_REQUIRE(workspace != nullptr && workspace_bytes >= sy_spp_maxpool_backward_workspace_bytes(x.n, x.h, x.w, x.c) &&
                 ((uintptr_t)workspace % 16) == 0,
             SY_EWORKSPACE, "spp_backward: workspace too small or misaligned");
  const long long total = (long long)x.n * x.h * x.w * (x.c / 8);
  spp_argmax_kernel<<<grid_cap(total, 128), 128, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x.ptr), x.pitch, x.n, x.h, x.w,
                                                              x.c, reinterpret_cast<uint8_t*>(workspace));
  spp_bwd_gather_kernel<<<grid_cap(total, 128), 128, 0, stream>>>(
      reinterpret_cast<const uint8_t*>(workspace), reinterpret_cast<const __nv_bfloat16*>(d5.ptr), d5.pitch,
      reinterpret_cast<const __nv_bfloat16*>(d9.ptr), d9.pitch, reinterpret_cast<const __nv_bfloat16*>(d13.ptr), d13.pitch, x.n, x.h,
      x.w, x.c, reinterpret_cast<__nv_bfloat16*>(dx.ptr), dx.pitch);
  return launch_status("spp backward kernels");
}
