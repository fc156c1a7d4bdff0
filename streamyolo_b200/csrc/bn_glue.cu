// BatchNorm(train) finalize / apply+SiLU, nearest upsample, SPP max pools, strided copy, per-image select:
// vectorised (16-byte) HBM-bound kernels over NHWC bf16 views.  The upsample, the copy and the select only move 16-bit
// values and serve fp16 views unchanged; the SPP max pools compare values and have an fp16 instantiation (sy_spp_maxpool_f16).
#include <math.h>
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"

namespace sy {

// block = 32 channels x 32 row-lanes.  Deterministic: every thread sums a fixed strided subset of the
// partial rows in fp64, the 32 row-lanes are then combined in a fixed order.
__global__ void __launch_bounds__(1024)
bn_finalize_kernel(const float* __restrict__ partials, int P, int p_split, int groups,
                   double count, int C, const float* __restrict__ gamma,
                   const float* __restrict__ beta, float* running_mean, float* running_var,
                   long long* nbt, float momentum, float eps, float* scale_out, float* shift_out) {
  __shared__ double red[2][32][33];
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  if (blockIdx.x == 0 && threadIdx.x == 0 && nbt != nullptr) *nbt += groups;
  float rm = 0.f, rv = 1.f;
  if (rl == 0 && c < C) {
    rm = running_mean ? running_mean[c] : 0.f;
    rv = running_var ? running_var[c] : 1.f;
  }
  for (int g = 0; g < groups; ++g) {
    const int pa = (g == 0) ? 0 : p_split, pb = (g == 0 && groups > 1) ? p_split : P;
    double s1 = 0.0, s2 = 0.0;
    if (c < C) {
      for (int q = pa + rl; q < pb; q += 32) {
        s1 += (double)partials[(size_t)q * 2 * C + c];
        s2 += (double)partials[(size_t)q * 2 * C + C + c];
      }
    }
    red[0][rl][cl] = s1;
    red[1][rl][cl] = s2;
    __syncthreads();
    if (rl == 0 && c < C) {
      s1 = 0.0; s2 = 0.0;
      for (int r = 0; r < 32; ++r) { s1 += red[0][r][cl]; s2 += red[1][r][cl]; }
      const double mean = s1 / count;
      double var = s2 / count - mean * mean;
      if (var < 0.0) var = 0.0;
      const float sc = gamma[c] * (float)(1.0 / sqrt(var + (double)eps));
      scale_out[g * C + c] = sc;
      shift_out[g * C + c] = beta[c] - (float)mean * sc;
      const double unbiased = count > 1.0 ? var * (count / (count - 1.0)) : var;
      rm = (1.f - momentum) * rm + momentum * (float)mean;
      rv = (1.f - momentum) * rv + momentum * (float)unbiased;
    }
    __syncthreads();
  }
  if (rl == 0 && c < C) {
    if (running_mean) running_mean[c] = rm;
    if (running_var) running_var[c] = rv;
  }
}

__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  f[0] = bf16_lo(v.x); f[1] = bf16_hi(v.x); f[2] = bf16_lo(v.y); f[3] = bf16_hi(v.y);
  f[4] = bf16_lo(v.z); f[5] = bf16_hi(v.z); f[6] = bf16_lo(v.w); f[7] = bf16_hi(v.w);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}

// y = act(x * scale[grp] + shift[grp]) (+ res), act = the SY_ACT_* code ACT, 16 bytes (8 channels) per thread and pixel.
// A thread keeps ONE channel chunk for its whole life (scale/shift of both statistics groups live in registers, no
// per-element index division) and walks the pixels with kApplyUnroll independent 16-byte loads in flight.
constexpr int kApplyThreads = 256;
constexpr int kApplyUnroll = 4;
template <int ACT, bool RES>
__global__ void __launch_bounds__(kApplyThreads, 3)
bn_act_apply_kernel(const __nv_bfloat16* __restrict__ x, long long xp, const float* __restrict__ scale,
                    const float* __restrict__ shift, long long split_pix,
                    const __nv_bfloat16* res, long long rp, __nv_bfloat16* y, long long yp,
                    long long npix, int C, long long y_goff1, long long r_goff1) {
  pdl_launch_dependents();
  const int G = C >> 3;                           // 16-byte chunks per pixel (<= 256)
  const int ppb = kApplyThreads / G;              // pixels per block pass
  const int prow = (int)threadIdx.x / G, g = (int)threadIdx.x - prow * G;
  if (prow >= ppb) return;
  pdl_wait();                                     // x, scale, shift (and res) come from the preceding kernels
  // scale/shift of the statistics group the thread is currently in (pixels are ordered group 0 then group 1, so a
  // thread switches at most once)
  float sc[8], sh[8];
  int cur = -1;
  auto load_group = [&](int grp) {
    const float4* a = reinterpret_cast<const float4*>(scale + (long long)grp * C + g * 8);
    const float4* b = reinterpret_cast<const float4*>(shift + (long long)grp * C + g * 8);
    const float4 a0 = a[0], a1 = a[1], b0 = b[0], b1 = b[1];
    sc[0] = a0.x; sc[1] = a0.y; sc[2] = a0.z; sc[3] = a0.w; sc[4] = a1.x; sc[5] = a1.y; sc[6] = a1.z; sc[7] = a1.w;
    sh[0] = b0.x; sh[1] = b0.y; sh[2] = b0.z; sh[3] = b0.w; sh[4] = b1.x; sh[5] = b1.y; sh[6] = b1.z; sh[7] = b1.w;
    cur = grp;
  };
  const long long step = (long long)gridDim.x * ppb;
  const __nv_bfloat16* xg = x + g * 8;
  const __nv_bfloat16* rg = RES ? res + g * 8 : nullptr;
  __nv_bfloat16* yg = y + g * 8;
  for (long long pix0 = (long long)blockIdx.x * ppb + prow; pix0 < npix; pix0 += step * kApplyUnroll) {
    uint4 v[kApplyUnroll], rv[kApplyUnroll];
#pragma unroll
    for (int j = 0; j < kApplyUnroll; ++j) {
      const long long pix = pix0 + j * step;
      if (pix < npix) v[j] = *reinterpret_cast<const uint4*>(xg + pix * xp);
    }
    if (RES) {
#pragma unroll
      for (int j = 0; j < kApplyUnroll; ++j) {
        const long long pix = pix0 + j * step;
        if (pix < npix) rv[j] = *reinterpret_cast<const uint4*>(rg + pix * rp + (pix >= split_pix ? r_goff1 : 0));
      }
    }
#pragma unroll
    for (int j = 0; j < kApplyUnroll; ++j) {
      const long long pix = pix0 + j * step;
      if (pix >= npix) continue;
      const bool g1 = pix >= split_pix;
      if ((int)g1 != cur) load_group((int)g1);
      float f[8];
      unpack8(v[j], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float t = f[i] * sc[i] + sh[i];
        f[i] = act_f(ACT, t);
      }
      if (RES) {
        float r[8];
        unpack8(rv[j], r);
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] += r[i];
      }
      *reinterpret_cast<uint4*>(yg + pix * yp + (g1 ? y_goff1 : 0)) = pack8(f);
    }
  }
}

// PyTorch legacy "nearest": src = min((int)floorf(dst * scale), in - 1), scale = (float)in / out
// One block pass per output row (n, oy): the source row is resolved once, the threads walk (ox, chunk) with 32-bit index
// arithmetic (the first version did five 64-bit divisions per 16-byte chunk and was bound by them, not by memory).
__global__ void upsample_nearest_kernel(const __nv_bfloat16* __restrict__ x, long long xp, int N, int Hi, int Wi,
                                        __nv_bfloat16* y, long long yp, int Ho, int Wo, int C) {
  const int G = C / 8;
  const float sh = (float)Hi / (float)Ho, sw = (float)Wi / (float)Wo;
  const int rows = N * Ho, per_row = Wo * G;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const int n = row / Ho, oy = row - n * Ho;
    const int iy = min((int)floorf(__fmul_rn((float)oy, sh)), Hi - 1);
    const __nv_bfloat16* src = x + ((long long)n * Hi + iy) * Wi * xp;
    __nv_bfloat16* dst = y + (long long)row * Wo * yp;
    for (int e = threadIdx.x; e < per_row; e += blockDim.x) {
      const int ox = e / G, g = e - ox * G;
      const int ix = min((int)floorf(__fmul_rn((float)ox, sw)), Wi - 1);
      *reinterpret_cast<uint4*>(dst + (long long)ox * yp + g * 8) = *reinterpret_cast<const uint4*>(src + (long long)ix * xp + g * 8);
    }
  }
}

// element-wise maximum of eight packed bf16 (F16: fp16) values
template <bool F16>
__device__ __forceinline__ uint4 bmax(const uint4 a, const uint4 b) {
  using T2 = typename std::conditional<F16, __half2, __nv_bfloat162>::type;
  uint4 r;
  const T2* pa = reinterpret_cast<const T2*>(&a);
  const T2* pb = reinterpret_cast<const T2*>(&b);
  T2* pr = reinterpret_cast<T2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) pr[i] = __hmax2(pa[i], pb[i]);
  return r;
}

// stride-1 same-padded max pools k = 5, 9, 13 (-inf padding) as a cascade of separable 5-wide pools
// (5 o 5 = 9, 5 o 5 o 5 = 13 for max with -inf padding).  One block = one (image, 8-channel group) plane
// held in shared memory; every pass is a 5-tap row or column max on packed bf16 | fp16 (exact).
constexpr int kSppMaxPix = 1024;
template <bool F16>
__global__ void __launch_bounds__(256)
spp_maxpool_kernel(const __nv_bfloat16* __restrict__ x, long long xp, int H, int W, int C,
                   __nv_bfloat16* y5, long long p5, __nv_bfloat16* y9, long long p9,
                   __nv_bfloat16* y13, long long p13) {
  __shared__ uint4 bufA[kSppMaxPix], bufB[kSppMaxPix];
  const int G = C / 8;
  const int n = blockIdx.x / G, g = blockIdx.x % G;
  const int HW = H * W;
  const long long base = (long long)n * HW;
  for (int i = threadIdx.x; i < HW; i += blockDim.x)
    bufA[i] = *reinterpret_cast<const uint4*>(x + (base + i) * xp + g * 8);
  __syncthreads();
  __nv_bfloat16* outs[3] = {y5, y9, y13};
  const long long pitches[3] = {p5, p9, p13};
#pragma unroll 1
  for (int lvl = 0; lvl < 3; ++lvl) {
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {      // row pass
      const int yy = i / W, xx = i - yy * W;
      uint4 m = bufA[i];
#pragma unroll
      for (int d = -2; d <= 2; ++d)
        if (d != 0 && xx + d >= 0 && xx + d < W) m = bmax<F16>(m, bufA[i + d]);
      bufB[i] = m;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {      // column pass
      const int yy = i / W;
      uint4 m = bufB[i];
#pragma unroll
      for (int d = -2; d <= 2; ++d)
        if (d != 0 && yy + d >= 0 && yy + d < H) m = bmax<F16>(m, bufB[i + d * W]);
      bufA[i] = m;
      *reinterpret_cast<uint4*>(outs[lvl] + (base + i) * pitches[lvl] + g * 8) = m;
    }
    __syncthreads();
  }
}

// large planes (not used by the 600x960 configs): direct nested-window version
template <bool F16>
__global__ void spp_maxpool_direct_kernel(const __nv_bfloat16* __restrict__ x, long long xp, int N, int H, int W, int C,
                                          __nv_bfloat16* y5, long long p5, __nv_bfloat16* y9, long long p9,
                                          __nv_bfloat16* y13, long long p13) {
  const int G = C / 8;
  const long long total = (long long)N * H * W * G;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(idx % G);
    const long long pix = idx / G;
    const int ox = (int)(pix % W), oy = (int)((pix / W) % H);
    const int n = (int)(pix / ((long long)W * H));
    uint4 m5 = *reinterpret_cast<const uint4*>(x + pix * xp + g * 8), m9 = m5, m13 = m5;
    for (int dy = -6; dy <= 6; ++dy) {
      const int iy = oy + dy;
      if (iy < 0 || iy >= H) continue;
      for (int dx = -6; dx <= 6; ++dx) {
        const int ix = ox + dx;
        if (ix < 0 || ix >= W) continue;
        const uint4 v = *reinterpret_cast<const uint4*>(x + (((long long)n * H + iy) * W + ix) * xp + g * 8);
        m13 = bmax<F16>(m13, v);
        const int ad = max(abs(dy), abs(dx));
        if (ad <= 4) m9 = bmax<F16>(m9, v);
        if (ad <= 2) m5 = bmax<F16>(m5, v);
      }
    }
    *reinterpret_cast<uint4*>(y5 + pix * p5 + g * 8) = m5;
    *reinterpret_cast<uint4*>(y9 + pix * p9 + g * 8) = m9;
    *reinterpret_cast<uint4*>(y13 + pix * p13 + g * 8) = m13;
  }
}

// A thread keeps its 16-byte channel chunk and walks the pixels (no per-element index division), four copies in flight.
__global__ void copy_kernel(const __nv_bfloat16* __restrict__ x, long long xp, __nv_bfloat16* y, long long yp,
                            long long npix, int C) {
  const int G = C / 8;
  if (G <= (int)blockDim.x) {
    const int ppb = (int)blockDim.x / G;
    const int prow = (int)threadIdx.x / G, g = (int)threadIdx.x - prow * G;
    if (prow >= ppb) return;
    const long long step = (long long)gridDim.x * ppb;
    for (long long pix0 = (long long)blockIdx.x * ppb + prow; pix0 < npix; pix0 += 4 * step) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (pix0 + j * step < npix) v[j] = *reinterpret_cast<const uint4*>(x + (pix0 + j * step) * xp + g * 8);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (pix0 + j * step < npix) *reinterpret_cast<uint4*>(y + (pix0 + j * step) * yp + g * 8) = v[j];
    }
  } else {                                        // more than 2048 channels: one pixel per block pass
    for (long long pix = blockIdx.x; pix < npix; pix += gridDim.x)
      for (int g = threadIdx.x; g < G; g += blockDim.x)
        *reinterpret_cast<uint4*>(y + pix * yp + g * 8) = *reinterpret_cast<const uint4*>(x + pix * xp + g * 8);
  }
}

// Per-image select of up to three views in one launch (the FPN levels of a streaming tick): blockIdx.z = view pair,
// blockIdx.y = image.  The flag is read on the device, so a captured launch follows the flags the host writes before each
// replay; every block of an image whose flag is clear returns at once.  Inside an image it is copy_kernel's walk.
struct SelectPair {
  const __nv_bfloat16* x;
  __nv_bfloat16* y;
  long long xp, yp;            // pixel pitches (elements)
  long long x_img, y_img;      // image strides (elements)
  long long npix;              // pixels per image
  int C;
};
struct SelectArgs {
  SelectPair p[3];
};

__global__ void __launch_bounds__(256) select_images_kernel(const __grid_constant__ SelectArgs a,
                                                            const int32_t* __restrict__ flags) {
  if (flags[blockIdx.y] == 0) return;
  const SelectPair& p = a.p[blockIdx.z];
  const __nv_bfloat16* x = p.x + (long long)blockIdx.y * p.x_img;
  __nv_bfloat16* y = p.y + (long long)blockIdx.y * p.y_img;
  const long long npix = p.npix;
  const int G = p.C / 8;
  if (G <= (int)blockDim.x) {
    const int ppb = (int)blockDim.x / G;
    const int prow = (int)threadIdx.x / G, g = (int)threadIdx.x - prow * G;
    if (prow >= ppb) return;
    const long long step = (long long)gridDim.x * ppb;
    for (long long pix0 = (long long)blockIdx.x * ppb + prow; pix0 < npix; pix0 += 4 * step) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (pix0 + j * step < npix) v[j] = *reinterpret_cast<const uint4*>(x + (pix0 + j * step) * p.xp + g * 8);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (pix0 + j * step < npix) *reinterpret_cast<uint4*>(y + (pix0 + j * step) * p.yp + g * 8) = v[j];
    }
  } else {                                        // more than 2048 channels: one pixel per block pass
    for (long long pix = blockIdx.x; pix < npix; pix += gridDim.x)
      for (int g = threadIdx.x; g < G; g += blockDim.x)
        *reinterpret_cast<uint4*>(y + pix * p.yp + g * 8) = *reinterpret_cast<const uint4*>(x + pix * p.xp + g * 8);
  }
}

static inline int grid_for(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 16;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

}  // namespace sy

using namespace sy;
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)

extern "C" int sy_bn_finalize(const float* partials, int32_t n_partials, int32_t p_split, int32_t groups,
                              int64_t count_per_group, int32_t c, const float* gamma, const float* beta,
                              float* running_mean, float* running_var, int64_t* nbt, float momentum, float eps,
                              float* scale_out, float* shift_out, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(partials && gamma && beta && scale_out && shift_out, SY_EINVAL, "bn_finalize: null pointer");
  SY_REQUIRE(groups == 1 || groups == 2, SY_EINVAL, "bn_finalize: groups=%d", groups);
  SY_REQUIRE(n_partials > 0 && count_per_group > 0 && c > 0, SY_EINVAL, "bn_finalize: empty input");
  SY_REQUIRE(groups == 1 || (p_split > 0 && p_split < n_partials), SY_EINVAL, "bn_finalize: p_split=%d of %d", p_split,
             n_partials);
  bn_finalize_kernel<<<cdiv(c, 32), 1024, 0, stream>>>(partials, n_partials, p_split, groups, (double)count_per_group, c,
                                                       gamma, beta, running_mean, running_var,
                                                       reinterpret_cast<long long*>(nbt), momentum, eps, scale_out,
                                                       shift_out);
  return launch_status("bn_finalize_kernel");
}

extern "C" int sy_bn_act_apply(SyTensor x, const float* scale, const float* shift, int32_t split_n, int32_t act,
                               SyTensor res, SyTensor y, int64_t y_goff1, int64_t r_goff1, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(view_ok(x) && view_ok(y) && scale && shift, SY_EINVAL, "bn_act_apply: bad view");
  SY_REQUIRE(x.n == y.n && x.h == y.h && x.w == y.w && x.c == y.c, SY_EINVAL, "bn_act_apply: x/y shape mismatch");
  SY_REQUIRE(((uintptr_t)scale % 16) == 0 && ((uintptr_t)shift % 16) == 0, SY_EINVAL, "bn_act_apply: scale/shift alignment");
  SY_REQUIRE((y_goff1 % 8) == 0 && (r_goff1 % 8) == 0, SY_EINVAL, "bn_act_apply: group offsets must be multiples of 8");
  SY_REQUIRE(act_ok(act), SY_EINVAL, "bn_act_apply: act=%d is not an SY_ACT_* code", act);
  const __nv_bfloat16* rp = nullptr;
  long long rpitch = 0;
  if (res.ptr) {
    SY_REQUIRE(view_ok(res) && res.n == x.n && res.h == x.h && res.w == x.w && res.c == x.c, SY_EINVAL,
               "bn_act_apply: residual mismatch");
    rp = CBF(res.ptr); rpitch = res.pitch;
  }
  const long long npix = (long long)x.n * x.h * x.w;
  const long long split_pix = (long long)split_n * x.h * x.w;
  SY_REQUIRE(x.c <= 8 * kApplyThreads, SY_EINVAL, "bn_act_apply: C=%d > %d", x.c, 8 * kApplyThreads);
  const int ppb = kApplyThreads / (x.c / 8);
  // enough blocks for one pass of kApplyUnroll pixels per thread, capped at one wave of 3 resident blocks per SM
  const long long want = (npix + (long long)ppb * kApplyUnroll - 1) / ((long long)ppb * kApplyUnroll);
  const long long cap = (long long)sm_count() * 3;
  const int grid = (int)(want < 1 ? 1 : (want < cap ? want : cap));
  const bool has_res = rp != nullptr;
  auto launch = [&](auto kernel) -> int {
    // L1/shared split: measured on the whole step (StreamYOLO-l, 8 pairs): carveout 0 (all L1) 6.40 ms, default and
    // 100 (all shared, the conv kernels' split) 6.51 ms.
    SY_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 0));
    SY_CUDA(launch_pdl(kernel, dim3(grid), dim3(kApplyThreads), 0, stream, CBF(x.ptr), (long long)x.pitch, scale, shift,
                       split_pix, rp, rpitch, BF(y.ptr), (long long)y.pitch, npix, x.c, (long long)y_goff1,
                       (long long)r_goff1));
    return SY_OK;
  };
  auto go = [&](auto code) -> int {
    constexpr int A = decltype(code)::value;
    return has_res ? launch(bn_act_apply_kernel<A, true>) : launch(bn_act_apply_kernel<A, false>);
  };
  int rc;
  switch (act) {
    case SY_ACT_NONE: rc = go(std::integral_constant<int, SY_ACT_NONE>{}); break;
    case SY_ACT_SILU: rc = go(std::integral_constant<int, SY_ACT_SILU>{}); break;
    case SY_ACT_RELU: rc = go(std::integral_constant<int, SY_ACT_RELU>{}); break;
    default: rc = go(std::integral_constant<int, SY_ACT_LRELU>{}); break;
  }
  if (rc != SY_OK) return rc;
  return launch_status("bn_act_apply_kernel");
}

extern "C" int sy_upsample_nearest(SyTensor x, SyTensor y, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(view_ok(x) && view_ok(y) && x.n == y.n && x.c == y.c, SY_EINVAL, "upsample: bad views");
  const long long total = (long long)y.n * y.h * y.w * (y.c / 8);
  (void)total;
  const int up_rows = y.n * y.h;
  upsample_nearest_kernel<<<up_rows < sm_count() * 8 ? up_rows : sm_count() * 8, 256, 0, stream>>>(CBF(x.ptr), x.pitch, x.n, x.h, x.w, BF(y.ptr),
                                                                                     y.pitch, y.h, y.w, x.c);
  return launch_status("upsample_nearest_kernel");
}

template <bool F16>
static int spp_maxpool(SyTensor x, SyTensor y5, SyTensor y9, SyTensor y13, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(view_ok(x) && view_ok(y5) && view_ok(y9) && view_ok(y13), SY_EINVAL, "spp: bad views");
  SY_REQUIRE(y5.c == x.c && y9.c == x.c && y13.c == x.c && y5.h == x.h && y5.w == x.w && y5.n == x.n, SY_EINVAL,
             "spp: shape mismatch");
  if (x.h * x.w <= kSppMaxPix) {
    spp_maxpool_kernel<F16><<<x.n * (x.c / 8), 256, 0, stream>>>(CBF(x.ptr), x.pitch, x.h, x.w, x.c, BF(y5.ptr), y5.pitch,
                                                            BF(y9.ptr), y9.pitch, BF(y13.ptr), y13.pitch);
  } else {
    const long long total = (long long)x.n * x.h * x.w * (x.c / 8);
    spp_maxpool_direct_kernel<F16><<<grid_for(total, 128), 128, 0, stream>>>(CBF(x.ptr), x.pitch, x.n, x.h, x.w, x.c,
                                                                        BF(y5.ptr), y5.pitch, BF(y9.ptr), y9.pitch,
                                                                        BF(y13.ptr), y13.pitch);
  }
  return launch_status("spp_maxpool_kernel");
}

extern "C" int sy_spp_maxpool(SyTensor x, SyTensor y5, SyTensor y9, SyTensor y13, sy_stream_t stream) {
  return spp_maxpool<false>(x, y5, y9, y13, stream);
}

extern "C" int sy_spp_maxpool_f16(SyTensor x, SyTensor y5, SyTensor y9, SyTensor y13, sy_stream_t stream) {
  return spp_maxpool<true>(x, y5, y9, y13, stream);
}

extern "C" int sy_copy(SyTensor x, SyTensor y, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(view_ok(x) && view_ok(y) && x.n == y.n && x.h == y.h && x.w == y.w && x.c == y.c, SY_EINVAL,
             "copy: view mismatch");
  const long long npix = (long long)x.n * x.h * x.w;
  {
    const int G = x.c / 8, ppb = G <= 256 ? 256 / G : 1;
    const long long want = (npix + 4LL * ppb - 1) / (4LL * ppb);
    copy_kernel<<<(int)(want < 1 ? 1 : (want < sm_count() * 8 ? want : sm_count() * 8)), 256, 0, stream>>>(CBF(x.ptr), x.pitch, BF(y.ptr), y.pitch,
                                                                                          npix, x.c);
  }
  return launch_status("copy_kernel");
}

extern "C" int sy_select_images(const SySelectImagesDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->flags != nullptr && d->n_pairs >= 1 && d->n_pairs <= 3, SY_EINVAL,
             "select_images: needs device flags and 1-3 view pairs");
  SelectArgs a{};
  const int n = d->src[0].n;
  SY_REQUIRE(n >= 1 && n <= 65535, SY_EINVAL, "select_images: %d images (1..65535)", n);
  long long most = 1;                               // 16-byte chunks per image of the largest pair
  for (int k = 0; k < d->n_pairs; ++k) {
    const SyTensor s = d->src[k], t = d->dst[k];
    SY_REQUIRE(view_ok(s) && view_ok(t) && s.n == n && t.n == n && s.h == t.h && s.w == t.w && s.c == t.c, SY_EINVAL,
               "select_images: pair %d: bad or mismatched views", k);
    const long long npix = (long long)s.h * s.w;
    a.p[k] = SelectPair{CBF(s.ptr), BF(t.ptr), (long long)s.pitch, (long long)t.pitch, npix * s.pitch, npix * t.pitch,
                        npix, s.c};
    const long long chunks = npix * (s.c / 8);
    most = chunks > most ? chunks : most;
  }
  // one pass of 4 chunks per thread over the largest image; the smaller pairs' surplus blocks return at once
  const long long want = (most + 4LL * 256 - 1) / (4LL * 256);
  const int gx = (int)(want < 1024 ? want : 1024);
  select_images_kernel<<<dim3(gx, n, d->n_pairs), 256, 0, stream>>>(a, d->flags);
  return launch_status("select_images_kernel");
}
