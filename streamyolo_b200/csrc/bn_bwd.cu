// Backward of BatchNorm(train) + activation behind every [yolox] BaseConv (what autograd runs for loss.backward(),
// /root/reference/exps/train_utils/double_trainer.py:114):   y = act(z),  z = gamma * xhat + beta,
// xhat = (raw - mean_g) * invstd_g  with the batch statistics of the pixel's statistics group g (current / support frames,
// see DESIGN.md section 3), raw = the conv output.
//
//   dz      = dy * act'(z)        SiLU:  s (1 + z (1 - s)),  s = sigmoid(z)
//                                 ReLU:  z > 0 ? 1 : 0       LeakyReLU(0.1):  z > 0 ? 1 : 0.1     identity: 1
//   dbeta   = sum dz             dgamma = sum dz * xhat               (over both groups)
//   draw    = gamma * invstd_g * (dz - mean_g(dz) - xhat * mean_g(dz * xhat))
//
// Three launches: partial sums (up to 296 rows per statistics group so that the pass fills the GPU whatever the map size;
// deterministic, fixed order), a finalize (one warp per channel) that produces dgamma, dbeta and the per-(group, channel)
// coefficients, and the element-wise pass that writes draw in bf16 for the conv's data / weight gradient kernels.
// HBM-bound 16-byte accesses over NHWC bf16 views.  The reduce and apply kernels come in two instantiations: KINK = false
// (identity / SiLU, the element loop of the SiLU-only kernels unchanged) and KINK = true (ReLU / LeakyReLU: the
// derivative is a select on z > 0 with the launch's code, uniform across the grid; no SFU work).
#include <math.h>

#include "common.cuh"

namespace sy {

constexpr int kBwdRowsPerGroup = 296;   // partial rows per statistics group (2 per SM): fills the GPU whatever the map size
constexpr int kBwdThreads = 256;
constexpr int kBwdUnroll = 4;

__device__ __forceinline__ void unpack8b(const uint4& v, float* f) {
  f[0] = bf16_lo(v.x); f[1] = bf16_hi(v.x); f[2] = bf16_lo(v.y); f[3] = bf16_hi(v.y);
  f[4] = bf16_lo(v.z); f[5] = bf16_hi(v.z); f[6] = bf16_lo(v.w); f[7] = bf16_hi(v.w);
}
struct BwdArgs {
  const __nv_bfloat16* raw; long long raw_pitch;
  const __nv_bfloat16* dy; long long dy_pitch;
  const float* scale; const float* shift; const float* mean; const float* invstd;   // [2 groups][C]
  long long npix, split_pix;       // pixels [0, split_pix) = statistics group 0, the rest group 1
  int C, act;
  int rows0, rows1;                // partial rows of group 0 / group 1
};

// Partial rows [rows0 + rows1][2 (sum dz | sum dz * xhat)][C].  Row r of a group covers an equal share of the group's
// pixels; inside the block a thread owns one 8-channel chunk and every (256 / G)-th pixel (kBwdUnroll 16-byte load pairs in
// flight), then the pixel lanes are combined through shared memory in a fixed order (deterministic).
template <bool KINK>
__global__ void __launch_bounds__(kBwdThreads, 2) bn_act_bwd_reduce_kernel(const BwdArgs q, float* partials) {
  __shared__ float red[kBwdThreads][17];
  const int grp = (int)blockIdx.x >= q.rows0 ? 1 : 0;
  const int row = grp ? (int)blockIdx.x - q.rows0 : (int)blockIdx.x, nrows = grp ? q.rows1 : q.rows0;
  const long long gbeg = grp ? q.split_pix : 0, gend = grp ? q.npix : q.split_pix;
  const long long share = (gend - gbeg + nrows - 1) / nrows;
  const long long p0 = gbeg + (long long)row * share, p1 = min(gend, p0 + share);
  const int C = q.C, G = C >> 3;
  float* out = partials + (size_t)blockIdx.x * 2 * C;
  const int lanes = G < kBwdThreads ? G : kBwdThreads, PL = kBwdThreads / lanes;
  const int gl = (int)threadIdx.x % lanes, pl = (int)threadIdx.x / lanes;
  for (int g0 = 0; g0 < G; g0 += lanes) {
    const int g = g0 + gl;
    float s[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) s[i] = 0.f;
    if (g < G && pl < PL) {
      float sc[8], sh[8], k1[8], k0[8];          // z = r * sc + sh,  xhat = r * k1 + k0
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = grp * C + g * 8 + i;
        sc[i] = q.scale[c]; sh[i] = q.shift[c];
        k1[i] = q.invstd[c]; k0[i] = -q.mean[c] * q.invstd[c];
      }
      const __nv_bfloat16* rp = q.raw + g * 8;
      const __nv_bfloat16* dp = q.dy + g * 8;
      for (long long pp = p0 + pl; pp < p1; pp += (long long)PL * kBwdUnroll) {
        uint4 rv[kBwdUnroll], dv[kBwdUnroll];
#pragma unroll
        for (int j = 0; j < kBwdUnroll; ++j) {
          const long long pix = pp + (long long)j * PL;
          if (pix < p1) {
            rv[j] = *reinterpret_cast<const uint4*>(rp + pix * q.raw_pitch);
            dv[j] = *reinterpret_cast<const uint4*>(dp + pix * q.dy_pitch);
          }
        }
#pragma unroll
        for (int j = 0; j < kBwdUnroll; ++j) {
          if (pp + (long long)j * PL >= p1) continue;
          float r[8], d[8];
          unpack8b(rv[j], r);
          unpack8b(dv[j], d);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float z = r[i] * sc[i] + sh[i];
            const float dz = KINK ? d[i] * dact_f(q.act, z) : (q.act ? d[i] * dsilu(z) : d[i]);
            s[i] += dz;
            s[8 + i] += dz * (r[i] * k1[i] + k0[i]);
          }
        }
      }
    }
    if (PL > 1) {
#pragma unroll
      for (int i = 0; i < 16; ++i) red[threadIdx.x][i] = s[i];
      __syncthreads();
      // 16 values x `lanes` chunks, each summed over the PL pixel lanes in order: spread over all threads
      for (int o = (int)threadIdx.x; o < lanes * 16; o += kBwdThreads) {
        const int l = o >> 4, i = o & 15;
        if (g0 + l < G) {
          float a = 0.f;
          for (int k = 0; k < PL; ++k) a += red[k * lanes + l][i];
          out[(i >> 3) * C + (g0 + l) * 8 + (i & 7)] = a;
        }
      }
      __syncthreads();
    } else if (g < G) {
#pragma unroll
      for (int i = 0; i < 16; ++i) out[(i >> 3) * C + g * 8 + (i & 7)] = s[i];
    }
  }
}

// One WARP per channel: lane l sums the partial rows l, l + 32, ... of each group in order (fp64), a fixed shuffle tree
// combines the lanes (deterministic).  Writes dgamma / dbeta ((+)= sums over both groups) and, per (group, channel), the
// four coefficients of the element-wise pass:  z = r * A + B,  draw = A * dz + C1 * r + C0
//   with A = scale, B = shift, C1 = -scale * mb * invstd, C0 = -scale * (ma - mb * mean * invstd),
//   ma = mean_g(dz), mb = mean_g(dz * xhat)     (draw = scale * (dz - ma - xhat * mb), xhat = (r - mean) * invstd)
// coef layout [2 groups][4 (A | B | C1 | C0)][C].
__global__ void __launch_bounds__(256) bn_act_bwd_finalize_kernel(const float* __restrict__ partials, int rows0, int rows1, double inv_cnt0,
                                                                  double inv_cnt1, int C, const float* __restrict__ scale,
                                                                  const float* __restrict__ shift, const float* __restrict__ mean,
                                                                  const float* __restrict__ invstd, float* dgamma, float* dbeta,
                                                                  int accumulate, float* coef) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  double s[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
  // a lane owns at most ceil(296 / 32) = 10 rows per group: all loads first, then the sums in row order (one L2 round trip
  // per group instead of ten dependent ones)
  constexpr int kPerLane = (kBwdRowsPerGroup + 31) / 32;
  float v0[2][kPerLane], v1[2][kPerLane];
#pragma unroll
  for (int g = 0; g < 2; ++g) {                  // the loads of BOTH groups first (40 independent requests per lane)
    const int rb = g ? rows0 : 0, re = g ? rows0 + rows1 : rows0;
#pragma unroll
    for (int j = 0; j < kPerLane; ++j) {
      const int r = rb + lane + 32 * j;
      v0[g][j] = r < re ? __ldg(partials + (size_t)r * 2 * C + c) : 0.f;
      v1[g][j] = r < re ? __ldg(partials + (size_t)r * 2 * C + C + c) : 0.f;
    }
  }
#pragma unroll
  for (int g = 0; g < 2; ++g) {
#pragma unroll
    for (int j = 0; j < kPerLane; ++j) {
      s[g][0] += (double)v0[g][j];
      s[g][1] += (double)v1[g][j];
    }
  }
#pragma unroll
  for (int g = 0; g < 2; ++g)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) s[g][i] += __shfl_xor_sync(0xffffffffu, s[g][i], m);
  if (lane != 0) return;
  for (int g = 0; g < 2; ++g) {
    const double inv_cnt = g ? inv_cnt1 : inv_cnt0;       // 1 / pixels of the group, host-computed (0: empty group) -- no fp64
    const float ma = (float)(s[g][0] * inv_cnt), mb = (float)(s[g][1] * inv_cnt);   // division on the device (software, ~1 us)
    const float A = scale[g * C + c], B = shift[g * C + c], mu = mean[g * C + c], is = invstd[g * C + c];
    coef[(g * 4 + 0) * C + c] = A;
    coef[(g * 4 + 1) * C + c] = B;
    coef[(g * 4 + 2) * C + c] = -A * mb * is;
    coef[(g * 4 + 3) * C + c] = -A * (ma - mb * mu * is);
  }
  const float db = (float)(s[0][0] + s[1][0]), dg = (float)(s[0][1] + s[1][1]);
  dbeta[c] = accumulate ? dbeta[c] + db : db;
  dgamma[c] = accumulate ? dgamma[c] + dg : dg;
}

// draw = A * dz + C1 * r + C0 (bf16), dz = dy * act'(r * A + B).  Same thread mapping as the forward normalise pass: a
// thread owns one 8-channel chunk for its whole life (coefficients in registers), kBwdUnroll load pairs in flight.
template <bool KINK>
__global__ void __launch_bounds__(kBwdThreads, 2) bn_act_bwd_apply_kernel(const BwdArgs q, const float* __restrict__ coef,
                                                                       __nv_bfloat16* draw, long long draw_pitch) {
  const int C = q.C, G = C >> 3;
  const int ppb = kBwdThreads / G;
  const int prow = (int)threadIdx.x / G, g = (int)threadIdx.x - prow * G;
  if (prow >= ppb) return;
  float A[8], B[8], C1[8], C0[8];
  int cur = -1;
  auto load_group = [&](int grp) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      A[i] = coef[(grp * 4 + 0) * C + g * 8 + i]; B[i] = coef[(grp * 4 + 1) * C + g * 8 + i];
      C1[i] = coef[(grp * 4 + 2) * C + g * 8 + i]; C0[i] = coef[(grp * 4 + 3) * C + g * 8 + i];
    }
    cur = grp;
  };
  const long long step = (long long)gridDim.x * ppb;
  const __nv_bfloat16* rp = q.raw + g * 8;
  const __nv_bfloat16* dp = q.dy + g * 8;
  __nv_bfloat16* op = draw + g * 8;
  for (long long pix0 = (long long)blockIdx.x * ppb + prow; pix0 < q.npix; pix0 += step * kBwdUnroll) {
    uint4 rv[kBwdUnroll], dv[kBwdUnroll];
#pragma unroll
    for (int j = 0; j < kBwdUnroll; ++j) {
      const long long pix = pix0 + j * step;
      if (pix < q.npix) {
        rv[j] = *reinterpret_cast<const uint4*>(rp + pix * q.raw_pitch);
        dv[j] = *reinterpret_cast<const uint4*>(dp + pix * q.dy_pitch);
      }
    }
#pragma unroll
    for (int j = 0; j < kBwdUnroll; ++j) {
      const long long pix = pix0 + j * step;
      if (pix >= q.npix) continue;
      const int grp = pix >= q.split_pix ? 1 : 0;
      if (grp != cur) load_group(grp);
      float r[8], d[8], o[8];
      unpack8b(rv[j], r);
      unpack8b(dv[j], d);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float z = r[i] * A[i] + B[i];
        const float dz = KINK ? d[i] * dact_f(q.act, z) : (q.act ? d[i] * dsilu(z) : d[i]);
        o[i] = A[i] * dz + (C1[i] * r[i] + C0[i]);
      }
      *reinterpret_cast<uint4*>(op + pix * draw_pitch) =
          make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7]));
    }
  }
}

}  // namespace sy

using namespace sy;

// Partial rows of one statistics group.  A block's 256 threads cover `lanes` = min(C / 8, 256) channel chunks x PL = 256 / lanes
// pixel lanes, kBwdUnroll pixels per lane and loop iteration; a row gets two iterations' worth of pixels (so that small feature
// maps still spread over the whole GPU: the first version gave every row >= 256 pixels, i.e. 9 - 72 blocks with 32 dependent
// iterations each on the 19 x 30 / 38 x 60 maps: 17 - 53 us per launch, where the traffic needs 3 - 8 us), capped at 296 rows.
static int bwd_rows_for(long long npix_group, int C) {
  if (npix_group <= 0) return 0;
  const int G = C >> 3, lanes = G < kBwdThreads ? G : kBwdThreads, PL = kBwdThreads / (lanes > 0 ? lanes : 1);
  const long long per_row = (long long)PL * kBwdUnroll * 2;
  long long r = (npix_group + per_row - 1) / per_row;
  if (r > kBwdRowsPerGroup) r = kBwdRowsPerGroup;
  return (int)r;
}

extern "C" int sy_bn_act_bwd_rows(int32_t n, int32_t hw) {
  (void)n; (void)hw;
  return 2 * kBwdRowsPerGroup;                       // upper bound for any split
}

extern "C" int sy_bn_act_backward(const SyBnActBwdDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  const SyTensor& raw = d->raw;
  const SyTensor& dy = d->dy;
  const SyTensor& dr = d->draw;
  SY_REQUIRE(view_ok(raw) && view_ok(dy) && view_ok(dr), SY_EINVAL, "bn_act_backward: bad view");
  SY_REQUIRE(dy.n == raw.n && dy.h == raw.h && dy.w == raw.w && dy.c == raw.c && dr.n == raw.n && dr.h == raw.h &&
                 dr.w == raw.w && dr.c == raw.c,
             SY_EINVAL, "bn_act_backward: shape mismatch");
  SY_REQUIRE(d->scale && d->shift && d->mean && d->invstd && d->dgamma && d->dbeta && d->partials && d->coef, SY_EINVAL,
             "bn_act_backward: null pointer");
  SY_REQUIRE(raw.c <= 8 * kBwdThreads, SY_EINVAL, "bn_act_backward: C=%d > %d", raw.c, 8 * kBwdThreads);
  SY_REQUIRE(act_ok(d->act), SY_EINVAL, "bn_act_backward: act=%d is not an SY_ACT_* code", d->act);
  const int hw = raw.h * raw.w;
  const int split = (d->split_n > 0 && d->split_n < raw.n) ? d->split_n : raw.n;
  BwdArgs q{};
  q.raw = reinterpret_cast<const __nv_bfloat16*>(raw.ptr); q.raw_pitch = raw.pitch;
  q.dy = reinterpret_cast<const __nv_bfloat16*>(dy.ptr); q.dy_pitch = dy.pitch;
  q.scale = d->scale; q.shift = d->shift; q.mean = d->mean; q.invstd = d->invstd;
  q.npix = (long long)raw.n * hw; q.split_pix = (long long)split * hw;
  q.C = raw.c; q.act = d->act;
  q.rows0 = bwd_rows_for(q.split_pix, raw.c); q.rows1 = bwd_rows_for(q.npix - q.split_pix, raw.c);
  const int rows = q.rows0 + q.rows1;
  SY_REQUIRE(d->n_partials >= rows, SY_EWORKSPACE, "bn_act_backward: %d partial rows, need %d", d->n_partials, rows);
  auto reduce = [&](auto kernel) { kernel<<<rows, kBwdThreads, 0, stream>>>(q, d->partials); };
  const bool kink = d->act == SY_ACT_RELU || d->act == SY_ACT_LRELU;
  if (kink) reduce(bn_act_bwd_reduce_kernel<true>);
  else reduce(bn_act_bwd_reduce_kernel<false>);
  const double inv0 = q.split_pix > 0 ? 1.0 / (double)q.split_pix : 0.0;
  const double inv1 = q.npix - q.split_pix > 0 ? 1.0 / (double)(q.npix - q.split_pix) : 0.0;
  // (plain launches: programmatic dependent launch of the backward kernels was measured SLOWER -- 17.16 vs 16.39 ms per
  //  StreamYOLO-l step: the early-scheduled dependents take SM slots from the multi-wave element-wise kernels)
  bn_act_bwd_finalize_kernel<<<cdiv(raw.c, 8), 256, 0, stream>>>(d->partials, q.rows0, q.rows1, inv0, inv1, raw.c, d->scale, d->shift, d->mean,
                                                                 d->invstd, d->dgamma, d->dbeta, d->accumulate, d->coef);
  const int G = raw.c / 8, ppb = kBwdThreads / G;
  long long blocks = (q.npix + (long long)ppb * kBwdUnroll - 1) / ((long long)ppb * kBwdUnroll);
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  auto apply = [&](auto kernel) {
    kernel<<<(int)blocks, kBwdThreads, 0, stream>>>(q, d->coef, reinterpret_cast<__nv_bfloat16*>(dr.ptr), dr.pitch);
  };
  if (kink) apply(bn_act_bwd_apply_kernel<true>);
  else apply(bn_act_bwd_apply_kernel<false>);
  return launch_status("bn_act_backward kernels");
}
