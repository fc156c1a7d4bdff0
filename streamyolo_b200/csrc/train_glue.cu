// Kernels around the training step that are neither convolutions nor BatchNorm:
//   * sy_pack_conv_weight      fp32 OIHW parameter -> bf16 GEMM operand of the tensor-core kernels (forward layout
//                              [Cout][taps][Cin], data-gradient layout = flipped taps + transposed channels, Focus-stem layout;
//                              the forward and stem layouts also in fp16 with SY_PACK_F16):
//                              one launch per parameter per optimiser step instead of an ATen permute + cast chain
//   * sy_sgd_nesterov_ema_step the optimiser step of the reference trainer as ONE launch over flat fp32 buffers:
//                              GradScaler unscale + weight decay + SGD momentum (nesterov) + ModelEMA
//                              (/root/reference/exps/train_utils/double_trainer.py:113-123, 173-175; [yolox 0.3.0]
//                              Exp.get_optimizer, ModelEMA)
//   * sy_nonfinite_flag        GradScaler's inf / NaN check of the flat gradient (double_trainer.py:115), feeding the
//                              step's skip-with-EMA mode
//   * sy_resize_bilinear       the multi-scale resize of Exp.preprocess (/root/reference/cfgs/s_s50_onex_dfp_tal_flip.py:160-171:
//                              F.interpolate(mode="bilinear", align_corners=False)) + sy_scale_labels for the box rescale
#include <math.h>

#include <type_traits>

#include "common.cuh"

namespace sy {

// mode 0: out[o][t][i]                      = w[o][i][r][s],               t = r * kw + s                (forward B operand)
// mode 1: out[i][(kh-1-r)*kw + (kw-1-s)][o] = w[o][i][r][s]   (row pitch out_pitch, column offset co_off: data gradient)
// mode 2: out[o][r][s * 16 + i]             = w[o][i][r][s], i < 12, 64 columns per (o, r), rest zero     (Focus stem)
// T: the operand's element type (bf16, or __half for SY_PACK_F16)
template <typename T>
__device__ __forceinline__ T round_to(float v) {
  if constexpr (std::is_same<T, __half>::value) return __float2half_rn(v); else return __float2bfloat16_rn(v);
}

template <typename T>
__global__ void pack_weight_kernel(const float* __restrict__ w, int O, int I, int kh, int kw, int mode, T* out,
                                   long long out_pitch, int co_off) {
  const int taps = kh * kw;
  if (mode == 2) {
    const long long total = (long long)O * kh * 64;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
      const int col = (int)(idx % 64);
      const int r = (int)((idx / 64) % kh);
      const int o = (int)(idx / (64 * kh));
      const int s = col >> 4, i = col & 15;
      float v = 0.f;
      if (s < kw && i < I) v = w[(((long long)o * I + i) * kh + r) * kw + s];
      out[idx] = round_to<T>(v);
    }
    return;
  }
  const long long total = (long long)O * I * taps;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    if (mode == 0) {                       // idx walks the OUTPUT: (o, t, i), i fastest (coalesced bf16 stores)
      const int i = (int)(idx % I);
      const int t = (int)((idx / I) % taps);
      const int o = (int)(idx / ((long long)I * taps));
      out[idx] = round_to<T>(w[((long long)o * I + i) * taps + t]);
    } else {                               // idx walks (i, t', o), o fastest
      const int o = (int)(idx % O);
      const int t2 = (int)((idx / O) % taps);
      const int i = (int)(idx / ((long long)O * taps));
      const int t = taps - 1 - t2;         // (kh-1-r)*kw + (kw-1-s) = taps - 1 - (r*kw + s)
      out[((long long)i * taps + t2) * out_pitch + co_off + o] = round_to<T>(w[((long long)o * I + i) * taps + t]);
    }
  }
}

// All conv operands of a model in ONE launch.  Work unit = TILE: 64 output channels x 32 input channels (x all taps) of one
// item (modes 0 / 1), or 64 output channels of a stem item (mode 2); items[k].begin = first tile of item k (prefix sum of
// sy_pack_item_tiles), found by binary search once per tile.  A tile is read with coalesced loads along the source's
// contiguous (ci, tap) run, converted, staged in shared memory and written with coalesced stores along the destination's
// contiguous dimension (ci for the forward operand, co for the data-gradient operand).  The first version moved one element
// per thread with the source index computed from the destination index: the data-gradient layout then read one 32-byte
// sector per element (1.19 ms for StreamYOLO-l; this version: the 660 MB of traffic at HBM speed).
constexpr int kPackTO = 64, kPackTI = 32, kPackMaxTaps = 9;
constexpr int kPackPitch = kPackTI * kPackMaxTaps + 2;      // bf16 elements; (pitch / 2) odd: column reads are conflict-free

__host__ __device__ inline long long pack_item_tiles(int cout, int cin, int mode) {
  const long long to = (cout + kPackTO - 1) / kPackTO;
  return mode == 2 ? to : to * ((cin + kPackTI - 1) / kPackTI);
}

__global__ void __launch_bounds__(256) pack_weights_batch_kernel(const SyPackItem* __restrict__ items, int n_items, long long total) {
  __shared__ __nv_bfloat16 tile[kPackTO][kPackPitch];
  __shared__ int s_item;
  for (long long tidx = blockIdx.x; tidx < total; tidx += gridDim.x) {
    if (threadIdx.x == 0) {
      int lo = 0, hi = n_items - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (items[mid].begin <= tidx) lo = mid; else hi = mid - 1;
      }
      s_item = lo;
    }
    __syncthreads();
    const SyPackItem it = items[s_item];
    const int l = (int)(tidx - it.begin);
    const int taps = it.taps, O = it.cout, I = it.cin;
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(it.out);
    if (it.mode == 2) {                                     // Focus stem: out[o][r][s * 16 + i], 64 columns per (o, r)
      const int kh = it.kh, kw = taps / kh;
      const int o0 = l * kPackTO, no = min(kPackTO, O - o0);
      const int n = no * kh * 64;
      for (int e = threadIdx.x; e < n; e += blockDim.x) {
        const int col = e % 64, r = (e / 64) % kh, o = o0 + e / (64 * kh);
        const int sx = col >> 4, i = col & 15;
        float v = 0.f;
        if (sx < kw && i < I) v = it.w[(((long long)o * I + i) * kh + r) * kw + sx];
        out[(long long)o0 * kh * 64 + e] = __float2bfloat16_rn(v);
      }
    } else if (taps > kPackMaxTaps) {                       // (no such conv in the path: element-wise fallback)
      const int tiles_i = (I + kPackTI - 1) / kPackTI;
      const int o0 = (l / tiles_i) * kPackTO, i0 = (l % tiles_i) * kPackTI;
      const int no = min(kPackTO, O - o0), ni = min(kPackTI, I - i0);
      for (int e = threadIdx.x; e < no * ni * taps; e += blockDim.x) {
        const int t = e % taps, i = i0 + (e / taps) % ni, o = o0 + e / (taps * ni);
        const __nv_bfloat16 v = __float2bfloat16_rn(it.w[((long long)o * I + i) * taps + t]);
        if (it.mode == 0) out[((long long)o * taps + t) * I + i] = v;
        else out[((long long)i * taps + (taps - 1 - t)) * it.out_pitch + it.co_offset + o] = v;
      }
    } else {
      const int tiles_i = (I + kPackTI - 1) / kPackTI;
      const int o0 = (l / tiles_i) * kPackTO, i0 = (l % tiles_i) * kPackTI;
      const int no = min(kPackTO, O - o0), ni = min(kPackTI, I - i0);
      const int cols = ni * taps;                           // contiguous floats of source row o: w[o][i0 .. i0 + ni)[taps]
      // (warp-per-row loops, lanes along the contiguous dimension: no per-element divisions -- with index arithmetic of the
      //  form e / cols, e % ni the kernel was bound by its integer divisions: 0.77 ms for StreamYOLO-l)
      const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
      for (int o = warp; o < no; o += 8) {
        const float* src = it.w + ((long long)(o0 + o) * I + i0) * taps;
        // nine loads in flight per lane (a whole 3x3 row in one pass): one load per iteration left the tile latency-bound
        for (int c0 = 0; c0 < cols; c0 += 32 * kPackMaxTaps) {
          float v[kPackMaxTaps];
#pragma unroll
          for (int j = 0; j < kPackMaxTaps; ++j) {
            const int c = c0 + 32 * j + lane;
            v[j] = c < cols ? src[c] : 0.f;
          }
#pragma unroll
          for (int j = 0; j < kPackMaxTaps; ++j) {
            const int c = c0 + 32 * j + lane;
            if (c < cols) tile[o][c] = __float2bfloat16_rn(v[j]);
          }
        }
      }
      __syncthreads();
      if (it.mode == 0) {                                   // out[o][t][i]: runs of ni consecutive input channels
        for (int o = warp; o < no; o += 8) {
          __nv_bfloat16* dst = out + (long long)(o0 + o) * taps * I + i0;
          for (int t = 0; t < taps; ++t)
            if (lane < ni) dst[(long long)t * I + lane] = tile[o][lane * taps + t];
        }
      } else {                                              // out[i][taps - 1 - t][co_offset + o]: runs of no consecutive output channels
        for (int i = warp; i < ni; i += 8) {
          for (int t2 = 0; t2 < taps; ++t2) {
            __nv_bfloat16* dst = out + ((long long)(i0 + i) * taps + t2) * it.out_pitch + it.co_offset + o0;
            const int c = i * taps + (taps - 1 - t2);
            for (int o = lane; o < no; o += 32) dst[o] = tile[o][c];
          }
        }
      }
    }
    __syncthreads();                                        // the tile (and s_item) are reused by the next iteration
  }
}

// One thread per element of the flat state.  Elements [0, n_param) are parameters (gradient, momentum), of which
// [decay_begin, n_param) get weight decay; elements [n_param, n_total) are floating-point buffers (BatchNorm running
// statistics) that only the EMA tracks.  Arithmetic mirrors torch.optim.SGD (foreach) and yolox ModelEMA step by step,
// including which operations are fused multiply-adds there (a.add(b, alpha) -> fma) and which are two roundings.
__global__ void sgd_ema_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ mbuf,
                               float* __restrict__ ema, long long n_param, long long n_total, long long decay_begin, float lr,
                               float momentum, float wd, float inv_scale, int nesterov, float ema_d, float ema_1md,
                               const float* __restrict__ found_inf, int found_inf_ema, const float* __restrict__ hyper) {
  // GradScaler.step skips the optimiser update on inf / nan.  found_inf_ema = 0: the whole launch is skipped, EMA included;
  // otherwise parameters and momentum stay, and the EMA still moves towards them (ModelEMA.update runs on a skipped step)
  bool skip = false;
  if (found_inf != nullptr && *found_inf != 0.f) {
    if (!found_inf_ema) return;
    skip = true;
  }
  if (hyper != nullptr) {                                          // graph-replay safe hyper-parameters
    lr = hyper[0]; momentum = hyper[1]; wd = hyper[2]; inv_scale = hyper[3]; ema_d = hyper[4]; ema_1md = hyper[5];
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_total; i += (long long)gridDim.x * blockDim.x) {
    float v = p[i];
    if (i < n_param && !skip) {
      float d = g[i];
      if (inv_scale != 1.0f) d = __fmul_rn(d, inv_scale);         // GradScaler.unscale_: grad.mul_(inv_scale)
      if (i >= decay_begin && wd != 0.f) d = fmaf(wd, v, d);      // grad.add(param, alpha=wd)
      float b = __fadd_rn(__fmul_rn(mbuf[i], momentum), d);       // buf.mul_(momentum).add_(grad)
      mbuf[i] = b;
      d = nesterov ? fmaf(momentum, b, d) : b;                    // grad.add(buf, alpha=momentum)
      v = fmaf(-lr, d, v);                                        // param.add_(grad, alpha=-lr)
      p[i] = v;
    }
    if (ema != nullptr) ema[i] = __fadd_rn(__fmul_rn(ema[i], ema_d), __fmul_rn(ema_1md, v));   // v *= d; v += (1 - d) * model
  }
}

// Any NaN / +-inf among x[0, n) -> *flag = 1 and ++*count, once per launch: the block that turns the flag from 0 to 1
// counts.  The flag is zeroed by the host entry point (a memset node in a captured graph) before this runs.  Four floats
// per load (x 16-byte aligned), the n % 4 tail by the first threads.  Non-finite = all exponent bits set (FLT_MAX and
// subnormals are finite), tested on the bits so that no compiler flag changes it.
__device__ __forceinline__ bool nonfinite_bits(float v) { return (__float_as_uint(v) & 0x7f800000u) == 0x7f800000u; }

__global__ void __launch_bounds__(256) nonfinite_flag_kernel(const float* __restrict__ x, long long n, float* flag,
                                                             int* count) {
  const long long n4 = n >> 2;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  bool bad = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = __ldg(x4 + i);
    bad |= nonfinite_bits(v.x) | nonfinite_bits(v.y) | nonfinite_bits(v.z) | nonfinite_bits(v.w);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) bad |= nonfinite_bits(x[(n4 << 2) + threadIdx.x]);
  if (__syncthreads_or(bad) && threadIdx.x == 0 && atomicExch(flag, 1.f) == 0.f) atomicAdd(count, 1);
}

// F.interpolate(x, size=(Ho, Wo), mode="bilinear", align_corners=False) on NCHW fp32 (ATen upsample_bilinear2d:
// src = max(0, scale * (dst + 0.5) - 0.5), scale = in / out, lambda from the fractional part, index clamped at the border)
__global__ void resize_bilinear_kernel(const float* __restrict__ x, int NC, int Hi, int Wi, float* __restrict__ y, int Ho, int Wo) {
  const float sh = (float)Hi / (float)Ho, sw = (float)Wi / (float)Wo;
  const long long total = (long long)NC * Ho * Wo;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(idx % Wo), oy = (int)((idx / Wo) % Ho);
    const long long nc = idx / ((long long)Wo * Ho);
    const float fy = fmaxf(sh * ((float)oy + 0.5f) - 0.5f, 0.f);     // contracted like ATen's own kernel
    const float fx = fmaxf(sw * ((float)ox + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < Hi - 1 ? 1 : 0), x1 = x0 + (x0 < Wi - 1 ? 1 : 0);
    const float ly = fy - (float)y0, lx = fx - (float)x0;
    const float hy = 1.f - ly, hx = 1.f - lx;
    const float* s = x + nc * (long long)Hi * Wi;
    const float a = s[(long long)y0 * Wi + x0], b = s[(long long)y0 * Wi + x1];
    const float c = s[(long long)y1 * Wi + x0], d = s[(long long)y1 * Wi + x1];
    y[idx] = hy * (hx * a + lx * b) + ly * (hx * c + lx * d);
  }
}

// labels [rows][5] (cls, cx, cy, w, h): x-like columns (1, 3) *= sx, y-like columns (2, 4) *= sy
// (targets[..., 1::2] *= scale_x; targets[..., 2::2] *= scale_y)
__global__ void scale_labels_kernel(float* lab, long long rows, int cols, float sx, float sy) {
  const long long total = rows * cols;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cols);
    if (c == 0) continue;
    lab[idx] = lab[idx] * ((c & 1) ? sx : sy);
  }
}

static int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  if (g > (long long)sm_count() * 16) g = (long long)sm_count() * 16;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace sy

using namespace sy;

extern "C" int sy_pack_conv_weight(const float* w, int32_t cout, int32_t cin, int32_t kh, int32_t kw, int32_t mode, void* out,
                                   int64_t out_pitch, int32_t co_offset, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(w != nullptr && out != nullptr && cout > 0 && cin > 0 && kh > 0 && kw > 0, SY_EINVAL, "pack_conv_weight: bad arguments");
  const bool f16 = (mode & SY_PACK_F16) != 0;
  mode &= ~SY_PACK_F16;
  SY_REQUIRE(mode >= 0 && mode <= 2 && !(f16 && mode == 1), SY_EINVAL, "pack_conv_weight: mode %d%s", mode,
             f16 ? " | SY_PACK_F16 (fp16: forward and stem layouts only)" : "");
  if (mode == 1) SY_REQUIRE(out_pitch >= co_offset + cout, SY_EINVAL, "pack_conv_weight: pitch %lld < %d + %d", (long long)out_pitch, co_offset, cout);
  if (mode == 2) SY_REQUIRE(cin <= 16 && kw <= 4, SY_EINVAL, "pack_conv_weight(stem): cin %d kw %d", cin, kw);
  const long long total = mode == 2 ? (long long)cout * kh * 64 : (long long)cout * cin * kh * kw;
  if (f16)
    pack_weight_kernel<<<grid_for(total, 256), 256, 0, stream>>>(w, cout, cin, kh, kw, mode, reinterpret_cast<__half*>(out),
                                                                out_pitch, co_offset);
  else
    pack_weight_kernel<<<grid_for(total, 256), 256, 0, stream>>>(w, cout, cin, kh, kw, mode,
                                                                reinterpret_cast<__nv_bfloat16*>(out), out_pitch, co_offset);
  return launch_status("pack_weight_kernel");
}

extern "C" int64_t sy_pack_item_tiles(int32_t cout, int32_t cin, int32_t mode) { return pack_item_tiles(cout, cin, mode); }

extern "C" int sy_pack_conv_weights_batch(const SyPackItem* items_dev, int32_t n_items, int64_t total, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(items_dev != nullptr && n_items > 0 && total > 0, SY_EINVAL, "pack_conv_weights_batch: bad arguments");
  const int grid = (int)(total < (long long)sm_count() * 8 ? total : (long long)sm_count() * 8);
  pack_weights_batch_kernel<<<grid, 256, 0, stream>>>(items_dev, n_items, total);
  return launch_status("pack_weights_batch_kernel");
}

extern "C" int sy_sgd_nesterov_ema_step(const SySgdEmaDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->param != nullptr && d->n_total > 0, SY_EINVAL, "sgd_ema_step: null state");
  SY_REQUIRE(d->n_param >= 0 && d->n_param <= d->n_total && d->decay_begin >= 0 && d->decay_begin <= d->n_param, SY_EINVAL,
             "sgd_ema_step: bad segment bounds");
  SY_REQUIRE(d->n_param == 0 || (d->grad != nullptr && d->momentum_buf != nullptr), SY_EINVAL, "sgd_ema_step: null grad / momentum");
  sgd_ema_kernel<<<grid_for(d->n_total, 256), 256, 0, stream>>>(d->param, d->grad, d->momentum_buf, d->ema, d->n_param, d->n_total,
                                                               d->decay_begin, d->lr, d->momentum, d->weight_decay,
                                                               d->inv_scale, d->nesterov, d->ema_decay, d->ema_one_minus_decay,
                                                               d->found_inf, d->found_inf_ema, d->hyper);
  return launch_status("sgd_ema_kernel");
}

extern "C" int sy_nonfinite_flag(const float* x, int64_t n, float* flag, int32_t* count, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(x != nullptr && flag != nullptr && count != nullptr && n > 0, SY_EINVAL, "nonfinite_flag: bad arguments");
  SY_REQUIRE(reinterpret_cast<uintptr_t>(x) % 16 == 0, SY_EINVAL, "nonfinite_flag: x must be 16-byte aligned");
  if (cudaMemsetAsync(flag, 0, sizeof(float), stream) != cudaSuccess) return launch_status("nonfinite_flag memset");
  nonfinite_flag_kernel<<<grid_for((n + 3) / 4, 256), 256, 0, stream>>>(x, n, flag, count);
  return launch_status("nonfinite_flag_kernel");
}

extern "C" int sy_resize_bilinear(const float* x, int32_t nc, int32_t hi, int32_t wi, float* y, int32_t ho, int32_t wo,
                                  sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(x != nullptr && y != nullptr && nc > 0 && hi > 0 && wi > 0 && ho > 0 && wo > 0, SY_EINVAL, "resize_bilinear: bad arguments");
  resize_bilinear_kernel<<<grid_for((long long)nc * ho * wo, 256), 256, 0, stream>>>(x, nc, hi, wi, y, ho, wo);
  return launch_status("resize_bilinear_kernel");
}

extern "C" int sy_scale_labels(float* labels, int64_t rows, int32_t cols, float sx, float sy_, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(labels != nullptr && rows > 0 && cols > 0, SY_EINVAL, "scale_labels: bad arguments");
  scale_labels_kernel<<<grid_for(rows * cols, 256), 256, 0, stream>>>(labels, rows, cols, sx, sy_);
  return launch_status("scale_labels_kernel");
}
