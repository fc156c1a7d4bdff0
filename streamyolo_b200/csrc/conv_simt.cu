// CUDA-core kernels: direct convolution (device-side cross-check of the wgmma kernel and
// the path for shapes it rejects), the Focus stem, and per-channel statistic partials.
#include "common.cuh"

namespace sy {

struct SimtConvParams {
  const __nv_bfloat16* x; long long x_pitch;
  const __nv_bfloat16* w;
  __nv_bfloat16* y; long long y_pitch;
  const __nv_bfloat16* res; long long res_pitch;
  const float* scale; const float* shift;
  int N, H, W, Cin, Ho, Wo, Cout, kh, kw, stride, pad_h, pad_w, mode, act;
};

// one thread = one output pixel x 8 consecutive output channels; fp32 accumulation in (tap, ci) order
__global__ void conv_simt_kernel(const SimtConvParams p) {
  const int G = p.Cout / 8;
  const long long total = (long long)p.N * p.Ho * p.Wo * G;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(idx % G);
    const long long pix = idx / G;
    const int ox = (int)(pix % p.Wo);
    const int oy = (int)((pix / p.Wo) % p.Ho);
    const int n = (int)(pix / ((long long)p.Wo * p.Ho));
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    const int taps = p.kh * p.kw;
    for (int t = 0; t < taps; ++t) {
      const int iy = oy * p.stride + t / p.kw - p.pad_h;
      const int ix = ox * p.stride + t % p.kw - p.pad_w;
      if (iy < 0 || iy >= p.H || ix < 0 || ix >= p.W) continue;
      const __nv_bfloat16* xp = p.x + (((long long)n * p.H + iy) * p.W + ix) * p.x_pitch;
      for (int c0 = 0; c0 < p.Cin; c0 += 8) {
        const uint4 xv = *reinterpret_cast<const uint4*>(xp + c0);
        const float xf[8] = {bf16_lo(xv.x), bf16_hi(xv.x), bf16_lo(xv.y), bf16_hi(xv.y),
                             bf16_lo(xv.z), bf16_hi(xv.z), bf16_lo(xv.w), bf16_hi(xv.w)};
#pragma unroll
        for (int o = 0; o < 8; ++o) {
          const __nv_bfloat16* wp = p.w + ((long long)(g * 8 + o) * taps + t) * p.Cin + c0;
          const uint4 wv = *reinterpret_cast<const uint4*>(wp);
          acc[o] += xf[0] * bf16_lo(wv.x); acc[o] += xf[1] * bf16_hi(wv.x);
          acc[o] += xf[2] * bf16_lo(wv.y); acc[o] += xf[3] * bf16_hi(wv.y);
          acc[o] += xf[4] * bf16_lo(wv.z); acc[o] += xf[5] * bf16_hi(wv.z);
          acc[o] += xf[6] * bf16_lo(wv.w); acc[o] += xf[7] * bf16_hi(wv.w);
        }
      }
    }
    if (p.mode == SY_CONV_FUSED) {
#pragma unroll
      for (int o = 0; o < 8; ++o) {
        const int c = g * 8 + o;
        float t = acc[o] * (p.scale ? p.scale[c] : 1.f) + (p.shift ? p.shift[c] : 0.f);
        acc[o] = act_f(p.act, t);
      }
      if (p.res) {
        const uint4 rv = *reinterpret_cast<const uint4*>(p.res + pix * p.res_pitch + g * 8);
        acc[0] += bf16_lo(rv.x); acc[1] += bf16_hi(rv.x); acc[2] += bf16_lo(rv.y); acc[3] += bf16_hi(rv.y);
        acc[4] += bf16_lo(rv.z); acc[5] += bf16_hi(rv.z); acc[6] += bf16_lo(rv.w); acc[7] += bf16_hi(rv.w);
      }
    }
    uint4 out = make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]), pack_bf16(acc[4], acc[5]),
                           pack_bf16(acc[6], acc[7]));
    *reinterpret_cast<uint4*>(p.y + pix * p.y_pitch + g * 8) = out;
  }
}

// Focus space-to-depth (TL, BL, TR, BR order) from the NCHW fp32 frame-pair batch into NHWC bf16, already
// gathered along W for the 3x3 stem conv: pixel (y, x) holds taps x-1, x, x+1 (zero outside the image), each
// 12 focus channels + 4 zero channels, plus 16 zero channels = 64 channels = one 128-byte row per pixel (TMA boxes
// whose inner extent runs past a 96-byte pixel were measured 2.6x slower: 354 vs 133 us for the stem conv), so that
// the stem is a 3x1 conv with three 64-deep K blocks for the tensor-core kernel.  thread = (pixel, tap | pad).
// Input pixels are rounded to bf16 (F16: to fp16, for the stem of an fp16-storage forward).
// One block pass per output row (image, oy); threads walk (ox, tap) with shifts only (the first version resolved
// (tap, ox, oy, image, frame) from a flat index with five 64-bit divisions per thread).
template <bool F16>
__global__ void focus_pack_kernel(const float* __restrict__ x, int B, int in_ch, int H, int W, int frames,
                                  uint16_t* y, long long y_pitch) {
  const int Ho = H / 2, Wo = W / 2;
  const int rows = frames * B * Ho;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const int n = row / Ho, oy = row - n * Ho;
    const int frame = n / B, b = n - frame * B;
    const float* xb = x + ((long long)b * in_ch + frame * 3) * H * W;
    for (int e = threadIdx.x; e < Wo * 4; e += blockDim.x) {
      const int s = e & 3, ox = e >> 2;
      const int fx = ox + s - 1;
      float v[12];
      if (s < 3 && fx >= 0 && fx < Wo) {
#pragma unroll
        for (int fc = 0; fc < 12; ++fc) {
          const int qd = fc / 3, c = fc % 3;
          const int dy = qd & 1, dx = qd >> 1;   // TL(0,0) BL(1,0) TR(0,1) BR(1,1)
          v[fc] = __ldg(xb + ((long long)c * H + (2 * oy + dy)) * W + 2 * fx + dx);
        }
      } else {
#pragma unroll
        for (int fc = 0; fc < 12; ++fc) v[fc] = 0.f;
      }
      uint4* dst = reinterpret_cast<uint4*>(y + ((long long)row * Wo + ox) * y_pitch + s * 16);
      dst[0] = make_uint4(st_pack<F16>(v[0], v[1]), st_pack<F16>(v[2], v[3]), st_pack<F16>(v[4], v[5]),
                          st_pack<F16>(v[6], v[7]));
      dst[1] = make_uint4(st_pack<F16>(v[8], v[9]), st_pack<F16>(v[10], v[11]), 0u, 0u);
    }
  }
}

// partial (sum, sumsq) per channel over a chunk of <= kStatChunk pixels of one image
constexpr int kStatChunk = 512;
__global__ void channel_stats_kernel(const __nv_bfloat16* x, long long pitch, int HW, int C, float* partials) {
  __shared__ float red[256][17];
  const int chunks = cdiv(HW, kStatChunk);
  const int n = blockIdx.x / chunks, ch = blockIdx.x % chunks;
  const int p0 = ch * kStatChunk, p1 = min(HW, p0 + kStatChunk);
  const int G = C / 8;
  const int lanes = G < 256 ? G : 256;       // threads across channel groups
  const int PL = 256 / lanes;                // threads across pixels
  const int gl = threadIdx.x % lanes, pl = threadIdx.x / lanes;
  float* out = partials + (size_t)blockIdx.x * 2 * C;
  for (int g0 = 0; g0 < G; g0 += lanes) {
    const int g = g0 + gl;
    float s[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) s[i] = 0.f;
    if (g < G && pl < PL) {
      for (int pp = p0 + pl; pp < p1; pp += PL) {
        const uint4 v = *reinterpret_cast<const uint4*>(x + ((long long)n * HW + pp) * pitch + g * 8);
        const float f[8] = {bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y),
                            bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w)};
#pragma unroll
        for (int i = 0; i < 8; ++i) { s[i] += f[i]; s[8 + i] += f[i] * f[i]; }
      }
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) red[threadIdx.x][i] = s[i];
    __syncthreads();
    if (pl == 0 && g < G) {
      for (int i = 0; i < 16; ++i) {
        float a = 0.f;
        for (int q = 0; q < PL; ++q) a += red[q * lanes + gl][i];
        out[(i >> 3) * C + g * 8 + (i & 7)] = a;
      }
    }
    __syncthreads();
  }
}

}  // namespace sy

using namespace sy;

extern "C" int sy_conv2d_simt(const SyConvDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  const SyTensor& x = d->x;
  const SyTensor& y = d->y;
  SY_REQUIRE(view_ok(x) && view_ok(y) && d->w != nullptr, SY_EINVAL, "conv2d_simt: bad x/y view or null weights");
  SY_REQUIRE((d->kh == 1 || d->kh == 3) && (d->kw == 1 || d->kw == 3) && (d->stride == 1 || d->stride == 2), SY_EINVAL,
             "conv2d_simt: kernel %dx%d stride %d unsupported", d->kh, d->kw, d->stride);
  SY_REQUIRE(d->storage == SY_STORAGE_BF16, SY_EINVAL, "conv2d_simt: bf16 storage only (storage %d)", d->storage);
  SY_REQUIRE(act_ok(d->act), SY_EINVAL, "conv2d_simt: act=%d is not an SY_ACT_* code", d->act);
  SimtConvParams p{};
  p.pad_h = (d->kh - 1) / 2; p.pad_w = (d->kw - 1) / 2;
  p.N = x.n; p.H = x.h; p.W = x.w; p.Cin = x.c; p.Cout = y.c; p.kh = d->kh; p.kw = d->kw; p.stride = d->stride;
  p.Ho = (x.h + 2 * p.pad_h - d->kh) / d->stride + 1;
  p.Wo = (x.w + 2 * p.pad_w - d->kw) / d->stride + 1;
  SY_REQUIRE(y.n == x.n && y.h == p.Ho && y.w == p.Wo, SY_EINVAL, "conv2d_simt: output view mismatch");
  p.x = reinterpret_cast<const __nv_bfloat16*>(x.ptr); p.x_pitch = x.pitch;
  p.w = reinterpret_cast<const __nv_bfloat16*>(d->w);
  p.y = reinterpret_cast<__nv_bfloat16*>(y.ptr); p.y_pitch = y.pitch;
  p.mode = d->mode; p.act = d->act; p.scale = d->scale; p.shift = d->shift;
  if (d->mode == SY_CONV_FUSED && d->res.ptr) {
    SY_REQUIRE(view_ok(d->res) && d->res.c == y.c && d->res.h == y.h && d->res.w == y.w && d->res.n == y.n, SY_EINVAL,
               "conv2d_simt: residual view mismatch");
    p.res = reinterpret_cast<const __nv_bfloat16*>(d->res.ptr); p.res_pitch = d->res.pitch;
  }
  const long long total = (long long)p.N * p.Ho * p.Wo * (p.Cout / 8);
  const int blocks = (int)((total + 127) / 128 < sm_count() * 16 ? (total + 127) / 128 : sm_count() * 16);
  conv_simt_kernel<<<blocks, 128, 0, stream>>>(p);
  return launch_status("conv_simt_kernel");
}

template <bool F16>
static int focus_pack(const float* x, int32_t b, int32_t in_ch, int32_t h, int32_t w_px, int32_t frames, SyTensor y,
                      sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(x && view_ok(y), SY_EINVAL, "focus_pack: null input or bad output view");
  SY_REQUIRE(h % 2 == 0 && w_px % 2 == 0 && frames >= 1 && frames * 3 <= in_ch, SY_EINVAL,
             "focus_pack: h=%d w=%d must be even, frames=%d in_ch=%d", h, w_px, frames, in_ch);
  SY_REQUIRE(y.n == frames * b && y.h == h / 2 && y.w == w_px / 2 && y.c == 64, SY_EINVAL,
             "focus_pack: output view must be [frames*b, h/2, w/2, 64]");
  const int rows = y.n * y.h;                                   // one block pass per output row
  const int blocks = rows < sm_count() * 16 ? rows : sm_count() * 16;
  focus_pack_kernel<F16><<<blocks, 256, 0, stream>>>(x, b, in_ch, h, w_px, frames, reinterpret_cast<uint16_t*>(y.ptr),
                                                     y.pitch);
  return launch_status("focus_pack_kernel");
}

extern "C" int sy_focus_pack(const float* x, int32_t b, int32_t in_ch, int32_t h, int32_t w_px, int32_t frames,
                             SyTensor y, sy_stream_t stream) {
  return focus_pack<false>(x, b, in_ch, h, w_px, frames, y, stream);
}

extern "C" int sy_focus_pack_f16(const float* x, int32_t b, int32_t in_ch, int32_t h, int32_t w_px, int32_t frames,
                                 SyTensor y, sy_stream_t stream) {
  return focus_pack<true>(x, b, in_ch, h, w_px, frames, y, stream);
}

extern "C" int sy_stats_num_partials(int32_t n, int32_t hw) { return n * cdiv(hw, kStatChunk); }

extern "C" int sy_channel_stats(SyTensor x, float* partials, int32_t n_partials, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(view_ok(x) && partials, SY_EINVAL, "channel_stats: bad view");
  const int P = sy_stats_num_partials(x.n, x.h * x.w);
  SY_REQUIRE(n_partials >= P, SY_EWORKSPACE, "channel_stats: %d partial rows, need %d", n_partials, P);
  channel_stats_kernel<<<P, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x.ptr), x.pitch, x.h * x.w, x.c,
                                              partials);
  return launch_status("channel_stats_kernel");
}
