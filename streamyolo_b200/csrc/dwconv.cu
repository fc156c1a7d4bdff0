// Depthwise k x k convolution (groups = channels) behind [yolox] DWConv = BaseConv(in, in, k, stride, groups=in) followed by a
// 1x1 pointwise BaseConv (/root/reference/exps/model/darknet.py:109, dfp_pafpn.py:31, tal_head.py:53 select it with
// depthwise=True; no shipped cfg does).  2 * k * k FLOP per output element against 2 + 2 bytes: tensor cores do not pay, so
// this is a coalesced, vectorised HBM kernel on the CUDA cores: NHWC bf16, one thread = one output pixel x 8 channels, every
// tap one 16-byte load (neighbouring pixels / rows come from L1/L2), weights [taps][C] bf16, fp32 accumulation in tap
// order.  Same RAW / FUSED epilogue contract as sy_conv2d_tc (RAW: bf16 conv result for the train-mode BatchNorm passes;
// FUSED: act(acc * scale + shift) (+ residual) for eval with folded BatchNorm).  F16: activations, residual and weights in
// fp16 (the eval / streaming forwards with fp16 storage; FUSED only).
#include <type_traits>

#include "common.cuh"

namespace sy {

struct DwParams {                          // 16-bit elements of the kernel's storage type (bf16 | fp16)
  const uint16_t* x; long long x_pitch;
  const uint16_t* w;                       // [taps][C]
  uint16_t* y; long long y_pitch;
  const uint16_t* res; long long res_pitch;
  const float* scale; const float* shift;
  int N, H, W, C, Ho, Wo, k, stride, pad, mode, act;
};

template <int K, bool F16>
__global__ void __launch_bounds__(256) dwconv_kernel(const DwParams p) {
  const int G = p.C >> 3;
  const long long total = (long long)p.N * p.Ho * p.Wo * G;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(idx % G);
    const long long pix = idx / G;
    const int ox = (int)(pix % p.Wo), oy = (int)((pix / p.Wo) % p.Ho);
    const int n = (int)(pix / ((long long)p.Wo * p.Ho));
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int r = 0; r < K; ++r) {
      const int iy = oy * p.stride + r - p.pad;
      if (iy < 0 || iy >= p.H) continue;
#pragma unroll
      for (int s = 0; s < K; ++s) {
        const int ix = ox * p.stride + s - p.pad;
        if (ix < 0 || ix >= p.W) continue;
        const uint4 xv = *reinterpret_cast<const uint4*>(p.x + (((long long)n * p.H + iy) * p.W + ix) * p.x_pitch + g * 8);
        const uint4 wv = __ldg(reinterpret_cast<const uint4*>(p.w + (long long)(r * K + s) * p.C + g * 8));
        float xf[8], wf[8];
        st_unpack8<F16>(xv, xf);
        st_unpack8<F16>(wv, wf);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += xf[i] * wf[i];
      }
    }
    if (p.mode == SY_CONV_FUSED) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = g * 8 + i;
        const float t = acc[i] * (p.scale ? p.scale[c] : 1.f) + (p.shift ? p.shift[c] : 0.f);
        acc[i] = act_f(p.act, t);
      }
      if (p.res != nullptr) {
        const uint4 rv = *reinterpret_cast<const uint4*>(p.res + pix * p.res_pitch + g * 8);
        float rf[8];
        st_unpack8<F16>(rv, rf);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += rf[i];
      }
    }
    *reinterpret_cast<uint4*>(p.y + pix * p.y_pitch + g * 8) =
        make_uint4(st_pack<F16>(acc[0], acc[1]), st_pack<F16>(acc[2], acc[3]), st_pack<F16>(acc[4], acc[5]),
                   st_pack<F16>(acc[6], acc[7]));
  }
}

}  // namespace sy

using namespace sy;

extern "C" int sy_dwconv2d(const SyConvDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  const SyTensor& x = d->x;
  const SyTensor& y = d->y;
  SY_REQUIRE(view_ok(x) && view_ok(y) && d->w != nullptr, SY_EINVAL, "dwconv2d: bad x/y view or null weights");
  SY_REQUIRE(d->kh == d->kw && (d->kh == 1 || d->kh == 3 || d->kh == 5) && (d->stride == 1 || d->stride == 2), SY_EINVAL,
             "dwconv2d: kernel %dx%d stride %d unsupported", d->kh, d->kw, d->stride);
  const int pad = (d->kh - 1) / 2;
  const int ho = (x.h + 2 * pad - d->kh) / d->stride + 1, wo = (x.w + 2 * pad - d->kw) / d->stride + 1;
  SY_REQUIRE(y.n == x.n && y.h == ho && y.w == wo && y.c == x.c, SY_EINVAL, "dwconv2d: output view %dx%dx%dx%d, expected %dx%dx%dx%d",
             y.n, y.h, y.w, y.c, x.n, ho, wo, x.c);
  SY_REQUIRE(((uintptr_t)d->w % 16) == 0, SY_EINVAL, "dwconv2d: weights not 16B aligned");
  SY_REQUIRE(d->storage == SY_STORAGE_BF16 || (d->storage == SY_STORAGE_F16 && d->mode == SY_CONV_FUSED), SY_EINVAL,
             "dwconv2d: storage %d in mode %d unsupported (fp16: FUSED only)", d->storage, d->mode);
  SY_REQUIRE(act_ok(d->act), SY_EINVAL, "dwconv2d: act=%d is not an SY_ACT_* code", d->act);
  DwParams p{};
  p.x = reinterpret_cast<const uint16_t*>(x.ptr); p.x_pitch = x.pitch;
  p.w = reinterpret_cast<const uint16_t*>(d->w);
  p.y = reinterpret_cast<uint16_t*>(y.ptr); p.y_pitch = y.pitch;
  p.res = nullptr;
  if (d->mode == SY_CONV_FUSED && d->res.ptr != nullptr) {
    SY_REQUIRE(view_ok(d->res) && d->res.n == y.n && d->res.h == ho && d->res.w == wo && d->res.c == y.c, SY_EINVAL,
               "dwconv2d: residual view mismatch");
    p.res = reinterpret_cast<const uint16_t*>(d->res.ptr); p.res_pitch = d->res.pitch;
  }
  p.scale = d->scale; p.shift = d->shift;
  p.N = x.n; p.H = x.h; p.W = x.w; p.C = x.c; p.Ho = ho; p.Wo = wo; p.k = d->kh; p.stride = d->stride; p.pad = pad;
  p.mode = d->mode; p.act = d->act;
  const long long total = (long long)x.n * ho * wo * (x.c / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)sm_count() * 32) blocks = (long long)sm_count() * 32;
  if (blocks < 1) blocks = 1;
  auto go = [&](auto f16) {
    constexpr bool F16 = decltype(f16)::value;
    switch (d->kh) {
      case 1: dwconv_kernel<1, F16><<<(int)blocks, 256, 0, stream>>>(p); break;
      case 3: dwconv_kernel<3, F16><<<(int)blocks, 256, 0, stream>>>(p); break;
      default: dwconv_kernel<5, F16><<<(int)blocks, 256, 0, stream>>>(p); break;
    }
  };
  if (d->storage == SY_STORAGE_F16) go(std::true_type{});
  else go(std::false_type{});
  return launch_status("dwconv_kernel");
}
