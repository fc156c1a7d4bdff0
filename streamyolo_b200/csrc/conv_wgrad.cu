// Weight gradient of a convolution on the Hopper tensor cores (sm_90a, wgmma):
//
//   dW[co][tap][ci] = sum over output pixels p of  dy[p][co] * x[p @ tap][ci]
//
// as one GEMM per filter tap with  M = output channels (128 per tile, 64 per consumer warpgroup),  N = input channels (BN),
// K = output pixels.  In NHWC both operands have K (pixels) as the strided dimension, so they are staged "MN-major"
// (wgmma's transposed operand form): every shared-memory row is one pixel holding 64 contiguous channels -- exactly what a
// TMA load of a [64 px][64 ch] box with the 128B swizzle writes.  Descriptor LBO = 8192 B (next 64-channel box),
// SBO = 1024 B (next 8 pixels), +2048 B per K = 16 step.
//   * dy tile: plain 2-D TMA boxes of the [pixels][Cout] view;
//   * x tile for tap (r, s): im2col-mode TMA (the forward kernel's loader) of the same 64 output pixels' input positions
//     shifted by the tap -- stride-2 convs and the zero padding come for free.
// The pixel range is split over CTAs (split-K); every CTA writes an fp32 partial [128][BN] per work item and a second
// kernel reduces the partials in a fixed order (deterministic) into the optimizer's fp32 OIHW layout.
//
// Replaces the cuDNN backward-filter call behind loss.backward() (exps/train_utils/double_trainer.py:114 of StreamYOLO)
// for every [yolox] BaseConv (exps/model/darknet.py:115-165, dfp_pafpn.py:33-105, tal_head.py:55-104).
#include <cuda.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace sy {
namespace wg {

using namespace tc;

constexpr int kThreads = 288;            // warps 0-7: two MMA + epilogue warpgroups (rows 0-63, 64-127), warp 8: TMA producer
constexpr int kPixK = 64;                // pixels per pipeline stage (K block)
constexpr int kBoxBytes = kPixK * 128;   // one [64 px][64 ch] box
constexpr int kMaxStages = 8;
static const int kSmemLimit = 232448;

struct WParams {
  int P_total, Ho, Wo, stride, pad_h, pad_w, kw;
  int Cout, Cin;
  int m_tiles, n_tiles, taps, ksplit, kb_total, kb_per_split, items;
  FastDiv fd_hw, fd_wo;
  float* partial;                        // [items][128][BN]
  int stages;
};

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// MN-major, 128B-swizzled operand: rows = K (pixels) of 128 bytes, 8-row groups 1 KiB apart, 64-channel boxes 8 KiB apart
__device__ __forceinline__ uint64_t make_desc_mn(uint32_t saddr) { return make_gmma_desc(saddr, kBoxBytes, 1024u); }

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX, const WParams p) {
  constexpr int kXBoxes = BN / 64;
  constexpr int kStageBytes = (2 + kXBoxes) * kBoxBytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int S = p.stages;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S * kStageBytes);
  const uint32_t bar0 = smem_u32(bars);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (kMaxStages + s); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 8 * 32) {
    prefetch_tmap(&tmDY);
    prefetch_tmap(&tmX);
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);                // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int hw = p.Ho * p.Wo;

  auto decode = [&](int item, int& m_tile, int& n_tile, int& tap, int& kb0, int& kb1) {
    const int ks = item % p.ksplit;
    int rest = item / p.ksplit;
    tap = rest % p.taps; rest /= p.taps;
    n_tile = rest % p.n_tiles;
    m_tile = rest / p.n_tiles;
    kb0 = ks * p.kb_per_split;
    kb1 = min(kb0 + p.kb_per_split, p.kb_total);
  };

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
      int m_tile, n_tile, tap, kb0, kb1;
      decode(item, m_tile, n_tile, tap, kb0, kb1);
      const int r = tap / p.kw, sx = tap - r * p.kw;
      for (int kb = kb0; kb < kb1; ++kb) {
        const int p0 = kb * kPixK;
        const int img = fdiv(p0, p.fd_hw), rem = p0 - img * hw;
        const int oh = fdiv(rem, p.fd_wo), ow = rem - oh * p.Wo;
        mbar_wait(empty_bar(stage), phase ^ 1u);
        uint8_t* st = smem + stage * kStageBytes;
        if (elect_one()) {
          mbar_expect_tx(full_bar(stage), (uint32_t)kStageBytes);
#pragma unroll
          for (int j = 0; j < 2; ++j) tma_load_2d(smem_u32(st + j * kBoxBytes), &tmDY, full_bar(stage), m_tile * 128 + j * 64, p0);
#pragma unroll
          for (int j = 0; j < kXBoxes; ++j)
            tma_load_im2col_4d(smem_u32(st + (2 + j) * kBoxBytes), &tmX, full_bar(stage), n_tile * BN + j * 64,
                               ow * p.stride - p.pad_w, oh * p.stride - p.pad_h, img, (uint16_t)sx, (uint16_t)r);
        }
        __syncwarp();
        if (++stage == S) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA + epilogue: registers -> fp32 partial [128][BN]
    // Warpgroup g computes output channels [64 g, 64 g + 64) of the tile (its dy box); a ring stage goes back to the producer
    // one commit group late, so the next group's MMAs are queued while the last ones drain.
    const int g = warp >> 2;
    const bool lead = (threadIdx.x & 127) == 0;
    const int row0 = g * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
      int m_tile, n_tile, tap, kb0, kb1;
      decode(item, m_tile, n_tile, tap, kb0, kb1);
      int pend = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t a0 = smem_u32(smem + stage * kStageBytes) + (uint32_t)(g * kBoxBytes), b0 = smem_u32(smem + stage * kStageBytes) + 2 * kBoxBytes;
        wgmma_fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kPixK / 16; ++k)
          Wgmma<BN, 1, 1>::mma(acc, make_desc_mn(a0 + k * 2048), make_desc_mn(b0 + k * 2048), (kb != kb0) || (k != 0));
        wgmma_commit();
        wgmma_fence_operand(acc);
        wgmma_wait<1>();
        if (lead && pend >= 0) mbar_arrive(empty_bar(pend));
        pend = stage;
        if (++stage == S) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      if (lead && pend >= 0) mbar_arrive(empty_bar(pend));
      const bool empty = kb1 <= kb0;             // (cannot happen with the host's ksplit; keeps the output defined)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* dst = p.partial + ((size_t)item * 128 + row0 + 8 * h) * BN + cq;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
          *reinterpret_cast<float2*>(dst + 8 * j) = empty ? make_float2(0.f, 0.f) : make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
  }
}

// dw[co][ci][r][s] (+)= sum over the K splits, fixed order.  Threads walk (co, tap, ci) with ci fastest: the partial reads
// (the bulk: ksplit per output) are coalesced along the N = input-channel dimension; only the single store per output is
// strided (by the tap count) in the optimizer's OIHW layout.
// SG > 1 (layers with few outputs and many splits: the 1x1 convs have up to 296 splits for 16 K - 260 K outputs): a block's
// 256 threads are 256 / SG outputs x SG split groups; group g sums the splits [g * ksplit / SG, (g + 1) * ksplit / SG) and
// the first group adds the SG sums in group order (deterministic).  One thread per output walked its 296 partials in a
// dependent-latency chain: ~13 us per 1x1 layer for 16 MB of partials.
template <int SG>
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ partial, int BN, int m_tiles, int n_tiles, int taps,
                                                           int ksplit, int Cout, int Cin, float* dw, int accumulate) {
  constexpr int kOut = 256 / SG;                  // outputs per block pass
  __shared__ float part[SG][kOut];
  const int ol = (int)threadIdx.x % kOut, sg = (int)threadIdx.x / kOut;
  const long long total = (long long)Cout * Cin * taps;
  const int k0 = (int)((long long)ksplit * sg / SG), k1 = (int)((long long)ksplit * (sg + 1) / SG);
  for (long long base = (long long)blockIdx.x * kOut; base < total; base += (long long)gridDim.x * kOut) {
    const long long idx = base + ol;
    float acc = 0.f;
    long long o = 0;
    if (idx < total) {
      const int ci = (int)(idx % Cin);
      const int tap = (int)((idx / Cin) % taps);
      const int co = (int)(idx / ((long long)taps * Cin));
      const int m_tile = co / 128, row = co % 128, n_tile = ci / BN, col = ci % BN;
      const size_t item0 = ((size_t)(m_tile * n_tiles + n_tile) * taps + tap) * ksplit;
      const float* src = partial + (item0 * 128 + row) * BN + col;
      int ks = k0;
      for (; ks + 4 <= k1; ks += 4) {             // four loads in flight; summed in split order
        const float v0 = __ldg(src + (size_t)ks * 128 * BN), v1 = __ldg(src + (size_t)(ks + 1) * 128 * BN);
        const float v2 = __ldg(src + (size_t)(ks + 2) * 128 * BN), v3 = __ldg(src + (size_t)(ks + 3) * 128 * BN);
        acc += v0; acc += v1; acc += v2; acc += v3;
      }
      for (; ks < k1; ++ks) acc += __ldg(src + (size_t)ks * 128 * BN);
      o = ((long long)co * Cin + ci) * taps + tap;
    }
    if (SG > 1) {
      part[sg][ol] = acc;
      __syncthreads();
      if (sg == 0 && idx < total) {
        float t = part[0][ol];
#pragma unroll
        for (int g = 1; g < SG; ++g) t += part[g][ol];
        dw[o] = accumulate ? dw[o] + t : t;
      }
      __syncthreads();
    } else if (idx < total) {
      dw[o] = accumulate ? dw[o] + acc : acc;
    }
  }
}

struct Plan {
  int bn, m_tiles, n_tiles, taps, ksplit, kb_total, kb_per_split, items, ho, wo;
  size_t ws_bytes;
};

static int make_plan(const SyConvWgradDesc* d, Plan* pl) {
  const SyTensor& x = d->x;
  const SyTensor& dy = d->dy;
  SY_REQUIRE(view_ok(x) && view_ok(dy), SY_EINVAL, "conv2d_wgrad: bad x/dy view");
  SY_REQUIRE((d->kh == 1 || d->kh == 3) && (d->kw == 1 || d->kw == 3) && (d->stride == 1 || d->stride == 2), SY_EINVAL,
             "conv2d_wgrad: kernel %dx%d stride %d unsupported", d->kh, d->kw, d->stride);
  const int ph = (d->kh - 1) / 2, pw = (d->kw - 1) / 2;
  pl->ho = (x.h + 2 * ph - d->kh) / d->stride + 1;
  pl->wo = (x.w + 2 * pw - d->kw) / d->stride + 1;
  SY_REQUIRE(dy.n == x.n && dy.h == pl->ho && dy.w == pl->wo, SY_EINVAL, "conv2d_wgrad: dy view %dx%dx%d, expected %dx%dx%d",
             dy.n, dy.h, dy.w, x.n, pl->ho, pl->wo);
  SY_REQUIRE((long long)x.n * pl->ho * pl->wo < (1ll << 31) - 256, SY_EINVAL, "conv2d_wgrad: too many pixels");
  pl->bn = x.c <= 64 ? 64 : (x.c <= 128 ? 128 : 256);
  pl->m_tiles = cdiv(dy.c, 128);
  pl->n_tiles = cdiv(x.c, pl->bn);
  pl->taps = d->kh * d->kw;
  pl->kb_total = cdiv(x.n * pl->ho * pl->wo, kPixK);
  const int base = pl->m_tiles * pl->n_tiles * pl->taps;
  int ks = cdiv(2 * num_sms(), base);                      // about two waves of work items
  const int ks_max = pl->kb_total / 8 > 1 ? pl->kb_total / 8 : 1;   // at least 8 K blocks per split
  if (ks > ks_max) ks = ks_max;
  if (ks < 1) ks = 1;
  pl->kb_per_split = cdiv(pl->kb_total, ks);
  pl->ksplit = cdiv(pl->kb_total, pl->kb_per_split);        // no empty splits
  pl->items = base * pl->ksplit;
  pl->ws_bytes = (size_t)pl->items * 128 * pl->bn * sizeof(float);
  return SY_OK;
}

template <int BN>
static int launch(const CUtensorMap& tdy, const CUtensorMap& tx, WParams& p, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    SY_CUDA(cudaFuncSetAttribute(conv_wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    attr_set = true;
  }
  const int stage_bytes = (2 + BN / 64) * kBoxBytes;
  int stages = (kSmemLimit - 1024 - 512) / stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  p.stages = stages;
  const int smem = 1024 + 512 + stages * stage_bytes;   // align slack + barriers + ring
  const int grid = p.items < num_sms() ? p.items : num_sms();
  conv_wgrad_kernel<BN><<<grid, kThreads, smem, stream>>>(tdy, tx, p);
  return launch_status("conv_wgrad_kernel");
}

}  // namespace wg
}  // namespace sy

using namespace sy;

extern "C" size_t sy_conv2d_wgrad_workspace_bytes(const SyConvWgradDesc* d) {
  wg::Plan pl{};
  if (d == nullptr || wg::make_plan(d, &pl) != SY_OK) return 0;
  return pl.ws_bytes;
}

extern "C" int sy_conv2d_wgrad_tc(const SyConvWgradDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  wg::Plan pl{};
  const int rc = wg::make_plan(d, &pl);
  if (rc != SY_OK) return rc;
  SY_REQUIRE(d->dw != nullptr && d->workspace != nullptr, SY_EINVAL, "conv2d_wgrad: null dw / workspace");
  SY_REQUIRE(d->workspace_bytes >= pl.ws_bytes, SY_EWORKSPACE, "conv2d_wgrad: workspace %zu < %zu", d->workspace_bytes, pl.ws_bytes);
  SY_REQUIRE(((uintptr_t)d->workspace % 16) == 0, SY_EINVAL, "conv2d_wgrad: workspace must be 16B aligned");
  const SyTensor& x = d->x;
  const SyTensor& dy = d->dy;
  SY_REQUIRE(tc::get_encode() != nullptr && tc::get_encode_im2col() != nullptr, SY_EARCH,
             "tensor-map encoders not available from the driver");
  const int ph = (d->kh - 1) / 2, pw = (d->kw - 1) / 2;
  wg::WParams p{};
  p.P_total = x.n * pl.ho * pl.wo; p.Ho = pl.ho; p.Wo = pl.wo; p.stride = d->stride; p.pad_h = ph; p.pad_w = pw; p.kw = d->kw;
  p.Cout = dy.c; p.Cin = x.c;
  p.m_tiles = pl.m_tiles; p.n_tiles = pl.n_tiles; p.taps = pl.taps; p.ksplit = pl.ksplit; p.kb_total = pl.kb_total;
  p.kb_per_split = pl.kb_per_split; p.items = pl.items;
  p.fd_hw = tc::make_fastdiv((uint32_t)(pl.ho * pl.wo));
  p.fd_wo = tc::make_fastdiv((uint32_t)pl.wo);
  p.partial = reinterpret_cast<float*>(d->workspace);
  CUtensorMap tdy, tx;
  {
    // dy as (C, pixels): box (64 ch, 64 px); pixels past the end / channels past Cout read as zero
    const cuuint64_t dims[2] = {(cuuint64_t)dy.c, (cuuint64_t)p.P_total};
    const cuuint64_t strides[1] = {(cuuint64_t)dy.pitch * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)wg::kPixK};
    const CUresult r = tc::encode_tiled(&tdy, 2, dy.ptr, dims, strides, box);
    SY_REQUIRE(r == CUDA_SUCCESS, SY_ELAUNCH, "cuTensorMapEncodeTiled(dy) failed: %d", (int)r);
  }
  {
    // x in im2col mode, 64 base pixels per load (same bounding box as the forward kernel's linear tiles)
    const CUresult r = tc::encode_im2col_nhwc(&tx, x, d->kh, d->kw, d->stride, wg::kPixK);
    SY_REQUIRE(r == CUDA_SUCCESS, SY_ELAUNCH, "cuTensorMapEncodeIm2col(x) failed: %d", (int)r);
  }
  int lrc;
  switch (pl.bn) {
    case 64: lrc = wg::launch<64>(tdy, tx, p, stream); break;
    case 128: lrc = wg::launch<128>(tdy, tx, p, stream); break;
    default: lrc = wg::launch<256>(tdy, tx, p, stream); break;
  }
  if (lrc != SY_OK) return lrc;
  const long long total = (long long)dy.c * x.c * pl.taps;
  // split groups per output: enough threads to cover the GPU (SMs x 2048) and at least 8 splits per group
  int sg = 1;
  while (sg < 8 && total * sg < (long long)tc::num_sms() * 2048 && pl.ksplit >= 16 * sg) sg *= 2;
  const long long per_block = 256 / sg;
  const long long want = (total + per_block - 1) / per_block;
  const int blocks = (int)(want < tc::num_sms() * 8 ? want : tc::num_sms() * 8);
  switch (sg) {
    case 8: wg::wgrad_reduce_kernel<8><<<blocks, 256, 0, stream>>>(p.partial, pl.bn, pl.m_tiles, pl.n_tiles, pl.taps, pl.ksplit, dy.c, x.c, d->dw, d->accumulate); break;
    case 4: wg::wgrad_reduce_kernel<4><<<blocks, 256, 0, stream>>>(p.partial, pl.bn, pl.m_tiles, pl.n_tiles, pl.taps, pl.ksplit, dy.c, x.c, d->dw, d->accumulate); break;
    case 2: wg::wgrad_reduce_kernel<2><<<blocks, 256, 0, stream>>>(p.partial, pl.bn, pl.m_tiles, pl.n_tiles, pl.taps, pl.ksplit, dy.c, x.c, d->dw, d->accumulate); break;
    default: wg::wgrad_reduce_kernel<1><<<blocks, 256, 0, stream>>>(p.partial, pl.bn, pl.m_tiles, pl.n_tiles, pl.taps, pl.ksplit, dy.c, x.c, d->dw, d->accumulate); break;
  }
  return launch_status("wgrad_reduce_kernel");
}
