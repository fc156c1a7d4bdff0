// Implicit-GEMM convolution on the Hopper tensor cores (sm_90a, wgmma).
//
//   M = 128 output pixels: 128 consecutive pixels of the flattened (n, oh, ow) space ("linear" tiles, the default), or a
//       16 x 8 patch of one image with its input halo (3x3 stride-1 convs; template parameter AM, see below)
//   N = output channels (BN = 64/128 per tile, chosen per layer)
//   K = taps * Cin, walked as (tap, 64-channel block)
//
// Operand movement is im2col-free: for linear tiles ONE im2col-mode TMA load per (tap, channel block) brings the shifted
// input pixels [128][64ch] straight from the NHWC tensor into a 128B-swizzled shared-memory tile (out-of-bounds = zero
// padding = the conv padding; stride-2 convs use the tensor map's element strides), and one 3-D TMA load brings the
// [BN][64] weight slab.  Two consumer warpgroups issue wgmma.mma_async (M=64 each, N=BN, K=16) with both operands in
// shared memory and the fp32 accumulators in registers.
//
// Warp roles (640 threads = five warpgroups, persistent CTA, one per SM), one function each:
//   warps 0-7   mma_convert: warpgroup wg computes rows [64 wg, +64) of the tile, then per 64-column slab converts its
//               accumulators (raw | folded BN + SiLU + residual) to bf16 in a 128B-swizzled shared staging tile
//   warps 8-15  statistics: per-channel (sum, sum of squares) of the staged tile in per-lane register accumulators that persist
//               across slabs and tiles (overlaps the next slab's conversion)
//   warps 0-15  bn_tail after either role: partial row, grid barrier, BatchNorm finalize
//   warp 16 store_slabs: TMA store (one 4-D store per slab; the tensor map clips the tile to the tensor / the channel slice)
//   warp 17 barrier init + weight (B) loads   warp 18 activation (A) loads: load_linear | load_halo_b, load_halo_a
//   warp 19 idle
// The kernel body carves up shared memory, initialises the barriers and dispatches the roles; every role walks the tiles
// through TileWalk.  setmaxnreg at the start of each branch moves registers from warps 16-19 to the MMA and statistics
// warpgroups (kRegs*).
// BN = 256 is not offered: 64 x 256 fp32 accumulators are 128 registers per thread, more than the MMA warpgroups can hold.
//
// Train-mode BatchNorm is folded into this kernel as far as the grid-wide dependency allows:
// every CTA accumulates per-channel (sum, sum of squares) of the values it stored, per
// statistics group (current / support frames), and writes ONE partial row.  All CTAs of the
// persistent grid are co-resident (one per SM), so the kernel ends with a grid-wide barrier after
// which every CTA reduces a slice of the channels over the rows (one per SM) in a fixed order
// (deterministic), updates the running statistics and publishes scale/shift for the normalise+SiLU
// pass.  (Two such kernels must not run concurrently on one GPU: the barrier needs the whole grid.)
//
// Activation storage: conv_tc_kernel reads and writes bf16 (every mode).  conv_tc_f16_kernel runs the same roles on fp16
// activations and weights (wgmma .f16 inputs, fp16 tensor maps, fp16 epilogue pack / residual): the FUSED epilogue of the
// eval and streaming forwards only, so its statistics warps just cycle the staging-tile barriers and its tail is empty.
//
// Replaces the cuDNN conv + ATen BN/SiLU triplet behind [yolox] BaseConv
// (exps/model/darknet.py:115-165, dfp_pafpn.py:33-105, tal_head.py:55-104 of StreamYOLO).
#include <cuda.h>
#include <stdio.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace sy {
namespace tc {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;              // 16-bit elements = one 128-byte swizzle row
constexpr int kThreads = 640;       // five warpgroups
// registers per thread after setmaxnreg: the launch grants 96 x 640; the load/store warpgroup (warps 16-19) keeps 32 and
// hands the rest to the MMA warpgroups (accumulators: BN / 2 registers) and the statistics warpgroups (per-lane sums)
constexpr int kRegsLaunch = 96;
constexpr int kRegsMma = 104;
constexpr int kRegsStats = 120;
constexpr int kRegsIo = 32;
static_assert(2 * kRegsMma + 2 * kRegsStats + kRegsIo <= 5 * kRegsLaunch, "register budget of one CTA");
constexpr int kEpiThreads = 256;    // MMA + convert warps 0-7
constexpr int kTailThreads = 512;   // convert + statistics warps run the kernel tail (partials, grid barrier, finalize)
constexpr int kABytes = kBlockM * 128;   // 16 KiB per stage
constexpr int kMaxStages = 8;
// Linear tiles: a ring of four A+B stages (four 64-deep K blocks in flight), not as many as shared memory holds.
// bench.py's forward+loss step on an H100 80GB HBM3 at 700 W, ring depth capped at 3 / 4 / 5 / none (= 6 stages at
// BN = 128): 405 / 416 / 404 / 387 pairs/s.  Why deeper rings are slower has not been isolated; four is the measured optimum.
constexpr int kRingStages = 4;
// Halo tiles: a 16 x 8 output patch (one 8-pixel swizzle atom per patch row) and its 18 x 10 input halo, stored densely
// (kHaloPitch pixels = 1280 bytes per halo row: the MMA's swizzle follows the absolute shared address bits, exactly like the
// TMA that wrote the tile, so neither the atoms' stride nor their start needs 1 KiB alignment); three filter taps per
// weight-ring stage (one barrier round per filter row)
constexpr int kHaloTH = 16, kHaloTW = 8;
constexpr int kHaloPitch = kHaloTW + 2;
constexpr int kHaloTx = (kHaloTH + 2) * kHaloPitch * 128;           // bytes one halo load delivers
constexpr int kHaloBytes = (kHaloTx + 1023) / 1024 * 1024;          // halo ring stage stride (multiple of 1 KiB)
constexpr int kHaloTaps = 3;

struct BnSeg {
  const float* gamma; const float* beta;
  float* rmean; float* rvar; long long* nbt;
  int c_begin;
};

struct Params {
  int N, Ho, Wo, Cout;
  int kw, stride, pad_h, pad_w;
  int tiles_x, tiles_y;     // halo mode: 16 x 8 patches per image row / column
  int m_tiles, n_tiles;
  FastDiv fd_m_tiles, fd_per_img, fd_tiles_x;
  // tile walk (pick_walk; see TileWalk) and the statistics rows it fills
  int band, t_end, cls_step, cls_tiles;
  int stat_rows;            // partial rows the finalize sums (N-major: one per CTA; M-band: one per class)
  FastDiv fd_band, fd_cls_tiles;
  // linear tiles (LIN): an M tile is 128 consecutive output pixels of the flattened (n, oh, ow) space
  int P_total;              // N * Ho * Wo
  int gp;                   // first output pixel of statistics group 1 (== P_total: single group)
  FastDiv fd_hw, fd_wo;
  int cblocks, kblocks, stages;
  int stage_tiles;          // 1 or 2 epilogue staging tiles
  int stagesA;              // halo mode: halo ring depth
  int mode, act;
  const uint16_t* res;      // 16-bit elements of the kernel's storage type (bf16 | fp16)
  long long res_pitch;
  const float* scale;
  const float* shift;
  // statistics / BatchNorm finalize (RAW mode)
  int split_n;              // images >= split_n form statistics group 1
  float* partials;          // [gridDim][Cout][2 groups][2 (sum, sumsq)] or nullptr (no statistics)
  int n_seg;                // > 0: finalize BatchNorm in the kernel tail (grid barrier + parallel reduce)
  BnSeg seg[2];
  float momentum, eps;
  double inv_cnt[2];        // 1 / (values per channel) of statistics group 0 | 1 (host-computed: no fp64 division in the tail)
  float unbias[2];          // cnt / (cnt - 1) of each group: biased -> unbiased variance for the running statistics
  int updates;              // running-statistics updates per channel: 1, or 2 (two groups, or one group applied twice)
  float* ss;                // [2 (scale|shift)][2 groups][Cout]
  float* mi;                // optional [2 (mean|invstd)][2 groups][Cout] for the backward pass
  unsigned int* sync;       // two counters (grid barrier + exit ticket), zero between launches
  long long* timeline;      // debug: CTA 0 records (event id, clock) pairs; nullptr in production
  int timeline_cap;
  int debug_flags;          // debug: 2 = skip the TMA loads (barriers still cycle)
  float* dbg_f32;           // validation: fp32 accumulators [pixel][Cout] written next to the stored result (nullptr in production)
};

// debug timeline: event = role<<28 | phase<<24 | tile<<8 | kb ; written by CTA 0 only
template <bool TL>
__device__ __forceinline__ void tl_rec(const Params& p, int& n, int role, int phase, int tile, int kb) {
  if (TL && p.timeline != nullptr && blockIdx.x == 0 && n + 1 < p.timeline_cap) {
    p.timeline[2 * n] = ((long long)role << 28) | ((long long)phase << 24) | ((long long)(tile & 0xffff) << 8) | (kb & 0xff);
    p.timeline[2 * n + 1] = clock64();
    ++n;
  }
}

__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
// staging-tile hand-off between the 8 convert warps, the 8 statistics warps and the store warp: 256 + 256 + 32 threads
// One or two staging tiles (Params::stage_tiles; slab j uses tile j & 1 when there are two, so that the TMA store /
// statistics of one slab overlap the conversion of the next -- worth an operand stage only for epilogue-bound layers);
// named barriers 2,3 belong to tile 0 and 6,7 to tile 1.
// Producer/consumer protocol (PTX bar.arrive / bar.sync pairs, 256 + 256 + 32 = 544 threads per barrier):
//   free(b)   : store warp arrives when its TMA store has read tile b, statistics warps arrive when their loads of
//               tile b are done; the convert warps WAIT on it before overwriting the tile
//   staged(b) : convert warps arrive after writing tile b (+ proxy fence); store and statistics warps WAIT on it
// so the convert warps never wait for the statistics arithmetic or the store issue, only for the tile to be read.
__device__ __forceinline__ void bar_free_wait(int b, int n = 544) { asm volatile("bar.sync %0, %1;" ::"r"(2 + 4 * b), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_free_arrive(int b, int n = 544) { asm volatile("bar.arrive %0, %1;" ::"r"(2 + 4 * b), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_staged_wait(int b, int n = 544) { asm volatile("bar.sync %0, %1;" ::"r"(3 + 4 * b), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_staged_arrive(int b, int n = 544) { asm volatile("bar.arrive %0, %1;" ::"r"(3 + 4 * b), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_stats_done() { asm volatile("bar.sync 5, 512;" ::: "memory"); }

// K-major, 128B-swizzled operand tile: rows of 128 bytes, 8-row atoms `sbo` bytes apart (1 KiB for a TMA-written tile).
// The leading byte offset is unused by K-major swizzled layouts.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t sbo = 1024u, uint32_t base_offset = 0u) {
  return make_gmma_desc(saddr, 16u, sbo, base_offset);
}

constexpr int kSlabCols = 64;                  // epilogue slab: 64 bf16 columns = one 128-byte swizzled row
constexpr int kSlabBytes = kBlockM * 128;      // 16 KiB staging tile

template <int BN>
struct Cfg {
  static constexpr int kBBytes = BN * 128;
  static constexpr int kAcc = BN / 2;                               // fp32 accumulators per consumer thread (64 rows x BN)
  // fixed part of dynamic smem (everything but the A/B ring and the per-CTA statistic accumulators)
  // plus, after the barriers, ONE region that is scale/shift (FUSED, 2 KiB) or the statistic accumulators (RAW)
  static constexpr int kFixedBytes = 1024 /*align slack*/ + kSlabBytes + 256 /*barriers*/;
};

// Tile walk of this CTA (pick_walk).  Every member is an expression of the kernel parameters and blockIdx, not a stored
// value: those cost no registers.
//   band == 1 (N-major): walk index = tile index, M fastest.
//   band == n_tiles (M-band): CTA b = slot * band + N tile; walk index t = class * cls_tiles + k visits M tile rho + k *
//   stat_rows of class rho = slot + class * cls_step.
// decode() is false for walk indices that name no tile (every role skips them alike).
struct TileWalk {
  const Params& p;
  __device__ __forceinline__ int first() const { return p.band > 1 ? 0 : (int)blockIdx.x; }
  __device__ __forceinline__ int step() const { return p.band > 1 ? 1 : (int)gridDim.x; }
  __device__ __forceinline__ int end() const { return p.t_end; }
  __device__ __forceinline__ bool mband() const { return p.band > 1; }
  // M-band walk: this CTA's slot (a fast division: callers evaluate it once) and N tile, the class of walk index t
  __device__ __forceinline__ int slot() const { return fdiv((int)blockIdx.x, p.fd_band); }
  __device__ __forceinline__ int band_n_tile(int slot) const { return (int)blockIdx.x - slot * p.band; }
  __device__ __forceinline__ int cls(int t) const { return fdiv(t, p.fd_cls_tiles); }
  // partial row of class cls (M-tile class rho = slot + cls * cls_step): the N-major walk's CTA (n_tile * m_tiles + rho)
  // mod stat_rows
  __device__ __forceinline__ int class_row(int slot, int cls) const {
    return (int)(((long long)band_n_tile(slot) * p.m_tiles + slot + cls * p.cls_step) % p.stat_rows);
  }
  __device__ __forceinline__ bool decode(int t, int& n_tile, int& m_tile) const {
    if (p.band == 1) {
      n_tile = fdiv(t, p.fd_m_tiles);
      m_tile = t - n_tile * p.m_tiles;
      return true;
    }
    const int s = slot();
    n_tile = band_n_tile(s);
    const int c = cls(t);
    const int r = s + c * p.cls_step;
    m_tile = r + (t - c * p.cls_tiles) * p.stat_rows;
    return r < p.stat_rows && m_tile < p.m_tiles;
  }
};

// position in a ring of mbarrier-guarded stages: the stage and the parity of its current phase
struct RingCursor {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance(int depth) {
    if (++stage == depth) { stage = 0; phase ^= 1u; }
  }
};

// first output pixel of an M tile as (image, row, column): the top-left corner of a halo patch, the first of 128
// consecutive pixels of a linear tile
struct TileOrigin {
  int img, y, x;
};
__device__ __forceinline__ TileOrigin halo_origin(const Params& p, int m_tile) {
  const int img = fdiv(m_tile, p.fd_per_img), rem = m_tile - img * (p.tiles_x * p.tiles_y);
  const int py = fdiv(rem, p.fd_tiles_x), px = rem - py * p.tiles_x;
  return {img, py * kHaloTH, px * kHaloTW};
}
__device__ __forceinline__ TileOrigin linear_origin(const Params& p, int m_tile) {
  const int p0 = m_tile * kBlockM;
  const int img = fdiv(p0, p.fd_hw);
  const int rem = p0 - img * (p.Ho * p.Wo);
  const int oh = fdiv(rem, p.fd_wo), ow = rem - oh * p.Wo;
  return {img, oh, ow};
}

// the BatchNorm (segment) that channel c belongs to
__device__ __forceinline__ const BnSeg& bn_seg(const Params& p, int c) {
  return (p.n_seg > 1 && c >= p.seg[1].c_begin) ? p.seg[1] : p.seg[0];
}

// Shared memory of a CTA as the roles see it (carved up in conv_tc_kernel)
struct Smem {
  uint8_t* a;            // A ring: linear stages of kABytes | halo stages of kHaloBytes
  uint8_t* b;            // B ring: one weight slab per stage | halo mode: kHaloTaps slabs per stage
  uint8_t* stage;        // Params::stage_tiles epilogue staging tiles (1024-aligned: the rings are multiples of 1 KiB)
  float* acc;            // RAW: statistic accumulators [2 groups][2][Cout]; FUSED: [256] scale, [256] shift
  uint32_t bar0;         // mbarriers: [0,8) full, [8,16) empty, [16,19) halo full, [19,22) halo empty
  int sflip;             // slab parity toggles the staging tile iff there are two
  __device__ __forceinline__ uint32_t full(int s) const { return bar0 + 8u * s; }
  __device__ __forceinline__ uint32_t empty(int s) const { return bar0 + 8u * (kMaxStages + s); }
  __device__ __forceinline__ uint32_t full_a(int s) const { return bar0 + 8u * (2 * kMaxStages + s); }   // halo ring (<= 3)
  __device__ __forceinline__ uint32_t empty_a(int s) const { return bar0 + 8u * (2 * kMaxStages + 3 + s); }
};

// ---------------------------------------------------------------- warp 18, halo mode: activation (A) loads
// one halo box [18 rows][10 px][64 ch] per (tile, channel block)
__device__ __forceinline__ void load_halo_a(const Params& p, const Smem& sm, const CUtensorMap& tmA) {
  const TileWalk w{p};
  RingCursor ra;
  for (int tile = w.first(); tile < w.end(); tile += w.step()) {
    int n_tile, m_tile;
    if (!w.decode(tile, n_tile, m_tile)) continue;
    const TileOrigin o = halo_origin(p, m_tile);
    for (int cb = 0; cb < p.cblocks; ++cb) {
      mbar_wait(sm.empty_a(ra.stage), ra.phase ^ 1u);
      if (elect_one()) {
        if (p.debug_flags & 2) {
          mbar_arrive(sm.full_a(ra.stage));
        } else {
          mbar_expect_tx(sm.full_a(ra.stage), (uint32_t)kHaloTx);
          tma_load_4d(smem_u32(sm.a + ra.stage * kHaloBytes), &tmA, sm.full_a(ra.stage), cb * kBlockK, o.x - 1, o.y - 1, o.img);
        }
      }
      __syncwarp();
      ra.advance(p.stagesA);
    }
  }
}

// ---------------------------------------------------------------- warp 17, halo mode: weight (B) loads
// kHaloTaps [BN][64] weight slabs (one filter row) per (channel block, ring stage)
template <int BN>
__device__ __forceinline__ void load_halo_b(const Params& p, const Smem& sm, const CUtensorMap& tmB) {
  constexpr int kBB = Cfg<BN>::kBBytes;
  const TileWalk w{p};
  RingCursor rb;
  for (int tile = w.first(); tile < w.end(); tile += w.step()) {
    int n_tile, m_tile_unused;
    if (!w.decode(tile, n_tile, m_tile_unused)) continue;
    for (int cb = 0; cb < p.cblocks; ++cb) {
      for (int t0 = 0; t0 < 9; t0 += kHaloTaps) {
        mbar_wait(sm.empty(rb.stage), rb.phase ^ 1u);
        if (elect_one()) {
          if (p.debug_flags & 2) {
            mbar_arrive(sm.full(rb.stage));
          } else {
            mbar_expect_tx(sm.full(rb.stage), (uint32_t)(kHaloTaps * kBB));
#pragma unroll
            for (int j = 0; j < kHaloTaps; ++j)
              tma_load_3d(smem_u32(sm.b + (rb.stage * kHaloTaps + j) * kBB), &tmB, sm.full(rb.stage), cb * kBlockK, t0 + j,
                          n_tile * BN);
          }
        }
        __syncwarp();
        rb.advance(p.stages);
      }
    }
  }
}

// ---------------------------------------------------------------- warps 17 / 18, linear tiles: B / A loads
// Two issuing threads because a single thread needs a few hundred cycles per cp.async.bulk.tensor: the pair keeps a
// K block's issue time below its MMA time.  Both arrive (with their byte counts) on the same full barrier.
template <int BN, bool TL>
__device__ __forceinline__ void load_linear(const Params& p, const Smem& sm, const CUtensorMap& tmA, const CUtensorMap& tmB,
                                            bool is_a) {
  constexpr int kBB = Cfg<BN>::kBBytes;
  const TileWalk w{p};
  RingCursor ring;
  int tl_n = is_a ? 0 : p.timeline_cap / 8;
  for (int tile = w.first(); tile < w.end(); tile += w.step()) {
    int n_tile, m_tile;
    if (!w.decode(tile, n_tile, m_tile)) continue;
    const TileOrigin o = linear_origin(p, m_tile);
    const int y0 = o.y * p.stride - p.pad_h, x0 = o.x * p.stride - p.pad_w;
    // walk the (tap, channel block) K blocks, one per ring stage
    int r = 0, sx = 0, cb = 0;
    for (int kb = 0; kb < p.kblocks; ++kb) {
      mbar_wait(sm.empty(ring.stage), ring.phase ^ 1u);          // whole warp waits: control flow stays uniform
      if (elect_one()) {
        tl_rec<TL>(p, tl_n, is_a ? 0 : 3, 0, tile, kb);
        if (p.debug_flags & 2) mbar_arrive(sm.full(ring.stage));
        else mbar_expect_tx(sm.full(ring.stage), is_a ? (uint32_t)kABytes : (uint32_t)kBB);
        tl_rec<TL>(p, tl_n, is_a ? 0 : 3, 1, tile, kb);
      }
      if (!(p.debug_flags & 2) && elect_one()) {
        if (is_a)
          tma_load_im2col_4d(smem_u32(sm.a + ring.stage * kABytes), &tmA, sm.full(ring.stage), cb * kBlockK, x0, y0, o.img,
                             (uint16_t)sx, (uint16_t)r);
        else
          tma_load_3d(smem_u32(sm.b + ring.stage * kBB), &tmB, sm.full(ring.stage), cb * kBlockK, r * p.kw + sx, n_tile * BN);
      }
      if (++cb == p.cblocks) { cb = 0; if (++sx == p.kw) { sx = 0; ++r; } }
      if (TL && elect_one()) tl_rec<TL>(p, tl_n, is_a ? 0 : 3, 2, tile, kb);
      __syncwarp();
      ring.advance(p.stages);
    }
  }
}

// ---------------------------------------------------------------- warp 16: TMA store
// One 4-D TMA store per 64-column slab; the tensor map clips the patch to the image and to the
// channel slice.  Issuing it here keeps its issue + drain latency off the epilogue warps' path.
template <int BN, bool TL, int AM>
__device__ __forceinline__ void store_slabs(const Params& p, const Smem& sm, const CUtensorMap& tmY, int tid) {
  const int lane = tid & 31;
  const TileWalk w{p};
  const int sflip = sm.sflip;
  const uint32_t stage_base = smem_u32(sm.stage);
  int sbuf = 0, prev = -1;
  int tl_s = 7 * (p.timeline_cap / 8);
  const int nbar = 544;
  bar_free_arrive(0, nbar);                    // both tiles start out free
  if (sflip) bar_free_arrive(1, nbar);
  for (int tile = w.first(); tile < w.end(); tile += w.step()) {
    int n_tile, m_tile;
    if (!w.decode(tile, n_tile, m_tile)) continue;
    int c1, c2, c3;                            // store coordinates below the channel: (x, y, image) | (pixel, 0, 0)
    if constexpr (AM == 1) {
      c1 = m_tile * kBlockM; c2 = 0; c3 = 0;
    } else {
      const TileOrigin o = halo_origin(p, m_tile);
      c1 = o.x; c2 = o.y; c3 = o.img;
    }
    for (int slab = 0; slab < BN / kSlabCols; ++slab, sbuf ^= sflip) {
      bar_staged_wait(sbuf, nbar);
      if (lane == 0) tl_rec<TL>(p, tl_s, 6, 0, tile, slab);
      if (elect_one()) {
        tma_store_4d(&tmY, stage_base + (uint32_t)(sbuf * kSlabBytes), n_tile * BN + slab * kSlabCols, c1, c2, c3);
        bulk_commit();
        if (sflip) {
          if (prev >= 0) bulk_wait_read1();    // two tiles: the previous slab's store has read ITS tile
        } else {
          bulk_wait_read();                    // one tile: wait until this store has read it
        }
      }
      __syncwarp();
      if (lane == 0) tl_rec<TL>(p, tl_s, 6, 1, tile, slab);
      if (sflip) {
        if (prev >= 0) bar_free_arrive(prev, nbar);
        prev = sbuf;
      } else {
        bar_free_arrive(0, nbar);
      }
    }
  }
  if (sflip && prev >= 0) {
    if (elect_one()) bulk_wait_read();
    __syncwarp();
    bar_free_arrive(prev, nbar);
  }
  // the stores have read the staging tiles before the CTA's final __syncthreads; their writes complete with the grid
  if (lane == 0) bulk_wait_read();
  __syncwarp();
}

// ---------------------------------------------------------------- warps 8-15: statistics
// Warp ew reduces columns [8*ew, 8*ew+8) of every staged 64-column slab while the convert warps already
// convert the next slab; one owner lane per (column, sum|sumsq) accumulates in fixed order.
template <int BN, bool TL, int AM>
__device__ __forceinline__ void statistics(const Params& p, const Smem& sm, int tid) {
  const int warp = tid >> 5, lane = tid & 31;
  const TileWalk w{p};
  float* sAcc = sm.acc;
  const int sflip = sm.sflip;
  const int ew = warp - 8;
  const int st = tid - 256;                    // 0..255
  const uint32_t stage_base = smem_u32(sm.stage);
  const bool do_stats = (p.mode == SY_CONV_RAW) && (p.partials != nullptr);
  if (do_stats) {
    for (int i = st; i < 4 * p.Cout; i += 256) sAcc[i] = 0.f;
  }
  int sbuf = 0;
  int tl_t = (st == 0) ? 5 * (p.timeline_cap / 8) : p.timeline_cap;
  const int nbar = 544;
  bar_free_arrive(0, nbar);                    // both tiles start out free
  if (sflip) bar_free_arrive(1, nbar);
  // Warp ew owns columns [8*ew, 8*ew+8) of every 64-column slab; lane l reads rows l, l+32, l+64, l+96 (one 16-byte
  // chunk each).  The per-lane partial sums (8 columns x {sum, sum of squares}) stay in REGISTERS across slabs and tiles
  // -- one set per slab index of the tile -- and are only combined across the 32 lanes (recursive-halving shuffles) and
  // added to the CTA's shared-memory totals on a FLUSH: when the CTA moves to another n tile (N-major walk only) or
  // statistics group, on a tile that straddles the group boundary, and at the end.  (Per-slab shuffle reductions made the statistics warps the
  // bottleneck of every epilogue-bound layer: ~1400 cycles per slab.)
  constexpr int kSlabs = BN / kSlabCols;
  float acc[kSlabs][16];
#pragma unroll
  for (int j = 0; j < kSlabs; ++j)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[j][i] = 0.f;
  int pend_grp = -1, pend_n0 = 0;                          // what the register sums belong to (-1: nothing pending)
  // lanes combine a[16] (fixed shuffle tree: deterministic) and the 16 owner lanes add into the shared totals
  auto reduce_store = [&](float (&a)[16], int grp, int col_base) {
    float b8[8], c4[4], d2[2], e1;
    {
      const bool up = (lane & 16) != 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float send = up ? a[i] : a[8 + i], keep = up ? a[8 + i] : a[i];
        b8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
      }
    }
    {
      const bool up = (lane & 8) != 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float send = up ? b8[i] : b8[4 + i], keep = up ? b8[4 + i] : b8[i];
        c4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
      }
    }
    {
      const bool up = (lane & 4) != 0;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float send = up ? c4[i] : c4[2 + i], keep = up ? c4[2 + i] : c4[i];
        d2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
      }
    }
    {
      const bool up = (lane & 2) != 0;
      const float send = up ? d2[0] : d2[1], keep = up ? d2[1] : d2[0];
      e1 = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    }
    e1 += __shfl_xor_sync(0xffffffffu, e1, 1);
    if ((lane & 1) == 0) {               // 16 owner lanes: bit4 = sum | sumsq, bits 3..1 = column in the group
      const int col = col_base + ew * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
      if (col < p.Cout) sAcc[(grp * 2 + (lane >> 4)) * p.Cout + col] += e1;
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = 0.f;
  };
  auto flush = [&]() {
    if (pend_grp < 0) return;
#pragma unroll
    for (int j = 0; j < kSlabs; ++j) reduce_store(acc[j], pend_grp, pend_n0 + j * kSlabCols);
    pend_grp = -1;
  };
  // M-band walk: the CTA's tiles of one class rho are exactly those that one CTA of the N-major walk took for this N tile,
  // in the same order, so this CTA's sums of a class are that CTA's partial row for these BN columns, bit for bit.  The
  // row of class rho is the N-major walk's CTA (n_tile * m_tiles + rho) mod stat_rows; classes without tiles write zeros.
  auto write_class = [&](int cls, bool zero) {                 // all 256 statistics threads
    const int my_slot = w.slot();
    float4* dst = reinterpret_cast<float4*>(p.partials) + (size_t)w.class_row(my_slot, cls) * p.Cout;
    const int c = w.band_n_tile(my_slot) * BN + st;
    if (zero) {
      if (st < BN && c < p.Cout) dst[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      return;
    }
    asm volatile("bar.sync 8, 256;" ::: "memory");          // the owner lanes' shared-memory sums are complete
    if (st < BN && c < p.Cout) {
      dst[c] = make_float4(sAcc[c], sAcc[p.Cout + c], sAcc[2 * p.Cout + c], sAcc[3 * p.Cout + c]);
      sAcc[c] = 0.f; sAcc[p.Cout + c] = 0.f; sAcc[2 * p.Cout + c] = 0.f; sAcc[3 * p.Cout + c] = 0.f;
    }
    asm volatile("bar.sync 8, 256;" ::: "memory");
  };
  int pend_cls = -1;                                           // class whose sums sAcc holds (M-band walk)
  if (do_stats && w.mband()) {
    const int my_slot = w.slot();
    for (int cls = 0; my_slot + cls * p.cls_step < p.stat_rows; ++cls)
      if (my_slot + cls * p.cls_step >= p.m_tiles) write_class(cls, true);
  }
  for (int tile = w.first(); tile < w.end(); tile += w.step()) {
    int n_tile, m_tile;
    if (!w.decode(tile, n_tile, m_tile)) continue;
    const int n0 = n_tile * BN;
    // rows [0, cut) of the tile belong to statistics group 0, rows [cut, 128) to group 1 (a halo tile lies in one
    // image = one group; a linear tile can straddle the boundary; rows past the end of the tensor were staged as zeros)
    int cut;
    if constexpr (AM == 1) {
      cut = min(max(p.gp - m_tile * kBlockM, 0), kBlockM);
    } else {
      cut = fdiv(m_tile, p.fd_per_img) >= p.split_n ? 0 : kBlockM;
    }
    const bool pure = (cut <= 0) || (cut >= kBlockM);
    const int tgrp = cut <= 0 ? 1 : 0;
    if (do_stats && w.mband()) {                               // warp-uniform
      const int cls = w.cls(tile);
      if (pend_cls >= 0 && cls != pend_cls) {
        flush();
        write_class(pend_cls, false);
      }
      pend_cls = cls;
    }
    if (do_stats && (!pure || pend_grp != tgrp || pend_n0 != n0)) flush();     // warp-uniform
    for (int slab = 0; slab < kSlabs; ++slab, sbuf ^= sflip) {
      bar_staged_wait(sbuf, nbar);
      tl_rec<TL>(p, tl_t, 5, 0, tile, slab);
      const uint32_t tile_base = stage_base + (uint32_t)(sbuf * kSlabBytes);
      float x[4][8];
      if (do_stats) {
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
          const uint32_t r = (uint32_t)(lane + 32 * rr);
          const uint4 u = lds128(tile_base + r * 128u + ((((uint32_t)ew) ^ (r & 7u)) << 4));
          x[rr][0] = bf16_lo(u.x); x[rr][1] = bf16_hi(u.x); x[rr][2] = bf16_lo(u.y); x[rr][3] = bf16_hi(u.y);
          x[rr][4] = bf16_lo(u.z); x[rr][5] = bf16_hi(u.z); x[rr][6] = bf16_lo(u.w); x[rr][7] = bf16_hi(u.w);
        }
      }
      bar_free_arrive(sbuf, nbar);             // the values are in registers: the tile may be overwritten
      tl_rec<TL>(p, tl_t, 5, 1, tile, slab);
      if (do_stats) {
        if (pure) {
          float (&a)[16] = acc[slab];
#pragma unroll
          for (int rr = 0; rr < 4; ++rr) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { a[i] += x[rr][i]; a[8 + i] += x[rr][i] * x[rr][i]; }
          }
          pend_grp = tgrp; pend_n0 = n0;
        } else {
          // the tile straddles the group boundary (at most one M tile per layer and N tile): masked, reduced at once.
          // The sums go through acc[slab]: the flush before this tile left it zero, and reduce_store zeroes it again
          // (a separate scratch array made the BN = 64 statistics warps spill)
#pragma unroll 1
          for (int grp = 0; grp < 2; ++grp) {
            const int lo = grp ? cut : 0, hi = grp ? kBlockM : cut;
            float (&a)[16] = acc[slab];
#pragma unroll
            for (int rr = 0; rr < 4; ++rr) {
              const int r = lane + 32 * rr;
              if (r >= lo && r < hi) {
#pragma unroll
                for (int i = 0; i < 8; ++i) { a[i] += x[rr][i]; a[8 + i] += x[rr][i] * x[rr][i]; }
              }
            }
            reduce_store(a, grp, n0 + slab * kSlabCols);
          }
        }
      }
      tl_rec<TL>(p, tl_t, 5, 2, tile, slab);
    }
  }
  if (do_stats) flush();
  if (do_stats && w.mband() && pend_cls >= 0) write_class(pend_cls, false);
}

// ---------------------------------------------------------------- warps 0-7: MMA + convert
// Warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile: it issues the wgmma stream for them (accumulators in
// registers), then converts its rows of every 64-column slab into the staging tile.  A ring stage is handed back to the
// producers one commit group late (wgmma.wait_group 1), so the next group's MMAs are queued while the last ones drain.
// Returns the debug-timeline cursor of thread 0, which the kernel tail carries on.  F16: fp16 operands and output.
template <int BN, bool TL, int AM, bool F16, bool KINK>
__device__ __forceinline__ int mma_convert(const Params& p, const Smem& sm, int tid) {
  // the compiler knows this range for threadIdx.x but not for the argument; with it the FUSED scale/shift fill below is
  // one guarded pass instead of a loop
  __builtin_assume(tid >= 0 && tid < kThreads);
  using C = Cfg<BN>;
  constexpr bool LIN = (AM == 1);
  constexpr bool HALO = (AM == 2);
  constexpr int kBB = C::kBBytes;
  const TileWalk w{p};
  const int sflip = sm.sflip;
  float* sScale = sm.acc;
  float* sShift = sScale + 256;
  const int warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const int et = tid;                                            // 0..255
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);        // this thread's tile rows: r0 and r0 + 8
  const int cq = 2 * (lane & 3);                                 // its first column in every 8-column group
  const uint32_t stage_base = smem_u32(sm.stage);
  const bool lead = (tid & 127) == 0;                            // signals the warpgroup's ring releases
  // halo mode: this warpgroup's 8 output rows start 8 halo rows further down
  constexpr uint32_t row_bytes = HALO ? (uint32_t)kHaloPitch * 128u : 1024u;
  const uint32_t a_off = HALO ? (uint32_t)(wg * 8) * row_bytes : (uint32_t)wg * 8192u;
  float acc[C::kAcc];
  RingCursor ring, ring_a;                                       // B ring (linear: A+B ring) | halo ring
  int sbuf = 0;
  int tl_n = (et == 0) ? p.timeline_cap / 2 : p.timeline_cap;
  for (int tile = w.first(); tile < w.end(); tile += w.step()) {
    int n_tile, m_tile;
    if (!w.decode(tile, n_tile, m_tile)) continue;
    // this thread's output pixels in the flattened (n, oh, ow) space (evaluated where they are used: only the
    // validity flags stay live across the main loop)
    auto pixel = [&](int h, bool& ok) -> long long {
      if constexpr (LIN) {
        const long long px = (long long)m_tile * kBlockM + r0 + 8 * h;
        ok = px < p.P_total;
        return px;
      } else {
        const TileOrigin o = halo_origin(p, m_tile);
        const int row = r0 + 8 * h;
        const int oy = o.y + row / kHaloTW, ox = o.x + row % kHaloTW;
        ok = (oy < p.Ho) && (ox < p.Wo);
        return ((long long)o.img * p.Ho + oy) * p.Wo + ox;
      }
    };
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) pixel(h, valid[h]);
    const int n0 = n_tile * BN;
    tl_rec<TL>(p, tl_n, 2, 0, tile, 0);
    if (p.mode == SY_CONV_FUSED) {
      epi_bar();                               // previous tile's readers of sScale/sShift are done
      for (int c = et; c < BN; c += kEpiThreads) {
        const int cg = n0 + c;
        sScale[c] = (cg < p.Cout && p.scale) ? p.scale[cg] : 1.0f;
        sShift[c] = (cg < p.Cout && p.shift) ? p.shift[cg] : 0.0f;
      }
      epi_bar();
    }
    // ---- main loop
    int pend_b = -1, pend_a = -1;              // ring stages read by the commit group still in flight
    auto release = [&]() {
      if (lead) {
        if (pend_b >= 0) mbar_arrive(sm.empty(pend_b));
        if (pend_a >= 0) mbar_arrive(sm.empty_a(pend_a));
      }
    };
    if constexpr (HALO) {                      // K order = (channel block, tap)
      for (int cb = 0; cb < p.cblocks; ++cb) {
        mbar_wait(sm.full_a(ring_a.stage), ring_a.phase);
        const uint32_t halo = smem_u32(sm.a + ring_a.stage * kHaloBytes) + a_off;
        for (int t0 = 0; t0 < 9; t0 += kHaloTaps) {
          mbar_wait(sm.full(ring.stage), ring.phase);
          wgmma_fence_operand(acc);
          wgmma_fence();
#pragma unroll
          for (int j = 0; j < kHaloTaps; ++j) {
            const int tap = t0 + j;
            const int r = tap / 3, sx = tap - 3 * r;
            const uint32_t a_addr = halo + (uint32_t)r * row_bytes + (uint32_t)sx * 128u;
            const uint64_t da = make_smem_desc(a_addr, row_bytes);
            const uint64_t db = make_smem_desc(smem_u32(sm.b + (ring.stage * kHaloTaps + j) * kBB));
#pragma unroll
            for (int k = 0; k < kBlockK / 16; ++k)   // 16 bf16 = 32 bytes along K inside the swizzle row: +2 in (addr >> 4)
              Wgmma<BN, 0, 0, F16>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (cb | tap | k) != 0);
          }
          wgmma_commit();
          wgmma_fence_operand(acc);
          wgmma_wait<1>();
          release();
          pend_b = ring.stage;
          pend_a = (t0 + kHaloTaps >= 9) ? ring_a.stage : -1;     // the halo is free after its ninth tap
          ring.advance(p.stages);
        }
        ring_a.advance(p.stagesA);
      }
    } else {
      for (int kb = 0; kb < p.kblocks; ++kb) {
        mbar_wait(sm.full(ring.stage), ring.phase);
        wgmma_fence_operand(acc);
        wgmma_fence();
        const uint64_t da = make_smem_desc(smem_u32(sm.a + ring.stage * kABytes) + a_off);
        const uint64_t db = make_smem_desc(smem_u32(sm.b + ring.stage * kBB));
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k)
          Wgmma<BN, 0, 0, F16>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) != 0);
        wgmma_commit();
        wgmma_fence_operand(acc);
        wgmma_wait<1>();
        release();
        pend_b = ring.stage;
        ring.advance(p.stages);
      }
    }
    wgmma_wait<0>();
    wgmma_fence_operand(acc);
    release();
    tl_rec<TL>(p, tl_n, 2, 1, tile, 0);
    // ---- epilogue: per 64-column slab, registers -> (raw | folded BN + act + residual) -> bf16 | fp16 -> staging tile
#pragma unroll
    for (int slab = 0; slab < BN / kSlabCols; ++slab, sbuf ^= sflip) {
      tl_rec<TL>(p, tl_n, 2, 2, tile, slab);
      bar_free_wait(sbuf);                     // (A) staging tile free: its store has read it, the statistics loads are done
      // 16-byte chunk j of row r lives at r*128 + ((j ^ (r & 7)) << 4); this thread's rows r0 and r0 + 8 share r & 7,
      // so the chunk offset is (j << 4) ^ sw: one logic op, nothing kept live across the main loop
      const uint32_t tb = stage_base + (uint32_t)(sbuf * kSlabBytes) + (uint32_t)cq * 2u + (uint32_t)r0 * 128u;
      const uint32_t sw = ((uint32_t)r0 & 7u) << 4;
      if (p.mode == SY_CONV_RAW && p.dbg_f32 == nullptr) {
        // raw values (every conv of a training step): round, pack and stage -- no per-value pixel or column arithmetic.
        // (The host never runs the fp16 kernel in RAW mode; compiling the branch out of it made ptxas spill 32 bytes in
        // the BN = 128 halo instantiation.)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int J = slab * 8 + j;
#pragma unroll
          for (int h = 0; h < 2; ++h)
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(tb + (uint32_t)h * 1024u + ((((uint32_t)j) << 4) ^ sw)),
                         "r"(valid[h] ? st_pack<F16>(acc[4 * J + 2 * h], acc[4 * J + 2 * h + 1]) : 0u) : "memory");
        }
      } else {
        long long pix[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          bool ok;
          pix[h] = pixel(h, ok);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int J = slab * 8 + j;
          const int cl = slab * kSlabCols + j * 8 + cq;          // tile column of this thread's first value
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float v0 = acc[4 * J + 2 * h], v1 = acc[4 * J + 2 * h + 1];
            const bool inb = valid[h] && n0 + cl < p.Cout;
            if (p.dbg_f32 != nullptr && inb)     // validation only: the accumulators before any rounding
              *reinterpret_cast<float2*>(p.dbg_f32 + pix[h] * p.Cout + n0 + cl) = make_float2(v0, v1);
            if (p.mode != SY_CONV_RAW) {
              v0 = v0 * sScale[cl] + sShift[cl];
              v1 = v1 * sScale[cl + 1] + sShift[cl + 1];
              if constexpr (KINK) {                      // ReLU / LeakyReLU: conv_tc_kink_kernel only
                v0 = act_f(p.act, v0); v1 = act_f(p.act, v1);
              } else if (p.act) {                        // SiLU (SY_ACT_NONE: the backward's data-gradient convs)
                v0 = silu_f(v0); v1 = silu_f(v1);
              }
              if (p.res != nullptr && inb) {
                const uint32_t rv = *reinterpret_cast<const uint32_t*>(p.res + pix[h] * p.res_pitch + n0 + cl);
                v0 += st_lo<F16>(rv);
                v1 += st_hi<F16>(rv);
              }
            }
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(tb + (uint32_t)h * 1024u + ((((uint32_t)j) << 4) ^ sw)),
                         "r"(valid[h] ? st_pack<F16>(v0, v1) : 0u) : "memory");
          }
        }
      }
      fence_proxy_async();                     // generic-proxy writes -> visible to the TMA (async proxy)
      bar_staged_arrive(sbuf);                 // (B) staging tile complete: store + statistics warps take it from here
      tl_rec<TL>(p, tl_n, 2, 3, tile, slab);
    }
  }
  bar_free_wait(0);                                // drain the last arrivals (balanced barriers at exit)
  if (sflip) bar_free_wait(1);
  return tl_n;
}

// ---------------------------------------------------------------- warps 0-15: per-CTA partial row, grid barrier, BatchNorm finalize
// Run by the 16 convert + statistics warps (512 threads), called at the end of both of their roles so that each copy is
// compiled under that warpgroup's register budget.  tl: debug-timeline cursor (thread 0 records).
template <bool TL>
__device__ __forceinline__ void bn_tail(const Params& p, const Smem& sm, int tid, int& tl) {
  const int warp = tid >> 5, lane = tid & 31;
  const float* sAcc = sm.acc;
  const int et = tid;                                // 0..511
  const bool do_stats = (p.mode == SY_CONV_RAW) && (p.partials != nullptr);
  if (et == 0) tl_rec<TL>(p, tl, 4, 2, 0, 0);
  bar_stats_done();                                // every sAcc update is done
  if (!do_stats) return;
  // partial row of this CTA, channel-major: the four sums of a channel are one 16-byte word (the finalize below loads
  // one word per row and channel; with the shared-memory layout [4][Cout] in global memory it needed four loads, and the
  // 640 sector requests per warp made the partial-row sums the longest part of the tail)
  // (M-band walk: the statistics warps wrote this CTA's class rows already)
  if (p.band == 1) {
    float4* mine = reinterpret_cast<float4*>(p.partials) + (size_t)blockIdx.x * p.Cout;
    for (int c = et; c < p.Cout; c += kTailThreads)
      mine[c] = make_float4(sAcc[c], sAcc[p.Cout + c], sAcc[2 * p.Cout + c], sAcc[3 * p.Cout + c]);
  }
  if (p.n_seg == 0) return;
  if (et == 0) tl_rec<TL>(p, tl, 4, 5, 0, 0);
  // This CTA finalizes channels [b*cpc, (b+1)*cpc), one warp per channel.  The BatchNorm parameters and running
  // statistics of the warp's first channel do not depend on the other CTAs: load them BEFORE the grid barrier (they
  // come from DRAM -- behind the barrier their latency, twice in a row, was most of the finalize)
  const int groups = p.split_n < p.N ? 2 : 1;
  const int cpc = (p.Cout + (int)gridDim.x - 1) / (int)gridDim.x;
  const int c_end = min(p.Cout, ((int)blockIdx.x + 1) * cpc);
  const int c_first = (int)blockIdx.x * cpc + warp;
  float pre_gamma = 1.f, pre_beta = 0.f, pre_rm = 0.f, pre_rv = 1.f;
  if (c_first < c_end && lane < 2) {
    const BnSeg& sg = bn_seg(p, c_first);
    const int cs = c_first - sg.c_begin;
    pre_gamma = sg.gamma[cs];
    pre_beta = sg.beta[cs];
    if (lane == 0) {
      if (sg.rmean) pre_rm = sg.rmean[cs];
      if (sg.rvar) pre_rv = sg.rvar[cs];
    }
  }
  // grid barrier: all CTAs of the persistent grid are resident (1 per SM)
  __threadfence();
  bar_stats_done();
  if (et == 0) {
    atomicAdd(&p.sync[0], 1u);
    while (ld_acquire_u32(&p.sync[0]) < gridDim.x) __nanosleep(32);
  }
  bar_stats_done();
  if (et == 0) tl_rec<TL>(p, tl, 4, 6, 0, 0);
  // exit ticket (the last CTA past the barrier re-arms the counters): taken as early as possible -- right after the
  // barrier -- so that the atomic's round trip overlaps the finalize instead of ending the kernel
  unsigned int ticket = 0xffffffffu;
  if (et == 0) ticket = atomicAdd(&p.sync[1], 1u);
  // one WARP per channel (no block barriers): lane l sums the partial rows l, l+32, ... in order, a fixed shuffle tree
  // combines the lanes (deterministic), lanes 0 / 1 finalize one statistics group each.
  for (int c = c_first; c < c_end; c += kTailThreads / 32) {
    // all loads first (<= 160 rows: five per lane), then the sums in the same fixed order: one L2 round trip instead
    // of five serialised ones (the fp64 adds used to sit between the loads of consecutive rows)
    const float4* rows4 = reinterpret_cast<const float4*>(p.partials) + c;
    float4 buf[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const int r = lane + 32 * j;
      buf[j] = r < p.stat_rows ? __ldcg(rows4 + (size_t)r * p.Cout) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    double v[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      v[0] += (double)buf[j].x; v[1] += (double)buf[j].y; v[2] += (double)buf[j].z; v[3] += (double)buf[j].w;
    }
    if (et == 0) tl_rec<TL>(p, tl, 4, 8, 0, 0);
    for (int r = lane + 160; r < p.stat_rows; r += 32) {            // (more than 160 rows: not on an H100)
      const float4 q = __ldcg(rows4 + (size_t)r * p.Cout);
      v[0] += (double)q.x; v[1] += (double)q.y; v[2] += (double)q.z; v[3] += (double)q.w;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], m);
    }
    if (et == 0) tl_rec<TL>(p, tl, 4, 9, 0, 0);
    // every lane holds the four sums: lane g finalizes statistics group g (fp64 only for mean / E[x^2] - mean^2; the
    // reciprocal square root is IEEE fp32 -- the fp64 sqrt / divisions of the first version cost ~3 us per launch),
    // lane 0 then folds both groups into the running statistics in order
    const BnSeg& sg = bn_seg(p, c);
    const int cs = c - sg.c_begin;
    float mean_f = 0.f, var_f = 0.f;
    if (lane < groups) {
      const int g = lane;
      const double s1 = g ? v[2] : v[0], s2 = g ? v[3] : v[1];
      const double mean = s1 * p.inv_cnt[g];
      double var = s2 * p.inv_cnt[g] - mean * mean;
      if (var < 0.0) var = 0.0;
      mean_f = (float)mean;
      var_f = (float)var;
      const float istd = 1.0f / sqrtf(var_f + p.eps);
      const float sc = (c == c_first ? pre_gamma : sg.gamma[cs]) * istd;
      p.ss[(0 * 2 + g) * p.Cout + c] = sc;
      p.ss[(1 * 2 + g) * p.Cout + c] = (c == c_first ? pre_beta : sg.beta[cs]) - mean_f * sc;
      if (p.mi != nullptr) {
        p.mi[(0 * 2 + g) * p.Cout + c] = mean_f;
        p.mi[(1 * 2 + g) * p.Cout + c] = istd;
      }
    }
    // the second update: group 1's statistics, or group 0's again when the launch repeats its single group
    const float mean1 = __shfl_sync(0xffffffffu, mean_f, groups - 1), var1 = __shfl_sync(0xffffffffu, var_f, groups - 1);
    if (lane == 0) {
      float rm = pre_rm, rv = pre_rv;
      if (c != c_first) {
        rm = sg.rmean ? sg.rmean[cs] : 0.f;
        rv = sg.rvar ? sg.rvar[cs] : 1.f;
      }
      rm = (1.f - p.momentum) * rm + p.momentum * mean_f;
      rv = (1.f - p.momentum) * rv + p.momentum * (var_f * p.unbias[0]);
      if (p.updates == 2) {
        rm = (1.f - p.momentum) * rm + p.momentum * mean1;
        rv = (1.f - p.momentum) * rv + p.momentum * (var1 * p.unbias[1]);
      }
      if (sg.rmean) sg.rmean[cs] = rm;
      if (sg.rvar) sg.rvar[cs] = rv;
    }
  }
  if (et == 0) tl_rec<TL>(p, tl, 4, 7, 0, 0);
  if (et == 0 && blockIdx.x == 0) {
    for (int sgi = 0; sgi < p.n_seg; ++sgi)          // (a reduction: no round trip -- a load-add-store ended CTA 0 ~1 us late)
      if (p.seg[sgi].nbt) atomicAdd(reinterpret_cast<unsigned long long*>(p.seg[sgi].nbt), (unsigned long long)p.updates);
  }
  if (et == 0 && ticket == gridDim.x - 1) {   // every CTA is past the barrier: re-arm for the next launch
    p.sync[0] = 0u;
    p.sync[1] = 0u;
    __threadfence();
  }
}

// AM = how the A operand (activations) reaches shared memory:
//   1 linear : 128 consecutive output pixels, one im2col-mode TMA load per (tap, channel block)
//   2 halo   : 16 x 8 patch tiles, ONE tiled load per channel block of the 18 x (8+2) input halo; the nine taps are nine
//              shared-memory descriptors into that halo (every 8-pixel swizzle atom of a tap view is one halo row).
//              3x3 stride-1 only.  Each input pixel crosses L2 -> SM once per tile instead of nine times.
// The body of both kernels below: carves up shared memory, initialises the barriers, dispatches the warp roles.
template <int BN, bool TL, int AM, bool F16, bool KINK>
__device__ __forceinline__ void conv_tc_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmY,
                                             const Params& p) {
  constexpr bool HALO = (AM == 2);
  const int S = p.stages;                                  // linear: A+B ring depth; halo: B ring depth
  // weight slabs per ring stage: one 64-deep K block; halo mode: kHaloTaps filter taps
  constexpr int kSub = HALO ? kHaloTaps : 1;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B swizzle atoms; plain pointer arithmetic keeps the shared address space
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = sA + (HALO ? p.stagesA * kHaloBytes : S * kABytes);
  uint8_t* sStage = sB + S * kSub * Cfg<BN>::kBBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStage + p.stage_tiles * kSlabBytes);

  const int warp = threadIdx.x >> 5;
  pdl_launch_dependents();               // the next kernel on the stream may start its own prologue
  int tl_k = 3 * (p.timeline_cap / 4);
  if (threadIdx.x == 16 * 32) tl_rec<TL>(p, tl_k, 4, 0, 0, 0);
  const Smem sm{sA, sB, sStage, reinterpret_cast<float*>(bars + 32), smem_u32(bars), p.stage_tiles - 1};

  if (threadIdx.x == 17 * 32) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    prefetch_tmap(&tmY);
    for (int s = 0; s < S; ++s) {
      mbar_init(sm.full(s), HALO ? 1 : 2);     // A producer + B producer (halo: B only)
      mbar_init(sm.empty(s), 2);               // one arrival per consumer warpgroup
    }
    if (HALO) {
      for (int s = 0; s < p.stagesA; ++s) {
        mbar_init(sm.full_a(s), 1);
        mbar_init(sm.empty_a(s), 2);
      }
    }
    fence_barrier_init();
  }
  __syncthreads();
  // everything above touched only smem / kernel parameters; from here on we read what the previous kernels wrote
  pdl_wait();
  if (threadIdx.x == 16 * 32) tl_rec<TL>(p, tl_k, 4, 1, 0, 0);

  // every role's branch starts with its warpgroup's setmaxnreg: the register budget of a code region is what ptxas can
  // prove for every path into it
  if (warp >= 16) {
    reg_dealloc<kRegsIo>();
    if (warp == 18 || warp == 17) {
      if constexpr (HALO) {
        if (warp == 18) load_halo_a(p, sm, tmA);
        else load_halo_b<BN>(p, sm, tmB);
      } else {
        load_linear<BN, TL>(p, sm, tmA, tmB, warp == 18);
      }
    } else if (warp == 16) {
      store_slabs<BN, TL, AM>(p, sm, tmY, threadIdx.x);
    }
  } else if (warp >= 8) {
    reg_alloc<kRegsStats>();
    statistics<BN, TL, AM>(p, sm, threadIdx.x);
    int tl = p.timeline_cap;
    bn_tail<TL>(p, sm, threadIdx.x, tl);
  } else {
    reg_alloc<kRegsMma>();
    int tl = mma_convert<BN, TL, AM, F16, KINK>(p, sm, threadIdx.x);
    bn_tail<TL>(p, sm, threadIdx.x, tl);
  }
  __syncthreads();
  if (threadIdx.x == 16 * 32) tl_rec<TL>(p, tl_k, 4, 3, 0, 0);
}

// bf16 activations, every mode (TL: debug timeline)
template <int BN, bool TL, int AM>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmY, const Params p) {
  conv_tc_body<BN, TL, AM, false, false>(tmA, tmB, tmY, p);
}

// fp16 activations and weights, FUSED mode only (a kernel of its own: the bf16 kernel's name and instantiations stay as
// they are)
template <int BN, int AM>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_f16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmY, const Params p) {
  conv_tc_body<BN, false, AM, true, false>(tmA, tmB, tmY, p);
}

// FUSED mode with SY_ACT_RELU / SY_ACT_LRELU, bf16 or fp16: the same roles with the activation switch compiled into the
// epilogue.  A kernel of its own so that the SiLU / identity epilogue of the two kernels above (every eval conv, the
// backward's data-gradient convs) stays the code it was.
template <int BN, int AM, bool F16>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kink_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmY, const Params p) {
  conv_tc_body<BN, false, AM, F16, true>(tmA, tmB, tmY, p);
}

// ------------------------------------------------------------------ host side

// Tile width heuristic from a per-K-block cost model: one 64-deep K block of a 128-row tile costs about kblock_cycles()
// (MMA + barrier hand-shake + operand supply), the epilogue about kEpiCyclesPerSlab per 64-column slab, and the
// persistent grid runs ceil(tiles / SMs) rounds -- so wide tiles win unless they add a round.  The constants are a model,
// not H100 measurements; a tile_bn override (SyConvDesc) forces the width.
constexpr double kEpiCyclesPerSlab = 1900.0;

static double kblock_cycles(int bn) { return bn == 128 ? 515.0 : 560.0; }

static int pick_bn(int cout, int m_tiles, int kblocks, int tile_bn) {
  if (tile_bn != 0) return tile_bn;
  const int cands[2] = {128, 64};
  int best_bn = 64;
  double best = 1e30;
  for (int i = 0; i < 2; ++i) {
    const int bn = cands[i];
    if (bn > 64 && bn / 2 >= cout) continue;          // a narrower tile already covers every channel
    const int tiles = m_tiles * cdiv(cout, bn);
    const int rounds = cdiv(tiles, num_sms());
    const double main_c = kblocks * kblock_cycles(bn);
    const double epi = kEpiCyclesPerSlab * (bn / 64);
    // the epilogue of a tile does not overlap the main loop of the next one (the accumulators are the consumers' registers)
    const double t = rounds * (main_c + epi + 400.0);
    if (t < best) { best = t; best_bn = bn; }
  }
  return best_bn;
}

static const int kSmemLimit = 232448;   // 227 KiB opt-in maximum per CTA

// Order in which the persistent grid walks the (N tile, M tile) space.
//   N-major (band 1): CTA b takes tiles b, b + G, ... numbered M fastest.  The whole grid works on one or two N tiles at a
//     time, so every N tile re-streams the whole A tensor, from HBM whenever A does not fit in L2.
//   M-band (band n_tiles, S = SMs / n_tiles slots, grid S * n_tiles): CTA b = slot * n_tiles + N tile keeps its N tile for
//     its whole life.  The M tiles fall into SMs classes rho = m mod SMs; slot j owns the classes j, j + S, j + 2S, ... < SMs
//     and walks them one after the other, each class in increasing m.  The n_tiles CTAs of a slot walk the same M tiles at
//     about the same time, so A crosses HBM -> L2 about once per layer.
// One class of one N tile holds exactly the tiles that one CTA of the N-major walk (grid = SMs) takes for that N tile, in the
// same order, so the M-band walk writes the N-major walk's statistics rows bit for bit (statistics warps, write_class).
// M-band is taken whenever it does not add a round of the persistent grid (it never saves one).
struct Walk {
  int band, grid, t_end, stat_rows, cls_step, cls_tiles;
};
static Walk pick_walk(int m_tiles, int n_tiles) {
  const int sms = num_sms(), total = m_tiles * n_tiles;
  const int grid = min(total, sms);
  const Walk nmajor{1, grid, total, grid, 0, 1};
  if (n_tiles == 1 || total <= sms) return nmajor;
  const int slots = sms / n_tiles;
  int worst = 0;                                   // tiles of the busiest slot
  for (int j = 0; j < slots; ++j) {
    int w = 0;
    for (int rho = j; rho < sms; rho += slots)
      if (rho < m_tiles) w += cdiv(m_tiles - rho, sms);
    worst = max(worst, w);
  }
  if (worst > cdiv(total, sms)) return nmajor;
  const int cls_tiles = cdiv(m_tiles, sms);
  return {n_tiles, slots * n_tiles, cdiv(sms, slots) * cls_tiles, sms, slots, cls_tiles};
}

struct Plan {
  int smem, grid;
};

template <int BN, int AM, bool F16>
static bool set_smem_attr() {
  static int state = 0;                 // 0 = not tried, 1 = ok, -1 = failed
  if (state == 0) {
    bool ok;
    if constexpr (F16)
      ok = cudaFuncSetAttribute(conv_tc_f16_kernel<BN, AM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit) == cudaSuccess;
    else
      ok = cudaFuncSetAttribute(conv_tc_kernel<BN, false, AM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit) == cudaSuccess &&
           cudaFuncSetAttribute(conv_tc_kernel<BN, true, AM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(conv_tc_kink_kernel<BN, AM, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    kSmemLimit) == cudaSuccess;
    if (!ok) cudaGetLastError();
    state = ok ? 1 : -1;
  }
  return state == 1;
}

// Ring depth, staging tiles, shared-memory size and grid of one launch.
template <int BN, int AM>
static int make_plan(Params& p, Plan* out) {
  const int acc_bytes = (p.mode == SY_CONV_RAW && p.partials) ? 16 * p.Cout : 2048;
  // epilogue-bound layers (main loop of a tile shorter than its epilogue: 1x1 convs with few input channels, the
  // stem) get a second staging tile: the store + statistics of a slab then overlap the conversion of the next
  const bool main_loop_bound = !(p.kblocks * kblock_cycles(BN) < kEpiCyclesPerSlab * (BN / 64));
  p.stage_tiles = main_loop_bound ? 1 : 2;
  const int bbytes = Cfg<BN>::kBBytes;
  const int fixed_bytes = Cfg<BN>::kFixedBytes + (p.stage_tiles - 1) * kSlabBytes;
  int smem;
  if (AM == 2) {
    // halo ring (2-3 stages of 23 KiB) + weight-slab ring (the rest, kHaloTaps taps per stage)
    p.stagesA = (BN == 64 && p.cblocks > 1) ? 3 : 2;
    int stages = (kSmemLimit - fixed_bytes - acc_bytes - p.stagesA * kHaloBytes) / (kHaloTaps * bbytes);
    if (stages > kMaxStages) stages = kMaxStages;
    SY_REQUIRE(stages >= 2, SY_EINVAL, "conv2d_tc(halo): Cout=%d leaves no room for the weight ring", p.Cout);
    p.stages = stages;
    smem = fixed_bytes + acc_bytes + p.stagesA * kHaloBytes + stages * kHaloTaps * bbytes;
  } else {
    const int stage_bytes = kABytes + bbytes;
    const int fit = min(kMaxStages, (kSmemLimit - fixed_bytes - acc_bytes) / stage_bytes);
    const int stages = min(fit, kRingStages);
    SY_REQUIRE(stages >= 2, SY_EINVAL, "conv2d_tc: Cout=%d leaves no room for the operand ring", p.Cout);
    p.stages = stages;
    smem = fixed_bytes + acc_bytes + stages * stage_bytes;
  }
  out->smem = smem;
  const Walk wk = pick_walk(p.m_tiles, p.n_tiles);
  p.band = wk.band; p.t_end = wk.t_end; p.stat_rows = wk.stat_rows; p.cls_step = wk.cls_step; p.cls_tiles = wk.cls_tiles;
  p.fd_band = make_fastdiv((uint32_t)wk.band);
  p.fd_cls_tiles = make_fastdiv((uint32_t)wk.cls_tiles);
  out->grid = wk.grid;
  return SY_OK;
}

template <int BN, int AM, bool F16>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ty, Params& p, const Plan& pl, cudaStream_t stream) {
  const int smem = pl.smem, grid = pl.grid;
  SY_REQUIRE((set_smem_attr<BN, AM, F16>()), SY_ELAUNCH, "conv2d_tc: cannot opt in to %d bytes of shared memory", kSmemLimit);
  if (p.n_seg > 0) {
    // The BatchNorm tail ends in a grid-wide barrier: every CTA of this launch must be resident at once.  The launch is
    // not a cooperative launch (it carries the programmatic-dependent-launch attribute instead), so check what a
    // cooperative launch would check -- per (instantiation, shared-memory size), once.
    static int ok_smem[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    bool seen = false;
    for (int i = 0; i < 8; ++i) seen = seen || ok_smem[i] == smem;
    if (!seen) {
      int per_sm = 0;
      SY_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, conv_tc_kernel<BN, false, AM>, kThreads, (size_t)smem));
      SY_REQUIRE(per_sm >= 1 && per_sm * num_sms() >= grid, SY_ELAUNCH,
                 "conv2d_tc: %d CTAs cannot be co-resident (%d per SM x %d SMs): the BatchNorm grid barrier would hang", grid,
                 per_sm, num_sms());
      for (int i = 0; i < 8; ++i)
        if (ok_smem[i] == 0) { ok_smem[i] = smem; break; }
    }
  }
  if (p.mode == SY_CONV_FUSED && (p.act == SY_ACT_RELU || p.act == SY_ACT_LRELU)) {     // (no timeline: refused)
    SY_CUDA(launch_pdl(conv_tc_kink_kernel<BN, AM, F16>, dim3(grid), dim3(kThreads), (size_t)smem, stream, ta, tb, ty, p));
    return launch_status("conv_tc_kink_kernel");
  }
  if constexpr (F16) {                  // (no statistics, no timeline: the host side refused them)
    SY_CUDA(launch_pdl(conv_tc_f16_kernel<BN, AM>, dim3(grid), dim3(kThreads), (size_t)smem, stream, ta, tb, ty, p));
    return launch_status("conv_tc_f16_kernel");
  }
  if (p.timeline != nullptr)
    SY_CUDA(launch_pdl(conv_tc_kernel<BN, true, AM>, dim3(grid), dim3(kThreads), (size_t)smem, stream, ta, tb, ty, p));
  else
    SY_CUDA(launch_pdl(conv_tc_kernel<BN, false, AM>, dim3(grid), dim3(kThreads), (size_t)smem, stream, ta, tb, ty, p));
  return launch_status("conv_tc_kernel");
}

template <int AM>
static int plan_bn(int bn, Params& p, Plan* out) {
  return bn == 64 ? make_plan<64, AM>(p, out) : make_plan<128, AM>(p, out);
}

template <int AM, bool F16>
static int launch_bn(int bn, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ty, Params& p, const Plan& pl,
                     cudaStream_t stream) {
  return bn == 64 ? launch<64, AM, F16>(ta, tb, ty, p, pl, stream) : launch<128, AM, F16>(ta, tb, ty, p, pl, stream);
}

// Halo mode (conv_tc_kernel, AM = 2) for a 3x3 stride-1 convolution?  It needs 16 x 8 patch tiles (more tiles than the
// linear tiling on small feature maps) and pays off where the tap re-reads bound the main loop.  Modelled per-K-block
// costs (cycles): linear 515 / 560, halo 430 / 370 at BN = 128 / 64.
// tile_mode 2 forces it (every eligible conv), 1 disables it.
static bool use_halo(int n, int ho, int wo, int cout, int kblocks, int tile_mode, int tile_bn) {
  if (tile_mode != 0) return tile_mode == 2;
  const int tiles_l = cdiv(n * ho * wo, kBlockM), tiles_h = n * cdiv(ho, 16) * cdiv(wo, 8);
  const int bn = pick_bn(cout, tiles_l, kblocks, tile_bn);
  const double lin_c = bn == 128 ? 515.0 : 560.0, halo_c = bn == 128 ? 430.0 : 370.0;
  const int nt = cdiv(cout, bn);
  return cdiv(tiles_h * nt, num_sms()) * halo_c < cdiv(tiles_l * nt, num_sms()) * lin_c;
}

// The tiling of one layer shape, shared by sy_conv2d_tc and the host-only sy_conv2d_plan: halo mode where use_halo
// takes it, linear tiles otherwise.  The tile width is chosen on the linear tiling (the halo decision assumed that width).
// tile_mode / tile_bn (SyConvDesc; 0 = planner) override the choices; they are plan inputs only and never reach Params.
struct Tiling {
  bool halo;
  int bn, m_tiles, tiles_x, tiles_y, cblocks, kblocks;
};
static bool tiling_override_ok(int tile_mode, int tile_bn) {
  return tile_mode >= 0 && tile_mode <= 2 && (tile_bn == 0 || tile_bn == 64 || tile_bn == 128);
}
static Tiling pick_tiling(int n, int ho, int wo, int cin, int cout, int kh, int kw, int stride, int tile_mode, int tile_bn) {
  Tiling t{};
  t.cblocks = cdiv(cin, kBlockK);
  t.kblocks = kh * kw * t.cblocks;
  t.halo = kh == 3 && kw == 3 && stride == 1 && use_halo(n, ho, wo, cout, t.kblocks, tile_mode, tile_bn);
  t.tiles_y = cdiv(ho, kHaloTH);
  t.tiles_x = cdiv(wo, kHaloTW);
  const int lin_tiles = cdiv(n * ho * wo, kBlockM);
  t.m_tiles = t.halo ? n * t.tiles_y * t.tiles_x : lin_tiles;
  t.bn = pick_bn(cout, lin_tiles, t.kblocks, tile_bn);
  return t;
}

}  // namespace tc
}  // namespace sy

using namespace sy;

extern "C" int sy_conv_stat_rows(void) { return tc::num_sms(); }

extern "C" int sy_conv2d_tc(const SyConvDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  const SyTensor& x = d->x;
  const SyTensor& y = d->y;
  SY_REQUIRE(view_ok(x) && view_ok(y) && d->w != nullptr, SY_EINVAL, "conv2d_tc: bad x/y view or null weights");
  SY_REQUIRE((d->kh == 1 || d->kh == 3) && (d->kw == 1 || d->kw == 3) && (d->stride == 1 || d->stride == 2), SY_EINVAL,
             "conv2d_tc: kernel %dx%d stride %d unsupported", d->kh, d->kw, d->stride);
  const int ph = (d->kh - 1) / 2, pw = (d->kw - 1) / 2;
  const int ho = (x.h + 2 * ph - d->kh) / d->stride + 1, wo = (x.w + 2 * pw - d->kw) / d->stride + 1;
  SY_REQUIRE(y.n == x.n && y.h == ho && y.w == wo, SY_EINVAL, "conv2d_tc: output view %dx%dx%d, expected %dx%dx%d",
             y.n, y.h, y.w, x.n, ho, wo);
  SY_REQUIRE(((uintptr_t)d->w % 16) == 0, SY_EINVAL, "conv2d_tc: weights not 16B aligned");
  SY_REQUIRE(y.c <= 2048, SY_EINVAL, "conv2d_tc: Cout=%d > 2048", y.c);
  SY_REQUIRE(d->debug_flags == 0 || d->debug_flags == 2, SY_EINVAL, "conv2d_tc: debug_flags %d unsupported", d->debug_flags);
  SY_REQUIRE(tc::tiling_override_ok(d->tile_mode, d->tile_bn), SY_EINVAL, "conv2d_tc: tile_mode %d / tile_bn %d unsupported",
             d->tile_mode, d->tile_bn);
  SY_REQUIRE(d->storage == SY_STORAGE_BF16 || d->storage == SY_STORAGE_F16, SY_EINVAL, "conv2d_tc: storage %d unsupported",
             d->storage);
  SY_REQUIRE(act_ok(d->act), SY_EINVAL, "conv2d_tc: act=%d is not an SY_ACT_* code", d->act);
  SY_REQUIRE(!(d->mode == SY_CONV_FUSED && d->act >= SY_ACT_RELU && d->debug_timeline != nullptr), SY_EINVAL,
             "conv2d_tc: the debug timeline is not recorded for ReLU / LeakyReLU FUSED launches");
  const bool f16 = d->storage == SY_STORAGE_F16;
  SY_REQUIRE(!f16 || (d->mode == SY_CONV_FUSED && d->stat_partials == nullptr && d->bn[0].gamma == nullptr &&
                      d->debug_timeline == nullptr),
             SY_EINVAL, "conv2d_tc: fp16 storage runs the FUSED mode only (no statistics, BatchNorm finalize or timeline)");
  {
    const bool one_group = !(d->split_n > 0 && d->split_n < x.n);
    SY_REQUIRE(d->stat_updates >= 0 && d->stat_updates <= 2, SY_EINVAL, "conv2d_tc: stat_updates %d unsupported (0, 1 or 2)",
               d->stat_updates);
    SY_REQUIRE(d->stat_updates < 2 || (d->mode == SY_CONV_RAW && d->stat_partials != nullptr && d->bn[0].gamma != nullptr),
               SY_EINVAL, "conv2d_tc: stat_updates = 2 needs the BatchNorm finalize (RAW mode, stat_partials and bn[])");
    SY_REQUIRE(d->stat_updates < 2 || one_group, SY_EINVAL,
               "conv2d_tc: stat_updates = 2 repeats a single statistics group, but split_n = %d splits %d images in two",
               d->split_n, x.n);
  }
  SY_REQUIRE(tc::get_encode() != nullptr, SY_EARCH, "cuTensorMapEncodeTiled not available from the driver");

  tc::Params p{};
  p.debug_flags = d->debug_flags;
  p.N = x.n; p.Ho = ho; p.Wo = wo; p.Cout = y.c;
  p.kw = d->kw; p.stride = d->stride; p.pad_h = ph; p.pad_w = pw;
  SY_REQUIRE((long long)x.n * ho * wo < (1ll << 31) - 256, SY_EINVAL, "conv2d_tc: too many output pixels");
  const tc::Tiling t = tc::pick_tiling(x.n, ho, wo, x.c, y.c, d->kh, d->kw, d->stride, d->tile_mode, d->tile_bn);
  const bool halo = t.halo;
  const int bn = t.bn;
  p.P_total = x.n * ho * wo;
  p.tiles_y = t.tiles_y; p.tiles_x = t.tiles_x;
  p.m_tiles = t.m_tiles;
  p.fd_hw = tc::make_fastdiv((uint32_t)(ho * wo));
  p.fd_wo = tc::make_fastdiv((uint32_t)wo);
  p.cblocks = t.cblocks;
  p.kblocks = t.kblocks;
  p.n_tiles = cdiv(y.c, bn);
  p.fd_m_tiles = tc::make_fastdiv((uint32_t)p.m_tiles);
  p.fd_per_img = tc::make_fastdiv((uint32_t)(p.tiles_x * p.tiles_y));
  p.fd_tiles_x = tc::make_fastdiv((uint32_t)p.tiles_x);
  p.mode = d->mode; p.act = d->act;
  p.res = nullptr; p.res_pitch = 0;
  if (d->mode == SY_CONV_FUSED && d->res.ptr != nullptr) {
    SY_REQUIRE(view_ok(d->res) && d->res.n == y.n && d->res.h == ho && d->res.w == wo && d->res.c == y.c, SY_EINVAL,
               "conv2d_tc: residual view mismatch");
    p.res = reinterpret_cast<const uint16_t*>(d->res.ptr); p.res_pitch = d->res.pitch;
  }
  p.scale = d->scale; p.shift = d->shift;
  p.split_n = (d->split_n > 0 && d->split_n < x.n) ? d->split_n : x.n;
  p.gp = p.split_n * ho * wo;
  p.partials = (d->mode == SY_CONV_RAW) ? d->stat_partials : nullptr;
  if (p.partials) {
    SY_REQUIRE(((uintptr_t)p.partials % 16) == 0, SY_EINVAL, "conv2d_tc: statistic rows not 16B aligned");
    SY_REQUIRE(d->n_partials >= tc::num_sms(), SY_EWORKSPACE, "conv2d_tc: %d statistic rows, need %d (sy_conv_stat_rows)",
               d->n_partials, tc::num_sms());
  }
  p.dbg_f32 = d->debug_f32;
  p.timeline = reinterpret_cast<long long*>(d->debug_timeline);
  p.timeline_cap = d->debug_timeline ? d->debug_timeline_events : 0;
  p.n_seg = 0;
  if (p.partials && d->bn[0].gamma != nullptr) {
    SY_REQUIRE(d->sync && d->scale_shift, SY_EINVAL, "conv2d_tc: BN finalize needs sync counters and scale_shift");
    for (int sgi = 0; sgi < 2; ++sgi) {
      if (d->bn[sgi].gamma == nullptr) break;
      SY_REQUIRE(d->bn[sgi].beta != nullptr && d->bn[sgi].c_begin >= 0 && d->bn[sgi].c_begin < y.c, SY_EINVAL,
                 "conv2d_tc: bad BN segment %d", sgi);
      p.seg[sgi].gamma = d->bn[sgi].gamma; p.seg[sgi].beta = d->bn[sgi].beta;
      p.seg[sgi].rmean = d->bn[sgi].running_mean; p.seg[sgi].rvar = d->bn[sgi].running_var;
      p.seg[sgi].nbt = reinterpret_cast<long long*>(d->bn[sgi].num_batches_tracked);
      p.seg[sgi].c_begin = d->bn[sgi].c_begin;
      p.n_seg = sgi + 1;
    }
    SY_REQUIRE(p.seg[0].c_begin == 0, SY_EINVAL, "conv2d_tc: first BN segment must start at channel 0");
    p.momentum = d->momentum; p.eps = d->eps;
    {
      const int groups = p.split_n < x.n ? 2 : 1;
      for (int g = 0; g < 2; ++g) {
        const double cnt = (double)(g == 0 ? (groups == 2 ? p.split_n : x.n) : x.n - p.split_n) * ho * wo;
        p.inv_cnt[g] = cnt > 0.0 ? 1.0 / cnt : 0.0;
        p.unbias[g] = cnt > 1.0 ? (float)(cnt / (cnt - 1.0)) : 1.0f;
      }
      p.updates = (groups == 2 || d->stat_updates == 2) ? 2 : 1;
      if (groups == 1) p.unbias[1] = p.unbias[0];      // a repeated update uses group 0's count
    }
    p.ss = d->scale_shift;
    p.mi = d->mean_invstd;
    p.sync = d->sync;
  }
  tc::Plan pl{};
  {
    const int rc = halo ? tc::plan_bn<2>(bn, p, &pl) : tc::plan_bn<1>(bn, p, &pl);
    if (rc != SY_OK) return rc;
  }
  if (d->rows_written) *d->rows_written = p.stat_rows;

  CUtensorMap ta, tb, ty;
  const CUtensorMapDataType dt = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if (halo) {
    // A, halo mode: input view as (C, W, H, N), box (64 ch, 10 px, 18 rows, 1 image) at (x0 - 1, y0 - 1): out of bounds
    // = zero padding
    cuuint64_t dims[4], strides[3];
    tc::nhwc_dims(x, dims, strides);
    const cuuint32_t box[4] = {(cuuint32_t)tc::kBlockK, (cuuint32_t)tc::kHaloPitch, (cuuint32_t)(tc::kHaloTH + 2), 1};
    const CUresult r = tc::encode_tiled(&ta, 4, x.ptr, dims, strides, box, dt);
    SY_REQUIRE(r == CUDA_SUCCESS, SY_ELAUNCH, "cuTensorMapEncodeTiled(A halo) failed: %d", (int)r);
  } else {
    // A, im2col mode: one load = 128 consecutive base pixels x 64 channels, shifted by the tap offset
    SY_REQUIRE(tc::get_encode_im2col() != nullptr, SY_EARCH, "cuTensorMapEncodeIm2col not available from the driver");
    const CUresult r = tc::encode_im2col_nhwc(&ta, x, d->kh, d->kw, d->stride, tc::kBlockM, dt);
    SY_REQUIRE(r == CUDA_SUCCESS, SY_ELAUNCH, "cuTensorMapEncodeIm2col(A) failed: %d (c=%d w=%d h=%d n=%d pitch=%lld k=%dx%d s=%d)",
               (int)r, x.c, x.w, x.h, x.n, (long long)x.pitch, d->kh, d->kw, d->stride);
  }
  {
    const int taps = d->kh * d->kw;
    const cuuint64_t dims[3] = {(cuuint64_t)x.c, (cuuint64_t)taps, (cuuint64_t)y.c};
    const cuuint64_t strides[2] = {(cuuint64_t)x.c * 2, (cuuint64_t)x.c * 2 * taps};
    const cuuint32_t box[3] = {(cuuint32_t)tc::kBlockK, 1, (cuuint32_t)bn};
    const CUresult r = tc::encode_tiled(&tb, 3, d->w, dims, strides, box, dt);
    SY_REQUIRE(r == CUDA_SUCCESS, SY_ELAUNCH, "cuTensorMapEncodeTiled(B) failed: %d", (int)r);
  }
  if (!halo) {
    // Y: output view as (C, pixels, 1, 1), box (64, 128, 1, 1): the TMA store clips the last tile / the channel slice
    const cuuint64_t dims[4] = {(cuuint64_t)y.c, (cuuint64_t)p.P_total, 1, 1};
    const cuuint64_t strides[3] = {(cuuint64_t)y.pitch * 2, (cuuint64_t)y.pitch * 2 * p.P_total, (cuuint64_t)y.pitch * 2 * p.P_total};
    const cuuint32_t box[4] = {(cuuint32_t)tc::kSlabCols, (cuuint32_t)tc::kBlockM, 1, 1};
    const CUresult r = tc::encode_tiled(&ty, 4, y.ptr, dims, strides, box, dt);
    SY_REQUIRE(r == CUDA_SUCCESS, SY_ELAUNCH, "cuTensorMapEncodeTiled(Y linear) failed: %d", (int)r);
  } else {
    // Y: output view as (C, W, H, N), box (64, 8, 16, 1): the TMA store clips the patch to the image / slice
    cuuint64_t dims[4], strides[3];
    tc::nhwc_dims(y, dims, strides);
    const cuuint32_t box[4] = {(cuuint32_t)tc::kSlabCols, (cuuint32_t)tc::kHaloTW, (cuuint32_t)tc::kHaloTH, 1};
    const CUresult r = tc::encode_tiled(&ty, 4, y.ptr, dims, strides, box, dt);
    SY_REQUIRE(r == CUDA_SUCCESS, SY_ELAUNCH, "cuTensorMapEncodeTiled(Y) failed: %d", (int)r);
  }
  if (f16) return halo ? tc::launch_bn<2, true>(bn, ta, tb, ty, p, pl, stream) : tc::launch_bn<1, true>(bn, ta, tb, ty, p, pl, stream);
  return halo ? tc::launch_bn<2, false>(bn, ta, tb, ty, p, pl, stream) : tc::launch_bn<1, false>(bn, ta, tb, ty, p, pl, stream);
}

// Host-only query (no launch, works without a GPU): the tiling decisions sy_conv2d_tc takes for a layer shape and
// tiling override (both go through pick_tiling and pick_walk).
extern "C" int sy_conv2d_plan(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t kh, int32_t kw, int32_t stride,
                              int32_t tile_mode, int32_t tile_bn, SyConvPlan* out) {
  SY_REQUIRE(out != nullptr && n > 0 && h > 0 && w > 0 && cin > 0 && cout > 0, SY_EINVAL, "conv2d_plan: bad arguments");
  SY_REQUIRE((kh == 1 || kh == 3) && (kw == 1 || kw == 3) && (stride == 1 || stride == 2), SY_EINVAL,
             "conv2d_plan: kernel %dx%d stride %d unsupported", kh, kw, stride);
  SY_REQUIRE(tc::tiling_override_ok(tile_mode, tile_bn), SY_EINVAL, "conv2d_plan: tile_mode %d / tile_bn %d unsupported",
             tile_mode, tile_bn);
  const int ph = (kh - 1) / 2, pw = (kw - 1) / 2;
  const int ho = (h + 2 * ph - kh) / stride + 1, wo = (w + 2 * pw - kw) / stride + 1;
  const tc::Tiling t = tc::pick_tiling(n, ho, wo, cin, cout, kh, kw, stride, tile_mode, tile_bn);
  const int m_tiles = t.m_tiles;
  out->mode = t.halo ? 2 : 1;
  out->bn = t.bn;
  out->m_tiles = m_tiles;
  out->n_tiles = cdiv(cout, t.bn);
  out->rounds = cdiv(m_tiles * out->n_tiles, tc::num_sms());
  const tc::Walk wk = tc::pick_walk(m_tiles, out->n_tiles);
  out->walk = wk.band > 1 ? 1 : 0;
  out->grid = wk.grid;
  out->kblocks = t.kblocks;
  out->patch_h = t.halo ? tc::kHaloTH : 0;
  out->patch_w = t.halo ? tc::kHaloTW : 0;
  return SY_OK;
}
