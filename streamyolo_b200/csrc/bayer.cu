// sy_bayer_to_bgr_sized: 8-bit Bayer mosaics (RGGB, BGGR, GBRG, GRBG) -> uint8 BGR slots, bit-identical to
// cv2.cvtColor(raw, COLOR_Bayer*2BGR) (bilinear) and COLOR_Bayer*2BGR_EA (edge-aware); the arithmetic is stated in the header.
// A block demosaics a tile of 16 rows x 128 columns of one frame.  It stages the input rows the tile reads, plus a halo,
// in shared memory with aligned 16-byte loads (byte loads where a chunk straddles the frame's first or last byte, so
// nothing outside the frame's h * w bytes is read); then each thread computes a run of 16 pixels of one row and writes
// its 48 bytes with 16-byte stores where the run is whole and aligned.
// The border copy (column 0 = column 1, row 0 = row 1, ...) is folded in: pixel (y, x) is the interior pixel at
// (clamp(y, 1, h - 2), clamp(x, 1, w - 2)).
#include "common.cuh"

namespace sy {
namespace {

constexpr int kRun = 16;                  // columns per thread
constexpr int kRuns = 8;                  // runs per tile row
constexpr int kTileW = kRun * kRuns;      // 128 columns
constexpr int kTileH = 16;                // rows
constexpr int kChunks = 10;               // 16-byte chunks per staged row: input columns X0 - 2 .. X0 + 129 from any alignment
constexpr int kPitch = 16 * kChunks;

__device__ __forceinline__ uint32_t byte_at(const uint32_t* w, int k) { return (w[k >> 2] >> (8 * (k & 3))) & 255u; }

// the first 3 * n bytes of words o to q
__device__ __forceinline__ void store_run(uint8_t* __restrict__ q, const uint32_t (&o)[12], int n) {
  if (n == kRun && (reinterpret_cast<uintptr_t>(q) & 15) == 0) {
    uint4* d = reinterpret_cast<uint4*>(q);
    d[0] = make_uint4(o[0], o[1], o[2], o[3]);
    d[1] = make_uint4(o[4], o[5], o[6], o[7]);
    d[2] = make_uint4(o[8], o[9], o[10], o[11]);
    return;
  }
#pragma unroll
  for (int k = 0; k < 3 * kRun; ++k)
    if (k < 3 * n) q[k] = (uint8_t)byte_at(o, k);
}

// 20 staged bytes from byte b of a staged row: 6 word loads realigned by funnel shifts
__device__ __forceinline__ void load_window(uint32_t (&q)[5], const uint8_t* row, int b) {
  const uint32_t* p = reinterpret_cast<const uint32_t*>(row + (b & ~3));
  uint32_t v[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) v[i] = p[i];
#pragma unroll
  for (int i = 0; i < 5; ++i) q[i] = __funnelshift_r(v[i], v[i + 1], 8 * (b & 3));
}

// blockIdx.z = frame, (x, y) = tile of the slot grid; threadIdx (x, y) = (run, row) in the tile
template <int ALGO>
__global__ void __launch_bounds__(kRuns * kTileH) bayer_to_bgr_sized_kernel(const uint8_t* __restrict__ src,
                                                                           long long max_bytes,
                                                                           const int32_t* __restrict__ sizes, int pattern,
                                                                           int slot_h, int slot_w,
                                                                           uint8_t* __restrict__ out) {
  __shared__ __align__(16) uint8_t tile[kTileH + 2][kPitch];
  const int k = blockIdx.z;
  const int h = sizes[2 * k], w = sizes[2 * k + 1];
  const long long hw = (long long)h * w;
  if (h < 1 || w < 1 || h > slot_h || w > slot_w || hw > max_bytes) return;
  const int X0 = blockIdx.x * kTileW, Y0 = blockIdx.y * kTileH;
  if (X0 >= w || Y0 >= h) return;
  const int y = Y0 + threadIdx.y, x0 = X0 + kRun * threadIdx.x;
  const bool mine = y < h && x0 < w;
  const int n = min(kRun, w - x0);
  uint8_t* q_out = out + (long long)slot_h * slot_w * 3 * k + ((long long)y * slot_w + x0) * 3;
  uint32_t o[12];
  if (h < 3 || w < 3) {                              // cv2 makes such a frame black
    if (mine) {
#pragma unroll
      for (int i = 0; i < 12; ++i) o[i] = 0;
      store_run(q_out, o, n);
    }
    return;
  }
  // stage input rows oy .. oy + kTileH + 1 (those < h): the rows the tile's clamped centres read
  const uint8_t* f = src + max_bytes * k;
  const uintptr_t f0 = reinterpret_cast<uintptr_t>(f), f1 = f0 + hw;
  const int oy = min(max(Y0, 1), h - 2) - 1;
  for (int c = threadIdx.y * kRuns + threadIdx.x; c < (kTileH + 2) * kChunks; c += kRuns * kTileH) {
    const int r = c / kChunks, j = c % kChunks, iy = oy + r;
    if (iy >= h) continue;
    const uintptr_t a = ((f0 + (long long)iy * w + X0 - 2) & ~(uintptr_t)15) + 16 * j;
    uint4 v;
    if (a >= f0 && a + 16 <= f1) {
      v = __ldg(reinterpret_cast<const uint4*>(a));
    } else {
      uint32_t b[4] = {0, 0, 0, 0};
#pragma unroll
      for (int i = 0; i < 16; ++i)
        if (a + i >= f0 && a + i < f1) b[i >> 2] |= (uint32_t)__ldg(reinterpret_cast<const uint8_t*>(a + i)) << (8 * (i & 3));
      v = make_uint4(b[0], b[1], b[2], b[3]);
    }
    *reinterpret_cast<uint4*>(&tile[r][16 * j]) = v;
  }
  __syncthreads();
  if (!mine) return;

  // rows cy - 1, cy, cy + 1, columns x0 - 2 .. x0 + 17
  const int cy = min(max(y, 1), h - 2);
  uint32_t ra[5], rb[5], rc[5];
  {
    const int sr = cy - 1 - oy;
    const auto at = [&](int iy) { return (int)((f0 + (long long)iy * w + X0 - 2) & 15) + kRun * (int)threadIdx.x; };
    load_window(ra, tile[sr], at(cy - 1));
    load_window(rb, tile[sr + 1], at(cy));
    load_window(rc, tile[sr + 2], at(cy + 1));
  }
  // the site at column x0 + j is green iff (cy + j) & 1 == gpar (x0 is even); a row's other colour is red or blue
  const int gpar = pattern == SY_BAYER_RGGB || pattern == SY_BAYER_BGGR;
  const bool first_red = pattern == SY_BAYER_RGGB || pattern == SY_BAYER_GRBG;
  const bool row_red = ((cy & 1) == 0) == first_red;
  const int qpar = (cy ^ gpar) & 1;                  // green iff (j & 1) == qpar

  // px[c]: the interior pixel at column x0 + c - 1, c = 0 .. 16
  uint32_t pb[kRun + 1], pg[kRun + 1], pr[kRun + 1];
#pragma unroll
  for (int c = 0; c <= kRun; ++c) {
    const int u = byte_at(ra, c + 1), d = byte_at(rc, c + 1), l = byte_at(rb, c), r = byte_at(rb, c + 2);
    const int ctr = byte_at(rb, c + 1);
    const int diag = (byte_at(ra, c) + byte_at(ra, c + 2) + byte_at(rc, c) + byte_at(rc, c + 2) + 2) >> 2;
    const int hor = (l + r + 1) >> 1, ver = (u + d + 1) >> 1;
    int cross;
    if constexpr (ALGO == SY_DEMOSAIC_BILINEAR)
      cross = (u + d + l + r + 2) >> 2;
    else
      cross = abs(l - r) > abs(u - d) ? ver : hor;
    const bool green = ((c - 1) & 1) == qpar;
    const int own = green ? hor : ctr, other = green ? ver : diag;   // the row's colour, the other one
    pg[c] = green ? ctr : cross;
    pr[c] = row_red ? own : other;
    pb[c] = row_red ? other : own;
  }
  // column x takes the interior pixel at clamp(x, 1, w - 2)
#pragma unroll
  for (int i = 0; i < 12; ++i) o[i] = 0;
#pragma unroll
  for (int j = 0; j < kRun; ++j) {
    uint32_t b = pb[j + 1], g = pg[j + 1], r = pr[j + 1];
    if (x0 + j == w - 1) b = pb[j], g = pg[j], r = pr[j];
    if (j == 0 && x0 == 0) b = pb[2], g = pg[2], r = pr[2];
    o[(3 * j) >> 2] |= b << (8 * ((3 * j) & 3));
    o[(3 * j + 1) >> 2] |= g << (8 * ((3 * j + 1) & 3));
    o[(3 * j + 2) >> 2] |= r << (8 * ((3 * j + 2) & 3));
  }
  store_run(q_out, o, n);
}

}  // namespace
}  // namespace sy

using namespace sy;

extern "C" int sy_bayer_to_bgr_sized(const SyBayerToBgrSizedDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->src != nullptr && d->sizes != nullptr && d->out != nullptr, SY_EINVAL,
             "bayer_to_bgr_sized: null pointer");
  SY_REQUIRE(d->pattern >= SY_BAYER_RGGB && d->pattern <= SY_BAYER_GRBG, SY_EINVAL,
             "bayer_to_bgr_sized: unknown pattern %d", d->pattern);
  SY_REQUIRE(d->algo == SY_DEMOSAIC_BILINEAR || d->algo == SY_DEMOSAIC_EA, SY_EINVAL,
             "bayer_to_bgr_sized: unknown demosaicing %d", d->algo);
  SY_REQUIRE(d->n > 0 && d->n <= 65535 && d->max_bytes > 0 && d->slot_h > 0 && d->slot_w > 0 &&
                 cdiv(d->slot_h, kTileH) <= 65535,
             SY_EINVAL, "bayer_to_bgr_sized: bad sizes (n %d, max_bytes %lld, slot %dx%d)", d->n,
             (long long)d->max_bytes, d->slot_h, d->slot_w);
  const dim3 block(kRuns, kTileH), grid(cdiv(d->slot_w, kTileW), cdiv(d->slot_h, kTileH), d->n);
  if (d->algo == SY_DEMOSAIC_BILINEAR)
    bayer_to_bgr_sized_kernel<SY_DEMOSAIC_BILINEAR><<<grid, block, 0, stream>>>(
        d->src, d->max_bytes, d->sizes, d->pattern, d->slot_h, d->slot_w, d->out);
  else
    bayer_to_bgr_sized_kernel<SY_DEMOSAIC_EA><<<grid, block, 0, stream>>>(
        d->src, d->max_bytes, d->sizes, d->pattern, d->slot_h, d->slot_w, d->out);
  return launch_status("bayer_to_bgr_sized_kernel");
}
