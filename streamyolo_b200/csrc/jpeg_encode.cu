// sy_jpeg_encode: uint8 BGR images of their own sizes -> JPEG files, byte-identical to cv2.imencode(".jpg", img,
// [IMWRITE_JPEG_QUALITY, q]) with cv2's defaults (libjpeg-turbo: baseline SOF0, 4:2:0, standard Huffman tables, no restart
// interval, JFIF 1.01).  oracle/jpeg_encode_oracle.py restates every stage in numpy.
//
//   jpeg_enc_transform  one CTA per 4 MCUs (64 x 16 pixels): jccolor.c RGB -> YCbCr, edge replication, jcsample.c h2v2
//                       downsample (bias 1, 2, 1, 2, ...), jfdctint.c islow FDCT, rounding division by 8 * qtable, the
//                       dummy blocks of partial MCUs (jccoefct.c: no AC, the DC of the block before them); int16
//                       coefficients in zigzag order, blocks in MCU interleave order (Y0 Y1 Y2 Y3 Cb Cr)
//   jpeg_enc_bits       one warp per block: DC difference against the previous block of its component and the block's
//                       coded length (DC, AC runs, ZRL, EOB)
//   jpeg_enc_scan       one CTA per image: the blocks' bit offsets (exclusive prefix sum) and the scan's byte length
//   jpeg_enc_zero       zeroes the words the scan's bits are ORed into
//   jpeg_enc_emit       one warp per block: every coefficient's code at its offset, then the 1-bit padding to a byte
//   jpeg_enc_count_ff   FF bytes per 4 KB chunk of the scan
//   jpeg_enc_finish     one CTA per image: the chunks' stuffed offsets, the file's length and its status
//   jpeg_enc_write      the headers (SOF0 with the image's size from the device table), the scan with a 00 after every
//                       FF, and EOI
// Nothing reads the sizes on the host: a captured graph follows sizes written before each replay.
#include <algorithm>

#include "common.cuh"

namespace sy {
namespace {

constexpr int kMaxBlockBits = 11 + 11 + 63 * (16 + 10);   // longest DC code + 11 bits, 63 x (longest AC code + 10 bits)
constexpr int kChunk = 4096;                               // scan bytes per jpeg_enc_count_ff / jpeg_enc_write CTA
constexpr int kHeaderBytes = 623;                          // SOI APP0 DQT DQT SOF0 DHT x 4 SOS
constexpr int kSofSize = 163;                              // offset of SOF0's height in the header (then the width)
constexpr int kMcusPerCta = 4;

// zigzag index -> natural index
__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Annex K.3 tables (jstdhuff.c): code counts per length 1..16, then the symbols
struct HuffSpec {
  uint8_t counts[16];
  uint8_t symbols[162];
};
constexpr HuffSpec kSpec[4] = {
    {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}},
    {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
     {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
      0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
      0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
      0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
      0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
      0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
      0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
      0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
      0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}},
    {{0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}},
    {{0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77},
     {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
      0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
      0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
      0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
      0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
      0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
      0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
      0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
      0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}}};
constexpr int kSpecCount[4] = {12, 162, 12, 162};

// symbol -> code / length (jchuff.c jpeg_make_c_derived_tbl); tables 0 = DC luma, 1 = AC luma, 2 = DC chroma, 3 = AC chroma
struct HuffTabs {
  uint16_t code[4][256];
  uint8_t len[4][256];
};
constexpr HuffTabs make_huff() {
  HuffTabs t{};
  for (int k = 0; k < 4; ++k) {
    int code = 0, s = 0;
    for (int ln = 1; ln <= 16; ++ln) {
      for (int i = 0; i < kSpec[k].counts[ln - 1]; ++i, ++s, ++code) {
        t.code[k][kSpec[k].symbols[s]] = (uint16_t)code;
        t.len[k][kSpec[k].symbols[s]] = (uint8_t)ln;
      }
      code <<= 1;
    }
  }
  return t;
}
__constant__ HuffTabs kHuff = make_huff();

struct Quant {
  int16_t div[2][64];   // 8 * qtable, natural order: luma, chroma
};
struct Header {
  uint8_t b[kHeaderBytes];
};

// per-image workspace, every array 256-byte aligned
struct Layout {
  int mx, my;            // MCUs of the slot
  size_t nblk, words, chunks;
  size_t coef, blen, word, ff, info, stride;
};
__host__ __device__ inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }
__host__ __device__ inline Layout make_layout(int max_h, int max_w, long long max_bytes) {
  Layout l{};
  l.mx = (max_w + 15) / 16, l.my = (max_h + 15) / 16;
  l.nblk = (size_t)6 * l.mx * l.my;
  const unsigned long long scan = l.nblk * (unsigned long long)kMaxBlockBits / 8 + 1;   // bytes the scan can take
  const unsigned long long cap = scan < (unsigned long long)max_bytes ? scan : (unsigned long long)max_bytes;
  l.words = (cap + 15) / 16 * 4 + 4;                                                      // whole uint4s
  l.chunks = (l.words * 4 + kChunk - 1) / kChunk;
  l.coef = 0;
  l.blen = align256(l.nblk * 128);
  l.word = l.blen + align256(l.nblk * 4);
  l.ff = l.word + align256(l.words * 4);
  l.info = l.ff + align256(l.chunks * 4);
  l.stride = l.info + 256;
  return l;
}

// info words of an image
enum { kInfoBits = 0, kInfoScanBytes = 1, kInfoOk = 2, kInfoFF = 3 };

__device__ __forceinline__ bool image_size(const int32_t* sizes, int k, int max_h, int max_w, int& h, int& w) {
  h = sizes[2 * k], w = sizes[2 * k + 1];
  return h >= 1 && w >= 1 && h <= max_h && w <= max_w;
}

// jccolor.c rgb_ycc_convert, SCALEBITS = 16
__device__ __forceinline__ int ycc_y(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16; }
__device__ __forceinline__ int ycc_cb(int r, int g, int b) {
  return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
}
__device__ __forceinline__ int ycc_cr(int r, int g, int b) {
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// jfdctint.c jpeg_fdct_islow, one pass over 8 values with stride s (CONST_BITS 13, PASS1_BITS 2)
template <bool kPass1>
__device__ __forceinline__ void fdct_1d(int* d, int s) {
  const int tmp0 = d[0] + d[7 * s], tmp7 = d[0] - d[7 * s];
  const int tmp1 = d[s] + d[6 * s], tmp6 = d[s] - d[6 * s];
  const int tmp2 = d[2 * s] + d[5 * s], tmp5 = d[2 * s] - d[5 * s];
  const int tmp3 = d[3 * s] + d[4 * s], tmp4 = d[3 * s] - d[4 * s];
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  constexpr int sh = kPass1 ? 11 : 15;
  if (kPass1) {
    d[0] = (tmp10 + tmp11) * 4;
    d[4 * s] = (tmp10 - tmp11) * 4;
  } else {
    d[0] = descale(tmp10 + tmp11, 2);
    d[4 * s] = descale(tmp10 - tmp11, 2);
  }
  int z1 = (tmp12 + tmp13) * 4433;
  d[2 * s] = descale(z1 + tmp13 * 6270, sh);
  d[6 * s] = descale(z1 - tmp12 * 15137, sh);
  z1 = tmp4 + tmp7;
  int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
  const int z5 = (z3 + z4) * 9633;
  const int t4 = tmp4 * 2446, t5 = tmp5 * 16819, t6 = tmp6 * 25172, t7 = tmp7 * 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  d[7 * s] = descale(t4 + z1 + z3, sh);
  d[5 * s] = descale(t5 + z2 + z4, sh);
  d[3 * s] = descale(t6 + z2 + z3, sh);
  d[s] = descale(t7 + z1 + z4, sh);
}

// grid (cdiv(slot MCU columns, 4), slot MCU rows, n), 256 threads
__global__ void __launch_bounds__(256) jpeg_enc_transform(const uint8_t* __restrict__ src, const int32_t* __restrict__ sizes,
                                                          int max_h, int max_w, Quant quant, uint8_t* __restrict__ ws,
                                                          size_t stride, Layout lay) {
  __shared__ int ys[16][kMcusPerCta * 16];
  __shared__ int cs[2][8][kMcusPerCta * 8];
  const int k = blockIdx.z, t = threadIdx.x;
  int h, w;
  if (!image_size(sizes, k, max_h, max_w, h, w)) return;
  const int mx = (w + 15) / 16, my = (h + 15) / 16;
  const int mcu0 = blockIdx.x * kMcusPerCta, mrow = blockIdx.y;
  if (mcu0 >= mx || mrow >= my) return;
  const uint8_t* img = src + (size_t)k * max_h * max_w * 3;
  // colour conversion: thread t takes the 2x2 pixel group (gy, gx) and its chroma sample
  {
    const int gy = t >> 5, gx = t & 31;
    const int y0 = mrow * 16 + 2 * gy, x0 = mcu0 * 16 + 2 * gx;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const uint8_t* p = img + ((size_t)min(y0 + dy, h - 1) * max_w + min(x0 + dx, w - 1)) * 3;
        ys[2 * gy + dy][2 * gx + dx] = ycc_y(p[2], p[1], p[0]) - 128;
      }
    // h2v2_downsample of the edge-expanded planes; output rows past the image's repeat its last one (jcprepct.c)
    const int r = min(mrow * 8 + gy, (h + 1) / 2 - 1), c = mcu0 * 8 + gx;
    const int bias = 1 + (c & 1);
    int scb = bias, scr = bias;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const uint8_t* p = img + ((size_t)min(2 * r + dy, h - 1) * max_w + min(2 * c + dx, w - 1)) * 3;
        scb += ycc_cb(p[2], p[1], p[0]);
        scr += ycc_cr(p[2], p[1], p[0]);
      }
    cs[0][gy][gx] = (scb >> 2) - 128;
    cs[1][gy][gx] = (scr >> 2) - 128;
  }
  __syncthreads();
  // block b = 6 * MCU + j of this CTA; thread t < 192 takes row / column t & 7 of block t >> 3
  const int b = t >> 3, i = t & 7, m = b / 6, j = b - 6 * m;
  int* base = nullptr;
  int pitch = 0;
  if (b < 6 * kMcusPerCta) {
    if (j < 4) {
      base = &ys[(j >> 1) * 8][m * 16 + (j & 1) * 8], pitch = kMcusPerCta * 16;
    } else {
      base = &cs[j - 4][0][m * 8], pitch = kMcusPerCta * 8;
    }
    fdct_1d<true>(base + i * pitch, 1);
  }
  __syncthreads();
  __shared__ int16_t q[6 * kMcusPerCta][64];
  if (b < 6 * kMcusPerCta) {
    fdct_1d<false>(base + i, pitch);
    const int16_t* div = quant.div[j < 4 ? 0 : 1];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int v = base[i + r * pitch], dv = div[r * 8 + i];
      const int a = (abs(v) + (dv >> 1)) / dv;
      q[b][r * 8 + i] = (int16_t)(v < 0 ? -a : a);
    }
  }
  __syncthreads();
  // jccoefct.c: Y blocks past ceil(w / 8) x ceil(h / 8) are dummies, with no AC and the DC of the block before them
  if (t < kMcusPerCta) {
    const int bx = 2 * (mcu0 + t), by = 2 * mrow, nbx = (w + 7) / 8, nby = (h + 7) / 8;
    for (int jj = 1; jj < 4; ++jj)
      if (by + (jj >> 1) >= nby || bx + (jj & 1) >= nbx) {
        for (int e = 1; e < 64; ++e) q[6 * t + jj][e] = 0;
        q[6 * t + jj][0] = q[6 * t + jj - 1][0];
      }
  }
  __syncthreads();
  // out: the CTA's MCUs are consecutive in the image's block order; zigzag order, two coefficients per 32-bit store
  const int nm = min(kMcusPerCta, mx - mcu0);
  uint32_t* out = reinterpret_cast<uint32_t*>(ws + stride * k + lay.coef) + ((size_t)mrow * mx + mcu0) * 6 * 32;
  for (int e = t; e < nm * 6 * 32; e += 256) {
    const int bb = e >> 5, z = 2 * (e & 31);
    out[e] = (uint32_t)(uint16_t)q[bb][kZigzag[z]] | ((uint32_t)(uint16_t)q[bb][kZigzag[z + 1]] << 16);
  }
}

__device__ __forceinline__ int category(int v) { return 32 - __clz(abs(v)); }

// bit k of the result = bit k / 2 of even (k even) or odd (k odd)
__device__ __forceinline__ uint64_t interleave(uint32_t even, uint32_t odd) {
  auto spread = [](uint64_t x) {
    x = (x | (x << 16)) & 0x0000FFFF0000FFFFull;
    x = (x | (x << 8)) & 0x00FF00FF00FF00FFull;
    x = (x | (x << 4)) & 0x0F0F0F0F0F0F0F0Full;
    x = (x | (x << 2)) & 0x3333333333333333ull;
    x = (x | (x << 1)) & 0x5555555555555555ull;
    return x;
  };
  return spread(even) | (spread(odd) << 1);
}

// One warp per block: lane l holds zigzag coefficients 2l and 2l + 1.  Each nonzero AC coefficient codes the zero run
// since the previous nonzero one (ZRLs for every 16, then (run, size) and its bits); lane 0 also codes the DC difference.
struct BlockCode {
  uint32_t val[2];       // (code << size) | magnitude bits of the lane's two coefficients
  int len[2], zrl[2];    // their lengths and the ZRLs before each
  int lane_bits;         // all of the lane's bits, ZRLs included (lane 0: the DC code first)
  int dc_val, dc_len;    // lane 0
  bool eob;
};

__device__ __forceinline__ BlockCode code_block(const uint32_t* __restrict__ coef, int blk, int prev, int lane) {
  const int comp = blk % 6 < 4 ? 0 : 1;
  const uint32_t pair = coef[(size_t)blk * 32 + lane];
  const int v[2] = {(int)(int16_t)(pair & 0xffff), (int)(int16_t)(pair >> 16)};
  const uint64_t nz = interleave(__ballot_sync(~0u, v[0] != 0), __ballot_sync(~0u, v[1] != 0)) & ~1ull;   // AC only
  BlockCode c{};
  const int ac = 2 * comp + 1, zrl_len = kHuff.len[ac][0xF0];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int kk = 2 * lane + e;
    if (kk == 0 || v[e] == 0) continue;
    const uint64_t below = nz & ((1ull << kk) - 1);
    const int run = kk - 1 - (below ? 63 - __clzll(below) : 0);
    const int s = category(v[e]), sym = ((run & 15) << 4) | s;
    const int mag = (v[e] < 0 ? v[e] - 1 : v[e]) & ((1 << s) - 1);
    c.zrl[e] = run >> 4;
    c.len[e] = kHuff.len[ac][sym] + s;
    c.val[e] = ((uint32_t)kHuff.code[ac][sym] << s) | (uint32_t)mag;
    c.lane_bits += c.zrl[e] * zrl_len + c.len[e];
  }
  if (lane == 0) {
    const int diff = v[0] - prev, s = category(diff), dc = 2 * comp;
    c.dc_len = kHuff.len[dc][s] + s;
    c.dc_val = (int)(((uint32_t)kHuff.code[dc][s] << s) | (uint32_t)((diff < 0 ? diff - 1 : diff) & ((1 << s) - 1)));
    c.lane_bits += c.dc_len;
  }
  c.eob = !(nz >> 63);
  return c;
}

// the DC of the block before block blk of its component in MCU interleave order (0 for the first)
__device__ __forceinline__ int prev_dc(const uint32_t* __restrict__ coef, int blk) {
  const int m = blk / 6, j = blk - 6 * m;
  const int p = j >= 1 && j < 4 ? blk - 1 : (m == 0 ? -1 : 6 * (m - 1) + (j == 0 ? 3 : j));
  return p < 0 ? 0 : (int)(int16_t)(coef[(size_t)p * 32] & 0xffff);
}

// grid (cdiv(slot blocks, 8), n), 256 threads: warp = block
__global__ void __launch_bounds__(256) jpeg_enc_bits(const int32_t* __restrict__ sizes, int max_h, int max_w,
                                                     uint8_t* __restrict__ ws, size_t stride, Layout lay) {
  const int k = blockIdx.y, lane = threadIdx.x & 31, blk = blockIdx.x * 8 + (threadIdx.x >> 5);
  int h, w;
  if (!image_size(sizes, k, max_h, max_w, h, w)) return;
  if (blk >= 6 * ((w + 15) / 16) * ((h + 15) / 16)) return;
  uint8_t* wsk = ws + stride * k;
  const uint32_t* coef = reinterpret_cast<const uint32_t*>(wsk + lay.coef);
  const BlockCode c = code_block(coef, blk, lane == 0 ? prev_dc(coef, blk) : 0, lane);
  int bits = c.lane_bits;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) bits += __shfl_xor_sync(~0u, bits, o);
  if (lane == 0)
    reinterpret_cast<uint32_t*>(wsk + lay.blen)[blk] = bits + (c.eob ? kHuff.len[blk % 6 < 4 ? 1 : 3][0x00] : 0);
}

// exclusive sum over the 1024 threads of a CTA; total to *total
__device__ __forceinline__ uint32_t block_exclusive_sum(uint32_t v, uint32_t* total) {
  __shared__ uint32_t warp_sum[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(~0u, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[wid] = x;
  __syncthreads();
  if (wid == 0) {
    const int nw = blockDim.x >> 5;
    uint32_t s = lane < nw ? warp_sum[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(~0u, s, o);
      if (lane >= o) s += y;
    }
    if (lane < nw) warp_sum[lane] = s;
  }
  __syncthreads();
  const uint32_t before = (wid ? warp_sum[wid - 1] : 0) + x - v;
  if (total) *total = warp_sum[(blockDim.x >> 5) - 1];
  __syncthreads();
  return before;
}

// grid (n), 1024 threads: blen -> exclusive bit offsets in place; the scan's bits and bytes; whether it can fit
__global__ void __launch_bounds__(1024) jpeg_enc_scan(const int32_t* __restrict__ sizes, int max_h, int max_w,
                                                      long long max_bytes, uint8_t* __restrict__ ws, size_t stride,
                                                      Layout lay, int64_t* __restrict__ lengths,
                                                      int32_t* __restrict__ status) {
  const int k = blockIdx.x, t = threadIdx.x;
  uint8_t* wsk = ws + stride * k;
  uint32_t* info = reinterpret_cast<uint32_t*>(wsk + lay.info);
  int h, w;
  if (!image_size(sizes, k, max_h, max_w, h, w)) {
    if (t == 0) {
      info[kInfoOk] = 0;
      lengths[k] = 0;
      status[k] = SY_JPEG_ENCODE_ESIZE;
    }
    return;
  }
  const int nb = 6 * ((w + 15) / 16) * ((h + 15) / 16);
  const int per = (nb + 1023) / 1024, b0 = min(t * per, nb), b1 = min(b0 + per, nb);
  uint32_t* blen = reinterpret_cast<uint32_t*>(wsk + lay.blen);
  uint32_t s = 0;
  for (int b = b0; b < b1; ++b) s += blen[b];
  uint32_t total;
  uint32_t off = block_exclusive_sum(s, &total);
  for (int b = b0; b < b1; ++b) {
    const uint32_t l = blen[b];
    blen[b] = off;
    off += l;
  }
  if (t == 0) {
    const uint32_t scan = (total + 7) / 8;
    const bool fits = (long long)kHeaderBytes + scan + 2 <= max_bytes;
    info[kInfoBits] = total;
    info[kInfoScanBytes] = scan;
    info[kInfoOk] = fits;
    if (!fits) {
      lengths[k] = 0;
      status[k] = SY_JPEG_ENCODE_EOVERFLOW;
    }
  }
}

// grid (cdiv(slot words, 1024), n), 256 threads: the image's scan words (whole uint4s) to zero
__global__ void __launch_bounds__(256) jpeg_enc_zero(uint8_t* __restrict__ ws, size_t stride, Layout lay) {
  uint8_t* wsk = ws + stride * blockIdx.y;
  const uint32_t* info = reinterpret_cast<const uint32_t*>(wsk + lay.info);
  if (!info[kInfoOk]) return;
  const size_t q = (size_t)blockIdx.x * 256 + threadIdx.x;           // uint4 index
  if (q * 16 < info[kInfoScanBytes]) reinterpret_cast<uint4*>(wsk + lay.word)[q] = make_uint4(0, 0, 0, 0);
}

// OR the top len bits of val (len <= 32) into the big-endian bit stream at bit pos
__device__ __forceinline__ void put_bits(uint32_t* __restrict__ words, uint32_t pos, uint32_t val, int len) {
  if (len == 0) return;
  const uint64_t v = (uint64_t)val << (64 - len - (pos & 31));
  atomicOr(words + (pos >> 5), (uint32_t)(v >> 32));
  if ((uint32_t)v) atomicOr(words + (pos >> 5) + 1, (uint32_t)v);
}

// grid (cdiv(slot blocks, 8), n), 256 threads: warp = block
__global__ void __launch_bounds__(256) jpeg_enc_emit(const int32_t* __restrict__ sizes, int max_h, int max_w,
                                                     uint8_t* __restrict__ ws, size_t stride, Layout lay) {
  const int k = blockIdx.y, lane = threadIdx.x & 31, blk = blockIdx.x * 8 + (threadIdx.x >> 5);
  int h, w;
  if (!image_size(sizes, k, max_h, max_w, h, w)) return;
  uint8_t* wsk = ws + stride * k;
  const uint32_t* info = reinterpret_cast<const uint32_t*>(wsk + lay.info);
  if (!info[kInfoOk]) return;
  uint32_t* words = reinterpret_cast<uint32_t*>(wsk + lay.word);
  if (blk == 0 && lane == 0) {                                       // jchuff.c flush_bits: 1-bits to a byte boundary
    const uint32_t bits = info[kInfoBits], pad = (8 - (bits & 7)) & 7;
    put_bits(words, bits, (1u << pad) - 1, pad);
  }
  if (blk >= 6 * ((w + 15) / 16) * ((h + 15) / 16)) return;
  const uint32_t* coef = reinterpret_cast<const uint32_t*>(wsk + lay.coef);
  const BlockCode c = code_block(coef, blk, lane == 0 ? prev_dc(coef, blk) : 0, lane);
  uint32_t x = c.lane_bits;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(~0u, x, o);
    if (lane >= o) x += y;
  }
  const uint32_t start = reinterpret_cast<const uint32_t*>(wsk + lay.blen)[blk];
  uint32_t pos = start + x - c.lane_bits;
  const int ac = blk % 6 < 4 ? 1 : 3;
  if (lane == 0) {
    put_bits(words, pos, (uint32_t)c.dc_val, c.dc_len);
    pos += c.dc_len;
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    for (int z = 0; z < c.zrl[e]; ++z) {
      put_bits(words, pos, kHuff.code[ac][0xF0], kHuff.len[ac][0xF0]);
      pos += kHuff.len[ac][0xF0];
    }
    put_bits(words, pos, c.val[e], c.len[e]);
    pos += c.len[e];
  }
  if (lane == 31 && c.eob) put_bits(words, pos, kHuff.code[ac][0x00], kHuff.len[ac][0x00]);
}

__device__ __forceinline__ uint32_t scan_byte(const uint32_t* words, uint32_t j) {
  return (words[j >> 2] >> (24 - 8 * (j & 3))) & 255u;
}

// grid (slot chunks, n), 256 threads x 16 bytes: FF bytes per chunk
__global__ void __launch_bounds__(256) jpeg_enc_count_ff(uint8_t* __restrict__ ws, size_t stride, Layout lay) {
  uint8_t* wsk = ws + stride * blockIdx.y;
  const uint32_t* info = reinterpret_cast<const uint32_t*>(wsk + lay.info);
  const uint32_t scan = info[kInfoScanBytes];
  if (!info[kInfoOk] || (size_t)blockIdx.x * kChunk >= scan) return;
  const uint32_t* words = reinterpret_cast<const uint32_t*>(wsk + lay.word);
  const uint32_t j0 = blockIdx.x * kChunk + threadIdx.x * 16;
  int n = 0;
  for (uint32_t j = j0; j < min(j0 + 16, scan); ++j) n += scan_byte(words, j) == 255u;
  __shared__ int sum;
  if (threadIdx.x == 0) sum = 0;
  __syncthreads();
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(~0u, n, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(&sum, n);
  __syncthreads();
  if (threadIdx.x == 0) reinterpret_cast<uint32_t*>(wsk + lay.ff)[blockIdx.x] = sum;
}

// grid (n), 1024 threads: chunk FF counts -> exclusive offsets; the file's length and status
__global__ void __launch_bounds__(1024) jpeg_enc_finish(long long max_bytes, uint8_t* __restrict__ ws, size_t stride,
                                                        Layout lay, int64_t* __restrict__ lengths,
                                                        int32_t* __restrict__ status) {
  const int k = blockIdx.x, t = threadIdx.x;
  uint8_t* wsk = ws + stride * k;
  uint32_t* info = reinterpret_cast<uint32_t*>(wsk + lay.info);
  if (!info[kInfoOk]) return;
  const uint32_t scan = info[kInfoScanBytes];
  const int nc = (int)((scan + kChunk - 1) / kChunk);
  const int per = (nc + 1023) / 1024, c0 = min(t * per, nc), c1 = min(c0 + per, nc);
  uint32_t* ff = reinterpret_cast<uint32_t*>(wsk + lay.ff);
  uint32_t s = 0;
  for (int c = c0; c < c1; ++c) s += ff[c];
  uint32_t total;
  uint32_t off = block_exclusive_sum(s, &total);
  for (int c = c0; c < c1; ++c) {
    const uint32_t l = ff[c];
    ff[c] = off;
    off += l;
  }
  if (t == 0) {
    const long long len = (long long)kHeaderBytes + scan + total + 2;
    const bool fits = len <= max_bytes;
    info[kInfoOk] = fits;
    info[kInfoFF] = total;
    lengths[k] = fits ? len : 0;
    status[k] = fits ? SY_JPEG_ENCODE_OK : SY_JPEG_ENCODE_EOVERFLOW;
  }
}

// grid (slot chunks, n), 256 threads x 16 bytes: the stuffed scan; CTA 0 also the headers and EOI
__global__ void __launch_bounds__(256) jpeg_enc_write(const int32_t* __restrict__ sizes, Header hdr,
                                                      uint8_t* __restrict__ out, long long max_bytes,
                                                      uint8_t* __restrict__ ws, size_t stride, Layout lay) {
  const int k = blockIdx.y, t = threadIdx.x;
  uint8_t* wsk = ws + stride * k;
  const uint32_t* info = reinterpret_cast<const uint32_t*>(wsk + lay.info);
  const uint32_t scan = info[kInfoScanBytes];
  if (!info[kInfoOk] || (size_t)blockIdx.x * kChunk >= scan) return;
  uint8_t* o = out + (size_t)max_bytes * k;
  const uint32_t* words = reinterpret_cast<const uint32_t*>(wsk + lay.word);
  const uint32_t* ff = reinterpret_cast<const uint32_t*>(wsk + lay.ff);
  if (blockIdx.x == 0) {
    const int h = sizes[2 * k], w = sizes[2 * k + 1];
    for (int i = t; i < kHeaderBytes; i += 256) {
      uint8_t v = hdr.b[i];
      if (i == kSofSize) v = (uint8_t)(h >> 8);
      if (i == kSofSize + 1) v = (uint8_t)h;
      if (i == kSofSize + 2) v = (uint8_t)(w >> 8);
      if (i == kSofSize + 3) v = (uint8_t)w;
      o[i] = v;
    }
    if (t == 0) {
      const size_t end = (size_t)kHeaderBytes + scan + info[kInfoFF];
      o[end] = 0xFF;
      o[end + 1] = 0xD9;
    }
  }
  const uint32_t j0 = blockIdx.x * kChunk + t * 16, j1 = min(j0 + 16, scan);
  uint32_t n = 0;
  for (uint32_t j = j0; j < j1; ++j) n += scan_byte(words, j) == 255u;
  uint32_t pos = kHeaderBytes + j0 + ff[blockIdx.x] + block_exclusive_sum(n, nullptr);
  for (uint32_t j = j0; j < j1; ++j) {
    const uint32_t v = scan_byte(words, j);
    o[pos++] = (uint8_t)v;
    if (v == 255u) o[pos++] = 0;
  }
}

// jcparam.c jpeg_quality_scaling + jpeg_add_quant_table(force_baseline): the tables as libjpeg stores them
void quant_tables(int quality, int (&qt)[2][64]) {
  static const int std_tab[2][64] = {
      {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,
       69, 56, 14, 17, 22,  29,  51,  87,  80, 62, 18, 22, 37,  56,  68,  109, 103, 77, 24, 35, 55, 64,
       81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
      {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
       99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
       99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int c = 0; c < 2; ++c)
    for (int i = 0; i < 64; ++i) qt[c][i] = std::min(std::max((std_tab[c][i] * scale + 50) / 100, 1), 255);
}

// SOI, APP0 JFIF 1.01 (density 1:1), DQT 0, DQT 1 (zigzag), SOF0 (size patched per image), DHT DC0 AC0 DC1 AC1, SOS
Header make_header(const int (&qt)[2][64]) {
  static const uint8_t zz[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  Header hd{};
  int p = 0;
  auto put = [&](int v) { hd.b[p++] = (uint8_t)v; };
  auto seg = [&](int marker, int len) { put(0xFF), put(marker), put(len >> 8), put(len & 255); };
  put(0xFF), put(0xD8);
  seg(0xE0, 16);
  for (int v : {0x4A, 0x46, 0x49, 0x46, 0, 1, 1, 0, 0, 1, 0, 1, 0, 0}) put(v);   // "JFIF\0", 1.01, density 1:1
  for (int c = 0; c < 2; ++c) {
    seg(0xDB, 67);
    put(c);
    for (int i = 0; i < 64; ++i) put(qt[c][zz[i]]);
  }
  seg(0xC0, 17);
  for (int v : {8, 0, 0, 0, 0, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1}) put(v);
  const int order[4] = {0, 1, 2, 3}, cls[4] = {0x00, 0x10, 0x01, 0x11};
  for (int k : order) {
    seg(0xC4, 2 + 1 + 16 + kSpecCount[k]);
    put(cls[k]);
    for (int i = 0; i < 16; ++i) put(kSpec[k].counts[i]);
    for (int i = 0; i < kSpecCount[k]; ++i) put(kSpec[k].symbols[i]);
  }
  seg(0xDA, 12);
  for (int v : {3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0}) put(v);
  return hd;
}

bool slot_ok(int n, int max_h, int max_w, long long max_bytes) {
  if (n <= 0 || n > 65535 || max_h <= 0 || max_w <= 0 || max_h > 65535 || max_w > 65535) return false;
  if (max_bytes <= 0 || max_bytes > (1ll << 31)) return false;
  const unsigned long long nblk = 6ull * ((max_w + 15) / 16) * ((max_h + 15) / 16);
  return nblk * kMaxBlockBits < (1ull << 32) && nblk <= 65535ull * 8;    // 32-bit bit offsets; the blocks' grid.x
}

}  // namespace
}  // namespace sy

using namespace sy;

extern "C" int64_t sy_jpeg_encode_max_bytes(int32_t h, int32_t w) {
  if (h <= 0 || w <= 0 || h > 65535 || w > 65535) return 0;
  const long long blocks = 6ll * ((h + 15) / 16) * ((w + 15) / 16);
  return kHeaderBytes + 2 * ((blocks * kMaxBlockBits + 7) / 8) + 2;
}

extern "C" size_t sy_jpeg_encode_workspace_bytes(int32_t n, int32_t max_h, int32_t max_w, int64_t max_bytes) {
  if (!slot_ok(n, max_h, max_w, max_bytes)) return 0;
  return make_layout(max_h, max_w, max_bytes).stride * (size_t)n;
}

extern "C" int sy_jpeg_encode(const SyJpegEncodeDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->src != nullptr && d->sizes != nullptr && d->out != nullptr && d->lengths != nullptr &&
                 d->status != nullptr && d->workspace != nullptr, SY_EINVAL, "jpeg_encode: null pointer");
  SY_REQUIRE(d->quality >= 1 && d->quality <= 100, SY_EINVAL, "jpeg_encode: quality %d not in 1..100", d->quality);
  SY_REQUIRE(slot_ok(d->n, d->max_h, d->max_w, d->max_bytes), SY_EINVAL,
             "jpeg_encode: bad sizes (n %d, slot %dx%d, max_bytes %lld)", d->n, d->max_h, d->max_w,
             (long long)d->max_bytes);
  SY_REQUIRE((uintptr_t)d->sizes % 4 == 0 && (uintptr_t)d->lengths % 8 == 0 && (uintptr_t)d->status % 4 == 0, SY_EINVAL,
             "jpeg_encode: misaligned sizes, lengths or status");
  const size_t need = sy_jpeg_encode_workspace_bytes(d->n, d->max_h, d->max_w, d->max_bytes);
  SY_REQUIRE(d->workspace_bytes >= need && ((uintptr_t)d->workspace % 256) == 0, SY_EINVAL,
             "jpeg_encode: workspace of %zu bytes (need %zu, 256-byte aligned)", d->workspace_bytes, need);
  const Layout lay = make_layout(d->max_h, d->max_w, d->max_bytes);
  int qt[2][64];
  quant_tables(d->quality, qt);
  Quant quant{};
  for (int c = 0; c < 2; ++c)
    for (int i = 0; i < 64; ++i) quant.div[c][i] = (int16_t)(8 * qt[c][i]);
  const Header hdr = make_header(qt);
  uint8_t* ws = static_cast<uint8_t*>(d->workspace);
  const size_t st = lay.stride;
  const int n = d->n;
  const unsigned blk_ctas = (unsigned)cdiv((int)lay.nblk, 8);
  jpeg_enc_transform<<<dim3(cdiv(lay.mx, kMcusPerCta), lay.my, n), 256, 0, stream>>>(d->src, d->sizes, d->max_h,
                                                                                     d->max_w, quant, ws, st, lay);
  jpeg_enc_bits<<<dim3(blk_ctas, n), 256, 0, stream>>>(d->sizes, d->max_h, d->max_w, ws, st, lay);
  jpeg_enc_scan<<<n, 1024, 0, stream>>>(d->sizes, d->max_h, d->max_w, d->max_bytes, ws, st, lay, d->lengths, d->status);
  jpeg_enc_zero<<<dim3((unsigned)((lay.words + 1023) / 1024), n), 256, 0, stream>>>(ws, st, lay);
  jpeg_enc_emit<<<dim3(blk_ctas, n), 256, 0, stream>>>(d->sizes, d->max_h, d->max_w, ws, st, lay);
  jpeg_enc_count_ff<<<dim3((unsigned)lay.chunks, n), 256, 0, stream>>>(ws, st, lay);
  jpeg_enc_finish<<<n, 1024, 0, stream>>>(d->max_bytes, ws, st, lay, d->lengths, d->status);
  jpeg_enc_write<<<dim3((unsigned)lay.chunks, n), 256, 0, stream>>>(d->sizes, hdr, d->out, d->max_bytes, ws, st, lay);
  return launch_status("jpeg_encode kernels");
}
