// Batched baseline JPEG decode on the device, bit-identical to cv2.imread (libjpeg-turbo's default decompression):
//   1. jpeg_parse_kernel     one thread per image walks the markers (SOI, APPn, DQT, SOF0/1, DHT, DRI, SOS), builds the
//                            Huffman lookup tables and the quantisation tables in the workspace and sets the status.
//   2. jpeg_ecs_kernel       one CTA per image: drops the byte stuffing (FF 00) and fill bytes of the entropy-coded
//                            segment, finds its end and splits it at the RSTn markers (one pass to count, one to write).
//   3. jpeg_huffman_kernel   one 8-CTA cluster per image.  With restart intervals every interval decodes on its own thread.
//                            Without them the stream is cut into up to 4096 subsequences of equal bit length, decoded by
//                            self-synchronising subsequence decoding (Weissenberger & Schmidt, ICPP 2018 / HiPC 2021):
//                            every thread decodes its subsequence from a start state (bit position, block in MCU,
//                            coefficient index), hands its end state to its successor through distributed shared memory,
//                            and the round repeats until no start state changes.  Subsequence 0 starts exactly, so the
//                            fixpoint is the sequential decode; Huffman codes resynchronise within a few codewords, so it
//                            is reached in a few rounds.  A cluster-wide prefix sum of the per-subsequence block counts and
//                            DC differences (per component) gives every thread its first block and DC predictions, and a
//                            last pass writes the quantised coefficients in zigzag order.
//   4. jpeg_idct_kernel      dequantise + jidctint.c's integer "islow" IDCT with its range-limit table, 8 threads per block.
//   5. jpeg_color_kernel     jdsample.c's chroma upsampling ("fancy" triangle filter for 2x1 / 2x2, plain replication when
//                            the chroma plane is at most 2 samples wide) and jdcolor.c's fixed-point YCbCr -> BGR; it also
//                            publishes each image's status.
// sy_jpeg_decode gives every image the batch's size; sy_jpeg_decode_sized gives image i its own expected size and a slot of
// max_h x max_w in the output.  Both run the same five kernels: each image's MCU geometry, restart bookkeeping, upsampling
// and colour conversion read the size stored in its JpegImage by the parse.
// oracle/jpeg_oracle.py restates every stage in numpy; tests/test_jpeg_decode.py pins it to cv2.imdecode.
#include <cooperative_groups.h>
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace sy {
namespace {

constexpr int kClusterCtas = 8;
constexpr int kHuffThreads = 512;
constexpr int kMaxSubseq = kClusterCtas * kHuffThreads;  // subsequences of a stream without restart intervals
constexpr int kMinSubseqBits = 2048;
constexpr int kEcsThreads = 1024;
constexpr int kIdctBlocksPerCta = 16;
constexpr int kErrPos = -1;                               // end state of a subsequence whose decode failed

struct HuffTab {
  uint16_t fast[512];   // 9-bit lookahead: (length << 8) | symbol, 0 = longer code or invalid
  int32_t maxcode[18];  // largest code of each length, -1 when there is none
  int32_t valoff[18];   // symbol index of a code of that length = code + valoff
  uint8_t vals[256];
};

struct JpegImage {
  int32_t status, done;
  int32_t h, w;         // the image's own size (SOF)
  int32_t h0, v0, mcux, mcuy, bpm, total_blocks;
  int32_t ri, n_units, unit_bits, ecs_bits;
  int32_t scan_begin;
  int32_t comp_q[3], comp_dc[3], comp_ac[3];
  uint16_t q[4][64];    // natural order
  HuffTab dc[4], ac[4];
};

// per-image slices of the workspace
struct Layout {
  size_t image_stride, off_ecs, off_seg, off_coef, off_planes;
  int32_t max_units;
};

__host__ __device__ inline size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

__device__ __forceinline__ JpegImage* image_of(uint8_t* ws, const Layout& L, int i) {
  return reinterpret_cast<JpegImage*>(ws + L.image_stride * i);
}

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t kUnzig[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42,
                                   3,  8,  12, 17, 25, 30, 41, 43, 9,  11, 18, 24, 31, 40, 44, 53,
                                   10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60,
                                   21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};  // natural -> zigzag

// ------------------------------------------------------------------------------------------------------------------
// 1. marker parse

__device__ __forceinline__ int u16be(const uint8_t* b, int i) { return (b[i] << 8) | b[i + 1]; }

// EXIF orientation of an APP1 payload [s, s + len): 1 when absent or unreadable
__device__ int exif_orientation(const uint8_t* s, int len) {
  if (len < 14 || s[0] != 'E' || s[1] != 'x' || s[2] != 'i' || s[3] != 'f' || s[4] != 0 || s[5] != 0) return 1;
  const uint8_t* t = s + 6;
  const int tl = len - 6;
  bool le;
  if (t[0] == 'I' && t[1] == 'I' && t[2] == 42 && t[3] == 0) le = true;
  else if (t[0] == 'M' && t[1] == 'M' && t[2] == 0 && t[3] == 42) le = false;
  else return 1;
  auto rd = [&](int i, int n) -> uint32_t {
    uint32_t v = 0;
    for (int k = 0; k < n; ++k) v |= (uint32_t)t[i + k] << (8 * (le ? k : n - 1 - k));
    return v;
  };
  const uint32_t ifd = rd(4, 4);
  if (ifd + 2 > (uint32_t)tl) return 1;
  const int cnt = (int)rd((int)ifd, 2);
  for (int e = 0; e < cnt; ++e) {
    const uint32_t p = ifd + 2 + 12u * e;
    if (p + 12 > (uint32_t)tl) return 1;
    if (rd((int)p, 2) == 0x0112) return rd((int)p + 2, 2) == 3 ? (int)rd((int)p + 8, 2) : 1;
  }
  return 1;
}

// canonical Huffman table (JPEG Annex C) from the 16 code-length counts and the symbols; false if over-subscribed
__device__ bool build_huff(HuffTab* t, const uint8_t* counts, const uint8_t* vals, int total) {
  for (int k = 0; k < 512; ++k) t->fast[k] = 0;
  for (int k = 0; k < total; ++k) t->vals[k] = vals[k];
  int code = 0, k = 0;
  for (int len = 1; len <= 16; ++len) {
    const int nl = counts[len - 1];
    t->valoff[len] = k - code;
    for (int j = 0; j < nl; ++j, ++k, ++code) {
      if (code >= (1 << len)) return false;
      if (len <= 9)
        for (int f = code << (9 - len), e = (code + 1) << (9 - len); f < e; ++f) t->fast[f] = (uint16_t)((len << 8) | vals[k]);
    }
    t->maxcode[len] = nl ? code - 1 : -1;
    code <<= 1;
  }
  t->maxcode[0] = t->maxcode[17] = -1;
  return true;
}

// h x w: the size every image must have, or with ``sizes`` the output slot, and image i must be sizes[i] = (h_i, w_i) and
// fit the slot
__global__ void __launch_bounds__(32) jpeg_parse_kernel(const uint8_t* __restrict__ bytes, const int32_t* __restrict__ lengths,
                                                        int64_t max_bytes, int h, int w, const int32_t* __restrict__ sizes,
                                                        uint8_t* ws, Layout L) {
  if (threadIdx.x != 0) return;
  const int i = blockIdx.x;
  JpegImage* im = image_of(ws, L, i);
  const uint8_t* b = bytes + max_bytes * i;
  const int64_t n64 = lengths[i];
  int status = SY_JPEG_EHEADER;
  im->done = 0;
  auto finish = [&](int s) { im->status = s; };
  if (n64 < 4 || n64 > max_bytes || b[0] != 0xFF || b[1] != 0xD8) return finish(SY_JPEG_EHEADER);
  const int n = (int)n64;
  bool have_sof = false, jfif = false;
  int adobe = -1, ri = 0, qdef = 0, dcdef = 0, acdef = 0;
  int ih = 0, iw = 0, cid[3], ch[3], cv[3], cq[3];
  int p = 2;
  for (;;) {
    if (p >= n || b[p] != 0xFF) return finish(status);
    while (p < n && b[p] == 0xFF) ++p;
    if (p >= n) return finish(status);
    const int m = b[p++];
    if (m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD9)) return finish(status);
    if (p + 2 > n) return finish(status);
    const int ln = u16be(b, p);
    if (ln < 2 || p + ln > n) return finish(status);
    const uint8_t* s = b + p + 2;
    const int sl = ln - 2;
    p += ln;
    if (m == 0xC0 || m == 0xC1) {
      if (have_sof || sl < 6) return finish(status);
      if (s[0] != 8) return finish(SY_JPEG_EUNSUPPORTED);
      ih = u16be(s, 1), iw = u16be(s, 3);
      if (s[5] != 3) return finish(SY_JPEG_EUNSUPPORTED);
      if (sl != 6 + 9) return finish(status);
      for (int k = 0; k < 3; ++k) cid[k] = s[6 + 3 * k], ch[k] = s[7 + 3 * k] >> 4, cv[k] = s[7 + 3 * k] & 15, cq[k] = s[8 + 3 * k];
      if (ih == 0 || iw == 0) return finish(SY_JPEG_EUNSUPPORTED);
      const bool luma_ok = (ch[0] == 1 && cv[0] == 1) || (ch[0] == 2 && cv[0] == 1) || (ch[0] == 2 && cv[0] == 2);
      if (!luma_ok || ch[1] != 1 || cv[1] != 1 || ch[2] != 1 || cv[2] != 1) return finish(SY_JPEG_EUNSUPPORTED);
      if (cq[0] > 3 || cq[1] > 3 || cq[2] > 3) return finish(status);
      have_sof = true;
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8) {
      return finish(SY_JPEG_EUNSUPPORTED);                 // progressive, lossless, hierarchical, arithmetic (and DAC)
    } else if (m == 0xDB) {
      for (int o = 0; o < sl;) {
        const int pq = s[o] >> 4, tq = s[o] & 15, sz = 64 * (pq + 1);
        if (pq > 1 || tq > 3 || o + 1 + sz > sl) return finish(status);
        for (int k = 0; k < 64; ++k)
          im->q[tq][kZigzag[k]] = pq ? (uint16_t)u16be(s, o + 1 + 2 * k) : (uint16_t)s[o + 1 + k];
        qdef |= 1 << tq;
        o += 1 + sz;
      }
    } else if (m == 0xC4) {
      for (int o = 0; o < sl;) {
        if (o + 17 > sl) return finish(status);
        const int tc = s[o] >> 4, th = s[o] & 15;
        int tot = 0;
        for (int k = 0; k < 16; ++k) tot += s[o + 1 + k];
        if (tc > 1 || th > 3 || tot > 256 || o + 17 + tot > sl) return finish(status);
        if (tc == 0)
          for (int k = 0; k < tot; ++k)
            if (s[o + 17 + k] > 15) return finish(status);
        if (!build_huff(tc == 0 ? &im->dc[th] : &im->ac[th], s + o + 1, s + o + 17, tot)) return finish(status);
        (tc == 0 ? dcdef : acdef) |= 1 << th;
        o += 17 + tot;
      }
    } else if (m == 0xDD) {
      if (sl != 2) return finish(status);
      ri = u16be(s, 0);
    } else if (m == 0xE0) {
      jfif = jfif || (sl >= 5 && s[0] == 'J' && s[1] == 'F' && s[2] == 'I' && s[3] == 'F' && s[4] == 0);
    } else if (m == 0xE1) {
      if (exif_orientation(s, sl) != 1) return finish(SY_JPEG_EORIENTATION);
    } else if (m == 0xEE) {
      if (sl >= 12 && s[0] == 'A' && s[1] == 'd' && s[2] == 'o' && s[3] == 'b' && s[4] == 'e') adobe = s[11];
    } else if (m == 0xDA) {
      if (!have_sof) return finish(status);
      const int ns = sl > 0 ? s[0] : 0;
      if (sl != 4 + 2 * ns) return finish(status);
      if (ns != 3) return finish(SY_JPEG_EUNSUPPORTED);
      if (s[7] != 0 || s[8] != 63 || s[9] != 0) return finish(status);
      for (int k = 0; k < 3; ++k) {
        if (s[1 + 2 * k] != cid[k]) return finish(SY_JPEG_EUNSUPPORTED);
        im->comp_dc[k] = s[2 + 2 * k] >> 4, im->comp_ac[k] = s[2 + 2 * k] & 15, im->comp_q[k] = cq[k];
      }
      if (adobe == 0 || (!jfif && adobe < 0 && cid[0] == 82 && cid[1] == 71 && cid[2] == 66))
        return finish(SY_JPEG_EUNSUPPORTED);
      for (int k = 0; k < 3; ++k)
        if (!((qdef >> cq[k]) & 1) || im->comp_dc[k] > 3 || im->comp_ac[k] > 3 || !((dcdef >> im->comp_dc[k]) & 1) ||
            !((acdef >> im->comp_ac[k]) & 1))
          return finish(status);
      break;
    }
    // APPn, COM and other segments: skipped
  }
  const int eh = sizes != nullptr ? sizes[2 * i] : h, ew = sizes != nullptr ? sizes[2 * i + 1] : w;
  if (ih != eh || iw != ew || ih > h || iw > w) return finish(SY_JPEG_ESIZE);
  im->h = ih, im->w = iw;
  im->h0 = ch[0], im->v0 = cv[0];
  im->mcux = cdiv(iw, 8 * ch[0]), im->mcuy = cdiv(ih, 8 * cv[0]);
  im->bpm = ch[0] * cv[0] + 2;
  im->total_blocks = im->mcux * im->mcuy * im->bpm;
  im->ri = ri;
  im->scan_begin = p;
  finish(SY_JPEG_OK);
}

// ------------------------------------------------------------------------------------------------------------------
// 2. entropy-coded segment: destuff, find the end, split at RSTn

// what byte j of [begin, end) contributes: kept as data, an RSTn marker (at its FF), or nothing (stuffed 00, fill FF)
__device__ __forceinline__ void classify(const uint8_t* b, int j, int begin, int end, bool& keep, bool& rst) {
  const int c = b[j];
  const int nx = j + 1 < end ? b[j + 1] : -1;
  if (c != 0xFF) {
    keep = !(j > begin && b[j - 1] == 0xFF);      // the 00 of a stuffed FF or the code byte of an RSTn marker
    rst = false;
  } else {
    keep = nx == 0;
    rst = nx >= 0xD0 && nx <= 0xD7;
  }
}

__global__ void __launch_bounds__(kEcsThreads) jpeg_ecs_kernel(const uint8_t* __restrict__ bytes,
                                                               const int32_t* __restrict__ lengths, int64_t max_bytes,
                                                               uint8_t* ws, Layout L) {
  using Scan = cub::BlockScan<int, kEcsThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_end, s_bad, s_kept, s_rst;
  const int i = blockIdx.x, t = threadIdx.x;
  JpegImage* im = image_of(ws, L, i);
  if (im->status != SY_JPEG_OK) return;
  const uint8_t* b = bytes + max_bytes * i;
  const int len = lengths[i], begin = im->scan_begin;
  uint8_t* ecs = ws + L.image_stride * i + L.off_ecs;
  int32_t* seg = reinterpret_cast<int32_t*>(ws + L.image_stride * i + L.off_seg);
  const int chunk = cdiv(max(len - begin, 1), kEcsThreads);
  const int lo = begin + t * chunk, hi = min(lo + chunk, len);
  if (t == 0) s_end = len, s_bad = 0;
  __syncthreads();
  // pass 1: the first marker other than RSTn ends the segment; count kept bytes and markers before it
  int kept = 0, rst = 0, my_end = hi;
  for (int j = lo; j < hi; ++j) {
    if (b[j] == 0xFF && j + 1 < len) {
      const int nx = b[j + 1];
      if (nx != 0 && nx != 0xFF && !(nx >= 0xD0 && nx <= 0xD7)) {
        my_end = j;
        atomicMin(&s_end, j);
        break;
      }
    }
  }
  __syncthreads();
  const int end = s_end;
  for (int j = lo; j < min(my_end, end); ++j) {
    bool k, r;
    classify(b, j, begin, end, k, r);
    kept += k, rst += r;
  }
  int kept0, rst0;
  Scan(tmp).ExclusiveSum(kept, kept0);
  __syncthreads();
  Scan(tmp).ExclusiveSum(rst, rst0);
  if (t == kEcsThreads - 1) s_kept = kept0 + kept, s_rst = rst0 + rst;
  __syncthreads();
  if (s_rst + 1 > L.max_units) {                       // more restart intervals than MCUs
    if (t == 0) im->status = SY_JPEG_EDATA;
    return;
  }
  // pass 2: write the kept bytes and the restart intervals' byte offsets
  for (int j = lo; j < min(my_end, end); ++j) {
    bool k, r;
    classify(b, j, begin, end, k, r);
    if (k) ecs[kept0++] = b[j];
    if (r) {
      if (b[j + 1] - 0xD0 != (rst0 & 7)) s_bad = 1;
      seg[++rst0] = kept0;
    }
  }
  __syncthreads();
  if (t < 8) ecs[s_kept + t] = 0;
  if (t != 0) return;
  seg[0] = 0;
  const int total_mcus = im->mcux * im->mcuy;
  int units;
  if (im->ri > 0) {
    units = s_rst + 1;
    if (units != cdiv(total_mcus, im->ri)) s_bad = 1;
  } else {
    if (s_rst != 0) s_bad = 1;
    const int bits = 8 * s_kept;
    im->unit_bits = max(kMinSubseqBits, cdiv(cdiv(bits, kMaxSubseq), 32) * 32);
    units = max(1, cdiv(bits, im->unit_bits));
  }
  im->n_units = units;
  im->ecs_bits = 8 * s_kept;
  if (s_bad) im->status = SY_JPEG_EDATA;
}

// ------------------------------------------------------------------------------------------------------------------
// 3. Huffman decode

struct Tabs {
  HuffTab dc[3], ac[3];   // per component
  int comp_of[6];         // component of each block of an MCU
};

// 32 bits of the destuffed stream from bit ``pos`` (MSB first); the stream is padded so that this stays in bounds
__device__ __forceinline__ uint32_t peek32(const uint8_t* __restrict__ ecs, int pos) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(ecs) + (pos >> 5);
  const uint32_t hi = __byte_perm(w[0], 0, 0x0123), lo = __byte_perm(w[1], 0, 0x0123);
  return __funnelshift_l(lo, hi, pos & 31);
}

// one Huffman symbol and its extra bits at ``pos``: returns the symbol (or -1 for an invalid code), advances pos past
// both and sets ``val`` to the extended value of the extra bits (the low 4 bits of the symbol give their count)
__device__ __forceinline__ int huff_symbol(const HuffTab& t, const uint8_t* __restrict__ ecs, int& pos, int& val) {
  const uint32_t v = peek32(ecs, pos);
  const int e = t.fast[v >> 23];
  int len, sym;
  if (e) {
    len = e >> 8, sym = e & 255;
  } else {
    len = 10;
    while (len <= 16 && (int)(v >> (32 - len)) > t.maxcode[len]) ++len;
    if (len > 16) return -1;
    sym = t.vals[((int)(v >> (32 - len)) + t.valoff[len]) & 255];
  }
  const int s = sym & 15;
  val = 0;
  if (s) {
    const int bits = (int)((v << len) >> (32 - s));
    val = bits < (1 << (s - 1)) ? bits - (1 << s) + 1 : bits;
  }
  pos += len + s;
  return sym;
}

// Decode from state (pos, blk, z) until pos reaches ``stop_bit`` at a symbol boundary or, at a block boundary, ``g``
// reaches ``g_end`` (g = index of the next block to start).  dc0..dc2 accumulate component c's DC differences onto their start
// values.  WRITE stores every coefficient position the decode covers (zigzag order) and returns false on an invalid code,
// a coefficient index past 63 or a read past ``limit_bit``.  Without WRITE the start state may be a guess: an invalid code
// steps over one bit and an index past 63 ends the block, so that the decode keeps going until it resynchronises (the
// exact chain from subsequence 0 is checked by the WRITE pass); it fails only on a read past ``limit_bit``.
template <bool WRITE>
__device__ bool decode_run(const Tabs& T, int bpm, const uint8_t* __restrict__ ecs, int& pos, int& blk, int& z, int stop_bit,
                           int limit_bit, int& g, int g_end, int& dc0, int& dc1, int& dc2,
                           int16_t* __restrict__ coef) {
  int16_t* cb = WRITE && z > 0 ? coef + (size_t)(g - 1) * 64 : nullptr;
  while (pos < stop_bit) {
    const int c = T.comp_of[blk];
    int val;
    if (z == 0) {
      if (g >= g_end) return true;
      if (huff_symbol(T.dc[c], ecs, pos, val) < 0) {
        if (WRITE) return false;
        ++pos;                                     // a guessed state: step over the bit and keep resynchronising
        continue;
      }
      const int d = (c == 0 ? dc0 : c == 1 ? dc1 : dc2) + val;
      if (c == 0) dc0 = d; else if (c == 1) dc1 = d; else dc2 = d;
      if constexpr (WRITE) {
        cb = coef + (size_t)g * 64;
        cb[0] = (int16_t)d;
      }
      ++g;
      z = 1;
    } else {
      const int rs = huff_symbol(T.ac[c], ecs, pos, val);
      if (rs < 0) {
        if (WRITE) return false;
        ++pos;
        continue;
      }
      const int r = rs >> 4, s = rs & 15;
      int zn;
      if (s) {
        if (z + r > 63) {
          if (WRITE) return false;
          zn = 64;
        } else {
          zn = z + r + 1;
        }
      } else {
        zn = r == 15 ? min(z + 16, 64) : 64;
      }
      if constexpr (WRITE) {
        const int zeros_end = s ? z + r : zn;
        for (int k = z; k < zeros_end; ++k) cb[k] = 0;
        if (s) cb[z + r] = (int16_t)val;
      }
      z = zn;
      if (z == 64) z = 0, blk = blk + 1 == bpm ? 0 : blk + 1;
    }
    if (pos > limit_bit) return false;
  }
  return true;
}

__device__ __forceinline__ void load_tabs(Tabs& T, const JpegImage* im) {
  const int n_words = (int)(sizeof(HuffTab) / 4);
  for (int c = 0; c < 3; ++c) {
    const uint32_t* sd = reinterpret_cast<const uint32_t*>(&im->dc[im->comp_dc[c]]);
    const uint32_t* sa = reinterpret_cast<const uint32_t*>(&im->ac[im->comp_ac[c]]);
    uint32_t* dd = reinterpret_cast<uint32_t*>(&T.dc[c]);
    uint32_t* da = reinterpret_cast<uint32_t*>(&T.ac[c]);
    for (int k = threadIdx.x; k < n_words; k += blockDim.x) dd[k] = sd[k], da[k] = sa[k];
  }
  if (threadIdx.x < 6) {
    const int nl = im->h0 * im->v0;
    T.comp_of[threadIdx.x] = threadIdx.x < nl ? 0 : threadIdx.x - nl + 1;
  }
}

__device__ __forceinline__ void flag_data_error(JpegImage* im) { atomicCAS(&im->status, SY_JPEG_OK, SY_JPEG_EDATA); }

__global__ void __cluster_dims__(kClusterCtas, 1, 1) __launch_bounds__(kHuffThreads)
    jpeg_huffman_kernel(uint8_t* ws, Layout L) {
  __shared__ Tabs T;
  __shared__ int2 s_end[kHuffThreads];             // end state (pos, blk << 8 | z) of each of this CTA's subsequences
  __shared__ int s_changed[3];
  __shared__ int s_tot[5];                         // this CTA's totals: blocks, DC sums of the 3 components, spare
  using Scan = cub::BlockScan<int, kHuffThreads>;
  __shared__ typename Scan::TempStorage tmp;
  cg::cluster_group cluster = cg::this_cluster();
  const int img = blockIdx.y, rank = (int)cluster.block_rank(), t = threadIdx.x;
  JpegImage* im = image_of(ws, L, img);
  const uint8_t* ecs = ws + L.image_stride * img + L.off_ecs;
  const int32_t* seg = reinterpret_cast<const int32_t*>(ws + L.image_stride * img + L.off_seg);
  int16_t* coef = reinterpret_cast<int16_t*>(ws + L.image_stride * img + L.off_coef);
  if (im->status != SY_JPEG_OK) return;            // uniform over the cluster
  load_tabs(T, im);
  if (t < 3) s_changed[t] = 0;
  __syncthreads();
  const int bpm = im->bpm, total = im->total_blocks, n_units = im->n_units, bits = im->ecs_bits;
  if (im->ri > 0) {
    // restart intervals: every interval starts at a known byte with zero DC predictions
    const int per = im->ri * bpm;
    for (int u = rank * kHuffThreads + t; u < n_units; u += kMaxSubseq) {
      int pos = 8 * seg[u], blk = 0, z = 0, g = u * per, d0 = 0, d1 = 0, d2 = 0;
      const int limit = u + 1 < n_units ? 8 * seg[u + 1] : bits;
      const int g_end = min(g + per, total);
      if (!decode_run<true>(T, bpm, ecs, pos, blk, z, INT_MAX, limit, g, g_end, d0, d1, d2, coef) || g != g_end) flag_data_error(im);
      else if (g_end == total) im->done = 1;
    }
    return;
  }
  const int u = rank * kHuffThreads + t, ub = im->unit_bits;
  const bool active = u < n_units;
  int pos = u * ub, blk = 0, z = 0;                // start state: exact for u = 0, a guess for the others
  int nblk = 0, s0 = 0, s1 = 0, s2 = 0;          // blocks started and DC difference sums
  for (int it = 0;; ++it) {
    if (active && pos != kErrPos) {
      int p = pos, b = blk, zz = z, g = 0;
      s0 = s1 = s2 = 0;
      const bool ok = decode_run<false>(T, bpm, ecs, p, b, zz, min((u + 1) * ub, bits), bits, g, INT_MAX, s0, s1, s2, nullptr);
      nblk = g;
      s_end[t] = ok ? make_int2(p, (b << 8) | zz) : make_int2(kErrPos, 0);
    } else {
      nblk = s0 = s1 = s2 = 0;
      s_end[t] = make_int2(kErrPos, 0);
    }
    cluster.sync();
    int changed = 0;
    if (active && u > 0) {
      const int2* prev = t > 0 ? &s_end[t - 1] : cluster.map_shared_rank(&s_end[kHuffThreads - 1], rank - 1);
      const int2 e = *prev;
      const int nb = e.y >> 8, nz = e.y & 255;
      if (e.x != pos || (e.x != kErrPos && (nb != blk || nz != z))) changed = 1;
      pos = e.x, blk = nb, z = nz;
    }
    if (__syncthreads_or(changed) && t == 0) atomicOr(cluster.map_shared_rank(&s_changed[it % 3], 0), 1);
    cluster.sync();
    const int any = *cluster.map_shared_rank(&s_changed[it % 3], 0);
    if (rank == 0 && t == 0) s_changed[(it + 2) % 3] = 0;
    if (!any) break;
  }
  // every start state now is the sequential decode's: exclusive prefix sums over the cluster of the block counts and DC
  // differences give each subsequence its first block index and DC predictions
  int v[4] = {nblk, s0, s1, s2}, pre[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int agg;
    Scan(tmp).ExclusiveSum(v[k], pre[k], agg);
    __syncthreads();
    if (t == 0) s_tot[k] = agg;
  }
  cluster.sync();
  for (int r = 0; r < rank; ++r) {
    const int* o = cluster.map_shared_rank(s_tot, r);
#pragma unroll
    for (int k = 0; k < 4; ++k) pre[k] += o[k];
  }
  cluster.sync();                                  // no CTA leaves while others still read its shared memory
  // A failed predecessor reports its own failure when it lies before the last block.  A subsequence that starts past
  // the last block holds only the stream's padding.
  if (!active || pos == kErrPos || pre[0] > total) return;
  int g = pre[0];
  if (z > 0 && g == 0) return flag_data_error(im);
  if (!decode_run<true>(T, bpm, ecs, pos, blk, z, min((u + 1) * ub, bits), bits, g, total, pre[1], pre[2], pre[3], coef))
    flag_data_error(im);
  else if (g == total && z == 0) im->done = 1;
}

// ------------------------------------------------------------------------------------------------------------------
// 4. dequantise + islow IDCT into the component planes

constexpr int kF0298 = 2446, kF0390 = 3196, kF0541 = 4433, kF0765 = 6270, kF0899 = 7373, kF1175 = 9633, kF1501 = 12299,
              kF1847 = 15137, kF1961 = 16069, kF2053 = 16819, kF2562 = 20995, kF3072 = 25172;

// one 8-point pass of jidctint.c (int32 as libjpeg's JLONG holds these values) with the final descale
__device__ __forceinline__ void idct8(const int (&s)[8], int shift, int (&o)[8]) {
  int z2 = s[2], z3 = s[6];
  int z1 = (z2 + z3) * kF0541;
  const int tmp2a = z1 - z3 * kF1847, tmp3a = z1 + z2 * kF0765;
  const int tmp0a = (s[0] + s[4]) * 8192, tmp1a = (s[0] - s[4]) * 8192;
  const int t10 = tmp0a + tmp3a, t13 = tmp0a - tmp3a, t11 = tmp1a + tmp2a, t12 = tmp1a - tmp2a;
  int t0 = s[7], t1 = s[5], t2 = s[3], t3 = s[1];
  z1 = t0 + t3, z2 = t1 + t2, z3 = t0 + t2;
  int z4 = t1 + t3;
  const int z5 = (z3 + z4) * kF1175;
  t0 *= kF0298, t1 *= kF2053, t2 *= kF3072, t3 *= kF1501;
  z1 *= -kF0899, z2 *= -kF2562, z3 = z3 * -kF1961 + z5, z4 = z4 * -kF0390 + z5;
  t0 += z1 + z3, t1 += z2 + z4, t2 += z2 + z3, t3 += z1 + z4;
  const int rnd = 1 << (shift - 1);
  o[0] = (t10 + t3 + rnd) >> shift, o[7] = (t10 - t3 + rnd) >> shift;
  o[1] = (t11 + t2 + rnd) >> shift, o[6] = (t11 - t2 + rnd) >> shift;
  o[2] = (t12 + t1 + rnd) >> shift, o[5] = (t12 - t1 + rnd) >> shift;
  o[3] = (t13 + t0 + rnd) >> shift, o[4] = (t13 - t0 + rnd) >> shift;
}

__device__ __forceinline__ uint32_t range_limit(int x) {  // jdmaster.c's IDCT range-limit table
  return (uint32_t)min(max(((x + 512) & 1023) - 512 + 128, 0), 255);
}

__global__ void __launch_bounds__(8 * kIdctBlocksPerCta) jpeg_idct_kernel(uint8_t* ws, Layout L) {
  __shared__ int16_t s_coef[kIdctBlocksPerCta][64];
  __shared__ int s_ws[kIdctBlocksPerCta][64];
  const int img = blockIdx.y;
  JpegImage* im = image_of(ws, L, img);
  if (im->status != SY_JPEG_OK) return;
  if (!im->done) {                                 // the entropy decode did not reach the last block
    if (blockIdx.x == 0 && threadIdx.x == 0) flag_data_error(im);
    return;
  }
  const int total = im->total_blocks;
  const int lb = threadIdx.x >> 3, j = threadIdx.x & 7;
  const int blkid = blockIdx.x * kIdctBlocksPerCta + lb;
  if (blockIdx.x * kIdctBlocksPerCta >= total) return;
  const bool live = blkid < total;
  const int16_t* coef = reinterpret_cast<const int16_t*>(ws + L.image_stride * img + L.off_coef);
  if (live) reinterpret_cast<uint4*>(s_coef[lb])[j] = reinterpret_cast<const uint4*>(coef + (size_t)blkid * 64)[j];
  __syncwarp();
  const int bpm = im->bpm, h0 = im->h0, v0 = im->v0, mcux = im->mcux;
  const int mcu = blkid / bpm, k = blkid - mcu * bpm, nl = h0 * v0;
  const int comp = k < nl ? 0 : k - nl + 1;
  const uint16_t* q = im->q[im->comp_q[comp]];
  // pass 1: column j (CONST_BITS - PASS1_BITS descale)
  int s[8], o[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int nat = r * 8 + j;
    s[r] = live ? (int)s_coef[lb][kUnzig[nat]] * (int)q[nat] : 0;
  }
  idct8(s, 11, o);
#pragma unroll
  for (int r = 0; r < 8; ++r) s_ws[lb][r * 8 + j] = o[r];
  __syncwarp();
  // pass 2: row j (CONST_BITS + PASS1_BITS + 3 descale), range-limited
#pragma unroll
  for (int c = 0; c < 8; ++c) s[c] = s_ws[lb][j * 8 + c];
  idct8(s, 18, o);
  if (!live) return;
  const int my = mcu / mcux, mx = mcu - my * mcux;
  uint8_t* planes = ws + L.image_stride * img + L.off_planes;
  const int yw = mcux * h0 * 8, yh = im->mcuy * v0 * 8, cw = mcux * 8, chh = im->mcuy * 8;
  uint8_t* dst;
  if (comp == 0) {
    const int by = my * v0 + k / h0, bx = mx * h0 + k % h0;
    dst = planes + (size_t)(by * 8 + j) * yw + bx * 8;
  } else {
    dst = planes + (size_t)yw * yh + (size_t)(comp - 1) * cw * chh + (size_t)(my * 8 + j) * cw + mx * 8;
  }
  uint2 px;
  px.x = range_limit(o[0]) | range_limit(o[1]) << 8 | range_limit(o[2]) << 16 | range_limit(o[3]) << 24;
  px.y = range_limit(o[4]) | range_limit(o[5]) << 8 | range_limit(o[6]) << 16 | range_limit(o[7]) << 24;
  *reinterpret_cast<uint2*>(dst) = px;
}

// ------------------------------------------------------------------------------------------------------------------
// 5. chroma upsampling + YCbCr -> BGR

// chroma sample of output pixel (y, x) from a plane of pitch cw (jdsample.c)
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ p, int cw, int y, int x, int h, int w, int h0, int v0) {
  if (h0 == 1) return p[(size_t)y * cw + x];
  const int dw = (w + 1) >> 1, c = x >> 1;
  const int r = v0 == 2 ? y >> 1 : y;
  if (dw <= 2) return p[(size_t)r * cw + c];       // plain replication
  const bool odd = x & 1;
  const int cf = odd ? min(c + 1, dw - 1) : max(c - 1, 0);
  if (v0 == 1) {
    const uint8_t* row = p + (size_t)r * cw;
    return (3 * row[c] + row[cf] + (odd ? 2 : 1)) >> 2;
  }
  const int dh = (h + 1) >> 1;
  const int rf = (y & 1) ? min(r + 1, dh - 1) : max(r - 1, 0);
  const uint8_t* rn = p + (size_t)r * cw;
  const uint8_t* rr = p + (size_t)rf * cw;
  const int near = 3 * rn[c] + rr[c], far = 3 * rn[cf] + rr[cf];
  return (3 * near + far + (odd ? 7 : 8)) >> 4;
}

// out: slots of slot_h x slot_w pixels, image img top-left in slot img
__global__ void __launch_bounds__(128) jpeg_color_kernel(uint8_t* ws, Layout L, int slot_h, int slot_w,
                                                          uint8_t* __restrict__ out, int32_t* __restrict__ status) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, img = blockIdx.z;
  const JpegImage* im = image_of(ws, L, img);
  if (x == 0 && y == 0) status[img] = im->status;
  if (im->status != SY_JPEG_OK) return;
  const int h = im->h, w = im->w;
  if (x >= w || y >= h) return;
  const int h0 = im->h0, v0 = im->v0, mcux = im->mcux;
  const uint8_t* planes = ws + L.image_stride * img + L.off_planes;
  const int yw = mcux * h0 * 8, yh = im->mcuy * v0 * 8, cw = mcux * 8, chh = im->mcuy * 8;
  const int Y = planes[(size_t)y * yw + x];
  const uint8_t* cbp = planes + (size_t)yw * yh;
  const int cb = chroma(cbp, cw, y, x, h, w, h0, v0) - 128;
  const int cr = chroma(cbp + (size_t)cw * chh, cw, y, x, h, w, h0, v0) - 128;
  const int R = Y + ((91881 * cr + 32768) >> 16);
  const int G = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int B = Y + ((116130 * cb + 32768) >> 16);
  uint8_t* o = out + (((size_t)img * slot_h + y) * slot_w + x) * 3;
  o[0] = (uint8_t)min(max(B, 0), 255);
  o[1] = (uint8_t)min(max(G, 0), 255);
  o[2] = (uint8_t)min(max(R, 0), 255);
}

// workspace layout for frames of h x w of any supported sampling (4:4:4 needs the most of everything)
Layout make_layout(int64_t max_bytes, int h, int w) {
  Layout L;
  const size_t b8y = (size_t)cdiv(h, 8), b8x = (size_t)cdiv(w, 8), b16y = (size_t)cdiv(h, 16), b16x = (size_t)cdiv(w, 16);
  const size_t blocks = std::max(std::max(3 * b8y * b8x, 4 * b8y * b16x), 6 * b16y * b16x);
  const size_t plane_bytes = std::max(std::max(3 * b8y * b8x, 4 * b8y * b16x), 6 * b16y * b16x) * 64;
  L.max_units = (int32_t)std::max<size_t>(kMaxSubseq, b8y * b8x);
  size_t off = align256(sizeof(JpegImage));
  L.off_ecs = off;
  off = align256(off + (size_t)max_bytes + 16);
  L.off_seg = off;
  off = align256(off + 4 * ((size_t)L.max_units + 1));
  L.off_coef = off;
  off = align256(off + blocks * 128);
  L.off_planes = off;
  off = align256(off + plane_bytes);
  L.image_stride = off;
  return L;
}

// the five kernels over n images in slots of h x w (sizes: each image's own size, or NULL for h x w)
int jpeg_launch(const uint8_t* bytes, const int32_t* lengths, int n, int64_t max_bytes, int h, int w, const int32_t* sizes,
                uint8_t* out, int32_t* status, void* workspace, cudaStream_t stream) {
  const Layout L = make_layout(max_bytes, h, w);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  jpeg_parse_kernel<<<n, 32, 0, stream>>>(bytes, lengths, max_bytes, h, w, sizes, ws, L);
  SY_CUDA(cudaGetLastError());
  jpeg_ecs_kernel<<<n, kEcsThreads, 0, stream>>>(bytes, lengths, max_bytes, ws, L);
  SY_CUDA(cudaGetLastError());
  jpeg_huffman_kernel<<<dim3(kClusterCtas, n), kHuffThreads, 0, stream>>>(ws, L);
  SY_CUDA(cudaGetLastError());
  const int max_blocks = (int)((L.off_planes - L.off_coef) / 128);
  jpeg_idct_kernel<<<dim3(cdiv(max_blocks, kIdctBlocksPerCta), n), 8 * kIdctBlocksPerCta, 0, stream>>>(ws, L);
  SY_CUDA(cudaGetLastError());
  jpeg_color_kernel<<<dim3(cdiv(w, 128), h, n), 128, 0, stream>>>(ws, L, h, w, out, status);
  return launch_status("jpeg_color_kernel");
}

}  // namespace
}  // namespace sy

using namespace sy;

extern "C" size_t sy_jpeg_decode_workspace_bytes(int32_t n, int64_t max_bytes, int32_t h, int32_t w) {
  if (n <= 0 || max_bytes <= 0 || max_bytes > (1ll << 28) || h <= 0 || w <= 0 || h > 65535 || w > 65535) return 0;
  return make_layout(max_bytes, h, w).image_stride * (size_t)n;
}

extern "C" int sy_jpeg_decode(const SyJpegDecodeDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->bytes != nullptr && d->lengths != nullptr && d->out != nullptr && d->status != nullptr &&
                 d->workspace != nullptr, SY_EINVAL, "jpeg_decode: null pointer");
  SY_REQUIRE(d->n > 0 && d->n <= 65535 && d->max_bytes > 0 && d->max_bytes <= (1ll << 28) && d->h > 0 && d->w > 0 &&
                 d->h <= 65535 && d->w <= 65535, SY_EINVAL, "jpeg_decode: bad sizes (n %d, max_bytes %lld, %dx%d)", d->n,
             (long long)d->max_bytes, d->h, d->w);
  const size_t need = sy_jpeg_decode_workspace_bytes(d->n, d->max_bytes, d->h, d->w);
  SY_REQUIRE(d->workspace_bytes >= need && ((uintptr_t)d->workspace % 256) == 0, SY_EINVAL,
             "jpeg_decode: workspace of %zu bytes (need %zu, 256-byte aligned)", d->workspace_bytes, need);
  return jpeg_launch(d->bytes, d->lengths, d->n, d->max_bytes, d->h, d->w, nullptr, d->out, d->status, d->workspace, stream);
}

extern "C" size_t sy_jpeg_decode_sized_workspace_bytes(int32_t n, int64_t max_bytes, int32_t max_h, int32_t max_w) {
  return sy_jpeg_decode_workspace_bytes(n, max_bytes, max_h, max_w);
}

extern "C" int sy_jpeg_decode_sized(const SyJpegDecodeSizedDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr && d->bytes != nullptr && d->lengths != nullptr && d->sizes != nullptr && d->out != nullptr &&
                 d->status != nullptr && d->workspace != nullptr, SY_EINVAL, "jpeg_decode_sized: null pointer");
  SY_REQUIRE(d->n > 0 && d->n <= 65535 && d->max_bytes > 0 && d->max_bytes <= (1ll << 28) && d->max_h > 0 &&
                 d->max_w > 0 && d->max_h <= 65535 && d->max_w <= 65535, SY_EINVAL,
             "jpeg_decode_sized: bad sizes (n %d, max_bytes %lld, slot %dx%d)", d->n, (long long)d->max_bytes, d->max_h,
             d->max_w);
  const size_t need = sy_jpeg_decode_sized_workspace_bytes(d->n, d->max_bytes, d->max_h, d->max_w);
  SY_REQUIRE(d->workspace_bytes >= need && ((uintptr_t)d->workspace % 256) == 0, SY_EINVAL,
             "jpeg_decode_sized: workspace of %zu bytes (need %zu, 256-byte aligned)", d->workspace_bytes, need);
  return jpeg_launch(d->bytes, d->lengths, d->n, d->max_bytes, d->max_h, d->max_w, d->sizes, d->out, d->status,
                     d->workspace, stream);
}
