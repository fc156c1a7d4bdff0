"""numpy restatement of the device JPEG encoder (streamyolo_b200/csrc/jpeg_encode.cu): the bytes
cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q]) returns for a uint8 BGR image, with cv2's defaults.

Test infrastructure only.  libjpeg-turbo's default compression, stage by stage: the quality-scaled Annex K tables
(jcparam.c jpeg_quality_scaling, clamped to 1..255 for baseline), the fixed-point RGB -> YCbCr of jccolor.c, edge
replication and the h2v2 downsample of jcsample.c (bias 1, 2, 1, 2, ... along each row), the integer "islow" forward DCT of
jfdctint.c, quantisation by 8 * qtable with rounding (jcdctmgr.c), the dummy blocks of partial MCUs (jccoefct.c) and the
standard Huffman tables of jchuff.c; baseline SOF0, 4:2:0, no restart interval, JFIF 1.01 APP0 with density 1:1.
tests/test_jpeg_encode.py pins it to cv2.imencode byte for byte.
"""
import numpy as np

from oracle.jpeg_oracle import ZIGZAG

# Annex K.1 (jcparam.c std_luminance_quant_tbl / std_chrominance_quant_tbl), natural order
STD_QUANT = (np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                       14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                       49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99]),
             np.array([17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
                       47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32))

# Annex K.3 (jstdhuff.c): (counts of codes of length 1..16, symbols) of the DC / AC tables, luminance then chrominance
STD_HUFF = {
    "dc0": ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12))),
    "dc1": ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12))),
    "ac0": ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [
        0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
        0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
        0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
        0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
        0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
        0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
        0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
        0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
        0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa]),
    "ac1": ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
        0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
        0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
        0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
        0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
        0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
        0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
        0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
        0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
        0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa]),
}

# the longest code any block can take: the longest DC code (11 bits, chrominance) and its 11 magnitude bits, then 63 AC
# coefficients each with the longest AC code (16 bits) and 10 magnitude bits; a ZRL (at most 11 bits) stands for 16 zero
# coefficients and an EOB only follows a zero, so neither makes a block longer
MAX_BLOCK_BITS = 11 + 11 + 63 * (16 + 10)


def quant_tables(quality):
    """jpeg_set_quality(quality, force_baseline=TRUE): the two tables, natural order, int64 [2, 64]"""
    if not 1 <= quality <= 100:
        raise ValueError(f"quality {quality} not in 1..100")
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.stack([np.clip((t * scale + 50) // 100, 1, 255) for t in STD_QUANT])


def huff_codes(counts, symbols):
    """jchuff.c jpeg_make_c_derived_tbl: symbol -> (code, length)"""
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            out[symbols[k]] = (code, ln)
            code += 1
            k += 1
        code <<= 1
    return out


HUFF = {k: huff_codes(*v) for k, v in STD_HUFF.items()}


def header(h, w, quality):
    """SOI, APP0 (JFIF 1.01, density 1:1), DQT x 2 (zigzag, 8-bit), SOF0 (4:2:0), DHT x 4, SOS: the bytes before the
    entropy-coded data"""
    seg = lambda m, body: bytes([0xFF, m]) + (len(body) + 2).to_bytes(2, "big") + body
    qt = quant_tables(quality)
    out = b"\xff\xd8" + seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for k in (0, 1):
        out += seg(0xDB, bytes([k]) + bytes(qt[k][ZIGZAG].astype(np.uint8)))
    out += seg(0xC0, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for cls, name in ((0x00, "dc0"), (0x10, "ac0"), (0x01, "dc1"), (0x11, "ac1")):
        counts, symbols = STD_HUFF[name]
        out += seg(0xC4, bytes([cls]) + bytes(counts) + bytes(symbols))
    return out + seg(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))


HEADER_BYTES = len(header(1, 1, 50))


def max_bytes(h, w):
    """a bound on the file's length for any h x w content and any quality: every block at MAX_BLOCK_BITS, every entropy
    byte followed by a stuffed zero, the headers and EOI"""
    blocks = 6 * -(-h // 16) * -(-w // 16)
    return HEADER_BYTES + 2 * -(-blocks * MAX_BLOCK_BITS // 8) + 2


def rgb_to_ycc(img):
    """jccolor.c rgb_ycc_convert (SCALEBITS = 16) of uint8 BGR [h, w, 3] -> int64 Y, Cb, Cr planes"""
    b, g, r = (img[..., k].astype(np.int64) for k in range(3))
    half, off = 1 << 15, 128 << 16
    y = (19595 * r + 38470 * g + 7471 * b + half) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + off + half - 1) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + off + half - 1) >> 16
    return y, cb, cr


def planes(img):
    """the three component planes at the MCU grid: Y [16 my, 16 mx] and Cb, Cr [8 my, 8 mx], edge-expanded as
    jcprepct.c / jcsample.c do (the padded-out parts of Y beyond its whole blocks are never coded: dummy blocks)"""
    h, w = img.shape[:2]
    my, mx = -(-h // 16), -(-w // 16)
    y, cb, cr = rgb_to_ycc(img)
    rows, cols = np.minimum(np.arange(16 * my), h - 1), np.minimum(np.arange(16 * mx), w - 1)
    yp = y[rows[:, None], cols[None, :]]
    # h2v2_downsample over the row pairs of the (even-padded) image, then the last output row repeated to the MCU height
    r = np.minimum(np.arange(8 * my), -(-h // 2) - 1)
    r0, r1 = np.minimum(2 * r, h - 1), np.minimum(2 * r + 1, h - 1)
    c0, c1 = cols[0::2], cols[1::2]
    bias = np.where(np.arange(8 * mx) & 1, 2, 1)

    def down(p):
        s = p[r0[:, None], c0] + p[r0[:, None], c1] + p[r1[:, None], c0] + p[r1[:, None], c1]
        return (s + bias) >> 2

    return yp, down(cb), down(cr)


_C = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
          f1961=16069, f2053=16819, f2562=20995, f3072=25172)


def _fdct_1d(d, pass1):
    """jfdctint.c jpeg_fdct_islow, one pass over axis -1 of int64 [.., 8] (CONST_BITS 13, PASS1_BITS 2)"""
    f = _C
    tmp0, tmp7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    tmp1, tmp6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    tmp2, tmp5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    tmp3, tmp4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    sh = 11 if pass1 else 15                                        # CONST_BITS -/+ PASS1_BITS
    desc = lambda x, n: (x + (1 << (n - 1))) >> n
    out = [None] * 8
    if pass1:
        out[0], out[4] = (tmp10 + tmp11) << 2, (tmp10 - tmp11) << 2
    else:
        out[0], out[4] = desc(tmp10 + tmp11, 2), desc(tmp10 - tmp11, 2)
    z1 = (tmp12 + tmp13) * f["f0541"]
    out[2] = desc(z1 + tmp13 * f["f0765"], sh)
    out[6] = desc(z1 - tmp12 * f["f1847"], sh)
    z1, z2, z3, z4 = tmp4 + tmp7, tmp5 + tmp6, tmp4 + tmp6, tmp5 + tmp7
    z5 = (z3 + z4) * f["f1175"]
    tmp4, tmp5, tmp6, tmp7 = tmp4 * f["f0298"], tmp5 * f["f2053"], tmp6 * f["f3072"], tmp7 * f["f1501"]
    z1, z2 = z1 * -f["f0899"], z2 * -f["f2562"]
    z3, z4 = z3 * -f["f1961"] + z5, z4 * -f["f0390"] + z5
    out[7], out[5] = desc(tmp4 + z1 + z3, sh), desc(tmp5 + z2 + z4, sh)
    out[3], out[1] = desc(tmp6 + z2 + z3, sh), desc(tmp7 + z1 + z4, sh)
    return np.stack(out, axis=-1)


def fdct_quant(blocks, qt):
    """uint8-range samples [n, 8, 8] -> quantised coefficients [n, 64] in zigzag order: islow FDCT of samples - 128, then
    each coefficient divided by 8 * qtable rounding half away from zero (jcdctmgr.c quantize)"""
    d = _fdct_1d(blocks.astype(np.int64) - 128, True)               # rows
    d = _fdct_1d(d.transpose(0, 2, 1), False).transpose(0, 2, 1)    # columns
    div = (8 * qt)[None, :]
    d = d.reshape(-1, 64)
    q = np.sign(d) * ((np.abs(d) + div // 2) // div)
    return q[:, ZIGZAG]


def coefficients(img, quality):
    """-> int64 [6 * mcus, 64] zigzag coefficients in MCU interleave order (Y0 Y1 Y2 Y3 Cb Cr per MCU), dummy blocks
    already holding the DC of the block before them and no AC"""
    h, w = img.shape[:2]
    my, mx = -(-h // 16), -(-w // 16)
    qt = quant_tables(quality)
    yp, cb, cr = planes(img)
    yb = fdct_quant(yp.reshape(2 * my, 8, 2 * mx, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8), qt[0]).reshape(my, 2, mx, 2, 64)
    cbb = fdct_quant(cb.reshape(my, 8, mx, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8), qt[1]).reshape(my, mx, 64)
    crb = fdct_quant(cr.reshape(my, 8, mx, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8), qt[1]).reshape(my, mx, 64)
    out = np.zeros((my, mx, 6, 64), np.int64)
    out[:, :, :4] = yb.transpose(0, 2, 1, 3, 4).reshape(my, mx, 4, 64)
    out[:, :, 4], out[:, :, 5] = cbb, crb
    # jccoefct.c compress_data: Y blocks past the image's ceil(w / 8) x ceil(h / 8) blocks are dummies
    by, bx = -(-h // 8), -(-w // 8)
    for j in range(1, 4):
        yy = 2 * np.arange(my)[:, None] + (j >> 1)
        xx = 2 * np.arange(mx)[None, :] + (j & 1)
        dummy = (yy >= by) | (xx >= bx)
        out[:, :, j][dummy] = 0
        out[:, :, j, 0] = np.where(dummy, out[:, :, j - 1, 0], out[:, :, j, 0])
    return out.reshape(-1, 64)


def _category(v):
    return int(abs(int(v))).bit_length()


def block_codes(coef, prev_dc, comp):
    """jchuff.c encode_one_block: the (code, length) pieces of one block, DC difference first"""
    dc, ac = HUFF["dc0" if comp == 0 else "dc1"], HUFF["ac0" if comp == 0 else "ac1"]
    out = []
    diff = int(coef[0]) - prev_dc
    s = _category(diff)
    out.append(dc[s])
    if s:
        out.append(((diff if diff >= 0 else diff - 1) & ((1 << s) - 1), s))
    run = 0
    for k in range(1, 64):
        v = int(coef[k])
        if v == 0:
            run += 1
            continue
        while run > 15:
            out.append(ac[0xF0])
            run -= 16
        s = _category(v)
        out.append(ac[(run << 4) | s])
        out.append(((v if v >= 0 else v - 1) & ((1 << s) - 1), s))
        run = 0
    if run:
        out.append(ac[0x00])
    return out


def entropy_bits(coef):
    """the scan's bits, a str of '0' / '1', for the blocks of ``coefficients``"""
    out = []
    pred = [0, 0, 0]
    comp_of = (0, 0, 0, 0, 1, 2)
    for b in range(coef.shape[0]):
        c = comp_of[b % 6]
        out.extend(format(code, f"0{ln}b") for code, ln in block_codes(coef[b], pred[c], c))
        pred[c] = int(coef[b, 0])
    return "".join(out)


def block_bits(coef):
    """the coded length in bits of every block of ``coefficients`` (the device's per-block lengths)"""
    pred = [0, 0, 0]
    comp_of = (0, 0, 0, 0, 1, 2)
    out = np.zeros(coef.shape[0], np.int64)
    for b in range(coef.shape[0]):
        c = comp_of[b % 6]
        out[b] = sum(ln for _, ln in block_codes(coef[b], pred[c], c))
        pred[c] = int(coef[b, 0])
    return out


def stuff(data):
    """a 00 byte after every FF"""
    return bytes(data).replace(b"\xff", b"\xff\x00")


def scan_bytes(img, quality):
    """the entropy-coded segment: the bits padded with 1s to a byte boundary, then byte-stuffed"""
    bits = entropy_bits(coefficients(img, quality))
    bits += "1" * (-len(bits) % 8)
    return stuff(np.packbits(np.frombuffer(bits.encode(), np.uint8) - 48).tobytes())


def encode(img, quality=95):
    """-> the bytes cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, quality]) gives for uint8 BGR [h, w, 3]"""
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3 or min(img.shape[:2]) < 1:
        raise ValueError(f"encode: img must be uint8 [h, w, 3] with h, w >= 1, not {img.dtype} {list(img.shape)}")
    h, w = img.shape[:2]
    if h > 65535 or w > 65535:
        raise ValueError(f"encode: {h}x{w} is larger than JPEG's 65535 x 65535")
    return header(h, w, quality) + scan_bytes(img, quality) + b"\xff\xd9"
