"""numpy restatement of the device JPEG decoder (streamyolo_b200/csrc/jpeg.cu): what cv2.imdecode(bytes, IMREAD_COLOR)
returns for the streams the device decodes, and the status code it gives the others.

Test infrastructure only.  The pixel stage is libjpeg-turbo's default decompression as cv2 4.x runs it: the integer "islow"
IDCT (jidctint.c) with its range-limit table, the "fancy" triangle-filter chroma upsampler (jdsample.c; plain replication
when the downsampled width is at most 2) and the fixed-point YCbCr -> RGB tables of jdcolor.c.  tests/test_jpeg_decode.py
pins it to cv2.imdecode bit for bit.
"""
import numpy as np

# per-image status codes (SY_JPEG_* in include/streamyolo_sm100.h)
OK, EHEADER, EUNSUPPORTED, EORIENTATION, ESIZE, EDATA = 0, 1, 2, 3, 4, 5
STATUS_NAMES = {OK: "ok", EHEADER: "malformed or truncated header", EUNSUPPORTED: "unsupported JPEG variant",
                EORIENTATION: "EXIF orientation other than 1", ESIZE: "image size differs from the batch size",
                EDATA: "corrupt or truncated entropy-coded data"}

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])          # zigzag index -> natural (row-major) index


class JpegError(Exception):
    def __init__(self, status, msg):
        super().__init__(msg)
        self.status = status


def _u16(b, i):
    return (b[i] << 8) | b[i + 1]


def _exif_orientation(seg):
    """orientation tag of an APP1 payload, 1 when absent or unreadable"""
    if len(seg) < 14 or seg[:6] != b"Exif\x00\x00":
        return 1
    t = seg[6:]
    if t[:4] == b"II*\x00":
        rd = lambda i, n: int.from_bytes(t[i:i + n], "little")
    elif t[:4] == b"MM\x00*":
        rd = lambda i, n: int.from_bytes(t[i:i + n], "big")
    else:
        return 1
    ifd = rd(4, 4)
    if ifd + 2 > len(t):
        return 1
    for e in range(rd(ifd, 2)):
        p = ifd + 2 + 12 * e
        if p + 12 > len(t):
            return 1
        if rd(p, 2) == 0x0112:
            return rd(p + 8, 2) if rd(p + 2, 2) == 3 else 1
    return 1


def parse(data):
    """-> header dict of a stream the decoder takes; raises JpegError(status) otherwise"""
    b = bytes(data)
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise JpegError(EHEADER, "no SOI")
    q, dc, ac = {}, {}, {}
    sof, ri, jfif, adobe = None, 0, False, None
    i = 2
    while True:
        if i >= n or b[i] != 0xFF:
            raise JpegError(EHEADER, "marker expected")
        while i < n and b[i] == 0xFF:
            i += 1
        if i >= n:
            raise JpegError(EHEADER, "truncated")
        m = b[i]
        i += 1
        if m in (0xD8, 0x01) or 0xD0 <= m <= 0xD7 or m == 0xD9:
            raise JpegError(EHEADER, f"unexpected marker {m:#x}")
        if i + 2 > n:
            raise JpegError(EHEADER, "truncated")
        ln = _u16(b, i)
        if ln < 2 or i + ln > n:
            raise JpegError(EHEADER, "segment runs past the end")
        seg = b[i + 2:i + ln]
        i += ln
        if m in (0xC0, 0xC1):
            if sof is not None or len(seg) < 6:
                raise JpegError(EHEADER, "bad SOF")
            if seg[0] != 8:
                raise JpegError(EUNSUPPORTED, "precision")
            h, w, nc = _u16(seg, 1), _u16(seg, 3), seg[5]
            if nc != 3:
                raise JpegError(EUNSUPPORTED, "components")
            if len(seg) != 6 + 3 * nc:
                raise JpegError(EHEADER, "bad SOF")
            comps = [(seg[6 + 3 * k], seg[7 + 3 * k] >> 4, seg[7 + 3 * k] & 15, seg[8 + 3 * k]) for k in range(3)]
            if h == 0 or w == 0:
                raise JpegError(EUNSUPPORTED, "DNL height")
            if (comps[0][1], comps[0][2]) not in ((1, 1), (2, 1), (2, 2)) or any(c[1:3] != (1, 1) for c in comps[1:]):
                raise JpegError(EUNSUPPORTED, "sampling")
            if any(c[3] > 3 for c in comps):
                raise JpegError(EHEADER, "quant table id")
            sof = dict(h=h, w=w, comps=comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise JpegError(EUNSUPPORTED, f"SOF{m - 0xC0}")
        elif m == 0xCC:
            raise JpegError(EUNSUPPORTED, "arithmetic conditioning")
        elif m == 0xDB:
            p = 0
            while p < len(seg):
                pq, tq = seg[p] >> 4, seg[p] & 15
                sz = 64 * (pq + 1)
                if pq > 1 or tq > 3 or p + 1 + sz > len(seg):
                    raise JpegError(EHEADER, "bad DQT")
                v = np.frombuffer(seg[p + 1:p + 1 + sz], dtype=">u2" if pq else np.uint8).astype(np.int64)
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = v
                q[tq] = t
                p += 1 + sz
        elif m == 0xC4:
            p = 0
            while p < len(seg):
                if p + 17 > len(seg):
                    raise JpegError(EHEADER, "bad DHT")
                tc, th = seg[p] >> 4, seg[p] & 15
                counts = list(seg[p + 1:p + 17])
                tot = sum(counts)
                if tc > 1 or th > 3 or tot > 256 or p + 17 + tot > len(seg):
                    raise JpegError(EHEADER, "bad DHT")
                vals = list(seg[p + 17:p + 17 + tot])
                if tc == 0 and any(v > 15 for v in vals):
                    raise JpegError(EHEADER, "bad DC table")
                (dc if tc == 0 else ac)[th] = _huff_table(counts, vals)
                p += 17 + tot
        elif m == 0xDD:
            if len(seg) != 2:
                raise JpegError(EHEADER, "bad DRI")
            ri = _u16(seg, 0)
        elif m == 0xE0:
            jfif = jfif or seg[:5] == b"JFIF\x00"
        elif m == 0xE1:
            if _exif_orientation(seg) != 1:
                raise JpegError(EORIENTATION, "EXIF orientation")
        elif m == 0xEE:
            if seg[:5] == b"Adobe" and len(seg) >= 12:
                adobe = seg[11]
        elif m == 0xDA:
            if sof is None:
                raise JpegError(EHEADER, "SOS before SOF")
            ns = seg[0] if seg else 0
            if len(seg) != 4 + 2 * ns:
                raise JpegError(EHEADER, "bad SOS")
            if ns != 3:
                raise JpegError(EUNSUPPORTED, "multi-scan")
            ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if (ss, se, ahal) != (0, 63, 0):
                raise JpegError(EHEADER, "bad spectral selection")
            tabs = []
            for k in range(3):
                cid, t = seg[1 + 2 * k], seg[2 + 2 * k]
                if cid != sof["comps"][k][0]:
                    raise JpegError(EUNSUPPORTED, "scan component order")
                tabs.append((t >> 4, t & 15))
            cids = [c[0] for c in sof["comps"]]
            if adobe == 0 or (not jfif and adobe is None and cids == [82, 71, 66]):
                raise JpegError(EUNSUPPORTED, "RGB colour space")
            try:
                qt = [q[c[3]] for c in sof["comps"]]
                hd = [(dc[td], ac[ta]) for td, ta in tabs]
            except KeyError:
                raise JpegError(EHEADER, "undefined table") from None
            return dict(sof, ri=ri, q=qt, huff=hd, scan=i)
        # APPn, COM and anything else: skipped


def _huff_table(counts, vals):
    """{(length, code): symbol}; raises on an over-subscribed table"""
    t, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            if code >= (1 << ln):
                raise JpegError(EHEADER, "bad Huffman table")
            t[(ln, code)] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return t


def split_scan(b, begin):
    """entropy-coded segment from ``begin``: the destuffed bytes of each restart interval"""
    segs, cur = [], bytearray()
    i, n = begin, len(b)
    expect = 0
    while i < n:
        c = b[i]
        if c != 0xFF:
            cur.append(c)
            i += 1
            continue
        nx = b[i + 1] if i + 1 < n else None
        if nx == 0x00:
            cur.append(0xFF)
            i += 2
        elif nx == 0xFF:
            i += 1
        elif nx is not None and 0xD0 <= nx <= 0xD7:
            if nx - 0xD0 != expect % 8:
                raise JpegError(EDATA, "restart marker out of order")
            expect += 1
            segs.append(bytes(cur))
            cur = bytearray()
            i += 2
        else:
            break
    segs.append(bytes(cur))
    return segs


class _Bits:
    def __init__(self, data):
        self.d = bytes(data) + bytes(8)
        self.n = 8 * len(data)
        self.p = 0

    def _peek32(self):
        i = self.p >> 3
        return (int.from_bytes(self.d[i:i + 5], "big") >> (8 - (self.p & 7))) & 0xFFFFFFFF

    def get(self, k):
        if self.p + k > self.n:
            raise JpegError(EDATA, "out of data")
        r = self._peek32() >> (32 - k) if k else 0
        self.p += k
        return r

    def sym(self, t):
        v = self._peek32()
        for ln in range(1, 17):
            s = t.get((ln, v >> (32 - ln)))
            if s is not None:
                if self.p + ln > self.n:
                    raise JpegError(EDATA, "out of data")
                self.p += ln
                return s
        raise JpegError(EDATA, "bad Huffman code")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def entropy_decode(hd, segs):
    """-> quantised coefficients [blocks, 64] (natural order) in MCU order, and the MCU geometry"""
    (_, h0, v0, _), h, w = hd["comps"][0], hd["h"], hd["w"]
    mx, my = -(-w // (8 * h0)), -(-h // (8 * v0))
    comp_of = [0] * (h0 * v0) + [1, 2]
    total = mx * my
    ri = hd["ri"] or total
    if len(segs) != -(-total // ri):
        raise JpegError(EDATA, "restart interval count")
    coef = np.zeros((total * len(comp_of), 64), np.int64)
    blk = 0
    for r, seg in enumerate(segs):
        bits, pred = _Bits(seg), [0, 0, 0]
        for _ in range(min(ri, total - r * ri)):
            for c in comp_of:
                dct, act = hd["huff"][c]
                s = bits.sym(dct)
                pred[c] += _extend(bits.get(s), s)
                coef[blk, 0] = pred[c]
                k = 1
                while k < 64:
                    rs = bits.sym(act)
                    rr, s = rs >> 4, rs & 15
                    if s:
                        k += rr
                        if k > 63:
                            raise JpegError(EDATA, "coefficient index")
                        coef[blk, ZIGZAG[k]] = _extend(bits.get(s), s)
                        k += 1
                    elif rr == 15:
                        k += 16
                    else:
                        break
                blk += 1
    return coef.astype(np.int16).astype(np.int64), (mx, my, h0, v0)


# jidctint.c constants (CONST_BITS = 13)
_F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
          f1961=16069, f2053=16819, f2562=20995, f3072=25172)


def _idct_1d(s, shift, pass2):
    """one islow pass over axis -1 of int64 [.., 8] (pass 2 feeds the workspace values straight in)"""
    f = _F
    z2, z3 = s[..., 2], s[..., 6]
    z1 = (z2 + z3) * f["f0541"]
    tmp2 = z1 + z3 * -f["f1847"]
    tmp3 = z1 + z2 * f["f0765"]
    tmp0 = (s[..., 0] + s[..., 4]) << 13
    tmp1 = (s[..., 0] - s[..., 4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = s[..., 7], s[..., 5], s[..., 3], s[..., 1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * f["f1175"]
    t0, t1, t2, t3 = t0 * f["f0298"], t1 * f["f2053"], t2 * f["f3072"], t3 * f["f1501"]
    z1, z2, z3, z4 = z1 * -f["f0899"], z2 * -f["f2562"], z3 * -f["f1961"] + z5, z4 * -f["f0390"] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    out = np.stack([t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3], axis=-1)
    return (out + (1 << (shift - 1))) >> shift


def idct_islow(coef, qt):
    """[blocks, 64] quantised coefficients (natural order) -> [blocks, 8, 8] uint8 samples"""
    d = (coef * qt).reshape(-1, 8, 8)
    ws = _idct_1d(d.transpose(0, 2, 1), 11, False).transpose(0, 2, 1)    # columns: CONST_BITS - PASS1_BITS
    x = _idct_1d(ws, 18, True)                                            # rows: CONST_BITS + PASS1_BITS + 3
    x = ((x + 512) & 1023) - 512                                          # range-limit table: 10-bit wrap, then clamp
    return np.clip(x + 128, 0, 255).astype(np.int64)


def _planes(coef, hd, geom):
    mx, my, h0, v0 = geom
    out = []
    blocks = coef.reshape(my, mx, h0 * v0 + 2, 64)
    # component 0: h0 x v0 blocks per MCU, row-major
    y = idct_islow(blocks[:, :, :h0 * v0].reshape(-1, 64), hd["q"][0]).reshape(my, mx, v0, h0, 8, 8)
    out.append(y.transpose(0, 2, 4, 1, 3, 5).reshape(my * v0 * 8, mx * h0 * 8))
    for c in (1, 2):
        p = idct_islow(blocks[:, :, h0 * v0 + c - 1].reshape(-1, 64), hd["q"][c]).reshape(my, mx, 8, 8)
        out.append(p.transpose(0, 2, 1, 3).reshape(my * 8, mx * 8))
    return out


def _upsample(p, h, w, h0, v0):
    """chroma plane -> [h, w] (jdsample.c: fullsize, h2v1 / h2v2 fancy, or plain replication for narrow planes)"""
    if (h0, v0) == (1, 1):
        return p[:h, :w]
    dw, dh = -(-w // 2), -(-h // v0)
    xs = np.arange(w)
    c = xs >> 1
    if dw <= 2:
        return p[(np.arange(h) // v0)[:, None], c[None, :]]
    lft, rgt = np.maximum(c - 1, 0), np.minimum(c + 1, dw - 1)
    odd = (xs & 1).astype(bool)
    if v0 == 1:
        row = p[:h]
        near, far = row[:, c], np.where(odd, row[:, rgt], row[:, lft])
        return np.where(odd, (3 * near + far + 2) >> 2, (3 * near + far + 1) >> 2)
    ys = np.arange(h)
    r = ys >> 1
    rf = np.where(ys & 1, np.minimum(r + 1, dh - 1), np.maximum(r - 1, 0))
    cs = 3 * p[r, :] + p[rf, :]                                     # column sums [h, plane width]
    near, far = cs[:, c], np.where(odd, cs[:, rgt], cs[:, lft])
    return np.where(odd, (3 * near + far + 7) >> 4, (3 * near + far + 8) >> 4)


def ycc_to_bgr(y, cb, cr):
    """jdcolor.c ycc_rgb_convert with its 16-bit fixed-point tables, BGR channel order"""
    cb, cr = cb - 128, cr - 128
    half = 1 << 15
    r = y + ((91881 * cr + half) >> 16)
    g = y + ((-22554 * cb + half - 46802 * cr) >> 16)
    b = y + ((116130 * cb + half) >> 16)
    return np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8)


def decode(data, hw=None):
    """-> (uint8 [H, W, 3] BGR or None, status)"""
    try:
        hd = parse(data)
        if hw is not None and (hd["h"], hd["w"]) != tuple(hw):
            raise JpegError(ESIZE, "size")
        segs = split_scan(bytes(data), hd["scan"])
        coef, geom = entropy_decode(hd, segs)
    except JpegError as e:
        return None, e.status
    h, w = hd["h"], hd["w"]
    yp, cbp, crp = _planes(coef, hd, geom)
    _, _, h0, v0 = geom
    return ycc_to_bgr(yp[:h, :w], _upsample(cbp, h, w, h0, v0), _upsample(crp, h, w, h0, v0)), OK
