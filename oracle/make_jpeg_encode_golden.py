"""Write tests/golden/jpeg_encode_small.npz and jpeg_encode_full.npz: what cv2.imencode(".jpg", img,
[cv2.IMWRITE_JPEG_QUALITY, q]) returns, the device encoder's fixtures (the GPU host may lack cv2).

    python -m oracle.make_jpeg_encode_golden

jpeg_encode_small.npz  per case ``<name>.bgr`` (the uint8 [h, w, 3] input), ``<name>.jpg`` (cv2's bytes) and
                ``<name>.q``: sizes 1x1 .. 37x53, qualities 1 .. 100, smooth, noisy, saturated / flat and +-255
                checkerboard content
jpeg_encode_full.npz   the 1200 x 1920 and 600 x 960 frames cv2.imdecode makes of jpeg_full_f420_q90.npz and
                jpeg_full_m420_q90_600x960.npz (not stored: the device decoder and oracle/jpeg_oracle.py rebuild them bit
                for bit), encoded at q 75 and 95: per case ``<name>.sha256`` and ``<name>.length`` of cv2's file, and
                ``<name>.bands`` / ``<name>.band_bits``, the CRC-32 and bit length of each MCU row band of its
                entropy-coded data (band_crcs), so that a mismatch names its first band
Both hold ``libjpeg_turbo``, the version cv2 was built with.
"""
import hashlib
import os
import re
import zlib

import numpy as np

from oracle import jpeg_oracle as jo
from oracle.make_jpeg_golden import GOLDEN, synth_frame

SIZES = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (33, 65), (37, 53)]
QUALITIES = [1, 10, 50, 75, 90, 95, 100]
CONTENTS = ("smooth", "noise", "flat", "checker")
FULL = {"f420_q90": ("jpeg_full_f420_q90.npz", (1200, 1920)),
        "m420_q90_600x960": ("jpeg_full_m420_q90_600x960.npz", (600, 960))}
FULL_QUALITIES = (75, 95)


def content(kind, h, w, seed):
    """uint8 BGR [h, w, 3] test content: camera-like, uniform noise, saturated blocks of 0 / 255 with flat areas, or a
    one-pixel 0 / 255 checkerboard (the largest AC coefficients)"""
    r = np.random.default_rng(seed)
    if kind == "smooth":
        return synth_frame(h, w, seed)
    if kind == "noise":
        return r.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "flat":
        img = np.full((h, w, 3), r.integers(0, 256, 3), np.uint8)
        img[: (h + 1) // 2, : (w + 1) // 2] = 255
        img[h // 2:, w // 2:, 1] = 0
        return img
    yy, xx = np.mgrid[0:h, 0:w]
    return np.repeat((((yy + xx) & 1) * 255).astype(np.uint8)[..., None], 3, axis=2)


def small_cases():
    """name -> (img, quality): every size at every quality, the content cycling with both, and the checkerboard at q = 100
    for every size"""
    out = {}
    for i, (h, w) in enumerate(SIZES):
        for j, q in enumerate(QUALITIES):
            kind = CONTENTS[(i + j) % len(CONTENTS)]
            out[f"{h}x{w}_q{q}_{kind}"] = (content(kind, h, w, 31 * i + j), q)
        if f"{h}x{w}_q100_checker" not in out:
            out[f"{h}x{w}_q100_checker"] = (content("checker", h, w, 0), 100)
    return out


def full_input(name, golden=GOLDEN):
    """the stored JPEG file whose cv2.imdecode is full case ``name``'s input, and its (h, w)"""
    fname, hw = FULL[name]
    with np.load(os.path.join(golden, fname)) as f:
        return f["jpg"], hw


def libjpeg_turbo_version():
    import cv2
    m = re.search(r"JPEG:\s+(.*)", cv2.getBuildInformation())
    return f"cv2 {cv2.__version__}: " + (m.group(1).strip() if m else "unknown")


def band_crcs(jpg):
    """(CRC-32, bit length) of each MCU row band of a baseline 4:2:0 file's entropy-coded data: the destuffed bits from
    the band's first MCU to the next band's, packed MSB first"""
    hd = jo.parse(jpg)
    seg = jo.split_scan(bytes(jpg), hd["scan"])
    assert len(seg) == 1 and hd["comps"][0][1:3] == (2, 2), "band_crcs takes 4:2:0 files without restart intervals"
    mx, my = -(-hd["w"] // 16), -(-hd["h"] // 16)
    bits = jo._Bits(seg[0])
    starts = []
    for m in range(mx * my):
        if m % mx == 0:
            starts.append(bits.p)
        for c in (0, 0, 0, 0, 1, 2):
            dct, act = hd["huff"][c]
            bits.get(bits.sym(dct))
            k = 1
            while k < 64:
                rs = bits.sym(act)
                if rs & 15:
                    bits.get(rs & 15)
                    k += (rs >> 4) + 1
                elif rs == 0xF0:
                    k += 16
                else:
                    break
    starts.append(bits.p)
    allbits = np.unpackbits(np.frombuffer(seg[0], np.uint8))
    crcs = [zlib.crc32(np.packbits(allbits[a:b]).tobytes()) for a, b in zip(starts[:-1], starts[1:])]
    return np.array(crcs, np.int64), np.diff(np.array(starts, np.int64))


def main():
    import cv2
    version = libjpeg_turbo_version()
    small = {"libjpeg_turbo": np.array(version)}
    for name, (img, q) in small_cases().items():
        ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])
        assert ok
        small[name + ".bgr"], small[name + ".jpg"], small[name + ".q"] = img, enc.reshape(-1), np.int32(q)
    full = {"libjpeg_turbo": np.array(version)}
    for name in FULL:
        jpg, hw = full_input(name)
        img = cv2.imdecode(jpg, cv2.IMREAD_COLOR)
        assert img.shape[:2] == hw
        for q in FULL_QUALITIES:
            b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()
            key = f"{name}_q{q}"
            full[key + ".sha256"] = np.frombuffer(hashlib.sha256(b).digest(), np.uint8)
            full[key + ".length"] = np.int64(len(b))
            full[key + ".bands"], full[key + ".band_bits"] = band_crcs(b)
    for fname, d in (("jpeg_encode_small.npz", small), ("jpeg_encode_full.npz", full)):
        np.savez_compressed(os.path.join(GOLDEN, fname), **d)
        print(fname, os.path.getsize(os.path.join(GOLDEN, fname)), "bytes,", version)


if __name__ == "__main__":
    main()
