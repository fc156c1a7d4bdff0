"""Write tests/golden/jpeg_streams.npz: JPEG files only cv2's writer makes here (4:2:2 and 4:4:4, optimised Huffman
tables, restart intervals of 1, of a count that does not divide the MCUs and of more than the MCUs, q100 noise) and what
cv2.imdecode returns for them.  tests/test_jpeg_decode_streams.py checks the device decoder against them (the GPU host
may lack cv2).

    python -m oracle.make_jpeg_streams_golden

Per case ``<name>.jpg`` (the file's bytes) and either ``<name>.bgr`` (cv2's uint8 [h, w, 3] output, small cases) or
``<name>.sha256`` of cv2's output and ``<name>.rows``, the CRC-32 of each MCU row of it (8 or 16 pixel rows), so that a
mismatch names its first row.  ``libjpeg_turbo`` is the version cv2 was built with.
"""
import hashlib
import os
import zlib

import numpy as np

from oracle.make_jpeg_encode_golden import content, libjpeg_turbo_version
from oracle.make_jpeg_golden import GOLDEN, encode

# name: (h, w, quality, sampling, restart interval in MCUs, optimised Huffman tables, content)
CASES = {
    "s444_q95_r1_37x53": (37, 53, 95, "444", 1, 0, "smooth"),
    "s444_q80_40x72": (40, 72, 80, "444", 0, 0, "smooth"),
    "s422_q90_opt_r7_45x77": (45, 77, 90, "422", 7, 1, "smooth"),     # 30 MCUs: 7 does not divide them
    "s422_q75_32x64": (32, 64, 75, "422", 0, 0, "flat"),
    "s420_q85_r1000_33x65": (33, 65, 85, "420", 1000, 0, "smooth"),  # one interval longer than the 15 MCUs
    "s420_q90_31x47": (31, 47, 90, "420", 0, 0, "smooth"),
    "s444_q100_opt_noise_24x40": (24, 40, 100, "444", 0, 1, "noise"),
    "s422_q100_r2_checker_16x24": (16, 24, 100, "422", 2, 0, "checker"),
    "m422_q100_noise_240x320": (240, 320, 100, "422", 0, 0, "noise"),
    "m444_q95_opt_r13_203x299": (203, 299, 95, "444", 13, 1, "smooth"),
    "f444_q50_r1_1200x1920": (1200, 1920, 50, "444", 1, 0, "smooth"),  # 36 000 restart intervals
}
SMALL_PIXELS = 64 * 96         # cases up to this size store cv2's pixels, the others their hashes


def band(samp):
    """pixel rows of one MCU row"""
    return 16 if samp == "420" else 8


def case_bytes(name):
    h, w, q, samp, ri, opt, kind = CASES[name]
    seed = 300 + sorted(CASES).index(name)
    return encode(content(kind, h, w, seed), q, samp, ri, opt)


def row_crcs(img, samp):
    b = band(samp)
    return np.array([zlib.crc32(np.ascontiguousarray(img[y:y + b]).tobytes()) for y in range(0, img.shape[0], b)],
                    np.int64)


def main():
    import cv2
    version = libjpeg_turbo_version()
    out = {"libjpeg_turbo": np.array(version)}
    for name, (h, w, q, samp, ri, opt, kind) in CASES.items():
        b = case_bytes(name)
        ref = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        assert ref.shape == (h, w, 3), name
        out[name + ".jpg"] = np.frombuffer(b, np.uint8)
        if h * w <= SMALL_PIXELS:
            out[name + ".bgr"] = ref
        else:
            out[name + ".sha256"] = np.frombuffer(hashlib.sha256(ref.tobytes()).digest(), np.uint8)
            out[name + ".rows"] = row_crcs(ref, samp)
    path = os.path.join(GOLDEN, "jpeg_streams.npz")
    np.savez_compressed(path, **out)
    print("jpeg_streams.npz", os.path.getsize(path), "bytes,", version)


if __name__ == "__main__":
    main()
