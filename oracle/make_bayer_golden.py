"""Write tests/golden/bayer_frames.npz: cv2.cvtColor's BGR frames of 8-bit Bayer mosaics in the four patterns and two
demosaicings StreamDetector(frame_format="bayer_*", demosaic=...) takes (tests/test_stream_bayer.py).  The GPU host may
lack cv2, so what cv2 computes is stored here.

    python -m oracle.make_bayer_golden

Per case ``<c>``, pattern ``<p>`` (bayer_oracle.PATTERNS) and algorithm ``<a>`` (bayer_oracle.ALGOS):
  ``<c>.hw``           the frame's (h, w)
  ``<c>.raw``          the uint8 [h, w] mosaic, for the small cases; the others are synth_frame(h, w, seed) and store
                       only ``<c>.seed`` and ``<c>.raw_sha256``.  One mosaic per case serves every pattern
  ``<p>.<a>.<c>.bgr``  cv2.cvtColor(raw, bayer_oracle.CV2_CODES[p, a]) for the small cases; ``<p>.<a>.<c>.sha256`` for
                       all, and ``<p>.<a>.<c>.crop`` a 32 x 32 crop at the frame's centre of the large ones
Cases: 2x2 and 2x9 (black, as cv2 makes frames of fewer than 3 rows or columns), 3x3, 5x8, 19x67 (odd sizes, a width
that is no multiple of 8, 16 or 32), 64x130 (more than one 128-column tile), 600x960 and 1200x1920 (camera frames), and
``edges`` (24x66): constant 0 and 255 blocks, so that every channel reaches 0 and 255, next to a field of 0, 1, 127, 128,
254 and 255 that makes the edge-aware gradient comparison tie often.
"""
import hashlib
import os

import numpy as np

from oracle.bayer_oracle import ALGOS, CV2_CODES, PATTERNS

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")

# case: (h, w, seed); seed None = stored verbatim from a seeded generator, else synth_frame
CASES = {"2x2": (2, 2, None), "2x9": (2, 9, None), "3x3": (3, 3, None), "5x8": (5, 8, None),
         "19x67": (19, 67, None), "64x130": (64, 130, 3), "600x960": (600, 960, 5), "1200x1920": (1200, 1920, 7)}
EDGES_HW = (24, 66)
EDGE_VALUES = np.array([0, 1, 127, 128, 254, 255], np.uint8)


def synth_frame(h, w, seed):
    """a uint8 [h, w] mosaic whose bytes are an integer hash of their index and ``seed`` (the same on every host)"""
    x = (np.arange(h * w, dtype=np.uint64) + np.uint64(seed)) * np.uint64(0x9E3779B97F4A7C15)
    x ^= x >> np.uint64(29)
    x *= np.uint64(0xBF58476D1CE4E5B9)
    x ^= x >> np.uint64(32)
    return (x & np.uint64(255)).astype(np.uint8).reshape(h, w)


def edge_frame():
    """0 and 255 blocks (8 x 8, so each holds every colour of the mosaic) above a field of extreme values"""
    h, w = EDGES_HW
    f = np.random.default_rng(77).choice(EDGE_VALUES, (h, w)).astype(np.uint8)
    f[:8] = np.where((np.arange(w) // 8) % 2 == 0, 0, 255)[None, :]
    return f


def frames():
    """case -> (h, w, raw, seed)"""
    rng = np.random.default_rng(2026)
    out = {}
    for c, (h, w, seed) in CASES.items():
        f = rng.integers(0, 256, (h, w), dtype=np.uint8) if seed is None else synth_frame(h, w, seed)
        out[c] = (h, w, f, seed)
    out["edges"] = (*EDGES_HW, edge_frame(), None)
    return out


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    import cv2
    g = {}
    for c, (h, w, f, seed) in frames().items():
        g[f"{c}.hw"] = np.array([h, w], np.int32)
        if seed is None:
            g[f"{c}.raw"] = f
        else:
            g[f"{c}.seed"] = np.array(seed, np.int64)
            g[f"{c}.raw_sha256"] = sha(f)
        for p in PATTERNS:
            for a in ALGOS:
                bgr = cv2.cvtColor(f, getattr(cv2, CV2_CODES[p, a]))
                assert bgr.shape == (h, w, 3) and bgr.dtype == np.uint8
                k = f"{p}.{a}.{c}"
                g[f"{k}.sha256"] = sha(bgr)
                if seed is None:
                    g[f"{k}.bgr"] = bgr
                else:
                    g[f"{k}.crop"] = bgr[h // 2 - 16:h // 2 + 16, w // 2 - 16:w // 2 + 16].copy()
    g["cv2_version"] = np.array(cv2.__version__)
    path = os.path.join(GOLDEN, "bayer_frames.npz")
    np.savez_compressed(path, **g)
    print(f"wrote {path} ({os.path.getsize(path)} bytes, cv2 {cv2.__version__})")


if __name__ == "__main__":
    main()
