"""Write tests/golden/yuv_frames.npz: cv2.cvtColor's BGR frames of raw YUV camera frames in the six formats
StreamDetector(frame_format=...) takes (tests/test_stream_yuv.py).  The GPU host may lack cv2, so what cv2 computes is
stored here.

    python -m oracle.make_yuv_golden

Per format ``<f>`` (yuv_oracle.FORMATS) and case ``<c>``:
  ``<f>.<c>.hw``       the frame's (h, w)
  ``<f>.<c>.yuv``      the uint8 frame in cv2's layout ([h * 3 // 2, w] for 4:2:0, [h, w, 2] for 4:2:2), for the small
                       cases; the others are synth_frame(f, h, w, seed) and store only ``<f>.<c>.yuv_sha256``
  ``<f>.<c>.bgr``      cv2.cvtColor(frame, yuv_oracle.CV2_CODES[f]) for the small cases; ``<f>.<c>.sha256`` for all, and
                       ``<f>.<c>.crop`` a 32 x 32 crop at the frame's centre of the large ones (to see a mismatch)
Cases: 2x2, 38x62 (a width that is no multiple of 8, 16 or 32), 120x162, 1200x1920 (a camera frame), and ``edges``
(16x62): Y below 16, at 16 and at 255 with every extreme chroma, so that every channel saturates at 0 and at 255.
"""
import hashlib
import os

import numpy as np

from oracle.yuv_oracle import CV2_CODES, FORMATS, frame_shape, is420

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")

# case: (h, w, seed); seed None = stored verbatim from a seeded generator, else synth_frame
CASES = {"2x2": (2, 2, None), "38x62": (38, 62, None), "120x162": (120, 162, 3), "1200x1920": (1200, 1920, 7)}
EDGES_HW = (16, 62)
Y_EDGES = np.array([0, 1, 15, 16, 17, 128, 235, 240, 254, 255], np.uint8)
C_EDGES = np.array([0, 1, 16, 127, 128, 129, 240, 255], np.uint8)


def synth_frame(fmt, h, w, seed):
    """a uint8 frame of ``fmt`` whose bytes are an integer hash of their index and ``seed`` (the same on every host)"""
    shape = frame_shape(fmt, h, w)
    x = (np.arange(int(np.prod(shape)), dtype=np.uint64) + np.uint64(seed)) * np.uint64(0x9E3779B97F4A7C15)
    x ^= x >> np.uint64(29)
    x *= np.uint64(0xBF58476D1CE4E5B9)
    x ^= x >> np.uint64(32)
    return (x & np.uint64(255)).astype(np.uint8).reshape(shape)


def pack(fmt, y, u, v):
    """planes -> the frame in cv2's layout: Y [h, w]; U, V [h / 2, w / 2] (4:2:0) or [h, w / 2] (4:2:2)"""
    h, w = y.shape
    if is420(fmt):
        if fmt in ("nv12", "nv21"):
            c = np.stack([u, v] if fmt == "nv12" else [v, u], -1).reshape(h // 2, w)
        else:
            c = np.concatenate([u.reshape(-1), v.reshape(-1)] if fmt == "i420" else [v.reshape(-1), u.reshape(-1)])
            c = c.reshape(h // 2, w)
        return np.ascontiguousarray(np.concatenate([y, c], 0), np.uint8)
    g = np.stack([y[:, 0::2], u, y[:, 1::2], v] if fmt == "yuyv" else [u, y[:, 0::2], v, y[:, 1::2]], -1)
    return np.ascontiguousarray(g.reshape(h, w, 2), np.uint8)


def edge_frame(fmt):
    """every (Y, U, V) of Y_EDGES x C_EDGES x C_EDGES that fits, chroma constant over each group"""
    h, w = EDGES_HW
    ch, cw = (h // 2, w // 2) if is420(fmt) else (h, w // 2)
    i = np.arange(ch * cw)
    u = C_EDGES[i % len(C_EDGES)].reshape(ch, cw)
    v = C_EDGES[(i // len(C_EDGES)) % len(C_EDGES)].reshape(ch, cw)
    y = Y_EDGES[np.arange(h * w) % len(Y_EDGES)].reshape(h, w)
    return pack(fmt, y, u, v)


def frames(fmt):
    """case -> (h, w, frame, seed)"""
    rng = np.random.default_rng(2024 + FORMATS.index(fmt))
    out = {}
    for c, (h, w, seed) in CASES.items():
        f = rng.integers(0, 256, frame_shape(fmt, h, w), dtype=np.uint8) if seed is None else synth_frame(fmt, h, w, seed)
        out[c] = (h, w, f, seed)
    out["edges"] = (*EDGES_HW, edge_frame(fmt), None)
    return out


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    import cv2
    g = {}
    for fmt in FORMATS:
        for c, (h, w, f, seed) in frames(fmt).items():
            bgr = cv2.cvtColor(f, getattr(cv2, CV2_CODES[fmt]))
            assert bgr.shape == (h, w, 3) and bgr.dtype == np.uint8
            k = f"{fmt}.{c}"
            g[f"{k}.hw"] = np.array([h, w], np.int32)
            g[f"{k}.sha256"] = sha(bgr)
            if seed is None:
                g[f"{k}.yuv"], g[f"{k}.bgr"] = f, bgr
            else:
                g[f"{k}.seed"] = np.array(seed, np.int64)
                g[f"{k}.yuv_sha256"] = sha(f)
                g[f"{k}.crop"] = bgr[h // 2 - 16:h // 2 + 16, w // 2 - 16:w // 2 + 16].copy()
    g["cv2_version"] = np.array(cv2.__version__)
    path = os.path.join(GOLDEN, "yuv_frames.npz")
    np.savez_compressed(path, **g)
    print(f"wrote {path} ({os.path.getsize(path)} bytes, cv2 {cv2.__version__})")


if __name__ == "__main__":
    main()
