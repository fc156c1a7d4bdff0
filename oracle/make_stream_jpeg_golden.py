"""Write tests/golden/stream_jpeg_files.npz: the fixtures of the streaming detector's JPEG input for camera streams of
different sizes (tests/test_stream_jpeg.py).  The GPU host may lack cv2, so everything cv2 computes is stored here.

    python -m oracle.make_stream_jpeg_golden

Per file ``<name>``:
  ``<name>.jpg``          the file's bytes (seeded synthetic frames written by cv2.imencode)
  ``<name>.hw``           its (h, w)
  ``<name>.sha256``       SHA-256 of cv2.imdecode's uint8 BGR frame (what cv2.imread returns), and ``<name>.crop`` a 32 x 32
                          crop of it at the frame's centre (to see a mismatch)
  ``<name>.seq``          SHA-256 of cv2's frame of requant(jpg, k), k = 0 .. SEQ - 1: the frames of a seeded sequence
  ``<name>.plain``        SHA-256 of the driver's preproc (streamyolo_det.py:57-60) at 600 x 960, as float32 [3, H, W]
  ``<name>.eval``         SHA-256 of the evaluation preproc (data_augment_flip.py:151-167) at 600 x 960, float32 [3, H, W]
  ``<name>.r``            the evaluation preproc's ratio r
The damaged file ``bad`` (a truncated entropy-coded segment) has only ``.jpg`` and ``.hw``.
"""
import hashlib
import os

import numpy as np

from oracle.make_jpeg_golden import encode

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
SIZE = (600, 960)
SEQ = 4

# name: (h, w, quality, sampling, restart interval in MCUs)
FILES = {
    "a420": (1200, 1920, 80, "420", 0),
    "b444": (2048, 1550, 75, "444", 0),
    "c420_r16": (1550, 2048, 80, "420", 16),
}


def scene(h, w, seed):
    """a smooth camera-like BGR frame with a few solid boxes (compresses to a small file)"""
    r = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.empty((h, w, 3))
    img[..., 0] = 80 + 90 * yy / (h - 1) + 25 * np.sin(xx / (41.0 + seed))
    img[..., 1] = 100 + 70 * np.cos(yy / 57.0) * np.sin(xx / (67.0 + seed))
    img[..., 2] = 60 + 130 * xx / (w - 1)
    for _ in range(24):
        y0, x0 = r.integers(0, h), r.integers(0, w)
        img[y0:y0 + r.integers(16, h // 5), x0:x0 + r.integers(16, w // 6)] = r.integers(0, 256, 3)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def requant(jpg, k):
    """the file with its first quantisation table's DC and first AC step raised by k: a valid file of the same size whose
    frame differs (brightness and texture) -- a sequence of distinct frames from one fixture, without an encoder"""
    b = bytearray(jpg)
    i = 2
    while b[i + 1] != 0xDB:
        i += 2 + ((b[i + 2] << 8) | b[i + 3])
    assert b[i + 4] >> 4 == 0, "8-bit tables"
    for z in (0, 1):
        b[i + 5 + z] = min(255, b[i + 5 + z] + k)
    return bytes(b)


def damaged(jpg):
    """the entropy-coded segment cut at its middle, then EOI"""
    return jpg[:len(jpg) // 2] + b"\xff\xd9"


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def preproc_plain(img, size):
    import cv2
    return cv2.resize(img, (size[1], size[0]), interpolation=cv2.INTER_LINEAR).transpose(2, 0, 1).astype(np.float32)


def preproc_eval(img, size):
    import cv2
    padded = np.ones((size[0], size[1], 3), dtype=np.uint8) * 114
    r = min(size[0] / img.shape[0], size[1] / img.shape[1])
    resized = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR)
    padded[:int(img.shape[0] * r), :int(img.shape[1] * r)] = resized
    return np.ascontiguousarray(padded.transpose(2, 0, 1), dtype=np.float32), r


def main():
    import cv2
    d = {}
    for seed, (name, (h, w, q, samp, rst)) in enumerate(FILES.items()):
        jpg = encode(scene(h, w, seed + 1), q, samp, rst, 0)
        img = cv2.imdecode(np.frombuffer(jpg, np.uint8), cv2.IMREAD_COLOR)
        assert img.shape == (h, w, 3)
        d[f"{name}.jpg"] = np.frombuffer(jpg, np.uint8)
        d[f"{name}.hw"] = np.array([h, w], np.int32)
        d[f"{name}.sha256"] = sha(img)
        d[f"{name}.crop"] = img[h // 2 - 16:h // 2 + 16, w // 2 - 16:w // 2 + 16].copy()
        seq = [cv2.imdecode(np.frombuffer(requant(jpg, k), np.uint8), cv2.IMREAD_COLOR) for k in range(SEQ)]
        assert len({sha(f).tobytes() for f in seq}) == SEQ, "requant gives distinct frames"
        d[f"{name}.seq"] = np.stack([sha(f) for f in seq])
        d[f"{name}.plain"] = sha(preproc_plain(img, SIZE))
        x, r = preproc_eval(img, SIZE)
        d[f"{name}.eval"] = sha(x)
        d[f"{name}.r"] = np.array(r, np.float64)
        print(f"{name}: {h}x{w} {samp} rst {rst}, {len(jpg)} bytes, r {r}")
    bad = damaged(bytes(d["c420_r16.jpg"]))
    d["bad.jpg"] = np.frombuffer(bad, np.uint8)
    d["bad.hw"] = d["c420_r16.hw"]
    path = os.path.join(GOLDEN, "stream_jpeg_files.npz")
    np.savez_compressed(path, **d)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
