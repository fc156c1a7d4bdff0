"""Write tests/golden/jpeg_small.npz, jpeg_full_<name>.npz and jpeg_bad.npz: JPEG files written by cv2 and what
cv2.imdecode returns for them (the device decoder's fixtures; the GPU host may lack cv2).

    python -m oracle.make_jpeg_golden

jpeg_small.npz  per case ``<name>.jpg`` (the file's bytes) and ``<name>.bgr`` (cv2's uint8 [h, w, 3] output)
jpeg_full_<name>.npz   one 1200 x 1920 frame (or 600 x 960) each, to keep every file small: ``jpg``, ``sha256`` of
                cv2's output and ``rows``, the CRC-32 of each MCU row of it (8 or 16 pixel rows), so a mismatch names its
                first row; load_full() merges them
jpeg_bad.npz    33 x 65 streams the decoder refuses: ``<name>.jpg`` and ``<name>.status`` (oracle/jpeg_oracle.py codes)
"""
import hashlib
import os
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")

SAMPLING = {"420": 0x221111, "422": 0x211111, "444": 0x111111, "411": 0x411111}   # cv2.IMWRITE_JPEG_SAMPLING_FACTOR_*

# name: (h, w, quality, sampling, restart interval in MCUs, optimised Huffman tables)
SMALL = {
    "s420_q75": (33, 65, 75, "420", 0, 0),
    "s422_q95_r1_opt": (33, 65, 95, "422", 1, 1),
    "s444_q50_r7": (33, 65, 50, "444", 7, 0),
    "s420_q100_opt": (33, 65, 100, "420", 0, 1),
    "s444_q90_17x23": (17, 23, 90, "444", 0, 0),
    "s420_q90_1x1": (1, 1, 90, "420", 0, 0),
    "s422_q85_15x31": (15, 31, 85, "422", 0, 0),
    "s420_q95_r3_8x8": (8, 8, 95, "420", 3, 1),
}
FULL = {
    "f420_q90": (1200, 1920, 90, "420", 0, 0),
    "f420_q85_r8": (1200, 1920, 85, "420", 8, 0),
    "f422_q90_opt": (1200, 1920, 90, "422", 0, 1),
    "f444_q80_r120": (1200, 1920, 80, "444", 120, 0),
    "m420_q90_600x960": (600, 960, 90, "420", 0, 0),
}


def synth_frame(h, w, seed):
    """a camera-like BGR frame: smooth sky / road gradients, a few solid boxes with edges, mild sensor noise"""
    r = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.empty((h, w, 3))
    img[..., 0] = 90 + 80 * yy / max(h - 1, 1) + 20 * np.sin(xx / 37.0)
    img[..., 1] = 110 + 60 * np.cos(yy / 53.0) * np.sin(xx / 71.0)
    img[..., 2] = 70 + 120 * xx / max(w - 1, 1)
    for _ in range(max(1, h * w // 40000)):
        y0, x0 = r.integers(0, h), r.integers(0, w)
        img[y0:y0 + r.integers(1, max(2, h // 6)), x0:x0 + r.integers(1, max(2, w // 8))] = r.integers(0, 256, 3)
    img += r.normal(0, 4.0, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def encode(img, q, samp, rst, opt, progressive=False):
    import cv2
    ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[samp],
                                         cv2.IMWRITE_JPEG_RST_INTERVAL, rst, cv2.IMWRITE_JPEG_OPTIMIZE, opt,
                                         cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)])
    assert ok
    return enc.tobytes()


def case_bytes(spec, seed):
    h, w, q, samp, rst, opt = spec
    return encode(synth_frame(h, w, seed), q, samp, rst, opt)


def find_marker(b, m):
    """offset of the first marker ``m`` (the FF byte) among the header segments"""
    i = 2
    while i + 4 <= len(b):
        if b[i + 1] == m:
            return i
        i += 2 + ((b[i + 2] << 8) | b[i + 3])
    raise ValueError(f"marker {m:#x} not found")


def exif_app1(orientation):
    """APP1 Exif segment (big-endian TIFF) holding one IFD0 entry: Orientation (SHORT) = orientation"""
    tiff = b"MM\x00*" + (8).to_bytes(4, "big") + (1).to_bytes(2, "big")
    tiff += (0x0112).to_bytes(2, "big") + (3).to_bytes(2, "big") + (1).to_bytes(4, "big") + orientation.to_bytes(2, "big") + b"\x00\x00"
    tiff += (0).to_bytes(4, "big")
    payload = b"Exif\x00\x00" + tiff
    return b"\xff\xe1" + (len(payload) + 2).to_bytes(2, "big") + payload


def bad_streams(h=33, w=65):
    """name -> bytes of streams outside the decoder's scope or damaged, all claiming (or being) h x w"""
    import cv2
    img = synth_frame(h, w, 7)
    good = encode(img, 90, "420", 0, 0)
    out = {"progressive": encode(img, 90, "420", 0, 0, progressive=True)}
    sof = find_marker(good, 0xC0)
    b = bytearray(good)
    b[sof + 1] = 0xC9
    out["arithmetic_sof9"] = bytes(b)
    b = bytearray(good)
    b[sof + 4] = 12
    out["precision_12"] = bytes(b)
    out["sampling_411"] = encode(img, 90, "411", 0, 0)
    ok, g = cv2.imencode(".jpg", cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), [cv2.IMWRITE_JPEG_QUALITY, 90])
    out["grayscale"] = g.tobytes()
    out["exif_orientation_6"] = good[:2] + exif_app1(6) + good[2:]
    out["size_mismatch"] = encode(synth_frame(h + 8, w, 7), 90, "420", 0, 0)
    sos = find_marker(good, 0xDA)
    for cut in (3, sof + 5, sos + 6, (sos + len(good)) // 2, len(good) - 40):
        out[f"cut_{cut}"] = good[:cut]
    return out


def load_full(golden=GOLDEN):
    """the full-size fixtures as one mapping: ``<name>.jpg``, ``<name>.sha256``, ``<name>.rows``"""
    out = {}
    for fname in sorted(os.listdir(golden)):
        if fname.startswith("jpeg_full_") and fname.endswith(".npz"):
            name = fname[len("jpeg_full_"):-len(".npz")]
            with np.load(os.path.join(golden, fname)) as f:
                out.update({f"{name}.{k}": f[k] for k in f})
    return out


def main():
    import cv2
    from oracle import jpeg_oracle
    small = {}
    for k, (name, spec) in enumerate(SMALL.items()):
        b = case_bytes(spec, 100 + k)
        small[name + ".jpg"] = np.frombuffer(b, np.uint8)
        small[name + ".bgr"] = cv2.imdecode(small[name + ".jpg"], cv2.IMREAD_COLOR)
    full = {}
    for k, (name, spec) in enumerate(FULL.items()):
        b = case_bytes(spec, 200 + k)
        ref = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        band = 16 if spec[3] == "420" else 8
        full[name] = {"jpg": np.frombuffer(b, np.uint8),
                      "sha256": np.frombuffer(hashlib.sha256(ref.tobytes()).digest(), np.uint8),
                      "rows": np.array([zlib.crc32(ref[y:y + band].tobytes()) for y in range(0, ref.shape[0], band)],
                                       np.int64)}
    bad = {}
    for name, b in bad_streams().items():
        bad[name + ".jpg"] = np.frombuffer(b, np.uint8)
        bad[name + ".status"] = np.int32(jpeg_oracle.decode(b, (33, 65))[1])
    files = [("jpeg_small.npz", small), ("jpeg_bad.npz", bad)] + [(f"jpeg_full_{n}.npz", d) for n, d in full.items()]
    for fname, d in files:
        np.savez_compressed(os.path.join(GOLDEN, fname), **d)
        print(fname, os.path.getsize(os.path.join(GOLDEN, fname)), "bytes")


if __name__ == "__main__":
    main()
