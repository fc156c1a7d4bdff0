"""Generate tests/golden/streaming_eval_script.npz -- TEST INFRASTRUCTURE.  Run in the build container, with the
StreamYOLO checkout at $STREAMYOLO_REF (default /root/reference), PIL and cv2 installed:

    python oracle/make_streaming_eval_golden.py

The UNMODIFIED sAP/det/streaming_eval.py main() is run under sys.argv on a fixture dataset in a temporary directory,
three times, always with --no-eval and --vis-dir.  oracle/ref_shim stands in for pycocotools and mmcv; this file adds
``imrescale`` to the mmcv stand-in, restated from mmcv's documented behaviour (mmcv.image.imrescale with a number:
rescale_size's ``int(w * scale + 0.5), int(h * scale + 0.5)``, then imresize's cv2.resize with INTER_LINEAR for
"bilinear").

The dataset: four sequences, each with the per-sequence pickle the detection driver writes (results_raw and
results_parsed per output, Python float timestamps, int input_fidx, runtime):
  s0  six 120 x 192 frames; raw rows as (float32 [n, 5] ltrb + score, int64 labels in 0..7), the annotation's
      coco_mapping dropping label 3 and permuting the others
  s1  five 75 x 131 frames (mmcv's size at 0.5 is 38 x 66, not an exact half)
  s2  the 1200 x 1920 frame of tests/golden/jpeg_full_f420_q90.npz
  s3  three 120 x 192 frames whose pickle has no results_raw (the script falls back to results_parsed)
The rows cover frames before the first output (miss), outputs with no rows (empty frames), boxes crossing every border
and wholly outside, reversed corners, zero-size boxes, half-integer corners (half to even after the 0.5 scale), labels
whose text is clipped at the top and left edges, and a timestamp equal to a frame's time.  The runs:
  raw     default pairing (results_raw, coco_mapping), --eta 0, --vis-scale 1, results into --result-dir
  parsed  --use-parsed, --eta -1, --vis-scale 0.5, --out-dir
  nomap   --no-class-mapping, --eta 0.5, --vis-scale 0.5, --out-dir
Stored: the inputs (JPEG bytes, the annotation file, the pickles), and per run the printed text, the bytes of
results_ccf.pkl and eval_assoc.pkl and every file written under --vis-dir (bytes; SHA-256 and length for s2's).
"""
import contextlib
import hashlib
import io
import json
import os
import pickle
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
REF = os.environ.get("STREAMYOLO_REF", "/root/reference")

from oracle.make_jpeg_encode_golden import content          # noqa: E402

CLASSES = ["person", "bicycle", "car", "motorcycle", "bus", "truck", "traffic_light", "stop_sign"]
COCO_MAPPING = [1, 0, 2, 100, 3, 4, 7, 6, 100, 5]           # raw label -> class; 3 and 8 are dropped
FPS = 30
SEQS = [("s0", "d0", (120, 192), 6, True), ("s1", "d1", (75, 131), 5, True), ("s2", "d2", (1200, 1920), 1, True),
        ("s3", "d3", (120, 192), 3, False)]
RUNS = [("raw", ["--eta", "0"], False),
        ("parsed", ["--use-parsed", "--eta", "-1", "--vis-scale", "0.5"], True),
        ("nomap", ["--no-class-mapping", "--eta", "0.5", "--vis-scale", "0.5"], True)]


def imrescale(img, scale, return_scale=False, interpolation="bilinear", backend=None):
    """mmcv.imrescale with a number ``scale`` and the cv2 backend"""
    import cv2
    if scale <= 0:
        raise ValueError(f"Invalid scale {scale}, must be positive.")
    h, w = img.shape[:2]
    size = int(w * float(scale) + 0.5), int(h * float(scale) + 0.5)
    codes = {"nearest": cv2.INTER_NEAREST, "bilinear": cv2.INTER_LINEAR}
    out = cv2.resize(img, size, interpolation=codes[interpolation])
    return (out, scale) if return_scale else out


def _rows(k, h, w, rng):
    """output k's rows of a frame of h x w: [(x1, y1, x2, y2), score, raw label]"""
    if k == 0:       # every border, reversed corners, zero size, labels clipped at the top and left
        return [((-6, 3, 40, 30), .91, 0), ((w - 30, 50, w + 12, 70), .5, 1), ((20, h - 10, 60, h + 15), .125, 2),
                ((70, 40, 50, 20), .875, 4), ((90, 60, 90, 60), .3, 5), ((-30, -30, -5, -5), .66, 6),
                ((100, 1, 140, 9), .705, 7), ((3, 80, 3.5, 100.5), .2, 3), ((-3, -2, w + 4, h + 3), .995, 5)]
    if k == 1:       # no rows
        return []
    if k == 2:       # half-integer corners, a label dropped by the mapping
        return [((10.5, 20.5, 30.5, 41.5), .6, 0), ((2.5, 3.5, 13.5, 16.5), .45, 3), ((51.5, 1.5, 60.5, 7.5), .05, 6)]
    out = []
    for i in range(30):
        x, y = rng.uniform(-0.2 * w, w), rng.uniform(-0.2 * h, h)
        bw, bh = rng.uniform(0, 0.5 * w), rng.uniform(0, 0.5 * h)
        out.append(((round(x * 2) / 2, round(y * 2) / 2, round((x + bw) * 2) / 2, round((y + bh) * 2) / 2),
                    float(rng.uniform(0, 1)), int(rng.integers(0, 8))))
    return out


def _pickle_dict(rows_per_output, timestamps, input_fidx, with_raw):
    """the driver's per-sequence pickle"""
    mapping = np.asarray(COCO_MAPPING)
    raw, parsed = [], []
    for rows in rows_per_output:
        bs = np.asarray([list(r[0]) + [r[1]] for r in rows], np.float32).reshape(-1, 5)
        lab = np.asarray([r[2] for r in rows], np.int64)
        raw.append((bs, lab))
        keep = mapping[lab] < len(CLASSES) if len(lab) else np.zeros(0, bool)
        parsed.append((bs[keep, :4].copy(), bs[keep, 4].copy(), mapping[lab][keep].astype(np.int32), None))
    d = {"results_parsed": parsed, "timestamps": timestamps, "input_fidx": input_fidx,
         "runtime": [0.02] * len(timestamps)}
    if with_raw:
        d = {"results_raw": raw, **d}
    return d


def fixture():
    """-> (annotation dict, {relative path: JPEG bytes}, {sequence: pickle dict})"""
    import cv2
    rng = np.random.default_rng(17)
    images, files, pickles = [], {}, {}
    img_id = 0
    for sid, (seq, d, (h, w), n, with_raw) in enumerate(SEQS):
        for fid in range(n):
            name = f"{fid:06d}.jpg"
            if h < 1000:
                ok, enc = cv2.imencode(".jpg", content("smooth", h, w, 300 + img_id), [cv2.IMWRITE_JPEG_QUALITY, 90])
                files[f"{d}/{name}"] = enc.tobytes()
            images.append({"id": img_id, "sid": sid, "fid": fid, "name": name, "width": w, "height": h})
            img_id += 1
        # outputs: the first after frame 1's time (frames 0 and 1 miss at eta 0), one exactly at frame 3's time
        if n == 1:
            timestamps, input_fidx = [0.0], [0]
        else:
            timestamps = [0.045, 0.07, 3 / FPS, 0.14, 0.16][:n - 1]
            input_fidx = [0, 1, 2, 3, 4][:n - 1]
        outputs = [_rows(k if n > 1 else 3, h, w, rng) for k in range(len(timestamps))]
        pickles[seq] = _pickle_dict(outputs, timestamps, input_fidx, with_raw)
    dataset = {"images": images, "annotations": [], "sequences": [s[0] for s in SEQS], "seq_dirs": [s[1] for s in SEQS],
               "categories": [{"id": i, "name": c} for i, c in enumerate(CLASSES)], "coco_mapping": COCO_MAPPING}
    return dataset, files, pickles


def full_frame():
    return np.load(os.path.join(ROOT, "tests", "golden", "jpeg_full_f420_q90.npz"))["jpg"].tobytes()


def import_script():
    """sAP/det/streaming_eval.py, imported as it is, with the stand-ins"""
    sys.path.insert(0, os.path.join(HERE, "ref_shim"))
    sys.path.insert(0, os.path.join(REF, "sAP"))
    import mmcv
    mmcv.imrescale = imrescale
    import det.streaming_eval as script
    return script


def run_script(script, dataset, files, pickles, extra, out_dir):
    """the script's main() on the fixture -> ({name: bytes} of the pickles, {relative vis path: bytes}, printed text)"""
    with tempfile.TemporaryDirectory() as tmp:
        for rel, b in list(files.items()) + [("d2/000000.jpg", full_frame())]:
            os.makedirs(os.path.join(tmp, "data", os.path.dirname(rel)), exist_ok=True)
            with open(os.path.join(tmp, "data", rel), "wb") as f:
                f.write(b)
        annot, res, vis, out = (os.path.join(tmp, v) for v in ("annot.json", "res", "vis", "out"))
        with open(annot, "w") as f:
            json.dump(dataset, f)
        os.makedirs(res)
        for seq, d in pickles.items():
            with open(os.path.join(res, seq + ".pkl"), "wb") as f:
                pickle.dump(d, f)
        argv, sys.argv = sys.argv, (["streaming_eval.py", "--data-root", os.path.join(tmp, "data"), "--annot-path", annot,
                                     "--fps", str(FPS), "--result-dir", res, "--vis-dir", vis, "--no-eval"]
                                    + (["--out-dir", out] if out_dir else []) + extra)
        printed = io.StringIO()
        try:
            with contextlib.redirect_stdout(printed):
                script.main()
        finally:
            sys.argv = argv
        got = {}
        for name in ("results_ccf.pkl", "eval_assoc.pkl"):
            with open(os.path.join(out if out_dir else res, name), "rb") as f:
                got[name] = f.read()
        written = {}
        for d, _, fs in os.walk(vis):
            for f in fs:
                with open(os.path.join(d, f), "rb") as fh:
                    written[os.path.relpath(os.path.join(d, f), vis)] = fh.read()
        return got, written, printed.getvalue().replace(vis, "<vis-dir>")


def golden():
    script = import_script()
    dataset, files, pickles = fixture()
    g = {"annot": np.frombuffer(json.dumps(dataset).encode(), np.uint8), "fps": np.int64(FPS)}
    for seq, d in pickles.items():
        g["pkl/" + seq] = np.frombuffer(pickle.dumps(d), np.uint8)
    for rel, b in files.items():
        g["in/" + rel] = np.frombuffer(b, np.uint8)
    for run, extra, out_dir in RUNS:
        got, written, printed = run_script(script, dataset, files, pickles, extra, out_dir)
        g[run + ".argv"] = np.asarray(extra + (["--out-dir"] if out_dir else []))
        g[run + ".printed"] = np.asarray(printed)
        for name, b in got.items():
            g[f"{run}.{name}"] = np.frombuffer(b, np.uint8)
        g[run + ".files"] = np.asarray(sorted(written))
        for rel, b in written.items():
            if rel.startswith("s2"):
                g[f"{run}/{rel}.sha256"] = np.frombuffer(hashlib.sha256(b).digest(), np.uint8)
                g[f"{run}/{rel}.len"] = np.int64(len(b))
            else:
                g[f"{run}/{rel}"] = np.frombuffer(b, np.uint8)
    return g


def main():
    path = os.path.join(ROOT, "tests", "golden", "streaming_eval_script.npz")
    np.savez_compressed(path, **golden())
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
