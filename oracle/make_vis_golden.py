"""Generate tests/golden/vis_script.npz and vis_record.npz -- TEST INFRASTRUCTURE.  Run in the build container, with the
StreamYOLO checkout at $STREAMYOLO_REF (default /root/reference), PIL and cv2 installed:

    python oracle/make_vis_golden.py

vis_script.npz: the UNMODIFIED sAP/vis/vis_det_th.py main() run under sys.argv on a fixture dataset in a temporary
directory, once on a result pickle (the default --score-th 0.3) and once with --gt; oracle/ref_shim stands in for
pycocotools, mmcv and skimage (whose find_boundaries only the mask branch calls).  The dataset has three sequences:
small frames of five sizes (cv2.imencode at q 90 of oracle/make_jpeg_encode_golden.py's content) and the 1200 x 1920
frame of tests/golden/jpeg_full_f420_q90.npz.  The result rows are streaming_eval.py's (float32 ltwh numpy rows, float32
scores, int32 labels), the annotations the same boxes as Python floats.  They cover overlapping boxes where the order
decides a pixel, reversed corners, zero-width, one-pixel and two-pixel boxes, boxes partly and wholly outside the frame and
touching each edge, half-integer coordinates, a score exactly float32(0.3) and one just below, a frame without rows, a
frame whose rows all fall below the threshold, and every palette entry.  Stored: the inputs (JPEG bytes, the annotation
file, the result pickle, the toolkit's class_palette entries for the fixture's coco_subset, as data), the files each run
wrote (bytes for the small frames, SHA-256 and length for the full-size one) and what it printed.

vis_record.npz: for StreamDetector(record_boxes=...): frames of three sizes, NMS rows as a tick holds them ([S, A, 7],
with ties at the threshold and at .5), and cv2.imencode(q 95) of oracle/vis_oracle.py's drawing of each stream's rows
(tick_rows, then draw with the palette in BGR order) on its frame."""
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

from oracle import vis_oracle as vo                         # noqa: E402
from oracle.make_jpeg_encode_golden import content          # noqa: E402

COCO_SUBSET = [0, 1, 2, 3, 4, 5, 6, 7, 9, 10, 11]           # 4 and 6 have no colour: 9 palette entries
SCORE_TH = 0.3
F32_TH = np.float32(SCORE_TH)
BELOW_TH = np.nextafter(F32_TH, np.float32(0))
SEQS = [("seqA", "dA", [(48, 64), (37, 53), (60, 80), (33, 65)]),
        ("seqB", "dB", [(24, 24), (60, 80), (37, 53)]),
        ("seqF", "dF", [(1200, 1920)])]


def _rows(k, h, w, rng, n_pal):
    """frame k's rows: (ltwh, score, label) with float coordinates"""
    if k == 0:       # overlapping, the order decides; reversed corners
        return [((5, 5, 25, 15), .9, 0), ((15, 10, 15, 15), .8, 1), ((20, 2, -10, 38), .7, 2), ((50, 40, -20, -15), .6, 3),
                ((12, 12, 3, 3), .5, 4)]
    if k == 1:       # zero-width, one- and two-pixel boxes; partly / wholly outside; each edge
        return [((10, 5, 0, 20), .9, 4), ((30, 30, 0, 0), .9, 5), ((40, 10, 1, 1), .9, 6), ((0, 10, 5, 5), .9, 7),
                ((47, 0, 5, 4), .9, 8), ((20, 32, 6, 4), .9, 0), ((-5, -5, 10, 10), .9, 1), ((60, 40, 5, 5), .9, 2),
                ((-20, -20, 5, 5), .9, 3), ((w - 1, h - 1, 4, 4), .9, 4), ((-1, 18, 1, 2), .9, 5), ((26, -1, 2, 0), .9, 6)]
    if k == 2:       # half-integers; the threshold exactly and just below
        return [((10.5, 20.5, 5.0, 6.0), F32_TH, 0), ((2.5, 3.5, 1.0, 1.0), .9, 1), ((2.3, 7.7, 0.2, 0.8), .9, 2),
                ((30.5, 40.5, 11.5, 0.5), .9, 3), ((50.5, 1.5, 20.0, 30.0), BELOW_TH, 4), ((60.5, 2.5, 7.5, 9.5), .95, 5)]
    if k == 3:       # no rows
        return []
    if k == 4:       # all below the threshold
        return [((2, 2, 10, 10), .1, 0), ((5, 5, 4, 4), BELOW_TH, 1)]
    n = 40 if h < 1000 else 24
    out = []
    for i in range(n):
        x, y = rng.uniform(-0.2 * w, w), rng.uniform(-0.2 * h, h)
        bw, bh = rng.uniform(0, 0.5 * w), rng.uniform(0, 0.5 * h)
        out.append(((round(x * 2) / 2, round(y * 2) / 2, round(bw * 2) / 2, round(bh * 2) / 2),
                    float(rng.uniform(0.2, 1.0)), i % n_pal))
    return out


def fixture(class_palette):
    """-> (annotation dict, {relative path: JPEG bytes} of the small frames, the result rows)"""
    import cv2
    rng = np.random.default_rng(7)
    n_pal = len([k for k in COCO_SUBSET if k in class_palette])
    images, anns, results, files = [], [], [], {}
    img_id = ann_id = 0
    k = 0
    for sid, (seq, d, sizes) in enumerate(SEQS):
        for fid, (h, w) in enumerate(sizes):
            name = f"{fid:06d}.jpg"
            if h < 1000:
                ok, enc = cv2.imencode(".jpg", content("smooth", h, w, 100 + k), [cv2.IMWRITE_JPEG_QUALITY, 90])
                files[f"{d}/{name}"] = enc.tobytes()
            images.append({"id": img_id, "sid": sid, "fid": fid, "name": name, "width": w, "height": h})
            for (ltwh, score, label) in _rows(k, h, w, rng, n_pal):
                results.append({"image_id": img_id, "bbox": np.asarray(ltwh, np.float32), "score": np.float32(score),
                                "category_id": np.int32(label)})
                anns.append({"id": ann_id, "image_id": img_id, "bbox": [float(v) for v in ltwh], "category_id": int(label),
                             "iscrowd": 0, "area": float(abs(ltwh[2] * ltwh[3]))})
                ann_id += 1
            img_id += 1
            k += 1
    dataset = {"images": images, "annotations": anns, "sequences": [s[0] for s in SEQS], "seq_dirs": [s[1] for s in SEQS],
               "categories": [{"id": c, "name": f"class{c}"} for c in COCO_SUBSET], "coco_subset": COCO_SUBSET}
    return dataset, files, results


def full_frame():
    return np.load(os.path.join(ROOT, "tests", "golden", "jpeg_full_f420_q90.npz"))["jpg"].tobytes()


def import_script():
    """sAP/vis/vis_det_th.py, imported as it is"""
    sys.path.insert(0, os.path.join(HERE, "ref_shim"))
    sys.path.insert(0, os.path.join(REF, "sAP"))
    import vis.vis_det_th as script
    return script


def run_script(script, dataset, files, results, extra):
    """the script's main() on the fixture -> ({relative output path: bytes}, printed text)"""
    with tempfile.TemporaryDirectory() as tmp:
        for rel, b in files.items():
            os.makedirs(os.path.join(tmp, "data", os.path.dirname(rel)), exist_ok=True)
            with open(os.path.join(tmp, "data", rel), "wb") as f:
                f.write(b)
        os.makedirs(os.path.join(tmp, "data", "dF"), exist_ok=True)
        with open(os.path.join(tmp, "data", "dF", "000000.jpg"), "wb") as f:
            f.write(full_frame())
        annot, res, out = (os.path.join(tmp, v) for v in ("annot.json", "res.pkl", "vis"))
        with open(annot, "w") as f:
            json.dump(dataset, f)
        with open(res, "wb") as f:
            pickle.dump(results, f)
        argv, sys.argv = sys.argv, ["vis_det_th.py", "--data-root", os.path.join(tmp, "data"), "--annot-path", annot,
                                    "--result-path", res, "--vis-dir", out, "--overwrite"] + extra
        printed = io.StringIO()
        try:
            with contextlib.redirect_stdout(printed):
                script.main()
        finally:
            sys.argv = argv
        written = {}
        for d, _, fs in os.walk(out):
            for f in fs:
                with open(os.path.join(d, f), "rb") as fh:
                    written[os.path.relpath(os.path.join(d, f), out)] = fh.read()
        return written, printed.getvalue().replace(out, "<vis-dir>")


def script_golden():
    script = import_script()
    keys = [k for k in COCO_SUBSET if k in script.class_palette]
    g = {"palette_keys": np.asarray(keys, np.int64),
         "palette_rgb": np.asarray([script.class_palette[k] for k in keys], np.uint8)}
    dataset, files, results = fixture(script.class_palette)
    g["annot"] = np.frombuffer(json.dumps(dataset).encode(), np.uint8)
    g["results"] = np.frombuffer(pickle.dumps(results), np.uint8)
    for rel, b in files.items():
        g["in/" + rel] = np.frombuffer(b, np.uint8)
    for run, extra in (("res", []), ("gt", ["--gt"])):
        written, printed = run_script(script, dataset, files, results, extra)
        g[run + ".printed"] = np.asarray(printed)
        g[run + ".files"] = np.asarray(sorted(written))
        for rel, b in written.items():
            if rel.startswith("seqF"):
                g[f"{run}/{rel}.sha256"] = np.frombuffer(hashlib.sha256(b).digest(), np.uint8)
                g[f"{run}/{rel}.len"] = np.int64(len(b))
            else:
                g[f"{run}/{rel}"] = np.frombuffer(b, np.uint8)
    return g


RECORD_SIZES = [(48, 64), (37, 53), (60, 80)]
RECORD_TH = 0.3


def record_rows(rng, h, w, a, n_pal, k):
    """[a, 7] NMS rows (x1, y1, x2, y2, obj, class_conf, class_pred) and their count"""
    det = np.zeros((a, 7), np.float32)
    n = a - 2 - k
    x1, y1 = rng.uniform(-8, w, n), rng.uniform(-8, h, n)
    det[:n, 0], det[:n, 1] = x1, y1
    det[:n, 2], det[:n, 3] = x1 + rng.uniform(0, 0.6 * w, n), y1 + rng.uniform(0, 0.6 * h, n)
    det[:n, :4] = np.where(rng.random((n, 4)) < 0.3, np.round(det[:n, :4] * 2) / 2, det[:n, :4])   # .5 ties
    det[:n, 4], det[:n, 5] = rng.uniform(0.2, 1, n), rng.uniform(0.3, 1, n)
    det[0, 4], det[0, 5] = F32_TH, 1.0                      # exactly the threshold
    det[1, 4], det[1, 5] = BELOW_TH, 1.0                    # just below
    det[2, 4], det[2, 5] = np.float32(0.5), np.float32(0.6)     # 0.3 after the fp32 product, or not
    det[:n, 6] = np.arange(n) % n_pal
    return det, n


def record_golden():
    import cv2
    rng = np.random.default_rng(11)
    palette = rng.integers(0, 256, (9, 3)).astype(np.uint8)                 # any colours, stored as data
    a = 24
    g = {"palette_rgb": palette, "score_th": np.float64(RECORD_TH), "quality": np.int64(95)}
    dets, counts = np.zeros((len(RECORD_SIZES), a, 7), np.float32), np.zeros(len(RECORD_SIZES), np.int32)
    for s, (h, w) in enumerate(RECORD_SIZES):
        frame = content("smooth" if s != 1 else "noise", h, w, 200 + s)
        det, n = record_rows(rng, h, w, a, len(palette), s)
        dets[s], counts[s] = det, n
        boxes, labels = vo.tick_rows(det, n, RECORD_TH)
        drawn = vo.draw(frame, boxes, labels, palette[:, ::-1])
        g[f"frame{s}"] = frame
        g[f"jpg{s}"] = np.frombuffer(cv2.imencode(".jpg", drawn, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes(), np.uint8)
    g["det"], g["count"] = dets, counts
    return g


def main():
    for name, g in (("vis_script", script_golden()), ("vis_record", record_golden())):
        path = os.path.join(ROOT, "tests", "golden", name + ".npz")
        np.savez_compressed(path, **g)
        print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
