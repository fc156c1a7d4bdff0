"""The sAP toolkit's detection visualisation (sAP/vis/vis_det_th.py) on the device: every frame of every sequence with
its detections drawn as boxes in class colours, written as JPEG files byte-identical to the script's.

    cd StreamYOLO/sAP                # the palette is read from the toolkit's vis/vis_det_th.py
    python -m streamyolo_b200.vis --data-root ... --annot-path .../val.json --result-path .../results_ccf.pkl \\
        --vis-dir ... [--seq 3 | --seq <name>] [--score-th 0.3] [--gt] [--make-video] [--overwrite]

It takes the script's arguments and writes the same files: ``<vis-dir>/<sequence>/%06d.jpg`` (the frame's index in its
sequence, from 1), what the script writes through PIL (``Image.fromarray(rgb).save(path)``, which is
``cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, 75])`` byte for byte), with vis_obj_fancy's boxes drawn
(show_label=False, show_score=False: no text).  Frames whose file exists are skipped without ``--overwrite``;
``--make-video`` runs make_videos_numbered.py's ffmpeg command per sequence; the closing line is the script's.

The host selects each frame's rows, turns ltwh into ltrb, applies the score threshold and rounds, with the script's own
numpy expressions on the rows' own dtypes (:228-242, :75-97: fp32 result rows and fp64 ``--gt`` annotations round their
ties differently, so this is never redone on the device).  The device decodes batches of frames (data.decode_jpeg_sized,
cv2.imread bit for bit), draws the boxes (data.draw_boxes, sy_draw_boxes) and encodes the files at quality 75
(data.encode_jpeg); a thread pool reads and writes the files while the device works.  A frame with no rows left is
re-encoded unchanged, as the script's early ``imwrite`` does (:89-92).

The colours are the toolkit's: ``class_palette`` is read (with ``ast``, never executed) from ``vis/vis_det_th.py`` under
``.`` or ``..``, the directories the script's own ``sys.path`` lines search, and ``color_palette`` is built from the
annotation file's ``coco_subset`` as the script builds it (:200-202).

Refused before anything is read or written:
  --vis-scale other than 1   ValueError.  The script calls ``cv2.resize(img, fx=, fy=, interpolation=)`` without
                             ``dsize``, which cv2 4.x rejects (cv2 4.13: "resize() missing required argument 'dsize'"),
                             so the script cannot run with it either.
  rows with 'segmentation'   NotImplementedError (vis_obj_fancy's mask branch)
  a label outside the palette  IndexError, as the script's ``color_palette[label]`` raises; negative labels too, which the
                             script's list index would wrap to the end of the palette.
A frame the device decoder refuses (not a baseline/progressive JPEG it reads, or not of the annotation's size) raises
RuntimeError naming its file and the reason.
"""
import argparse
import ast
import json
import os
import pickle
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import data

QUALITY = 75              # PIL's default JPEG quality, what the script's imwrite saves with
BATCH = 8                 # frames per device batch


def parse_args(argv=None):
    """vis_det_th.py's arguments (:25-40)"""
    p = argparse.ArgumentParser(prog="python -m streamyolo_b200.vis")
    p.add_argument("--data-root", type=str, required=True)
    p.add_argument("--annot-path", type=str, required=True)
    p.add_argument("--fps", type=float, default=30)
    p.add_argument("--result-path", type=str, default=None)
    p.add_argument("--gt", action="store_true", default=False)
    p.add_argument("--vis-dir", type=str, required=True)
    p.add_argument("--vis-scale", type=float, default=1)
    p.add_argument("--seq", type=str, default=None)
    p.add_argument("--score-th", type=float, default=0.3)
    p.add_argument("--make-video", action="store_true", default=False)
    p.add_argument("--overwrite", action="store_true", default=False)
    return p.parse_args(argv)


def read_class_palette(search=(".", "..")):
    """The toolkit's ``class_palette`` dict literal, read with ``ast`` from ``<dir>/vis/vis_det_th.py`` for the first of
    ``search`` that has it; RuntimeError when none does"""
    for d in search:
        path = os.path.join(d, "vis", "vis_det_th.py")
        if not os.path.isfile(path):
            continue
        with open(path) as f:
            tree = ast.parse(f.read(), path)
        for node in tree.body:
            if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "class_palette" for t in node.targets):
                return ast.literal_eval(node.value)
        raise RuntimeError(f"vis: {path} has no class_palette")
    raise RuntimeError("vis: the toolkit's vis/vis_det_th.py (its class_palette) was not found under "
                       f"{' or '.join(repr(d) for d in search)}: run from the toolkit's sAP directory")


def color_palette(class_palette, dataset):
    """vis_det_th.py:196, 200-202: the colours of the annotation file's classes, (R, G, B) each"""
    coco_subset = np.asarray(dataset["coco_subset"])
    return [class_palette[k] for k in coco_subset if k in class_palette]


def frame_rows(dets, score_th, gt):
    """One frame's rows -> the (int32 boxes [k, 4], labels [k]) vis_obj_fancy draws, k = 0 where it writes the frame
    unchanged: vis_det_th.py:229-242 and vis_obj_fancy :75-97, the same numpy expressions on the rows' own dtypes"""
    bboxes = np.array([d["bbox"] for d in dets])
    if len(bboxes):
        bboxes[:, 2:] += bboxes[:, :2]
        if any("segmentation" in d for d in dets):
            raise NotImplementedError("vis: rows with 'segmentation' take vis_obj_fancy's mask branch, which is not "
                                      "implemented")
    labels = np.array([d["category_id"] for d in dets])
    scores = None if gt else np.array([d["score"] for d in dets])
    empty = len(bboxes) == 0
    if not empty and scores is not None and score_th > 0:
        sel = scores >= score_th
        bboxes, labels = bboxes[sel], labels[sel]
        empty = len(bboxes) == 0
    if empty:
        return np.zeros((0, 4), np.int32), np.zeros((0,), np.int32)
    return bboxes.round().astype(np.int32), labels


class Frame:
    """one frame to draw: its file, (h, w) by the annotation, output path and rows"""

    def __init__(self, path, hw, out, boxes, labels):
        self.path, self.hw, self.out, self.boxes, self.labels = path, hw, out, boxes, labels


def plan(opts, dataset, results, n_colors):
    """main() of the script (:192-254) without the drawing -> [(sequence name, its frames to write)], every refusal
    raised here, before any file is read or written"""
    if opts.vis_scale != 1:
        raise ValueError(f"vis: --vis-scale {opts.vis_scale}: only 1 is supported (the script's cv2.resize call has no "
                         "dsize, which cv2 4.x rejects)")
    seqs, seq_dirs = dataset["sequences"], dataset["seq_dirs"]
    imgs = {}
    for img in dataset.get("images", []):           # pycocotools' db.imgs
        imgs[img["id"]] = img
    by_image = {}
    for r in results:
        by_image.setdefault(r["image_id"], []).append(r)
    if opts.seq is not None:
        idx = int(opts.seq) if opts.seq.isdigit() else seqs.index(opts.seq)
        seqs = [seqs[idx]]
    else:
        idx = None
    out = []
    for sid, seq in enumerate(seqs):
        if idx is not None:
            sid = idx
        frames = []
        for ii, img in enumerate(v for v in imgs.values() if v["sid"] == sid):
            vis_path = os.path.join(opts.vis_dir, seq, "%06d.jpg" % (ii + 1))
            dets = by_image.get(img["id"], [])
            boxes, labels = frame_rows(dets, opts.score_th, opts.gt)
            if not (opts.overwrite or not os.path.isfile(vis_path)):
                continue
            bad = [int(v) for v in np.asarray(labels).reshape(-1) if not 0 <= v < n_colors]
            if bad:
                raise IndexError(f"vis: {img['name']}: label {bad[0]} is outside the palette of {n_colors} colours")
            frames.append(Frame(os.path.join(opts.data_root, seq_dirs[sid], img["name"]),
                                (int(img["height"]), int(img["width"])), vis_path, boxes, labels))
        out.append((seq, frames))
    return out


def _pow2(n):
    return 1 << max(16, int(n - 1).bit_length())


def device_pass(files, frames, palette_bgr, device="cuda"):
    """The files' bytes of a batch of Frames -> the output files: decode (cv2.imread), draw, encode at quality 75"""
    sizes = [f.hw for f in frames]
    mh, mw = max(h for h, _ in sizes), max(w for _, w in sizes)
    rows, lengths = data.pack_jpeg(files, _pow2(max(len(b) for b in files)))
    img, status = data.decode_jpeg_sized(torch.from_numpy(rows).to(device), torch.from_numpy(lengths).to(device), sizes,
                                         (mh, mw))
    data.draw_boxes(img, [f.boxes for f in frames], [np.asarray(f.labels, np.int64) for f in frames], None,
                    palette_bgr, sizes)
    for f, s in zip(frames, status.tolist()):
        if s != 0:
            raise RuntimeError(f"vis: {f.path} did not decode: {data.JPEG_STATUS.get(s, f'status {s}')}")
    return data.encode_jpeg(img, QUALITY, sizes)


def make_video(d, fps):
    """make_videos_numbered.py's worker_func: the frames of directory ``d`` into ``d + '.mp4'``"""
    subprocess.run(
        ["ffmpeg", "-loglevel", "panic", "-y", "-framerate", str(fps), "-i", os.path.join(d, "%06d.jpg"), "-c:v",
         "libx264", "-pix_fmt", "yuv420p", "-vf", "pad=width=ceil(iw/2)*2:height=ceil(ih/2)*2", os.path.join(d + ".mp4")],
        check=True)


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _write(path, b):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(b)


def run(opts, device_pass=device_pass, search=(".", "..")):
    """The script's main() with the drawing on the device -> the number of files written; ``device_pass`` is the
    device half (tests pass an emulation)"""
    class_palette = read_class_palette(search)
    with open(opts.annot_path) as f:
        dataset = json.load(f)
    palette = color_palette(class_palette, dataset)
    if opts.gt:
        results = dataset["annotations"]
    else:
        with open(opts.result_path, "rb") as f:
            results = pickle.load(f)
    seqs = plan(opts, dataset, results, len(palette))
    os.makedirs(opts.vis_dir, exist_ok=True)
    palette_bgr = np.asarray(palette, np.uint8).reshape(-1, 3)[:, ::-1].copy() if palette else np.zeros((1, 3), np.uint8)
    written = 0
    with ThreadPoolExecutor(max_workers=4) as pool:
        for seq, frames in seqs:
            batches = [frames[k:k + BATCH] for k in range(0, len(frames), BATCH)]
            reads = [pool.submit(lambda b: [_read(f.path) for f in b], b) for b in batches[:1]]
            writes = []
            for k, batch in enumerate(batches):
                if k + 1 < len(batches):
                    reads.append(pool.submit(lambda b: [_read(f.path) for f in b], batches[k + 1]))
                files = device_pass(reads[k].result(), batch, palette_bgr)
                reads[k] = None
                writes += [pool.submit(_write, f.out, b) for f, b in zip(batch, files)]
            for w in writes:
                w.result()
            written += len(frames)
            if opts.make_video:
                seq_dir_out = os.path.join(opts.vis_dir, seq)
                if opts.overwrite or not os.path.isfile(seq_dir_out + ".mp4"):
                    make_video(seq_dir_out, opts.fps)
    if not opts.make_video:
        print(f'python vis/make_videos_numbered.py "{opts.vis_dir}" --fps {opts.fps}')
    return written


def main(argv=None):
    return run(parse_args(argv))


if __name__ == "__main__":
    main()
