"""The sAP toolkit's streaming evaluation (sAP/det/streaming_eval.py) with its --vis-dir frames drawn on the device:
every annotated frame paired with the last output at or before its time, the pairs written as the script's pickles and
scored by the toolkit's own ``det.eval_ccf`` (pycocotools), and with --vis-dir each frame written as a JPEG file
byte-identical to the script's.

    cd StreamYOLO/sAP                # det.eval_ccf is imported from here, as the script's sys.path lines find it
    python -m streamyolo_b200.streaming_eval --data-root ... --annot-path .../val.json --fps 30 --eta 0 \\
        --result-dir ... [--out-dir ...] [--vis-dir ... [--vis-scale 0.5]] [--no-class-mapping] [--no-eval] \\
        [--use-parsed] [--eval-mask] [--overwrite]

It takes the script's arguments and writes the same files:
  results_ccf.pkl, eval_assoc.pkl   byte-identical: the pairing (:69-148) is the script's own numpy and Python
                                    expressions on the pickles' own objects (the frame order of the annotation's images,
                                    ``(ii - eta) / fps``, ``results_raw`` unless --use-parsed or absent, parse_det_result
                                    with the annotation's ``coco_mapping`` unless --no-class-mapping, ltrb -> ltwh)
  eval_summary.pkl (_mask.pkl)      what the toolkit's det.eval_ccf returns; nothing is scored here
  <vis-dir>/<seq>/<name>.jpg        what vis_det (sAP/det/__init__.py:103-178) writes through PIL
each under the script's --overwrite / existing-file rule, in --out-dir (by default --result-dir), and it prints the
script's lines.  pycocotools' own loading messages appear only when it scores (--no-eval needs neither pycocotools nor
the toolkit).

--vis-dir.  Per frame the host takes vis_det's numpy steps on the paired rows (``out_scale * bboxes``, then
``.round().astype(np.int32)``, half to even; score_th is 0, so no row is dropped) and rasterises the labels
``"<class>|<score:.02f>"`` with cv2.putText (FONT_HERSHEY_COMPLEX, scale 0.5, thickness 1, LINE_8, origin (x1, y1 - 2))
into a one-channel canvas of the output frame's size: the glyph strokes exist only inside cv2, and clipping at the
frame's edges changes them, so no stamp of a glyph or a string could be exact.  The lit pixels go to the device as a
list.  The device decodes batches of frames (data.decode_jpeg_sized, which equals PIL's decode of these files), resizes
them at --vis-scale other than 1 to mmcv.imrescale's size (data.resize_sized, cv2's INTER_LINEAR bit for bit), draws the
1-pixel boxes and the label pixels in green (data.draw_outlines, sy_draw_outlines) and encodes at quality 75, PIL's
default (data.encode_jpeg).  A frame with no rows is re-encoded unchanged, as vis_det's early imwrite does.  A thread
pool reads the files, renders the labels (one reused canvas per thread, cleared where it was written) and writes the
files while the device works.  cv2 is imported only for --vis-dir.

Refused before anything is written:
  --vis-dir with a frame to draw whose rows carry masks   NotImplementedError (vis_det's mask branch draws colours from
                                                          numpy's global random state)
  --vis-dir with a frame to draw whose rows carry tracks  NotImplementedError (vis_track)
  --vis-scale <= 0 with --vis-dir                         ValueError, as mmcv.imrescale raises
  a missing pickle or frame, a label outside the annotation's classes   what the script raises (FileNotFoundError,
                                                          IndexError)
A frame the device decoder refuses raises RuntimeError naming the file and the reason.
"""
import argparse
import errno
import json
import os
import pickle
import sys
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import data
from .contrast import sof_size
from .vis import _pow2, _read, _write

QUALITY = 75              # PIL's default JPEG quality, what vis_det's imwrite saves with
BATCH = 8                 # frames per device batch
FONT_SCALE = 0.5          # vis_det's label font: FONT_HERSHEY_COMPLEX at 0.5, thickness 1, LINE_8
TEXT_PAD = 2              # pixels scanned around cv2.getTextSize's box of a label (its strokes stay inside the box)


def parse_args(argv=None):
    """streaming_eval.py's arguments (:27-43)"""
    p = argparse.ArgumentParser(prog="python -m streamyolo_b200.streaming_eval")
    p.add_argument("--data-root", type=str, required=True)
    p.add_argument("--annot-path", type=str, required=True)
    p.add_argument("--fps", type=float, default=30)
    p.add_argument("--eta", type=float, default=0, help="eta >= -1")
    p.add_argument("--result-dir", type=str, required=True)
    p.add_argument("--out-dir", type=str, default=None)
    p.add_argument("--vis-dir", type=str, default=None)
    p.add_argument("--vis-scale", type=float, default=1)
    p.add_argument("--no-class-mapping", action="store_true", default=False)
    p.add_argument("--no-eval", action="store_true", default=False)
    p.add_argument("--use-parsed", action="store_true", default=False)
    p.add_argument("--eval-mask", action="store_true", default=False)
    p.add_argument("--overwrite", action="store_true", default=False)
    return p.parse_args(argv)


def ltrb2ltwh(bboxes):
    """the toolkit's util.bbox.ltrb2ltwh: a copy with x2, y2 turned into w, h, on the array's own dtype"""
    bboxes = bboxes.copy()
    if len(bboxes):
        if bboxes.ndim == 1:
            bboxes[2:] -= bboxes[:2]
        else:
            bboxes[:, 2:] -= bboxes[:, :2]
    return bboxes


def parse_det_result(result, class_mapping, n_class):
    """the toolkit's det.parse_det_result(result, class_mapping, n_class) -> (bboxes, scores, labels, masks): labels
    mapped through ``class_mapping`` and rows mapped to n_class or beyond dropped; empty float32 boxes and scores when no
    row is left"""
    if len(result) > 2:
        bboxes_scores, labels, masks = result
    else:
        (bboxes_scores, labels), masks = result, None
    if class_mapping is not None:
        labels = class_mapping[labels]
        sel = labels < n_class
        bboxes_scores, labels = bboxes_scores[sel], labels[sel]
        if masks is not None:
            masks = masks[sel]
    if not len(labels):
        return np.empty((0, 4), dtype=np.float32), np.empty((0,), dtype=np.float32), labels, masks
    return bboxes_scores[:, :4], bboxes_scores[:, 4], labels, masks


class VisFrame:
    """one frame to draw: its file, output path, int32 boxes [k, 4] in output pixels and labels [(text, origin)]"""

    def __init__(self, path, out, boxes, texts):
        self.path, self.out, self.boxes, self.texts = path, out, boxes, texts
        self.hw = self.out_hw = self.points = None        # set once the file is read (render)


def vis_marks(bboxes, labels, class_names, masks, scores, out_scale, where):
    """vis_det's host steps (sAP/det/__init__.py:110-174) -> (int32 boxes [k, 4], [(label text, putText origin)]);
    k = 0 where it writes the frame unchanged"""
    bboxes = np.asarray(bboxes)
    labels = np.asarray(labels)
    if len(bboxes) == 0:
        return np.zeros((0, 4), np.int32), []
    if masks is not None:
        raise NotImplementedError(f"streaming_eval: {where}: --vis-dir with results that carry masks (vis_det's mask "
                                  "branch, whose colours come from numpy's global random state) is not implemented")
    if out_scale != 1:
        bboxes = out_scale * bboxes
    bboxes = bboxes.round().astype(np.int32)
    texts = []
    for i, (bbox, label) in enumerate(zip(bboxes, labels)):
        text = class_names[label]
        if scores is not None:
            text += f"|{scores[i]:.02f}"
        texts.append((text, (bbox[0], bbox[1] - 2)))
    return bboxes, texts


class Pairing:
    """main()'s loop (:62-148): results_ccf, the association counts and, with --vis-dir, the frames to draw"""

    def __init__(self, results_ccf, miss, in_time, mismatch, frames):
        self.results_ccf, self.miss, self.in_time, self.mismatch, self.frames = (results_ccf, miss, in_time, mismatch,
                                                                                 frames)


def pair(opts, dataset, imgs):
    """The script's pairing of every annotated frame with the last output whose timestamp is <= (ii - eta) / fps, on
    the annotation (``dataset``, ``imgs`` = pycocotools' db.imgs) and the pickles of --result-dir.  Every refusal is
    raised here, before any file is written."""
    vis_out = bool(opts.vis_dir)
    class_names = [c["name"] for c in dataset["categories"]]
    n_class = len(class_names)
    coco_mapping = None if opts.no_class_mapping else dataset.get("coco_mapping", None)
    if coco_mapping is not None:
        coco_mapping = np.asarray(coco_mapping)
    seqs, seq_dirs = dataset["sequences"], dataset["seq_dirs"]
    results_ccf, frames = [], []
    in_time = miss = mismatch = 0
    for sid, seq in enumerate(seqs):
        frame_list = [img for img in imgs.values() if img["sid"] == sid]
        with open(os.path.join(opts.result_dir, seq + ".pkl"), "rb") as f:
            results = pickle.load(f)
        results_raw = None
        if opts.use_parsed:
            results_parsed = results["results_parsed"]
        else:
            results_raw = results.get("results_raw", None)
            if results_raw is None:
                results_parsed = results["results_parsed"]
        timestamps = results["timestamps"]
        input_fidx = results["input_fidx"]
        tidx_p1 = 0
        for ii, img in enumerate(frame_list):
            t = (ii - opts.eta) / opts.fps
            while tidx_p1 < len(timestamps) and timestamps[tidx_p1] <= t:
                tidx_p1 += 1
            if tidx_p1 == 0:
                miss += 1
                bboxes, scores, labels = [], [], []
                masks, tracks = None, None
            else:
                tidx = tidx_p1 - 1
                ifidx = input_fidx[tidx]
                in_time += int(ii == ifidx)
                mismatch += ii - ifidx
                if opts.use_parsed or results_raw is None:
                    result = results_parsed[tidx]
                    bboxes, scores, labels, masks = result[:4]
                    tracks = result[4] if len(result) > 4 else None
                else:
                    bboxes, scores, labels, masks = parse_det_result(results_raw[tidx], coco_mapping, n_class)
                    tracks = None
            if vis_out:
                img_path = os.path.join(opts.data_root, seq_dirs[sid], img["name"])
                if not os.path.isfile(img_path):                        # the script's imread runs for every frame
                    raise FileNotFoundError(errno.ENOENT, os.strerror(errno.ENOENT), img_path)
                vis_path = os.path.join(opts.vis_dir, seq, img["name"][:-3] + "jpg")
                if opts.overwrite or not os.path.isfile(vis_path):
                    where = f"{seq}/{img['name']}"
                    if tracks is not None:
                        raise NotImplementedError(f"streaming_eval: {where}: --vis-dir with results that carry tracks "
                                                  "(vis_track) is not implemented")
                    boxes, texts = vis_marks(bboxes, labels, class_names, masks, scores, opts.vis_scale, where)
                    frames.append(VisFrame(img_path, vis_path, boxes, texts))
            n = len(bboxes)
            if n:
                bboxes_ltwh = ltrb2ltwh(bboxes)
            for i in range(n):
                result_dict = {
                    "image_id": img["id"],
                    "bbox": bboxes_ltwh[i],
                    "score": scores[i],
                    "category_id": labels[i],
                }
                if masks is not None:
                    result_dict["segmentation"] = masks[i]
                results_ccf.append(result_dict)
    return Pairing(results_ccf, miss, in_time, mismatch, frames)


_canvases = threading.local()


def text_points(texts, hw):
    """The pixels cv2.putText lights for vis_det's labels ``texts`` on an ``hw`` frame -> sorted int32 indices
    y * w + x.  Each thread keeps one canvas per size and clears only the boxes it scanned."""
    import cv2
    h, w = hw
    if not texts:
        return np.zeros((0,), np.int32)
    canvas = _canvases.__dict__.get(hw)
    if canvas is None:
        canvas = _canvases.__dict__[hw] = np.zeros(hw, np.uint8)
    boxes = []
    for text, org in texts:
        cv2.putText(canvas, text, org, cv2.FONT_HERSHEY_COMPLEX, FONT_SCALE, 255, 1, cv2.LINE_8)
        (tw, th), base = cv2.getTextSize(text, cv2.FONT_HERSHEY_COMPLEX, FONT_SCALE, 1)
        x, y = int(org[0]), int(org[1])
        r0, r1 = max(y - th - TEXT_PAD, 0), min(y + base + TEXT_PAD + 1, h)
        c0, c1 = max(x - TEXT_PAD, 0), min(x + tw + TEXT_PAD + 1, w)
        if r0 < r1 and c0 < c1:
            boxes.append((r0, r1, c0, c1))
    found = []
    for r0, r1, c0, c1 in boxes:
        roi = canvas[r0:r1, c0:c1]
        ys, xs = np.nonzero(roi)
        if len(ys):
            found.append((ys + r0).astype(np.int64) * w + (xs + c0))
            roi[ys, xs] = 0
    if not found:
        return np.zeros((0,), np.int32)
    return np.unique(np.concatenate(found)).astype(np.int32)


def render(frame, scale):
    """the host half of one frame, in a pool thread: its file's bytes, its size (the SOF header's), its output size and
    its label pixels"""
    b = _read(frame.path)
    hw = sof_size(b)
    if hw is None or min(hw) < 1:
        raise RuntimeError(f"streaming_eval: {frame.path} did not decode: {data.JPEG_STATUS[1]}")
    frame.hw = hw
    frame.out_hw = hw if scale == 1 else data.imrescale_size(hw[0], hw[1], scale)
    frame.points = text_points(frame.texts, frame.out_hw)
    return b


def device_pass(files, frames, scale, device="cuda"):
    """The files' bytes of a batch of rendered VisFrames -> the output files: decode (PIL's pixels), resize at a scale
    other than 1, draw, encode at quality 75"""
    sizes, out_sizes = [f.hw for f in frames], [f.out_hw for f in frames]
    mh, mw = max(h for h, _ in sizes), max(w for _, w in sizes)
    rows, lengths = data.pack_jpeg(files, _pow2(max(len(b) for b in files)))
    img, status = data.decode_jpeg_sized(torch.from_numpy(rows).to(device), torch.from_numpy(lengths).to(device), sizes,
                                         (mh, mw))
    if scale != 1:
        img = data.resize_sized(img, sizes, out_sizes)
    data.draw_outlines(img, [f.boxes for f in frames], [f.points for f in frames], out_sizes)
    for f, s in zip(frames, status.tolist()):
        if s != 0:
            raise RuntimeError(f"streaming_eval: {f.path} did not decode: {data.JPEG_STATUS.get(s, f'status {s}')}")
    return data.encode_jpeg(img, QUALITY, out_sizes)


def write_vis(frames, scale, device_pass=device_pass, workers=8):
    """Every VisFrame through the device in batches of BATCH, the next batch read and rendered while one runs"""
    batches = [frames[k:k + BATCH] for k in range(0, len(frames), BATCH)]
    with ThreadPoolExecutor(max_workers=workers) as pool:
        def submit(batch):
            return [pool.submit(render, f, scale) for f in batch]
        pending = [submit(batches[0])] if batches else []
        writes = []
        for k, batch in enumerate(batches):
            if k + 1 < len(batches):
                pending.append(submit(batches[k + 1]))
            files = [r.result() for r in pending[k]]
            pending[k] = None
            out = device_pass(files, batch, scale)
            writes += [pool.submit(_write, f.out, b) for f, b in zip(batch, out)]
        for w in writes:
            w.result()
    return len(frames)


def _dump(path, obj, overwrite):
    """the script's ``if opts.overwrite or not isfile(out_path): pickle.dump(obj, open(out_path, 'wb'))``"""
    if overwrite or not os.path.isfile(path):
        with open(path, "wb") as f:
            pickle.dump(obj, f)


def toolkit():
    """(det.eval_ccf, pycocotools.coco.COCO), the toolkit's det module found as the script's ``sys.path.insert(0, '..');
    sys.path.insert(0, '.')`` finds it; RuntimeError when either is missing"""
    for d in ("..", "."):
        if d not in sys.path:
            sys.path.insert(0, d)
    try:
        from det import eval_ccf
        from pycocotools.coco import COCO
    except ImportError as e:
        raise RuntimeError(f"streaming_eval: scoring needs the toolkit's det.eval_ccf and pycocotools ({e}): run from "
                           "the toolkit's sAP directory with pycocotools installed, or pass --no-eval") from e
    return eval_ccf, COCO


def run(opts, device_pass=device_pass):
    """The script's main() with the --vis-dir frames drawn on the device -> the Pairing; ``device_pass`` is the device
    half (tests pass an emulation)"""
    vis_out = bool(opts.vis_dir)
    if vis_out:
        if not opts.vis_scale > 0:
            raise ValueError(f"streaming_eval: --vis-scale {opts.vis_scale}: Invalid scale {opts.vis_scale}, must be "
                             "positive.")
        try:
            import cv2  # noqa: F401
        except ImportError as e:
            raise RuntimeError("streaming_eval: --vis-dir renders the labels with cv2.putText, and cv2 is not "
                               f"installed ({e})") from e
    db = None
    if not opts.no_eval:
        eval_ccf, COCO = toolkit()
        db = COCO(opts.annot_path)
        dataset, imgs = db.dataset, db.imgs
    else:
        with open(opts.annot_path) as f:
            dataset = json.load(f)
        imgs = {}
        for img in dataset["images"]:                 # pycocotools' db.imgs
            imgs[img["id"]] = img
    print("Pairing the output with the ground truth")
    p = pair(opts, dataset, imgs)
    out_dir = opts.out_dir if opts.out_dir else opts.result_dir
    if opts.out_dir:
        os.makedirs(out_dir, exist_ok=True)
    if vis_out:
        os.makedirs(opts.vis_dir, exist_ok=True)
        write_vis(p.frames, opts.vis_scale, device_pass)
    _dump(os.path.join(out_dir, "results_ccf.pkl"), p.results_ccf, opts.overwrite)
    _dump(os.path.join(out_dir, "eval_assoc.pkl"), {"miss": p.miss, "in_time": p.in_time, "mismatch": p.mismatch},
          opts.overwrite)
    if db is not None:
        _dump(os.path.join(out_dir, "eval_summary.pkl"), eval_ccf(db, p.results_ccf), opts.overwrite)
        if opts.eval_mask:
            print("Evaluating instance segmentation")
            _dump(os.path.join(out_dir, "eval_summary_mask.pkl"), eval_ccf(db, p.results_ccf, iou_type="segm"),
                  opts.overwrite)
    if vis_out:
        print(f'python vis/make_videos.py "{opts.vis_dir}" --fps {opts.fps}')
    return p


def main(argv=None):
    return run(parse_args(argv))


if __name__ == "__main__":
    main()
