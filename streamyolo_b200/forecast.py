"""The sAP toolkit's offline forecast (sAP/forecast/pps_forecast_kf.py) on the device: the per-sequence pickles of the
streaming driver in, ``results_ccf.pkl`` (and ``eval_summary.pkl``) out.

    cd StreamYOLO/sAP                # for det.eval_ccf; elsewhere pass --no-eval
    python -m streamyolo_b200.forecast --data-root ... --annot-path .../val.json --fps 30 --eta 0 \\
        --forecast-before-assoc --in-dir <the driver's --out-dir> --out-dir ... --overwrite

It takes the script's arguments.  ``--forecast-before-assoc`` is required (the script asserts it), ``--assoc given`` and
``--vis-dir`` raise NotImplementedError, ``--forecast-rt-ub`` and ``--vis-scale`` are accepted and unused, as there.

Each sequence's detections are its pickle's ``results_parsed`` (ltrb fp32 boxes in frame pixels, scores, labels), what
both this package's ``python -m streamyolo_b200.sap`` and the reference driver write; ``results_raw``, which the script
prefers and then cannot parse for StreamYOLO's head output, is not read.  Boxes and scores are carried in fp32, as the
script's torch state carries the boxes: the driver's fp32 scores come out unchanged, float64 scores rounded to fp32 (and
sorted as such).  The query schedule (which detection each
annotated frame sees, :155-170) is computed here on the host; the association, the Kalman filter and the extrapolation of
every sequence run on the device, one CTA per sequence (``ops.forecast_sequences``).  AP stays on the host: the toolkit's
``det.eval_ccf`` scores the rows when it is importable.

One divergence: with ``--eta`` < 0 a frame can see a detection while its sequence has no track yet (every detection so
far was empty).  The script then emits the previous frame's rows again -- even the previous sequence's -- since its
``if len(kf_x)`` branch leaves ``bboxes_t3`` as it was; this pass emits nothing for such a frame.
"""
import argparse
import json
import os
import pickle
import time

import numpy as np
import torch

from . import ops, sap

GROUP = 64                         # sequences per device launch (one CTA each)


def parse_args(argv=None):
    """pps_forecast_kf.py's arguments (:32-51)"""
    p = argparse.ArgumentParser(prog="python -m streamyolo_b200.forecast")
    p.add_argument("--data-root", type=str, required=True)
    p.add_argument("--annot-path", type=str, required=True)
    p.add_argument("--split", type=str, default="val")
    p.add_argument("--fps", type=float, default=30)
    p.add_argument("--eta", type=float, default=0, help="eta >= -1")
    p.add_argument("--assoc", type=str, default="iou")
    p.add_argument("--match-iou-th", type=float, default=0.3)
    p.add_argument("--forecast-rt-ub", type=float, default=0)
    p.add_argument("--forecast-before-assoc", action="store_true", default=False)
    p.add_argument("--in-dir", type=str, required=True)
    p.add_argument("--out-dir", type=str, required=True)
    p.add_argument("--vis-dir", type=str, default=None)
    p.add_argument("--vis-scale", type=float, default=1)
    p.add_argument("--no-eval", action="store_true", default=False)
    p.add_argument("--overwrite", action="store_true", default=False)
    opts = p.parse_args(argv)
    if not opts.forecast_before_assoc:
        p.error("--forecast-before-assoc is required (the forecast after association is not implemented, as in "
                "pps_forecast_kf.py)")
    if opts.assoc == "given":
        raise NotImplementedError("--assoc given: association by given track ids is not implemented, as in pps_forecast_kf.py")
    if opts.vis_dir:
        raise NotImplementedError("--vis-dir: visualisation is not implemented")
    return opts


def schedule(n_frames, timestamps, input_fidx, eta, fps):
    """Which detection each annotated frame sees (:155-170): the last one with ``timestamps[k] <= (ii - eta) / fps``.
    -> per frame (k or -1, k is new to the sequence, dt of its update (frames since the previous new detection's input
    frame, 0 for the first), dt of the query ``ii - input_fidx[k]``)"""
    out, p1, prev = [], 0, None
    for ii in range(n_frames):
        t = (ii - eta) / fps
        while p1 < len(timestamps) and timestamps[p1] <= t:
            p1 += 1
        if p1 == 0:
            out.append((-1, False, 0, 0))
            continue
        k = p1 - 1
        new = k != prev
        dt_up = int(input_fidx[k] - input_fidx[prev]) if new and prev is not None else 0
        if new:
            prev = k
        out.append((k, new, dt_up, int(ii - input_fidx[k])))
    return out


class Plan:
    """The host half of the offline pass for a group of sequences: the detections to upload, the frame table of
    sy_forecast_sequences and each frame's output room.

      rows        fp32 [R, 7]: every new detection's rows (x1, y1, x2, y2, score, 1, label)
      det_start   int32 [D], det_n int32 [D]: detection k's rows
      frames      int32 [F, 6]: (k or -1, dt of the update, dt of the query, first output row, W, H)
      seq_frames  int32 [S + 1]
      n_rows      the output room: the sum over frames of the sequence's track count after the frame's detection (a new
                  detection's n when n > 0, else unchanged; 0 before the first and where the frame sees none)
      max_tracks  the largest n (at least 1)
      image_ids   per frame; label_src per frame: the detection whose labels and scores the frame's tracks carry (their
                  dtypes are the output's), or -1"""

    def __init__(self, sequences, eta, fps):
        rows, det_start, det_n, frames, seq_frames, image_ids, label_src, dtypes = [], [], [], [], [0], [], [], []
        r = n_rows = 0
        max_tracks = 1
        for seq in sequences:
            parsed = seq["results_parsed"]
            n_tracks, src = 0, -1
            for img, (d, new, dt_up, dt_q) in zip(seq["images"], schedule(len(seq["images"]), seq["timestamps"],
                                                                          seq["input_fidx"], eta, fps)):
                k = -1
                if d >= 0:
                    if new:
                        bb, sc, lb = (np.asarray(v) for v in parsed[d][:3])
                        n = len(bb)
                        blk = np.zeros((n, 7), np.float32)
                        if n:
                            blk[:, :4] = bb.reshape(n, 4)
                            blk[:, 4], blk[:, 5], blk[:, 6] = sc, 1.0, lb
                        rows.append(blk)
                        det_start.append(r)
                        det_n.append(n)
                        dtypes.append((sc.dtype, lb.dtype))
                        r += n
                        if n:
                            n_tracks, src = n, len(det_n) - 1
                            max_tracks = max(max_tracks, n)
                    k = len(det_n) - 1
                frames.append((k, dt_up, dt_q, n_rows, img["width"], img["height"]))
                image_ids.append(img["id"])
                label_src.append(src if k >= 0 else -1)
                n_rows += n_tracks if k >= 0 else 0
            seq_frames.append(len(frames))
        self.rows = np.concatenate(rows) if rows else np.zeros((0, 7), np.float32)
        self.det_start = np.asarray(det_start, np.int32)
        self.det_n = np.asarray(det_n, np.int32)
        self.frames = np.asarray(frames, np.int64).reshape(-1, 6)
        self.seq_frames = np.asarray(seq_frames, np.int32)
        self.n_rows, self.max_tracks = n_rows, max_tracks
        self.image_ids, self.label_src, self.dtypes = image_ids, label_src, dtypes
        self.names = [seq.get("name", f"sequence {q}") for q, seq in enumerate(sequences)]
        if self.frames.size and (np.abs(self.frames).max() > np.iinfo(np.int32).max or n_rows > np.iinfo(np.int32).max):
            raise ValueError("forecast: frame indices or output rows exceed int32")
        self.frames = self.frames.astype(np.int32)


def device_pass(plan, match_iou_th, device="cuda"):
    """sy_forecast_sequences on a Plan -> numpy (box [n_rows, 4], score, label, track, rows per frame)"""
    s = len(plan.seq_frames) - 1
    if not plan.det_n.size:
        return (np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros(0, np.int32), np.zeros(0, np.int32),
                np.zeros(len(plan.frames), np.int32))
    state = ops.ForecastState(s, plan.max_tracks, device)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    rows = plan.rows if len(plan.rows) else np.zeros((1, 7), np.float32)
    out = ops.forecast_sequences(state, up(rows), up(plan.det_start), up(plan.det_n), up(plan.frames),
                                 up(plan.seq_frames), plan.n_rows, match_iou_th)
    res = tuple(t.cpu().numpy() for t in out)
    over = state.meta[:, 3].nonzero().flatten().tolist()
    if over:                    # max_tracks is the largest detection, so this means the plan and the kernel disagree
        raise RuntimeError(f"forecast: {plan.names[over[0]]}: a detection has more rows than the plan's max_tracks")
    return res


def results_ccf(plan, out):
    """the script's result dicts (:279-287) from the device pass: per frame, its rows in track order"""
    box, score, label, _, nrows = out
    res = []
    for f, iid in enumerate(plan.image_ids):
        n = int(nrows[f])
        if not n:
            continue
        o = int(plan.frames[f, 3])
        sdt, ldt = plan.dtypes[plan.label_src[f]]
        b = box[o:o + n]
        sc, lb = score[o:o + n].astype(sdt), label[o:o + n].astype(ldt)
        for i in range(n):
            res.append({"image_id": iid, "bbox": b[i], "score": sc[i], "category_id": lb[i]})
    return res


def load_sequences(opts):
    """-> (dataset, per sequence {images, results_parsed, timestamps, input_fidx}) from the annotation file and the
    pickles of ``--in-dir``"""
    with open(opts.annot_path) as f:
        dataset = json.load(f)
    seqs = []
    for name, imgs in zip(dataset["sequences"], sap.sequences(dataset)):
        with open(os.path.join(opts.in_dir, name + ".pkl"), "rb") as f:
            r = pickle.load(f)
        seqs.append({"name": name, "images": imgs, "results_parsed": r["results_parsed"], "timestamps": r["timestamps"],
                     "input_fidx": r["input_fidx"]})
    return dataset, seqs


def _eval_ccf():
    try:
        from det import eval_ccf              # the toolkit's, importable from its sAP directory
        from pycocotools.coco import COCO
    except ImportError:
        return None
    return eval_ccf, COCO


def run(opts, device_pass=device_pass):
    """main() of the script (:99-322) -> results_ccf; ``device_pass`` is the device half (tests pass an emulation)"""
    ev = None
    if not opts.no_eval:
        ev = _eval_ccf()
        if ev is None:
            raise RuntimeError("forecast: det.eval_ccf is not importable (run from the toolkit's sAP directory with "
                               "pycocotools installed), or pass --no-eval")
    os.makedirs(opts.out_dir, exist_ok=True)
    _, seqs = load_sequences(opts)
    res = []
    t0 = time.perf_counter()
    for g in range(0, len(seqs), GROUP):
        plan = Plan(seqs[g:g + GROUP], opts.eta, opts.fps)
        res += results_ccf(plan, device_pass(plan, opts.match_iou_th))
    print(f"forecast: {len(seqs)} sequences, {len(res)} rows, {1e3 * (time.perf_counter() - t0):.3g} ms")
    sap.dump(os.path.join(opts.out_dir, "results_ccf.pkl"), res, opts.overwrite)
    if ev is not None:
        eval_ccf, COCO = ev
        summary = eval_ccf(COCO(opts.annot_path), res)
        sap.dump(os.path.join(opts.out_dir, "eval_summary.pkl"), summary, opts.overwrite)
    return res


def main(argv=None):
    return run(parse_args(argv))


if __name__ == "__main__":
    main()
