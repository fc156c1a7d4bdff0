"""Generate tests/golden/forecast_eta0.npz and forecast_etam1.npz -- TEST INFRASTRUCTURE.  Run in the build container,
with the StreamYOLO checkout at $STREAMYOLO_REF (default /root/reference):

    python oracle/make_forecast_golden.py

Runs the UNMODIFIED sAP/forecast/pps_forecast_kf.py main() with --forecast-before-assoc --no-eval on synthetic sequences
(a small annotation json and driver pickles without ``results_raw``), on top of the stand-ins of oracle/ref_shim
(pycocotools' COCO image table, mask.iou, a COCOeval that refuses, an empty mmcv) and ``np.int = int`` for
extrap_clean_up.  ``track.iou_assoc`` is wrapped, not changed, to record every association decision and its margins.

Each file holds the inputs (``annot`` json text; per detection its sequence, boxes, scores, labels; per sequence
timestamps and input_fidx), the reference's results_ccf rows, and the decisions.  The sequences cover: det_stride gaps
(dt > 1); an empty detection at a sequence start and one mid-sequence after matches (keeps n_matched); a full restart
with no match; a label mismatch; an IoU of exactly 0.3 (inclusive) and equal IoUs from two tracks (the later wins), both
with exactly representable boxes; dropped tracks; boxes clipped at each border and removed by the 75-pixel rule; several
sequences.  With eta = -1 the last sequence starts with an empty detection that its first frame already sees, where the
reference emits the previous sequence's last rows again (the documented divergence).  Every other decision keeps its IoU
margins (to 0.3 and to the runner-up) >= 1e-4; the seeded search reruns to the same files."""
import json
import os
import pickle
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("STREAMYOLO_REF", "/root/reference")
W_IMG, H_IMG, FPS = 640, 480, 30.0


def crafted():
    """hand-built detections of sequence 0 (ltrb fp32, scores, labels) at input frames 0, 2, 4, ...: see the module doc"""
    f = np.float32
    D = []
    # 0: first detection of the sequence is empty
    D.append((np.zeros((0, 4), f), np.zeros(0, f), np.zeros(0, np.int32)))
    # 1: fresh tracks: A (0.9), tie pair T1 / T2 (0.8 / 0.7), clipped boxes at each border, a small box (< 75 px)
    D.append((np.array([[100, 100, 113, 110], [300, 300, 310, 310], [310, 300, 320, 310],
                        [-6, 200, 30, 240], [200, -4, 240, 30], [620, 100, 650, 140], [100, 460, 140, 490],
                        [400, 50, 408, 59]], f),
              np.array([0.9, 0.8, 0.7, 0.6, 0.55, 0.5, 0.45, 0.4], f), np.array([1, 2, 2, 0, 0, 0, 0, 0], np.int32)))
    # 2: IoU(A, .) = 0.3 exactly (inclusive match); a box between T1 and T2 at equal IoU 1/3 (the later track T2 wins);
    #    a box overlapping the first border box with another label (mismatch: new track); the others dropped
    D.append((np.array([[107, 100, 120, 110], [305, 300, 315, 310], [-6, 200, 30, 240]], f),
              np.array([0.95, 0.85, 0.35], f), np.array([1, 2, 3], np.int32)))
    # 3: empty mid-sequence: the predicted tracks and n_matched stay
    D.append((np.zeros((0, 4), f), np.zeros(0, f), np.zeros(0, np.int32)))
    # 4: far away from every track: a full restart, ids continue from the advanced counter
    D.append((np.array([[500, 300, 560, 350], [20, 380, 70, 420]], f), np.array([0.7, 0.65], f),
              np.array([1, 2], np.int32)))
    return D


def moving(rng, n_det, n_obj, stride):
    """detections of n_obj objects moving at constant velocity with noise, some missing per detection, input frames
    0, stride, 2 stride, ..."""
    p0 = rng.uniform([20, 20], [W_IMG - 120, H_IMG - 100], (n_obj, 2))
    v = rng.uniform(-6, 6, (n_obj, 2))
    wh = rng.uniform([25, 20], [110, 90], (n_obj, 2))
    lab = rng.integers(0, 3, n_obj)
    D = []
    for k in range(n_det):
        t = k * stride
        seen = rng.random(n_obj) > 0.15
        p = p0[seen] + v[seen] * t + rng.normal(0, 1.5, (seen.sum(), 2))
        s = wh[seen] * rng.uniform(0.95, 1.05, (seen.sum(), 2))
        b = np.concatenate((p, p + s), 1).astype(np.float32)
        sc = rng.permutation(np.linspace(0.2, 0.95, seen.sum())).astype(np.float32) + np.float32(k * 1e-3)
        D.append((b, sc.astype(np.float32), lab[seen].astype(np.int32)))
    return D


def build(seed, eta):
    """-> the fixture's sequences: list of (n_frames, detections, input_fidx, timestamps)"""
    rng = np.random.default_rng(seed)
    seqs = []
    d = crafted()
    fidx = [2 * k for k in range(len(d))]
    seqs.append((12, d, fidx, [(f + 1.5) / FPS for f in fidx]))                      # stride 2, runtime 1.5 frames
    for stride, n_obj, n_frames in ((1, 5, 24), (3, 7, 30)):
        n_det = (n_frames - 2) // stride
        d = moving(rng, n_det, n_obj, stride)
        fidx = [k * stride for k in range(n_det)]
        rt = rng.uniform(0.6, 2.4, n_det)
        ts = [(f + r) / FPS for f, r in zip(fidx, rt)]
        ts = list(np.maximum.accumulate(ts))
        seqs.append((n_frames, d, fidx, ts))
    if eta < 0:                                 # the divergence: the first frame sees an empty first detection
        d = [(np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros(0, np.int32))] + moving(rng, 4, 3, 2)[1:]
        fidx = [0, 2, 4, 6]
        seqs.append((9, d, fidx, [0.5 / FPS, 3.5 / FPS, 5.5 / FPS, 7.5 / FPS]))
    return seqs


def write_inputs(seqs, root):
    images, names, iid = [], [], 0
    for sid, (n_frames, _, _, _) in enumerate(seqs):
        names.append(f"seq{sid}")
        for ii in range(n_frames):
            images.append({"id": iid, "sid": sid, "fid": ii, "name": f"{ii:06d}.jpg", "width": W_IMG, "height": H_IMG})
            iid += 1
    annot = {"images": images, "annotations": [], "sequences": names, "seq_dirs": names,
             "categories": [{"id": c, "name": f"c{c}"} for c in range(4)]}
    path = os.path.join(root, "annot.json")
    with open(path, "w") as f:
        json.dump(annot, f)
    os.makedirs(os.path.join(root, "in"), exist_ok=True)
    for name, (_, d, fidx, ts) in zip(names, seqs):
        with open(os.path.join(root, "in", name + ".pkl"), "wb") as f:
            pickle.dump({"results_parsed": [(b, s, l, None) for b, s, l in d], "timestamps": ts, "input_fidx": fidx,
                         "runtime": [0.0] * len(ts)}, f)
    return path


def run_reference(seqs, eta):
    sys.path.insert(0, os.path.join(HERE, "ref_shim"))
    sys.path.insert(0, os.path.join(REF, "sAP"))
    np.int = int                                          # extrap_clean_up's astype(np.int), removed in numpy 1.24
    import track
    from forecast import pps_forecast_kf as ref
    from pycocotools.mask import iou
    decisions = []
    orig = track.iou_assoc

    def recorded(bboxes1, labels1, tracks1, tkidx, bboxes2, labels2, th, no_unmatched1=False):
        out = orig(bboxes1, labels1, tracks1, tkidx, bboxes2, labels2, th, no_unmatched1=no_unmatched1)
        ious = iou(bboxes1, bboxes2, [0] * len(bboxes2))
        margins = []
        for j in range(len(bboxes2)):
            e = sorted((ious[i, j] for i in range(len(bboxes1)) if labels1[i] == labels2[j]), reverse=True)
            margins.append(min(abs(e[0] - th) if e else np.inf, e[0] - e[1] if len(e) > 1 and e[1] >= th else np.inf))
        decisions.append((out[0], out[1], out[2], margins))
        return out

    ref.iou_assoc = recorded
    with tempfile.TemporaryDirectory() as root:
        annot = write_inputs(seqs, root)
        out = os.path.join(root, "out")
        argv = sys.argv
        sys.argv = ["pps_forecast_kf.py", "--data-root", root, "--annot-path", annot, "--fps", str(FPS), "--eta", str(eta),
                    "--forecast-before-assoc", "--in-dir", os.path.join(root, "in"), "--out-dir", out, "--no-eval",
                    "--overwrite"]
        try:
            ref.main()
        finally:
            sys.argv = argv
            ref.iou_assoc = orig
        with open(os.path.join(out, "results_ccf.pkl"), "rb") as f:
            ccf = pickle.load(f)
        with open(annot) as f:
            annot_text = f.read()
    return ccf, decisions, annot_text


def pack(seqs, eta, ccf, decisions, annot_text):
    g = {"eta": np.float64(eta), "annot": np.array(annot_text)}
    det_seq, det_box, det_score, det_label, det_n = [], [], [], [], []
    for q, (_, d, _, _) in enumerate(seqs):
        for b, s, l in d:
            det_seq.append(q), det_n.append(len(b)), det_box.append(b), det_score.append(s), det_label.append(l)
    g["det_seq"], g["det_n"] = np.array(det_seq, np.int32), np.array(det_n, np.int32)
    g["det_box"] = np.concatenate(det_box).astype(np.float32)
    g["det_score"], g["det_label"] = np.concatenate(det_score), np.concatenate(det_label)
    g["seq_frames"] = np.array([s[0] for s in seqs], np.int32)
    g["seq_ndet"] = np.array([len(s[1]) for s in seqs], np.int32)
    g["input_fidx"] = np.concatenate([np.asarray(s[2], np.int64) for s in seqs])
    g["timestamps"] = np.concatenate([np.asarray(s[3], np.float64) for s in seqs])
    g["ccf_image_id"] = np.array([r["image_id"] for r in ccf], np.int64)
    g["ccf_bbox"] = np.array([r["bbox"] for r in ccf], np.float32).reshape(-1, 4)
    g["ccf_score"] = np.array([r["score"] for r in ccf], np.float32)
    g["ccf_category"] = np.array([r["category_id"] for r in ccf], np.int64)
    g["dec_n_matched"] = np.array([d[2] for d in decisions], np.int32)
    g["dec_order1"] = np.concatenate([np.asarray(d[0], np.int32) for d in decisions] + [np.zeros(0, np.int32)])
    g["dec_order2"] = np.concatenate([np.asarray(d[1], np.int32) for d in decisions] + [np.zeros(0, np.int32)])
    g["dec_len1"] = np.array([len(d[0]) for d in decisions], np.int32)
    g["dec_len2"] = np.array([len(d[1]) for d in decisions], np.int32)
    g["dec_margin"] = np.concatenate([np.asarray(d[3], np.float64) for d in decisions] + [np.zeros(0)])
    return g


def main():
    for name, eta in (("eta0", 0.0), ("etam1", -1.0)):
        for seed in range(100):
            seqs = build(seed, eta)
            ccf, decisions, annot_text = run_reference(seqs, eta)
            m = np.concatenate([np.asarray(d[3], np.float64) for d in decisions])
            if np.all((m == 0) | (m >= 1e-4)):
                break
        else:
            raise RuntimeError("no seed keeps the margins")
        g = pack(seqs, eta, ccf, decisions, annot_text)
        path = os.path.join(ROOT, "tests", "golden", f"forecast_{name}.npz")
        np.savez_compressed(path, **g)
        print(f"{path}: seed {seed}, {len(ccf)} rows, {len(decisions)} associations, "
              f"{int((g['dec_n_matched'] > 0).sum())} with matches, min margin {m[m > 0].min():.3g}, "
              f"{int((m == 0).sum())} exact ties")


if __name__ == "__main__":
    main()
