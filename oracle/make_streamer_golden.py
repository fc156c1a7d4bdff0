"""Generate tests/golden/streamer_*.npz -- TEST INFRASTRUCTURE.  Run in the build container, with the StreamYOLO checkout
at $STREAMYOLO_REF (default /root/reference) and Cython installed:

    python oracle/make_streamer_golden.py

Runs the UNMODIFIED sAP/forecast/streamer.py main() on synthetic sequences, on a virtual clock:
  - ``perf_counter`` is the clock of oracle/streamer_oracle.py: it reads the virtual time, restarts at 0 at each
    sequence's ``t_start`` and, on two consecutive readings at the loop head (an idle iteration between them), moves to
    the first time of the next frame;
  - ``mp`` is an in-process fake: the detector process never starts, a frame sent at t completes at t + R, the result
    pipe's ``poll(w)`` returns at min(t + w, completion) and ``recv`` hands over the frame index; a detection still in
    flight when a sequence ends is dropped, as the script's wait for 'ready' drains it;
  - ``parse_det_result`` returns that frame's synthetic detection (ltrb fp32, fp32 scores, int32 labels);
  - ``det.det_apis`` is an empty stand-in (no mmdet), ``track.iou_assoc_cp`` is compiled from its .pyx with Cython into a
    temporary directory, and oracle/ref_shim stands in for pycocotools and mmcv;
  - ``iou_assoc`` is wrapped, not changed, to record every association decision and its IoU margins.

Every frame of every sequence has a detection, so any schedule finds one.  Sequence 0 is crafted: a first phase of
tracks (one moving, four clipped at the four borders, one below 75 pixels, one clipped below 75 pixels, one leaving the
image to the right), an empty phase (the streamer clears the tracks), the first phase again (fresh tracks, ids
continuing), a far-away phase (a restart with no match).  The others are moving objects with noise.  Each file keeps
every decision's IoU margins (to the threshold and to the runner-up) >= 1e-4; the seeded search reruns to the same
files."""
import importlib.util
import inspect
import json
import os
import pickle
import shutil
import subprocess
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
REF = os.environ.get("STREAMYOLO_REF", "/root/reference")
W_IMG, H_IMG, FPS = 640, 480, 30.0

from oracle.make_forecast_golden import moving          # noqa: E402
from oracle.streamer_oracle import next_frame_time       # noqa: E402

# name -> (runtime R in seconds, --dynamic-schedule, --eta, runtime samples of the --runtime pickle)
CASES = {
    "r20_eta0": (0.020, False, 0.0, [0.018, 0.022, 0.021]),
    "r75_eta0p3": (0.075, False, 0.3, [0.07, 0.08, 0.075]),
    "r75_dyn_eta0": (0.075, True, 0.0, [0.07, 0.08, 0.076]),
    "r45_dyn_etam0p5": (0.045, True, -0.5, [0.04, 0.05, 0.047]),
}


def crafted(rng):
    """sequence 0's detection of every frame: see the module doc"""
    f = np.float32
    base = np.array([[100, 100, 160, 150], [-20, 200, 30, 240], [200, -15, 240, 30], [610, 100, 660, 140],
                     [100, 450, 140, 500], [400, 50, 408, 59], [-60, 300, 2, 330], [560, 200, 600, 240]], f)
    vel = np.array([[2, 1], [0, 0], [0, 0], [0, 0], [0, 0], [0, 0], [0, 0], [12, 0]], f)
    lab = np.array([1, 0, 0, 2, 2, 0, 1, 3], np.int32)
    far = np.array([[450, 330, 520, 400], [20, 380, 90, 440]], f)
    D = []
    for k in range(28):
        if k < 8 or 12 <= k < 18:
            t = k if k < 8 else k - 12
            b = base + np.concatenate((vel, vel), 1) * t
            sc = (np.linspace(0.9, 0.3, len(b)) + 1e-3 * k).astype(f)
            D.append((b.astype(f), sc, lab.copy()))
        elif k < 12:
            D.append((np.zeros((0, 4), f), np.zeros(0, f), np.zeros(0, np.int32)))
        else:
            t = k - 18
            D.append(((far + np.array([3, 1, 3, 1], f) * t).astype(f), np.array([0.8, 0.7], f) + f(1e-3 * k),
                      np.array([1, 2], np.int32)))
    return D


def build(seed):
    """-> the sequences' detections: one list per sequence of (ltrb, scores, labels) per frame"""
    rng = np.random.default_rng(seed)
    seqs = [crafted(rng)]
    for n_obj, n_frames in ((5, 30), (7, 22)):
        seqs.append([(b, s, l.astype(np.int32)) for b, s, l in moving(rng, n_frames, n_obj, 1)])
    return seqs


def write_inputs(seqs, root, samples):
    images, names, iid = [], [], 0
    for sid, d in enumerate(seqs):
        names.append(f"seq{sid}")
        for ii in range(len(d)):
            images.append({"id": iid, "sid": sid, "fid": ii, "name": f"{ii:06d}.jpg", "width": W_IMG, "height": H_IMG})
            iid += 1
    annot = {"images": images, "annotations": [], "sequences": names, "seq_dirs": names,
             "categories": [{"id": c, "name": f"c{c}"} for c in range(4)]}
    path = os.path.join(root, "annot.json")
    with open(path, "w") as f:
        json.dump(annot, f)
    rt = os.path.join(root, "runtime.pkl")
    with open(rt, "wb") as f:
        pickle.dump({"type": "empirical", "samples": list(samples)}, f)
    return path, rt


def compile_iou_assoc(tmp):
    """track/iou_assoc_cp.pyx built with Cython in ``tmp`` -> the module, registered as track.iou_assoc_cp"""
    src = os.path.join(tmp, "iou_assoc_cp.pyx")
    shutil.copy(os.path.join(REF, "sAP", "track", "iou_assoc_cp.pyx"), src)
    subprocess.run([sys.executable, "-m", "Cython.Build.Cythonize", "-i", "-q", src], cwd=tmp, check=True,
                   stdout=subprocess.DEVNULL)
    so = next(os.path.join(tmp, f) for f in os.listdir(tmp) if f.startswith("iou_assoc_cp") and f.endswith(".so"))
    spec = importlib.util.spec_from_file_location("track.iou_assoc_cp", so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules["track.iou_assoc_cp"] = mod
    return mod


class World:
    """the virtual clock and the fake detector process of one run"""

    def __init__(self, runtime, fps, head_line, start_line):
        self.t, self.runtime, self.fps = 0.0, runtime, fps
        self.head, self.start = head_line, start_line
        self.last = None
        self.pending = None                   # (fidx, completion)
        self.msgs = []
        self.seq = -1

    def perf_counter(self):
        line = sys._getframe(1).f_lineno
        if line == self.start:
            self.t = 0.0
        elif line == self.head and self.last == self.head:
            self.t = next_frame_time(self.t, self.fps)
        self.last = line
        return self.t

    # frame_send
    def send(self, msg):
        if isinstance(msg, list):             # a new sequence: a result still in flight is drained before 'ready'
            self.seq += 1
            self.pending = None
            self.msgs.append("ready")
        elif msg is not None:
            assert self.pending is None, "a frame sent while one is in flight"
            self.pending = (msg[0], self.t + self.runtime)

    # det_res_recv
    def poll(self, w):
        if self.pending is not None and self.pending[1] <= self.t + w:
            self.t = max(self.t, self.pending[1])
            return True
        self.t = self.t + w
        return False

    def recv(self):
        if self.msgs:
            return self.msgs.pop(0)
        (fidx, done), self.pending = self.pending, None
        return [(self.seq, fidx), 0.0, done]


def run_reference(seqs, runtime, dynamic, eta, samples):
    sys.path.insert(0, os.path.join(HERE, "ref_shim"))
    sys.path.insert(0, os.path.join(REF, "sAP"))
    np.int = int                                          # extrap_clean_up's astype(np.int), removed in numpy 1.24
    import torch
    decisions, results = [], {}
    with tempfile.TemporaryDirectory() as tmp:
        if "track.iou_assoc_cp" not in sys.modules:
            compile_iou_assoc(tmp)
        apis = types.ModuleType("det.det_apis")
        apis.init_detector = apis.inference_detector = None
        sys.modules["det.det_apis"] = apis
        from forecast import streamer as ref
        from pycocotools.mask import iou
        lines = inspect.getsource(ref).splitlines()
        head = 1 + next(i for i, s in enumerate(lines) if s.strip() == "t1 = perf_counter()")
        start = 1 + next(i for i, s in enumerate(lines) if s.strip() == "t_start = perf_counter()")
        world = World(runtime, FPS, head, start)
        fake_mp = types.SimpleNamespace(set_start_method=lambda *a, **k: None,
                                        Pipe=lambda duplex=True: (world, world),
                                        Process=lambda target, args: types.SimpleNamespace(start=lambda: None))
        orig = ref.iou_assoc

        def recorded(bboxes1, labels1, tracks1, tkidx, bboxes2, labels2, th, no_unmatched1=False):
            out = orig(bboxes1, labels1, tracks1, tkidx, bboxes2, labels2, th, no_unmatched1=no_unmatched1)
            ious = iou(bboxes1, bboxes2, [0] * len(bboxes2))
            margins = []
            for j in range(len(bboxes2)):
                e = sorted((ious[i, j] for i in range(len(bboxes1)) if labels1[i] == labels2[j]), reverse=True)
                margins.append(min(abs(e[0] - th) if e else np.inf, e[0] - e[1] if len(e) > 1 and e[1] >= th else np.inf))
            decisions.append((out[0], out[1], out[2], margins))
            return out

        def parse(result, coco_mapping=None, n_class=None):
            q, fidx = result
            b, s, l = seqs[q][fidx]
            return b.copy(), s.copy(), l.copy(), None

        saved = (ref.mp, ref.perf_counter, ref.parse_det_result, ref.iou_assoc, torch.cuda.device_count)
        ref.mp, ref.perf_counter, ref.parse_det_result, ref.iou_assoc = fake_mp, world.perf_counter, parse, recorded
        torch.cuda.device_count = lambda: 1
        annot, rt = write_inputs(seqs, tmp, samples)
        out = os.path.join(tmp, "out")
        argv = sys.argv
        sys.argv = ["streamer.py", "--data-root", tmp, "--annot-path", annot, "--fps", str(FPS), "--eta", str(eta),
                    "--config", "none", "--weights", "none", "--runtime", rt, "--out-dir", out, "--overwrite"]
        if dynamic:
            sys.argv.append("--dynamic-schedule")
        try:
            ref.main()
        finally:
            sys.argv = argv
            ref.mp, ref.perf_counter, ref.parse_det_result, ref.iou_assoc, torch.cuda.device_count = saved
        for q in range(len(seqs)):
            with open(os.path.join(out, f"seq{q}.pkl"), "rb") as f:
                results[q] = pickle.load(f)
        with open(os.path.join(out, "time_info.pkl"), "rb") as f:
            time_info = pickle.load(f)
        with open(annot) as f:
            annot_text = f.read()
    return results, time_info, decisions, annot_text


def pack(seqs, case, results, time_info, decisions, annot_text):
    runtime, dynamic, eta, samples = case
    g = {"runtime": np.float64(runtime), "dynamic": np.bool_(dynamic), "eta": np.float64(eta), "fps": np.float64(FPS),
         "samples": np.asarray(samples, np.float64), "annot": np.array(annot_text)}
    det_n, det_box, det_score, det_label = [], [], [], []
    for d in seqs:
        for b, s, l in d:
            det_n.append(len(b)), det_box.append(b), det_score.append(s), det_label.append(l)
    g["seq_frames"] = np.array([len(d) for d in seqs], np.int32)
    g["det_n"] = np.array(det_n, np.int32)
    g["det_box"] = np.concatenate(det_box).astype(np.float32)
    g["det_score"], g["det_label"] = np.concatenate(det_score), np.concatenate(det_label)
    ts, fi, n_emit, n_rows, tracked, box, score, label, track = [], [], [], [], [], [], [], [], []
    for q in range(len(seqs)):
        r = results[q]
        ts += r["timestamps"]
        fi += r["input_fidx"]
        n_emit.append(len(r["timestamps"]))
        for b, s, l, m, tr in r["results_parsed"]:
            assert m is None and b.dtype == np.float32 and s.dtype == np.float32 and l.dtype == np.int32
            assert tr.dtype == (np.uint32 if tr.dtype == np.uint32 else np.int32)
            n_rows.append(len(b)), tracked.append(tr.dtype == np.uint32)
            box.append(b.reshape(-1, 4)), score.append(s), label.append(l), track.append(tr.astype(np.int64))
    g["timestamps"], g["input_fidx"] = np.asarray(ts, np.float64), np.asarray(fi, np.int64)
    g["seq_emit"], g["emit_rows"] = np.asarray(n_emit, np.int32), np.asarray(n_rows, np.int32)
    g["emit_tracked"] = np.asarray(tracked, bool)          # track ids are uint32 (tracks exist) or int32 (none)
    g["box"] = np.concatenate(box + [np.zeros((0, 4), np.float32)])
    g["score"] = np.concatenate(score + [np.zeros(0, np.float32)])
    g["label"] = np.concatenate(label + [np.zeros(0, np.int32)])
    g["track"] = np.concatenate(track + [np.zeros(0, np.int64)])
    g["n_total"] = np.int64(time_info["n_total"])
    g["time_counts"] = np.array([len(time_info[k]) for k in ("t_det", "t_send_frame", "t_recv_res", "t_assoc",
                                                             "t_forecast")], np.int64)
    g["dec_n_matched"] = np.array([d[2] for d in decisions], np.int32)
    g["dec_order1"] = np.concatenate([np.asarray(d[0], np.int32) for d in decisions] + [np.zeros(0, np.int32)])
    g["dec_order2"] = np.concatenate([np.asarray(d[1], np.int32) for d in decisions] + [np.zeros(0, np.int32)])
    g["dec_len1"] = np.array([len(d[0]) for d in decisions], np.int32)
    g["dec_len2"] = np.array([len(d[1]) for d in decisions], np.int32)
    g["dec_margin"] = np.concatenate([np.asarray(d[3], np.float64) for d in decisions] + [np.zeros(0)])
    return g


def main():
    for name, case in CASES.items():
        for seed in range(100):
            seqs = build(seed)
            results, time_info, decisions, annot_text = run_reference(seqs, case[0], case[1], case[2], case[3])
            m = np.concatenate([np.asarray(d[3], np.float64) for d in decisions] + [np.zeros(0)])
            if np.all(m >= 1e-4):
                break
        else:
            raise RuntimeError("no seed keeps the margins")
        g = pack(seqs, case, results, time_info, decisions, annot_text)
        path = os.path.join(ROOT, "tests", "golden", f"streamer_{name}.npz")
        np.savez_compressed(path, **g)
        print(f"{path}: seed {seed}, {len(g['timestamps'])} emissions, {int(g['emit_rows'].sum())} rows, "
              f"{len(decisions)} associations, {int((g['dec_n_matched'] > 0).sum())} with matches, "
              f"{int(((g['dec_len2'] == 0) & (g['dec_len1'] == 0)).sum())} empty, min margin {m.min():.3g}")


if __name__ == "__main__":
    main()
