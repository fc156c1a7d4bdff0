"""Generate tests/golden/srt_*.npz -- TEST INFRASTRUCTURE.  Run in the build container, with the StreamYOLO checkout at
$STREAMYOLO_REF (default /root/reference):

    python oracle/make_srt_golden.py

Runs the UNMODIFIED sAP/det/srt_det.py and sAP/det/srt_det_inf.py main() on a small synthetic annotation file and a
pickled empirical runtime distribution, with stand-ins for what needs a detector or the frames:
  - ``det.det_apis`` is a module of its own (no mmdet): ``init_detector`` returns a token and ``inference_detector``
    returns ``("result", frame)``, the frame ``imread`` gave it;
  - ``imread`` returns the frame's tag, (sequence directory, frame index) read from its path;
  - ``parse_det_result`` returns one box whose first coordinate is that frame index, so every result in the pickles
    names the frame it came from;
  - ``tqdm`` is the identity when it is not installed, ``torch.cuda.device_count`` returns 1 (the scripts assert a
    single GPU), and oracle/ref_shim stands in for pycocotools and mmcv.

Each file records, per sequence in the pickles' order: ``input_fidx``, ``timestamps``, ``runtime`` and the frame index of
each result (``result_fidx``, from ``results_raw``; ``results_parsed`` is checked to name the same frames), and the run's
time_info.pkl and printed summary.  The cases: two seeds; --perf-factor 1 and 1.37; --det-stride 1, 2 and 1.5;
--dynamic-schedule with a mean runtime above and below one frame interval; five sequences (one empty), so the draws
cross sequence boundaries; and two infinite-GPU runs, one whose samples are multiples of 0.1 s so that ``ii / fps +
draw`` ties and np.argsort's (unstable) order of the ties is pinned."""
import contextlib
import io
import json
import os
import pickle
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("STREAMYOLO_REF", "/root/reference")
FPS = 30.0
LENGTHS = [23, 0, 40, 7, 31]
# a wall-clock run's runtime_all (seconds): mean 40.2 ms, 1.2 frame intervals at 30 fps
SAMPLES = [0.0213, 0.0341, 0.0275, 0.0612, 0.0189, 0.0455, 0.0298, 0.0833]
# a faster detector: mean 21.6 ms, 0.65 frame intervals
FAST = [0.012, 0.025, 0.018, 0.031, 0.022]
# multiples of 0.1 s, three frame intervals: ii / 30 + draw lands on the same time from several frames
TIES = [0.1, 0.2, 0.3, 0.4]

# name -> (clock, --det-stride, --dynamic-schedule, samples, --perf-factor, --seed)
CASES = {
    "srt_seed0": ("simulated", 1, False, SAMPLES, 1, 0),
    "srt_seed5_stride2_pf1p37": ("simulated", 2, False, SAMPLES, 1.37, 5),
    "srt_stride1p5": ("simulated", 1.5, False, SAMPLES, 1, 5),
    "srt_dyn_above": ("simulated", 1, True, SAMPLES, 1, 0),
    "srt_dyn_below_pf1p37": ("simulated", 1, True, FAST, 1.37, 5),
    "srt_inf_ties": ("infinite", 1, False, TIES, 1, 0),
    "srt_inf_seed5_pf1p37": ("infinite", 1, False, SAMPLES, 1.37, 5),
}


def annotation(lengths):
    """the annotation file's text: sequence q has lengths[q] frames of 1920 x 1200 in directory d{q}"""
    images, k = [], 0
    for q, n in enumerate(lengths):
        for j in range(n):
            images.append({"id": k, "sid": q, "fid": j, "name": f"{j:06d}.jpg", "width": 1920, "height": 1200})
            k += 1
    return json.dumps({"sequences": [f"s{q}" for q in range(len(lengths))], "seq_dirs": [f"d{q}" for q in
                       range(len(lengths))], "images": images, "annotations": [], "categories": [{"id": 0, "name": "car"}]})


def import_scripts():
    """sAP/det/srt_det.py and srt_det_inf.py, imported as they are"""
    sys.path.insert(0, os.path.join(HERE, "ref_shim"))
    sys.path.insert(0, os.path.join(REF, "sAP"))
    try:
        import tqdm  # noqa: F401
    except ImportError:
        sys.modules["tqdm"] = types.SimpleNamespace(tqdm=lambda x, *a, **k: x)
    apis = types.ModuleType("det.det_apis")
    apis.init_detector = lambda opts: "model"
    apis.inference_detector = lambda model, frame: ("result", frame)
    sys.modules["det.det_apis"] = apis
    import det.srt_det as srt
    import det.srt_det_inf as srt_inf
    return srt, srt_inf


def imread(path):
    return os.path.basename(os.path.dirname(path)), int(os.path.basename(path)[:6])


def parse_det_result(result, class_mapping=None, n_class=None):
    _, (_, fidx) = result
    return (np.array([[fidx, 0, 1, 1]], np.float32), np.array([0.5], np.float32), np.array([0], np.int32), None)


def run_reference(script, case, annot_text):
    import torch
    clock, stride, dynamic, samples, perf_factor, seed = case
    with tempfile.TemporaryDirectory() as tmp:
        annot, rt, out = os.path.join(tmp, "annot.json"), os.path.join(tmp, "runtime.pkl"), os.path.join(tmp, "out")
        with open(annot, "w") as f:
            f.write(annot_text)
        with open(rt, "wb") as f:
            pickle.dump({"type": "empirical", "samples": list(samples)}, f)
        argv = ["srt", "--data-root", tmp, "--annot-path", annot, "--fps", str(FPS), "--config", "none", "--weights",
                "none", "--runtime", rt, "--perf-factor", str(perf_factor), "--seed", str(seed), "--out-dir", out,
                "--overwrite"]
        if clock == "simulated":
            argv += ["--det-stride", str(stride)] + (["--dynamic-schedule"] if dynamic else [])
        saved = (sys.argv, script.imread, script.parse_det_result, torch.cuda.device_count)
        sys.argv, script.imread, script.parse_det_result = argv, imread, parse_det_result
        torch.cuda.device_count = lambda: 1
        printed = io.StringIO()
        try:
            with contextlib.redirect_stdout(printed):
                script.main()
        finally:
            sys.argv, script.imread, script.parse_det_result, torch.cuda.device_count = saved
        results = []
        for q in range(len(LENGTHS)):
            with open(os.path.join(out, f"s{q}.pkl"), "rb") as f:
                results.append(pickle.load(f))
        with open(os.path.join(out, "time_info.pkl"), "rb") as f:
            time_info = pickle.load(f)
    return results, time_info, printed.getvalue()


def pack(case, annot_text, results, time_info, printed):
    clock, stride, dynamic, samples, perf_factor, seed = case
    g = {"clock": np.array(clock), "det_stride": np.float64(stride), "dynamic": np.bool_(dynamic),
         "samples": np.asarray(samples, np.float64), "perf_factor": np.float64(perf_factor), "seed": np.int64(seed),
         "fps": np.float64(FPS), "lengths": np.asarray(LENGTHS, np.int64), "annot": np.array(annot_text),
         "printed": np.array(printed)}
    n, fi, ts, rt, rf = [], [], [], [], []
    for r in results:
        assert sorted(r) == ["input_fidx", "results_parsed", "results_raw", "runtime", "timestamps"]
        got = [res[1][1] for res in r["results_raw"]]
        assert got == [int(p[0][0, 0]) for p in r["results_parsed"]]
        assert all(type(v) is int for v in r["input_fidx"]) and all(type(v) is np.float64 for v in r["runtime"])
        n.append(len(r["input_fidx"]))
        fi += r["input_fidx"]
        ts += r["timestamps"]
        rt += r["runtime"]
        rf += got
    g["seq_n"] = np.asarray(n, np.int64)
    g["input_fidx"], g["result_fidx"] = np.asarray(fi, np.int64), np.asarray(rf, np.int64)
    g["timestamps"], g["runtime"] = np.asarray(ts, np.float64), np.asarray(rt, np.float64)
    g["runtime_all"] = np.asarray(time_info["runtime_all"], np.float64)
    g["n_processed"], g["n_total"] = np.int64(time_info["n_processed"]), np.int64(time_info["n_total"])
    g["n_small_runtime"] = np.int64(time_info["n_small_runtime"])
    return g


def main():
    srt, srt_inf = import_scripts()
    annot_text = annotation(LENGTHS)
    for name, case in CASES.items():
        results, time_info, printed = run_reference(srt if case[0] == "simulated" else srt_inf, case, annot_text)
        g = pack(case, annot_text, results, time_info, printed)
        note = ""
        if case[0] == "infinite":
            ties = unstable = 0
            for res in results:             # the times in frame order, and the order a stable sort would give
                by_frame = sorted(zip(res["input_fidx"], res["runtime"]))
                raw = [ii / FPS + r for ii, r in by_frame]
                ties += len(raw) - len(set(raw))
                unstable += np.argsort(raw, kind="stable").tolist() != res["input_fidx"]
            note = f", {ties} tied times, {unstable} sequences whose ties are not in frame order"
            if name == "srt_inf_ties":
                assert ties > 0 and unstable > 0, "the tie case pins nothing"
        path = os.path.join(ROOT, "tests", "golden", f"{name}.npz")
        np.savez_compressed(path, **g)
        print(f"{path}: {int(g['n_processed'])}/{int(g['n_total'])} frames{note}")


if __name__ == "__main__":
    main()
