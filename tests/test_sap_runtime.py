"""Sampled detector runtimes in the sAP driver (``python -m streamyolo_b200.sap --runtime rt.pkl``): srt_det.py's draws
on the simulated clock and srt_det_inf.py's infinite GPUs (``--clock infinite``).

CPU (no GPU needed):
  * oracle/srt_oracle.py's srt_det / srt_det_inf equal the unmodified scripts' output (tests/golden/srt_*.npz, made by
    oracle/make_srt_golden.py) exactly: input_fidx, timestamps, runtime, time_info;
  * sap.simulated_schedule with a runtime distribution equals the oracle over strides, dynamic schedules, seeds, perf
    factors and sequence lengths, with the generator carried across sequences;
  * sap.run with an emulated detector writes the fixtures' pickles (each result the frame its row names; on the infinite
    clock each frame fused with the one before it), time_info and printed summary, on both clocks and at 1 and 3
    streams; a second run writes the same pickles (results_raw compared by value);
  * a one-sample distribution {samples: [R]} gives what --runtime-ms R * 1000 gives;
  * the global numpy generator is left as it was;
  * the arguments: exclusive runtime sources, --perf-factor / --seed need --runtime, infinite takes neither
    --det-stride nor --dynamic-schedule, --cached-res is not implemented, an unknown distribution type is named.

GPU (H100), the JPEG fixture sequences of tests/test_sap_driver.py:
  * --clock infinite at S = 1 equals the eager driver loop over every frame, reordered as srt_det_inf.py reorders;
  * at S = 4 each stream equals eager on_pipe calls at batch 4;
  * --clock simulated --runtime with several samples: each row is the eager driver loop's on the frame the schedule
    lists, and a second run writes the same pickles (results_raw by value: a pickled tensor carries its storage's
    address).
"""
import json
import os
import pickle
import sys

import numpy as np
import pytest
import torch

from oracle import sap_oracle, srt_oracle
from streamyolo_b200 import sap, stream

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith("srt_") and f.endswith(".npz"))
FPS = 30.0


def _golden(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    bounds = np.concatenate(([0], np.cumsum(g["seq_n"])))
    per_seq = [tuple(g[k][a:b].tolist() for k in ("input_fidx", "timestamps", "runtime", "result_fidx"))
               for a, b in zip(bounds[:-1], bounds[1:])]
    return g, per_seq


# ================================================================================================ emulated detector
class TagDetector:
    """StreamDetector's JPEG interface without a GPU, for files whose bytes are "q j" (sequence q, frame j): each result
    is one box [j, carried j, q, 0], the carried frame being the stream's previous one (its own after reset(i))"""

    def __init__(self, model, frame_hw=None, in_scale=0.5, frame_sizes=None, jpeg_max_bytes=None):
        self.streams = len(frame_sizes)
        self.prev, self.flags = [None] * self.streams, [1] * self.streams
        self.jpeg_max_bytes, self.ticks = jpeg_max_bytes, 0

    def reset(self, stream=None):
        for s in range(self.streams) if stream is None else [stream]:
            self.flags[s] = 1

    def step_jpeg(self, files):
        assert len(files) == self.streams and all(f is None or len(f) <= self.jpeg_max_bytes for f in files)
        out = []
        for s, f in enumerate(files):
            if f is None:
                out.append((np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros(0, np.int32)))
                continue
            q, j = map(int, f.tobytes().decode().split())
            if self.flags[s]:
                self.prev[s] = j
            out.append((np.array([[j, self.prev[s], q, 0]], np.float32), np.ones(1, np.float32), np.zeros(1, np.int32)))
            self.prev[s], self.flags[s] = j, 0
        self.raw = torch.tensor([[len(r[0]), r[0][0, 0] if len(r[0]) else -1] for r in out], dtype=torch.float16)[:, None]
        self.status = np.array([stream.NO_FRAME if f is None else 0 for f in files], np.int32)
        self.ticks += 1
        return out

    def last_raw(self):
        return self.raw.clone()

    def last_status(self):
        return self.status.copy()


def _dataset(tmp_path, annot_text):
    """the annotation file and a file "q j" for frame j of sequence q"""
    ann = json.loads(annot_text)
    root = tmp_path / "data"
    for img in ann["images"]:
        d = root / ann["seq_dirs"][img["sid"]]
        d.mkdir(parents=True, exist_ok=True)
        (d / img["name"]).write_bytes(f"{img['sid']} {img['fid']}".encode())
    path = tmp_path / "annot.json"
    path.write_text(annot_text)
    return root, path


def _runtime(tmp_path, samples, kind="empirical"):
    path = tmp_path / "rt.pkl"
    with open(path, "wb") as f:
        pickle.dump({"type": kind, "samples": list(samples)}, f)
    return path


def _opts(root, ann, out, *extra):
    return sap.parse_args(["--data-root", str(root), "--annot-path", str(ann), "--out-dir", str(out), "--config", "c",
                           "--weights", "w", "--overwrite", *extra])


def _load(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def _contents(out):
    """every file under ``out`` as bytes, the pickles' results_raw apart: a pickled tensor carries its storage's address,
    so those are compared by value -> ({name: bytes}, {name: [tensor]})"""
    files, raws = {}, {}
    for p in sorted(os.listdir(out)):
        d = _load(out / p)
        raws[p] = d.pop("results_raw", [])
        files[p] = pickle.dumps(d)
    return files, raws


def _same_contents(a, b):
    return a[0] == b[0] and a[1].keys() == b[1].keys() and all(
        len(a[1][k]) == len(b[1][k]) and all(torch.equal(x, y) for x, y in zip(a[1][k], b[1][k])) for k in a[1])


def _case_args(g, rt):
    args = ["--clock", str(g["clock"]), "--runtime", str(rt), "--fps", repr(float(g["fps"])), "--perf-factor",
            repr(float(g["perf_factor"])), "--seed", str(int(g["seed"]))]
    if str(g["clock"]) == "simulated":
        args += ["--det-stride", repr(float(g["det_stride"]))] + (["--dynamic-schedule"] if g["dynamic"] else [])
    return args


# ================================================================================================ CPU: oracle, schedules
@pytest.mark.parametrize("name", CASES)
def test_oracle_is_the_scripts(name):
    g, per_seq = _golden(name)
    lengths, samples, pf, seed = g["lengths"].tolist(), g["samples"].tolist(), float(g["perf_factor"]), int(g["seed"])
    if str(g["clock"]) == "simulated":
        got = srt_oracle.srt_det(lengths, float(g["fps"]), float(g["det_stride"]), bool(g["dynamic"]), samples, pf, seed)
    else:
        got = srt_oracle.srt_det_inf(lengths, float(g["fps"]), samples, pf, seed)
    assert [s[:3] for s in got] == [s[:3] for s in per_seq]
    assert all(fi == rf for fi, _, _, rf in per_seq)          # every result is the frame its row names
    assert [r for s in got for r in s[2]] == g["runtime_all"].tolist() and int(g["n_total"]) == sum(lengths)
    if name == "srt_inf_ties":                              # ties, and np.argsort did not keep them in frame order
        raw = [sorted(zip(fi, rt)) for fi, _, rt, _ in per_seq]
        raw = [[ii / FPS + r for ii, r in s] for s in raw]
        assert sum(len(t) - len(set(t)) for t in raw) > 0
        assert any(np.argsort(t, kind="stable").tolist() != s[0] for t, s in zip(raw, per_seq))


def test_the_fixtures_cover_the_protocol():
    g = {n: np.load(os.path.join(GOLDEN, n + ".npz")) for n in CASES}
    sim = [v for v in g.values() if str(v["clock"]) == "simulated"]
    assert {int(v["seed"]) for v in g.values()} == {0, 5} and {float(v["perf_factor"]) for v in g.values()} == {1, 1.37}
    assert {float(v["det_stride"]) for v in sim if not v["dynamic"]} == {1, 1.5, 2}
    rtf = {v["samples"].mean() / v["perf_factor"] * v["fps"] > 1 for v in sim if v["dynamic"]}
    assert rtf == {True, False}
    assert all(len(v["lengths"]) > 2 and (v["lengths"] == 0).any() for v in g.values())


@pytest.mark.parametrize("dynamic", [False, True], ids=["fixed", "dynamic"])
@pytest.mark.parametrize("stride", [1, 2, 1.5, 3])
def test_schedules_are_the_oracles(stride, dynamic):
    """sequences of 0 to 900 frames, seeds, perf factors and distributions below, around and above one frame: the
    schedules sap computes one after another from one generator equal the oracle's whole run"""
    lengths = [0, 1, 2, 7, 30, 31, 5, 900, 64]
    dists = [[0.011, 0.019, 0.03], [0.02, 0.033, 0.05, 0.09], [0.06, 0.11, 0.075], [1 / FPS]]
    for samples in dists:
        for seed in (0, 1, 12345):
            for pf in (1, 0.8, 1.37, 3.0):
                want = srt_oracle.srt_det(lengths, FPS, stride, dynamic, samples, pf, seed)
                dist = sap.Empirical(samples, pf, seed)
                got = [sap.simulated_schedule(n, FPS, stride, dynamic, dist) for n in lengths]
                assert got == want, (samples, seed, pf)
                assert all(type(r) is np.float64 for s in got for r in s[2])


def test_constant_runtime_keeps_its_form():
    """a number still gives (input_fidx, timestamps), the oracle's"""
    for rt in (0.02, 0.05):
        got = sap.simulated_schedule(31, FPS, 1, False, rt)
        assert got == sap_oracle.simulated_schedule(31, FPS, 1, False, rt) and len(got) == 2


# ================================================================================================ CPU: the command
@pytest.mark.parametrize("streams", [1, 3])
@pytest.mark.parametrize("name", CASES)
def test_run_writes_the_scripts_pickles(tmp_path, capsys, name, streams):
    g, per_seq = _golden(name)
    root, ann = _dataset(tmp_path, str(g["annot"]))
    out = tmp_path / "out"
    opts = _opts(root, ann, out, *_case_args(g, _runtime(tmp_path, g["samples"])), "--streams", str(streams))
    info = sap.run(opts, None, detector=TagDetector)
    infinite = str(g["clock"]) == "infinite"
    for q, (fi, ts, rt, rf) in enumerate(per_seq):
        d = _load(out / f"s{q}.pkl")
        assert sorted(d) == ["input_fidx", "results_parsed", "results_raw", "runtime", "timestamps"]
        assert (d["input_fidx"], d["timestamps"], d["runtime"]) == (fi, ts, rt), q
        assert all(type(v) is int for v in d["input_fidx"]) and all(type(v) is np.float64 for v in d["runtime"])
        assert [int(b[0, 0]) for b, *_ in d["results_parsed"]] == rf, q
        assert [int(r[0, 0, 1]) for r in d["results_raw"]] == rf, q
        if infinite:                                  # frame ii fused with ii - 1, frame 0 with itself
            assert all(int(b[0, 1]) == max(int(b[0, 0]) - 1, 0) and int(b[0, 2]) == q for b, *_ in d["results_parsed"])
    t = _load(out / "time_info.pkl")
    assert sorted(t) == ["n_processed", "n_small_runtime", "n_total", "runtime_all"]
    assert t["runtime_all"] == g["runtime_all"].tolist() and t["runtime_all"] == info["runtime_all"]
    assert (t["n_processed"], t["n_total"], t["n_small_runtime"]) == (int(g["n_processed"]), int(g["n_total"]),
                                                                       int(g["n_small_runtime"]))
    assert capsys.readouterr().out == str(g["printed"])
    # a second run writes the same bytes
    before = _contents(out)
    sap.run(opts, None, detector=TagDetector)
    capsys.readouterr()
    assert _same_contents(_contents(out), before)


@pytest.mark.parametrize("clock", ["simulated", "simulated_dynamic", "simulated_stride2"])
def test_one_sample_equals_runtime_ms(tmp_path, clock):
    """{samples: [R]} and --runtime-ms R * 1000: the same schedules, results and time_info"""
    extra = {"simulated": [], "simulated_dynamic": ["--dynamic-schedule"], "simulated_stride2": ["--det-stride", "2"]}[clock]
    root, ann = _dataset(tmp_path, json.dumps({
        "sequences": ["a", "b", "c"], "seq_dirs": ["a", "b", "c"],
        "images": [{"id": 100 * q + j, "sid": q, "fid": j, "name": f"{j:06d}.jpg", "width": 1920, "height": 1200}
                   for q, n in enumerate([31, 9, 44]) for j in range(n)]}))
    for r in (0.02, 1 / 30, 0.045, 0.11):
        assert r * 1000 / 1000.0 == r
        a, b = tmp_path / f"a{r}", tmp_path / f"b{r}"
        ia = sap.run(_opts(root, ann, a, "--clock", "simulated", "--runtime", str(_runtime(tmp_path, [r])), *extra),
                     None, detector=TagDetector)
        ib = sap.run(_opts(root, ann, b, "--clock", "simulated", "--runtime-ms", repr(r * 1000), *extra), None,
                     detector=TagDetector)
        for q in "abc":
            da, db = _load(a / f"{q}.pkl"), _load(b / f"{q}.pkl")
            assert da["input_fidx"] and (da["input_fidx"], da["timestamps"], da["runtime"]) == (
                db["input_fidx"], db["timestamps"], db["runtime"])
            assert all(torch.equal(x, y) for x, y in zip(da["results_raw"], db["results_raw"]))
            assert all(all(np.array_equal(x, y) for x, y in zip(u[:3], v[:3])) for u, v in
                       zip(da["results_parsed"], db["results_parsed"]))
        assert ia["runtime_all"] == ib["runtime_all"] and ia["n_small_runtime"] == ib["n_small_runtime"]


def test_global_generator_is_left_alone(tmp_path):
    g, _ = _golden("srt_seed0")
    root, ann = _dataset(tmp_path, str(g["annot"]))
    np.random.seed(77)
    before = np.random.get_state()
    for clock in ("simulated", "infinite"):
        sap.run(_opts(root, ann, tmp_path / clock, "--clock", clock, "--runtime",
                      str(_runtime(tmp_path, g["samples"])), "--seed", "3"), None, detector=TagDetector)
    after = np.random.get_state()
    assert all(np.array_equal(x, y) for x, y in zip(before, after))


# ================================================================================================ CPU: arguments
BASE = ["--data-root", "d", "--annot-path", "a", "--out-dir", "o", "--config", "c", "--weights", "w"]


def test_arguments():
    o = sap.parse_args(BASE + ["--clock", "simulated", "--runtime", "rt.pkl"])
    assert (o.runtime, o.runtime_ms, o.perf_factor, o.seed, o.det_stride, o.cached_res) == ("rt.pkl", None, 1, 0, 1, None)
    o = sap.parse_args(BASE + ["--clock", "simulated", "--runtime", "rt.pkl", "--perf-factor", "1.5", "--seed", "9",
                               "--det-stride", "1.5", "--dynamic-schedule", "--streams", "4"])
    assert (o.perf_factor, o.seed, o.det_stride, o.dynamic_schedule, o.streams) == (1.5, 9, 1.5, True, 4)
    o = sap.parse_args(BASE + ["--clock", "infinite", "--runtime", "rt.pkl", "--perf-factor", "2", "--seed", "1",
                               "--streams", "8"])
    assert (o.clock, o.perf_factor, o.seed, o.streams, o.det_stride, o.dynamic_schedule) == ("infinite", 2, 1, 8, 1, False)
    o = sap.parse_args(BASE + ["--clock", "simulated", "--runtime-ms", "30"])
    assert (o.runtime, o.perf_factor, o.seed) == (None, 1, 0)
    for bad in (["--clock", "simulated", "--runtime", "r", "--runtime-ms", "30"],     # two runtime sources
                ["--clock", "simulated"], ["--clock", "infinite"],                     # none
                ["--clock", "infinite", "--runtime-ms", "30"],
                ["--runtime", "r"], ["--runtime", "r", "--clock", "wall"],             # the wall clock measures
                ["--clock", "simulated", "--runtime-ms", "30", "--perf-factor", "2"],  # need --runtime
                ["--clock", "simulated", "--runtime-ms", "30", "--seed", "2"], ["--seed", "2"],
                ["--clock", "simulated", "--runtime", "r", "--perf-factor", "0"],
                ["--clock", "simulated", "--runtime", "r", "--perf-factor", "-1"],
                ["--clock", "infinite", "--runtime", "r", "--det-stride", "2"],
                ["--clock", "infinite", "--runtime", "r", "--det-stride", "1"],
                ["--clock", "infinite", "--runtime", "r", "--dynamic-schedule"],
                ["--clock", "infinite", "--runtime", "r", "--streams", "0"]):
        with pytest.raises(SystemExit):
            sap.parse_args(BASE + bad)
    with pytest.raises(NotImplementedError, match="depends on the frame processed before it"):
        sap.parse_args(BASE + ["--clock", "simulated", "--runtime", "r", "--cached-res", "c.pkl"])


def test_unknown_distribution_type(tmp_path):
    g, _ = _golden("srt_seed0")
    root, ann = _dataset(tmp_path, str(g["annot"]))
    for clock in ("simulated", "infinite"):
        rt = _runtime(tmp_path, [0.03], kind="gaussian")
        with pytest.raises(ValueError, match='Unknown distribution type "gaussian"'):
            sap.run(_opts(root, ann, tmp_path / "o", "--clock", clock, "--runtime", str(rt)), None, detector=TagDetector)


# ================================================================================================ GPU
SAMPLES = [0.021, 0.034, 0.028, 0.061, 0.019, 0.045, 0.1]


def _gpu_run(tmp_path, m, extra, detector=stream.StreamDetector):
    from test_sap_driver import LENGTHS, _jpeg_dataset
    root, ann = _jpeg_dataset(tmp_path, LENGTHS)
    out = tmp_path / "out"
    sap.run(_opts(root, ann, out, "--runtime", str(_runtime(tmp_path, SAMPLES)), *extra), m, detector=detector)
    return root, ann, out, [_load(out / f"s{q}.pkl") for q in range(len(LENGTHS))]


@pytest.mark.gpu
def test_infinite_one_stream_equals_the_eager_driver(tmp_path):
    """every frame through the driver's loop body, eagerly, then srt_det_inf's reordering: the same rows, bit for bit"""
    from test_sap_driver import LENGTHS, _eager, _model, _same
    m = _model("s")
    _, _, _, pk = _gpu_run(tmp_path, m, ["--clock", "infinite", "--seed", "4"])
    want = srt_oracle.srt_det_inf(LENGTHS, FPS, SAMPLES, 1, 4)
    n_dets = 0
    for q, (d, (fi, ts, rt)) in enumerate(zip(pk, want)):
        assert (d["input_fidx"], d["timestamps"], d["runtime"]) == (fi, ts, rt)
        eager = _eager(m, q, range(LENGTHS[q]))
        for k, ii in enumerate(d["input_fidx"]):
            res, parsed = eager[ii]
            assert torch.equal(d["results_raw"][k], res), (q, ii)
            assert _same(parsed + (None,), d["results_parsed"][k]), (q, ii)
            n_dets += len(parsed[2])
    assert n_dets > 0 and any(d["input_fidx"] != sorted(d["input_fidx"]) for d in pk)


@pytest.mark.gpu
def test_infinite_four_streams_equal_eager_batch(tmp_path):
    """five sequences on four streams, every frame: each stream's rows equal two eager on_pipe calls at batch 4 (its
    current features at a sequence start, its carried ones otherwise), placed where srt_det_inf's order puts them"""
    from test_sap_driver import LENGTHS, Recorder, _frame, _model, _same, IN_SCALE, SIZE
    from test_stream import driver_inference
    from streamyolo_b200 import data
    m = _model("s")
    dets = []

    def recorder(*a, **k):
        dets.append(Recorder(*a, **k))
        return dets[-1]

    _, _, _, pk = _gpu_run(tmp_path, m, ["--clock", "infinite", "--streams", "4"], detector=recorder)
    det, = dets
    ticks = sap.pack_ticks(LENGTHS, 4)
    assert det.streams == 4 and len(ticks) == len(det.log) and any(e is None for row in ticks for e in row)
    carried = None
    for t, (row, (x, present, resets)) in enumerate(zip(ticks, det.log)):
        assert present == [e is not None for e in row]
        assert resets == {s for s, e in enumerate(row) if e is not None and e[1] == 0}
        for s, e in enumerate(row):
            if e is not None:
                assert torch.equal(x[s], data.stream_frame(_frame(*e), SIZE)[0]), (t, s)
        with torch.no_grad():
            _, cur = m(x, mode="on_pipe")
            cur = tuple(c.clone() for c in cur)
            start = [e is not None and e[1] == 0 for e in row]
            mix = tuple(torch.stack([c[i] if start[i] or carried is None else p[i] for i in range(4)]).contiguous(
                memory_format=torch.channels_last) for c, p in zip(cur, carried or cur))
            result, _ = m(x, buffer=mix, mode="on_pipe")
        for s, e in enumerate(row):
            if e is not None:
                q, ii = e                             # the schedule is every frame: the k-th entry is frame k
                k = pk[q]["input_fidx"].index(ii)
                assert torch.equal(pk[q]["results_raw"][k][0], result[s]), (t, s)
                want = driver_inference(result[s].cpu(), m.head.num_classes, IN_SCALE)
                assert _same(want + (None,), pk[q]["results_parsed"][k]), (t, s)
        carried = tuple(torch.stack([c[i] if row[i] is not None else p[i] for i in range(4)]).contiguous(
            memory_format=torch.channels_last) for c, p in zip(cur, carried or cur))


@pytest.mark.gpu
def test_simulated_draws_run_the_scheduled_frames(tmp_path):
    """--clock simulated with a seven-sample distribution and --perf-factor: srt_det's schedule, and each row the eager
    driver loop's on the frames that schedule lists; a second run writes the same bytes"""
    from test_sap_driver import LENGTHS, _eager, _model, _same
    m = _model("s")
    extra = ["--clock", "simulated", "--perf-factor", "1.3", "--seed", "2"]
    _, _, out, pk = _gpu_run(tmp_path, m, extra)
    want = srt_oracle.srt_det(LENGTHS, FPS, 1, False, SAMPLES, 1.3, 2)
    assert any(len(fi) < n for (fi, _, _), n in zip(want, LENGTHS))        # frames were skipped
    for q, (d, (fi, ts, rt)) in enumerate(zip(pk, want)):
        assert (d["input_fidx"], d["timestamps"], d["runtime"]) == (fi, ts, rt)
        for (res, parsed), raw, got in zip(_eager(m, q, fi), d["results_raw"], d["results_parsed"]):
            assert torch.equal(raw, res) and _same(parsed + (None,), got), q
    before = _contents(out)
    _gpu_run(tmp_path, m, extra)
    assert _same_contents(_contents(out), before)
