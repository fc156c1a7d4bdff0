"""The sAP streaming driver on the device (streamyolo_b200.sap, ``python -m streamyolo_b200.sap``).

CPU (no GPU needed):
  * the wall clock's loop, driven by a fake clock and a fake detector whose ticks take scripted times (faster than,
    exactly, and slower than 1/fps, and ticks that run past the sequence's end), keeps the frames and timestamps of the
    driver's loop as oracle/sap_oracle.py restates it, for --det-stride 1, 2, 1.5 with --dynamic-schedule on and off;
  * the simulated clock's schedule is srt_det.py's for runtimes below, at and above 1/fps;
  * every argument the driver takes parses; the annotation file's order gives COCO.imgs' per-sequence frame lists;
  * with a fake detector: the pickles have the driver's keys, types and dtypes, --overwrite is respected, and packing
    sequences of different lengths onto fewer streams (idle streams included) gives each sequence what it gets alone.

GPU (H100), sequences made of the 1200x1920 JPEG fixture requantised into distinct frames (tests/golden):
  * wall clock with a fake clock, tiny and StreamYOLO-s models, fp16 storage: every result equals the eager driver loop
    (cv2's frame, preproc, model(x, buffer, mode='on_pipe'), inference()) on the same input_fidx, bit for bit;
  * simulated clock, one stream: the same results as the wall clock for the same schedule;
  * simulated clock, 4 streams: each stream equals eager on_pipe calls at batch 4, stream by stream;
  * a damaged file raises and names itself, on both clocks.
"""
import json
import os
import pickle
import sys
import zlib

import numpy as np
import pytest
import torch

from oracle.make_stream_jpeg_golden import SEQ, requant
from oracle.sap_oracle import simulated_schedule as oracle_simulated, wall_schedule as oracle_wall
from streamyolo_b200 import data, sap, stream

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FPS = 30.0
STRIDES = [1, 2, 1.5]


# ================================================================================================ fakes
class FakeClock:
    """perf_counter on a script: every read returns the time and moves it on by ``poll`` (FakeDetector adds its ticks)"""

    def __init__(self, poll):
        self.t, self.poll = 0.0, poll

    def __call__(self):
        t = self.t
        self.t += self.poll
        return t


def fake_result(content, previous):
    """a detector's output that depends on the frame and on the frame it is fused with (the carried one)"""
    h = zlib.crc32(bytes(content)) ^ (zlib.crc32(bytes(previous)) << 1)
    n = h % 5
    rng = np.random.default_rng(h)
    return (rng.random((n, 4)).astype(np.float32) * 1000, rng.random(n).astype(np.float32),
            rng.integers(0, 8, n).astype(np.int32))


class FakeDetector:
    """StreamDetector's interface without a GPU: each stream carries its previous frame, reset(i) makes its next frame
    fuse with itself; ``durations`` (seconds, cycled) are added to ``clock`` per ``step``"""

    def __init__(self, model, frame_hw=None, in_scale=0.5, frame_sizes=None, jpeg_max_bytes=None, clock=None,
                 durations=(0.0,)):
        self.streams = 1 if frame_sizes is None else len(frame_sizes)
        self.jpeg_max_bytes, self.clock, self.durations = jpeg_max_bytes, clock, durations
        self.prev, self.flags = [None] * self.streams, [1] * self.streams
        self.ticks, self.status, self.raw = 0, None, None

    def reset(self, stream=None):
        for s in range(self.streams) if stream is None else [stream]:
            self.flags[s] = 1

    def _tick(self, frames):
        out = []
        for s, f in enumerate(frames):
            if f is None:
                out.append((np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros(0, np.int32)))
                continue
            if self.flags[s]:
                self.prev[s] = f
            out.append(fake_result(f, self.prev[s]))
            self.prev[s], self.flags[s] = f, 0
        self.raw = torch.tensor([[float(len(r[0])), float(r[1].sum()) if len(r[1]) else 0.0] for r in out],
                                dtype=torch.float16)[:, None, :]
        self.status = np.array([stream.NO_FRAME if f is None else 0 for f in frames], np.int32)
        if self.clock is not None:
            self.clock.t += self.durations[self.ticks % len(self.durations)]
        self.ticks += 1
        return out

    def step(self, frame):
        return self._tick([np.asarray(frame, np.uint8).tobytes()])

    def step_jpeg(self, files):
        assert len(files) == self.streams and all(f is None or len(f) <= self.jpeg_max_bytes for f in files)
        return self._tick([None if f is None else f.tobytes() for f in files])

    def last_raw(self):
        return self.raw.clone()

    def last_status(self):
        return self.status.copy()


# ================================================================================================ CPU: schedules
# scripted tick durations: faster than 1/fps, exactly 1/fps, slower, and a mix whose long ticks cross the sequence's end
DURATIONS = {"fast": [0.011], "exact": [1 / FPS], "slow": [0.052, 0.047], "mixed": [0.02, 1 / FPS, 0.09, 0.004, 0.3]}


@pytest.mark.parametrize("durations", list(DURATIONS), ids=list(DURATIONS))
@pytest.mark.parametrize("dynamic", [False, True], ids=["fixed", "dynamic"])
@pytest.mark.parametrize("stride", STRIDES)
def test_wall_loop_is_the_drivers(durations, dynamic, stride):
    """wall_sequence on a fake clock (0.7 ms per read) = the driver's loop restated, for sequences of 1, 13 and 40 frames"""
    crossed = 0
    for n in (1, 13, 40):
        clock = FakeClock(0.0007)
        det = FakeDetector(None, clock=clock, durations=DURATIONS[durations])
        frames = [np.full((2, 2, 3), k, np.uint8) for k in range(n)]
        out = sap.wall_sequence(det, frames, n, FPS, stride, dynamic, clock)
        fidx, ts, ticks = oracle_wall(n, FPS, stride, dynamic, DURATIONS[durations], 0.0007)
        assert out["input_fidx"] == fidx and out["timestamps"] == ts and det.ticks == ticks, (n, out["input_fidx"], fidx)
        assert len(out["runtime"]) == len(fidx) and all(r > 0 for r in out["runtime"])
        crossed += ticks == len(fidx) + 1
        if dynamic is False and stride == 1 and durations == "fast" and n > 1:
            assert fidx == list(range(n)), fidx           # a detector faster than the camera sees every frame
    if durations == "mixed":
        assert crossed >= 1                               # a tick ran past the end and was dropped


@pytest.mark.parametrize("runtime", [0.02, 1 / FPS, 0.05, 0.11], ids=["below", "at", "above", "far_above"])
@pytest.mark.parametrize("dynamic", [False, True], ids=["fixed", "dynamic"])
@pytest.mark.parametrize("stride", STRIDES)
def test_simulated_schedule_is_srt_det(runtime, dynamic, stride):
    for n in (0, 1, 2, 7, 30, 31, 900):
        got = sap.simulated_schedule(n, FPS, stride, dynamic, runtime)
        assert got == oracle_simulated(n, FPS, stride, dynamic, runtime), n
        fidx, ts = got
        # not always increasing: after the idle jump to frame k (t = k / fps) srt_det's floor(t * fps) can give k - 1
        # again, and the oracle keeps that too
        assert all(0 <= f < n for f in fidx) and all(t < n / FPS for t in ts)


def test_simulated_schedule_examples():
    """schedules worked out by hand: at 20 ms every frame; at 50 ms (1.5 frames) frames 0, 1, 3, with frame 4's result
    due at the sequence's end and dropped; stride 2 every 2nd frame; with --dynamic-schedule at 50 ms a frame already
    half gone is waited out and the next one taken when it arrives"""
    assert sap.simulated_schedule(5, FPS, 1, False, 0.02)[0] == [0, 1, 2, 3, 4]
    assert sap.simulated_schedule(6, FPS, 1, False, 0.05)[0] == [0, 1, 3]
    assert sap.simulated_schedule(6, FPS, 2, False, 0.02)[0] == [0, 2, 4]
    assert sap.simulated_schedule(9, FPS, 1, True, 0.05) == ([0, 2, 4, 6], [0.05, 0.11666666666666667, 0.18333333333333335,
                                                                            0.25])


# ================================================================================================ CPU: arguments, order
DRIVER_ARGS = ["--data-root", "/d/tracking", "--annot-path", "/d/val.json", "--det-stride", "2", "--in_scale", "0.5",
               "--fps", "30", "--no-mask", "--no-class-mapping", "--cpu-pre", "--dynamic-schedule", "--out-dir", "/o",
               "--config", "/c.py", "--weights", "/w.pth", "--overwrite"]


def test_arguments():
    """every argument of the driver's parse_args (streamyolo_det.py:30-47), with its defaults; the three new ones"""
    o = sap.parse_args(DRIVER_ARGS)
    assert (o.data_root, o.annot_path, o.det_stride, o.in_scale, o.fps, o.out_dir, o.config, o.weights) == (
        "/d/tracking", "/d/val.json", 2.0, 0.5, 30.0, "/o", "/c.py", "/w.pth")
    assert o.no_mask and o.no_class_mapping and o.cpu_pre and o.dynamic_schedule and o.overwrite
    assert (o.clock, o.runtime_ms, o.streams) == ("wall", None, 1)
    o = sap.parse_args(["--data-root", "a", "--annot-path", "b", "--out-dir", "c", "--config", "d", "--weights", "e"])
    assert (o.det_stride, o.in_scale, o.fps, o.no_mask, o.dynamic_schedule, o.overwrite) == (1, 0.5, 30, False, False, False)
    o = sap.parse_args(DRIVER_ARGS + ["--clock", "simulated", "--runtime-ms", "33.3", "--streams", "8"])
    assert (o.clock, o.runtime_ms, o.streams) == ("simulated", 33.3, 8)
    for bad in (["--clock", "simulated"], ["--runtime-ms", "30"], ["--streams", "2"],
                ["--clock", "simulated", "--runtime-ms", "0"], ["--clock", "simulated", "--runtime-ms", "5", "--streams", "0"]):
        with pytest.raises(SystemExit):
            sap.parse_args(DRIVER_ARGS + bad)


def test_sequence_order_is_coco_imgs():
    """interleaved sequences, ids out of order and a repeated id: COCO.imgs (id -> image, insertion order of
    dataset['images'], a repeated id keeps its first place and its last dict) filtered by sid"""
    img = lambda i, sid, name: {"id": i, "sid": sid, "name": name, "width": 1920, "height": 1200}
    ds = {"sequences": ["a", "b", "c"], "seq_dirs": ["da", "db", "dc"],
          "images": [img(7, 1, "b0"), img(3, 0, "a0"), img(9, 1, "b1"), img(1, 0, "a1"), img(3, 0, "a0bis"),
                     img(2, 1, "b2"), img(0, 0, "a2")]}
    got = [[i["name"] for i in s] for s in sap.sequences(ds)]
    assert got == [["a0bis", "a1", "a2"], ["b0", "b1", "b2"], []]


# ================================================================================================ CPU: pickles, packing
def _dataset(tmp_path, lengths, name="seq"):
    """an annotation file and fake frame files: sequence q has lengths[q] frames"""
    root = tmp_path / "data"
    images, k = [], 0
    for q, n in enumerate(lengths):
        (root / f"dir{q}").mkdir(parents=True, exist_ok=True)
        for j in range(n):
            (root / f"dir{q}" / f"{j:06d}.jpg").write_bytes(f"{name} {q} frame {j}".encode() * (j + 1))
            images.append({"id": k, "sid": q, "fid": j, "name": f"{j:06d}.jpg", "width": 1920, "height": 1200})
            k += 1
    ann = tmp_path / "val.json"
    ann.write_text(json.dumps({"sequences": [f"s{q}" for q in range(len(lengths))],
                               "seq_dirs": [f"dir{q}" for q in range(len(lengths))], "images": images,
                               "categories": [{"id": 0, "name": "car"}]}))
    return root, ann


def _opts(root, ann, out, *extra):
    return sap.parse_args(["--data-root", str(root), "--annot-path", str(ann), "--out-dir", str(out), "--config", "c",
                           "--weights", "w", *extra])


def _load(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def test_pickles_have_the_drivers_layout_and_overwrite(tmp_path, capsys):
    root, ann = _dataset(tmp_path, [9, 0, 14])
    out = tmp_path / "out"
    opts = _opts(root, ann, out, "--clock", "simulated", "--runtime-ms", "40", "--streams", "2")
    info = sap.run(opts, None, detector=FakeDetector)
    for q, n in enumerate([9, 0, 14]):
        d = _load(out / f"s{q}.pkl")
        assert sorted(d) == ["input_fidx", "results_parsed", "results_raw", "runtime", "timestamps"]
        fidx, ts = sap.simulated_schedule(n, 30, 1, False, 0.04)
        assert d["input_fidx"] == fidx and d["timestamps"] == ts and d["runtime"] == [0.04] * len(fidx)
        assert all(type(v) is int for v in d["input_fidx"]) and all(type(v) is float for v in d["timestamps"] + d["runtime"])
        assert len(d["results_parsed"]) == len(d["results_raw"]) == len(fidx)
        for (b, s, l, m), raw in zip(d["results_parsed"], d["results_raw"]):
            assert b.dtype == np.float32 and b.ndim == 2 and b.shape[1] == 4 and s.dtype == np.float32 and s.shape == b.shape[:1]
            assert l.dtype == np.int32 and l.shape == s.shape and m is None
            assert torch.is_tensor(raw) and raw.shape[0] == 1
    t = _load(out / "time_info.pkl")
    assert sorted(t) == ["n_processed", "n_small_runtime", "n_total", "runtime_all"]
    assert t["n_total"] == 23 and t["n_processed"] == len(t["runtime_all"]) == info["n_processed"]
    assert t["n_small_runtime"] == 0 and isinstance(t["n_small_runtime"], np.integer)
    printed = capsys.readouterr().out
    assert f"{t['n_processed']}/23 frames processed" in printed and "Runtime (ms): mean: 40; std: " in printed
    assert "min: 40; max: 40\n" in printed
    assert "Runtime smaller than unit time interval: 0/" in printed
    # without --overwrite nothing is rewritten; with it, everything is
    before = {p: (out / p).read_bytes() for p in os.listdir(out)}
    opts2 = _opts(root, ann, out, "--clock", "simulated", "--runtime-ms", "20")
    sap.run(opts2, None, detector=FakeDetector)
    assert {p: (out / p).read_bytes() for p in os.listdir(out)} == before
    sap.run(_opts(root, ann, out, "--clock", "simulated", "--runtime-ms", "20", "--overwrite"), None, detector=FakeDetector)
    assert _load(out / "s0.pkl")["runtime"] == [0.02] * 9 and _load(out / "time_info.pkl")["n_small_runtime"] == 23


def test_pack_ticks():
    """three sequences on two streams: the third takes the first free stream at the next tick, idle streams get None;
    an empty sequence takes no stream"""
    ticks = sap.pack_ticks([2, 0, 4, 1], 2)
    assert ticks == [[(0, 0), (2, 0)], [(0, 1), (2, 1)], [(3, 0), (2, 2)], [None, (2, 3)]]
    assert sap.pack_ticks([3], 4) == [[(0, 0), None, None, None], [(0, 1), None, None, None], [(0, 2), None, None, None]]
    assert sap.pack_ticks([0, 0], 2) == []


@pytest.mark.parametrize("streams", [2, 3, 5, 8])
def test_packed_streams_equal_sequences_alone(tmp_path, streams):
    """sequences of different lengths (one empty, one of a single frame), more sequences than streams, streams idle at the
    end: with a detector whose results depend on each stream's carried frame, every sequence gets, in every pickle
    field, what it gets on one stream"""
    lengths = [17, 5, 0, 30, 1, 12, 9]
    root, ann = _dataset(tmp_path, lengths)
    with open(ann) as f:
        seqs, paths = sap.frame_paths(_opts(root, ann, tmp_path), json.load(f))
    schedules = [sap.simulated_schedule(len(p), FPS, 1, False, 0.045) for p in paths]
    results = {}
    for s in (1, streams):
        got = {}
        det = FakeDetector(None, frame_sizes=[(1200, 1920)] * s, jpeg_max_bytes=1 << 12)
        sap.run_simulated(det, paths, schedules, 0.045, lambda q, out: got.__setitem__(q, out))
        assert sorted(got) == list(range(len(lengths)))
        results[s] = got
    for q in range(len(lengths)):
        a, b = results[1][q], results[streams][q]
        assert a["input_fidx"] == b["input_fidx"] and a["timestamps"] == b["timestamps"] and a["runtime"] == b["runtime"]
        assert all(all(np.array_equal(x, y) for x, y in zip(u[:3], v[:3])) for u, v in
                   zip(a["results_parsed"], b["results_parsed"])), q
        assert all(torch.equal(u, v) for u, v in zip(a["results_raw"], b["results_raw"])), q


# ================================================================================================ GPU
DEV = "cuda"
G = np.load(os.path.join(ROOT, "tests", "golden", "stream_jpeg_files.npz"))
SIZE, IN_SCALE = (600, 960), 0.5


def _jpeg_dataset(tmp_path, lengths, damaged=None):
    """sequences of the 1200x1920 fixture requantised (frame j of sequence q: step (q + j) % SEQ); ``damaged``: (q, j)
    whose file is the damaged fixture"""
    root = tmp_path / "data"
    images, k = [], 0
    a420 = bytes(G["a420.jpg"])
    for q, n in enumerate(lengths):
        (root / f"dir{q}").mkdir(parents=True, exist_ok=True)
        for j in range(n):
            b = bytes(G["bad.jpg"]) if damaged == (q, j) else requant(a420, (q + j) % SEQ)
            (root / f"dir{q}" / f"{j:06d}.jpg").write_bytes(b)
            images.append({"id": k, "sid": q, "fid": j, "name": f"{j:06d}.jpg", "width": 1920, "height": 1200})
            k += 1
    ann = tmp_path / "val.json"
    ann.write_text(json.dumps({"sequences": [f"s{q}" for q in range(len(lengths))],
                               "seq_dirs": [f"dir{q}" for q in range(len(lengths))], "images": images}))
    return root, ann


def _model(tag):
    from test_gpu_model import build_product
    from test_stream import _model_s
    from oracle.make_golden import CASES
    from streamyolo_b200 import synth
    from streamyolo_b200.model import engine
    if tag == "s":
        return _model_s(torch.float16)
    tiny = CASES["tiny_120x160"]
    m = build_product(tiny["depth"], tiny["width"], momentum=1.0)
    engine.name_modules(m)
    m.cuda().train()
    x = synth.synth_frames(8, 600, 960, seed=99).cuda()
    fut, cur = synth.synth_labels(8, 600, 960, seed=11)
    with torch.no_grad():
        m(x, (fut.cuda(), cur.cuda()))
    m.eval()
    m.activation_dtype = torch.float16
    return m


def _frame(q, j):
    """cv2.imread's frame of sequence q's frame j (the device decode, checked against cv2's digest)"""
    rows, lengths = data.pack_jpeg([requant(bytes(G["a420.jpg"]), (q + j) % SEQ)], 1 << 19)
    f, st = data.decode_jpeg(torch.from_numpy(rows).to(DEV), torch.from_numpy(lengths).to(DEV), (1200, 1920))
    assert st.tolist() == [0]
    import hashlib
    assert hashlib.sha256(f[0].cpu().numpy().tobytes()).digest() == bytes(G["a420.seq"][(q + j) % SEQ])
    return f[0]


def _eager(m, q, fidx):
    """the driver's loop on the frames ``fidx`` of sequence q: -> [(result [1, A, 5 + nc], inference() tuple)]"""
    from test_stream import driver_inference
    buffer, out = None, []
    for j in fidx:
        with torch.no_grad():
            result, buffer = m(data.stream_frame(_frame(q, j), SIZE), buffer=buffer, mode="on_pipe")
        out.append((result.clone(), driver_inference(result[0].cpu(), m.head.num_classes, IN_SCALE)))
    return out


def _same(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a[:3], b[:3])) and b[3] is None


LENGTHS = [7, 4, 10, 3, 6]


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["tiny", "s"])
def test_wall_and_simulated_one_stream_equal_the_eager_driver(tmp_path, tag):
    """wall clock on a fake clock: every result equals the eager driver loop on the same input_fidx; the simulated clock
    on one stream, given that schedule, writes the same results"""
    m = _model(tag)
    root, ann = _jpeg_dataset(tmp_path, LENGTHS)
    out = tmp_path / "wall"
    # reads move the clock by 9 ms, 21 ms, 4 ms in turn: ticks of every kind, frames skipped, a tick past the end
    steps = iter(np.resize([0.009, 0.021, 0.004], 100000).tolist())
    t = [0.0]

    def clock():
        t[0] += next(steps)
        return t[0]

    sap.run(_opts(root, ann, out), m, clock=clock)
    with open(ann) as f:
        seqs, paths = sap.frame_paths(_opts(root, ann, out), json.load(f))
    wall = [_load(out / f"s{q}.pkl") for q in range(len(LENGTHS))]
    n_dets = 0
    for q, d in enumerate(wall):
        assert d["input_fidx"] and d["input_fidx"] == sorted(set(d["input_fidx"]))
        for (res, want), raw, got in zip(_eager(m, q, d["input_fidx"]), d["results_raw"], d["results_parsed"]):
            assert raw.is_cuda and torch.equal(raw, res), q
            assert _same(want + (None,), got), q
            n_dets += len(got[2])
    assert n_dets > 0
    # the simulated clock's runner on one JPEG stream, given the wall clock's schedules
    det = stream.StreamDetector(m, frame_sizes=[(1200, 1920)], in_scale=IN_SCALE, jpeg_max_bytes=1 << 19)
    sim = {}
    sap.run_simulated(det, paths, [(d["input_fidx"], d["timestamps"]) for d in wall], 0.03,
                      lambda q, o: sim.__setitem__(q, o))
    for q, d in enumerate(wall):
        assert sim[q]["input_fidx"] == d["input_fidx"]
        assert all(torch.equal(a, b) for a, b in zip(sim[q]["results_raw"], d["results_raw"]))
        assert all(_same(a, b) for a, b in zip(sim[q]["results_parsed"], d["results_parsed"]))
    # the CLI's simulated run on one stream keeps srt_det's schedule
    sap.run(_opts(root, ann, tmp_path / "sim", "--clock", "simulated", "--runtime-ms", "45"), m)
    for q, n in enumerate(LENGTHS):
        assert _load(tmp_path / "sim" / f"s{q}.pkl")["input_fidx"] == oracle_simulated(n, 30.0, 1, False, 0.045)[0]


class Recorder(stream.StreamDetector):
    """StreamDetector that keeps, per tick, its model input, the files it was given and the streams reset before it"""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.log, self._resets = [], set()

    def reset(self, stream=None):
        super().reset(stream)
        if stream is not None:
            self._resets.add(stream)

    def step_jpeg(self, files):
        got = super().step_jpeg(files)
        self.log.append((self._tick.x.clone(), [f is not None for f in files], set(self._resets)))
        self._resets = set()
        return got


@pytest.mark.gpu
def test_simulated_four_streams_equal_eager_batch(tmp_path):
    """five sequences of different lengths on four streams (a stream takes a second sequence, others go idle): each
    stream's results equal two eager on_pipe calls at batch 4 (current features, then the fusion with each stream's own
    support: its current features at a sequence start, its carried ones otherwise), as tests/test_stream_jpeg.py checks
    a rig; the inputs of the streams that have a frame are the driver's preproc of cv2's frame"""
    from test_stream import driver_inference
    m = _model("s")
    root, ann = _jpeg_dataset(tmp_path, LENGTHS)
    dets = []

    def recorder(*a, **k):
        dets.append(Recorder(*a, **k))
        return dets[-1]

    out = tmp_path / "out"
    sap.run(_opts(root, ann, out, "--clock", "simulated", "--runtime-ms", "50", "--streams", "4"), m, detector=recorder)
    det, = dets
    assert det.streams == 4
    schedules = [sap.simulated_schedule(n, 30.0, 1, False, 0.05) for n in LENGTHS]
    ticks = sap.pack_ticks([len(f) for f, _ in schedules], 4)
    assert len(ticks) == len(det.log) and any(e is None for row in ticks for e in row)
    pk = [_load(out / f"s{q}.pkl") for q in range(len(LENGTHS))]
    carried = None
    for t, (row, (x, present, resets)) in enumerate(zip(ticks, det.log)):
        assert present == [e is not None for e in row]
        assert resets == {s for s, e in enumerate(row) if e is not None and e[1] == 0}
        for s, e in enumerate(row):
            if e is not None:
                q, k = e
                assert torch.equal(x[s], data.stream_frame(_frame(q, schedules[q][0][k]), SIZE)[0]), (t, s)
        with torch.no_grad():
            _, cur = m(x, mode="on_pipe")
            cur = tuple(c.clone() for c in cur)
            start = [e is not None and e[1] == 0 for e in row]
            mix = tuple(torch.stack([c[i] if start[i] or carried is None else p[i] for i in range(4)]).contiguous(
                memory_format=torch.channels_last) for c, p in zip(cur, carried or cur))
            result, _ = m(x, buffer=mix, mode="on_pipe")
        for s, e in enumerate(row):
            if e is not None:
                q, k = e
                assert torch.equal(pk[q]["results_raw"][k][0], result[s]), (t, s)
                want = driver_inference(result[s].cpu(), m.head.num_classes, IN_SCALE)
                assert _same(want + (None,), pk[q]["results_parsed"][k]), (t, s)
        carried = tuple(torch.stack([c[i] if row[i] is not None else p[i] for i in range(4)]).contiguous(
            memory_format=torch.channels_last) for c, p in zip(cur, carried or cur))


@pytest.mark.gpu
@pytest.mark.parametrize("clock", ["wall", "simulated"])
def test_damaged_file_names_itself(tmp_path, clock):
    m = _model("tiny")
    root, ann = _jpeg_dataset(tmp_path, [3, 4], damaged=(1, 2))
    extra = [] if clock == "wall" else ["--clock", "simulated", "--runtime-ms", "10", "--streams", "2"]
    with pytest.raises(RuntimeError, match=r"dir1/000002\.jpg did not decode"):
        sap.run(_opts(root, ann, tmp_path / "out", *extra), m)
