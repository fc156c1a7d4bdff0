"""The sAP toolkit's streamer on the device (streamyolo_b200.streamer, ``python -m streamyolo_b200.streamer``).

CPU (no GPU needed), against tests/golden/streamer_*.npz (the unmodified streamer.py on a virtual clock, see
oracle/make_streamer_golden.py):
  * oracle/streamer_oracle.py reproduces every fixture exactly: emission times, input_fidx, rows and their dtypes,
    time_info counts and every association decision;
  * ``simulated_schedule`` gives the fixtures' emission times, input frames and counts;
  * ``wall_sequence`` on the virtual clock, with a detector emulated by the oracle's torch Kalman filter, writes the
    fixtures' pickles;
  * ``run`` on the simulated clock with an emulated StreamDetector (one and three streams) writes what the oracle
    streamer writes for each sequence, in streaming_eval.py's layout;
  * the streamer's arguments parse, and the clock-specific ones are checked.

GPU (H100):
  * sy_forecast_update's streamer mode equals the oracle on crafted detections (an empty one after matches clears the
    tracks, ids continue), and the pps mode still keeps the tracks there;
  * sy_forecast_extrap_queries is bit-identical to one sy_forecast_extrap per query for integer offsets, and equals the
    oracle's fp32 arithmetic bit for bit for fractional ones;
  * simulated clock, StreamYOLO-s on JPEG files, one and three streams: each stream's detections equal a forecast=False
    detector's bit for bit, and each sequence's pickle equals the oracle streamer fed those detections (boxes within
    the Kalman filter's fp32 rounding, everything else exactly);
  * one wall-clock run: timestamps increase, each output's input_fidx is the last received detection, each output is
    the oracle's extrapolation of that detection's tracks to its query.
"""
import copy
import inspect
import json
import os
import pickle
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import forecast_oracle as fo  # noqa: E402
from oracle import streamer_oracle as so  # noqa: E402
from oracle.make_streamer_golden import World  # noqa: E402
from streamyolo_b200 import ops, streamer  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["r20_eta0", "r75_eta0p3", "r75_dyn_eta0", "r45_dyn_etam0p5"]
BOX_ATOL = 1e-2          # pixels: the device's Kalman update sums in another order than torch's (see test_forecast.py)


def golden(name):
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", f"streamer_{name}.npz")))
    annot = json.loads(str(g["annot"]))
    img0 = next(i for i in annot["images"] if i["id"] == 0)
    seqs, k, r = [], 0, 0
    for n_frames in g["seq_frames"]:
        d = []
        for _ in range(n_frames):
            n = int(g["det_n"][k])
            d.append((g["det_box"][r:r + n], g["det_score"][r:r + n], g["det_label"][r:r + n]))
            k, r = k + 1, r + n
        seqs.append(d)
    rtf = np.asarray(g["samples"]).mean() * float(g["fps"]) if g["dynamic"] else None
    return g, seqs, (img0["width"], img0["height"]), rtf


def golden_pickles(g):
    """the fixture's per-sequence pickles"""
    out, e, r = [], 0, 0
    for n_emit in g["seq_emit"]:
        rows = []
        for j in range(e, e + n_emit):
            n = int(g["emit_rows"][j])
            rows.append((g["box"][r:r + n], g["score"][r:r + n], g["label"][r:r + n], None,
                         g["track"][r:r + n].astype(np.uint32 if g["emit_tracked"][j] else np.int32)))
            r += n
        out.append({"results_parsed": rows, "timestamps": g["timestamps"][e:e + n_emit].tolist(),
                    "input_fidx": g["input_fidx"][e:e + n_emit].tolist()})
        e += n_emit
    return out


def assert_rows_equal(got, want, what, atol=0.0):
    assert len(got) == len(want), what
    for j, (a, b) in enumerate(zip(got, want)):
        assert a[3] is None and b[3] is None, (what, j)
        for x, y in zip(a[:3] + a[4:], b[:3] + b[4:]):
            assert x.dtype == y.dtype and x.shape == y.shape, (what, j, x.dtype, y.dtype, x.shape, y.shape)
        if atol:
            np.testing.assert_allclose(a[0], b[0], rtol=0, atol=atol, err_msg=f"{what} {j}")
        else:
            np.testing.assert_array_equal(a[0].view(np.int32), b[0].view(np.int32), err_msg=f"{what} {j}")
        for x, y in zip(a[1:3] + a[4:], b[1:3] + b[4:]):
            np.testing.assert_array_equal(x, y, err_msg=f"{what} {j}")


def assert_pickle_equal(got, want, what, atol=0.0):
    assert set(got) == {"results_parsed", "timestamps", "input_fidx"}, what
    assert got["timestamps"] == want["timestamps"], what
    assert got["input_fidx"] == want["input_fidx"], what
    assert_rows_equal(got["results_parsed"], want["results_parsed"], what, atol)


def oracle_sequence(g, d, wh, rtf, log=None):
    return so.sequence(lambda f: d[f], len(d), *wh, fps=float(g["fps"]), eta=float(g["eta"]),
                       runtime=float(g["runtime"]), dynamic_schedule=bool(g["dynamic"]), mean_rtf=rtf, log=log)


# ================================================================================================ CPU
@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_reference(name):
    g, seqs, wh, rtf = golden(name)
    log, counts = [], np.zeros(5, np.int64)
    for d, want in zip(seqs, golden_pickles(g)):
        got, c = oracle_sequence(g, d, wh, rtf, log)
        assert_pickle_equal(got, want, name)
        counts += [c["t_det"]] * 4 + [c["t_forecast"]]
    np.testing.assert_array_equal(counts[[0, 1, 2, 3, 4]], g["time_counts"])
    assert int(g["n_total"]) == sum(len(d) for d in seqs)
    dec = [e for e in log if e[1] > 0]                 # the reference associates only when tracks exist
    assert [e[2] for e in dec] == g["dec_n_matched"].tolist()
    o1 = np.split(g["dec_order1"], np.cumsum(g["dec_len1"])[:-1])
    o2 = np.split(g["dec_order2"], np.cumsum(g["dec_len2"])[:-1])
    for e, a, b in zip(dec, o1, o2):
        assert list(e[3]) == a.tolist() and list(e[4]) == b.tolist()


def test_fixtures_cover_cases():
    seen = set()
    for name in NAMES:
        g, _, _, _ = golden(name)
        R = float(g["runtime"])
        seen.add("fast" if R < 1 / float(g["fps"]) else "slow")
        seen.add("dynamic" if g["dynamic"] else "static")
        seen.add("eta0" if float(g["eta"]) == 0 else "eta_frac")
        empty_after_match = (g["dec_len1"] == 0) & (g["dec_len2"] == 0)
        assert empty_after_match.any(), name                    # an empty detection with tracks: cleared
        assert ((g["dec_n_matched"] == 0) & (g["dec_len2"] > 0)).any(), name     # a restart with no match
        assert g["dec_margin"].min() >= 1e-4, name
        assert (~g["emit_tracked"]).any() and g["emit_tracked"].any(), name
        box = g["box"]
        ltrb_w = box[:, 2] - box[:, 0]
        assert (box[:, 0] == 0).any() and (box[:, 1] == 0).any() and (box[:, 2] == 640).any() and (box[:, 3] == 480).any()
        assert (ltrb_w > 0).all()
        assert len(g["seq_frames"]) >= 3
    assert seen == {"fast", "slow", "dynamic", "static", "eta0", "eta_frac"}


@pytest.mark.parametrize("name", NAMES)
def test_simulated_schedule_is_the_reference_loop(name):
    g, seqs, _, rtf = golden(name)
    counts = np.zeros(5, np.int64)
    for d, want in zip(seqs, golden_pickles(g)):
        sch = streamer.simulated_schedule(len(d), float(g["fps"]), float(g["runtime"]), 0.003, bool(g["dynamic"]), rtf)
        assert sch["timestamps"] == want["timestamps"]
        assert [sch["det_fidx"][k] for k in sch["emit_det"]] == want["input_fidx"]
        assert sch["emit_det"] == sorted(sch["emit_det"])
        counts += [len(sch["det_fidx"])] * 4 + [sch["n_forecast"]]
    np.testing.assert_array_equal(counts, g["time_counts"])


def test_next_frame_time_advances_the_frame():
    for fps in (30.0, 29.97, 10.0, 7.0):
        for f in range(0, 2000, 7):
            t = f / fps
            u = streamer.next_frame_time(t, fps)
            assert np.floor(u * fps) == np.floor(t * fps) + 1 and u >= t


class Emulated:
    """a one-stream detector for wall_sequence on World's virtual clock: the oracle's torch Kalman filter with the
    streamer's empty-detection rule, the sequence's detections by frame"""

    def __init__(self, world, dets, wh):
        self.world, self.dets, self.wh = world, dets, wh
        self.log = []

    def reset(self):
        self.tracks, self.last, self.pub = so.StreamerTracks(), None, None

    def submit(self, frame, fidx):
        assert frame == fidx and self.world.pending is None
        self.world.pending = (fidx, self.world.t + self.world.runtime)

    def poll(self, w):
        return self.world.poll(w)

    def receive(self):
        (fidx, _), self.world.pending = self.world.pending, None
        b, s, lab = self.dets[fidx]
        self.tracks.update(b, s, lab, 0 if self.last is None else fidx - self.last)
        self.last = fidx
        self.log.append(fidx)

    def publish(self):
        self.pub = copy.deepcopy(self.tracks)

    def query(self, dt):
        return [self.pub.query(dt, *self.wh)]


def _wall_lines():
    src, first = inspect.getsourcelines(streamer.wall_sequence)
    head = first + next(i for i, s in enumerate(src) if s.strip() == "t1 = clock()")
    start = first + next(i for i, s in enumerate(src) if s.strip() == "t_start = clock()")
    return head, start


@pytest.mark.parametrize("name", NAMES)
def test_wall_sequence_on_the_virtual_clock_is_the_reference(name):
    g, seqs, wh, rtf = golden(name)
    head, start = _wall_lines()
    counts = np.zeros(5, np.int64)
    for d, want in zip(seqs, golden_pickles(g)):
        world = World(float(g["runtime"]), float(g["fps"]), head, start)
        det = Emulated(world, d, wh)
        got, times = streamer.wall_sequence(det, list(range(len(d))), len(d), float(g["fps"]), float(g["eta"]), 0.003,
                                            bool(g["dynamic"]), rtf, clock=world.perf_counter)
        assert_pickle_equal(got, want, name)
        counts += [len(times[k]) for k in ("t_det", "t_send_frame", "t_recv_res", "t_assoc", "t_forecast")]
        assert all(abs(v - float(g["runtime"])) < 1e-9 for v in times["t_det"])
    np.testing.assert_array_equal(counts - [0, 0, 0, 0, 0], g["time_counts"])


class EmulatedDetector:
    """StreamDetector(jpeg_max_bytes, forecast=True, clear_on_empty=True, queries=Q) on the host: each file's bytes name
    its (sequence, frame), whose detection comes from ``DETS``; per stream the oracle's Kalman filter"""
    DETS, made = None, []

    def __init__(self, model, frame_sizes=None, jpeg_max_bytes=None, queries=0, forecast=False, clear_on_empty=False,
                 in_scale=0.5, match_iou_th=0.3, max_tracks=1024):
        assert forecast and clear_on_empty and queries >= 1 and jpeg_max_bytes
        self.streams, self.queries = len(frame_sizes), queries
        self.wh = [(w, h) for h, w in frame_sizes]
        self.tracks, self.last = [None] * self.streams, [None] * self.streams
        self.flags = [True] * self.streams
        EmulatedDetector.made.append(self)

    def reset(self, stream=None):
        self.flags[stream] = True

    def step_jpeg(self, files, fidx, query_dt):
        self.status, self.q = [], []
        for s, f in enumerate(files):
            if f is None:
                self.status.append(-1), self.q.append([])
                continue
            assert len(query_dt[s]) <= self.queries
            q, j = map(int, bytes(f).decode().split(","))
            if self.flags[s]:
                self.tracks[s], self.last[s], self.flags[s] = so.StreamerTracks(), fidx[s], False
            t = self.tracks[s]
            b, sc, lab = self.DETS[q][j]
            t.update(b, sc, lab, fidx[s] - self.last[s])
            self.last[s] = fidx[s]
            self.status.append(0)
            self.q.append([t.query(dt, *self.wh[s]) for dt in query_dt[s]])
        return [None] * self.streams

    def last_status(self):
        return np.asarray(self.status)

    def last_queries(self):
        return self.q


def _jpeg_free_dataset(tmp_path, seqs):
    """annotation file of 1200 x 1920 frames whose files hold "q,j" """
    root = tmp_path / "data"
    images, k = [], 0
    for q, d in enumerate(seqs):
        (root / f"dir{q}").mkdir(parents=True)
        for j in range(len(d)):
            (root / f"dir{q}" / f"{j:06d}.jpg").write_bytes(f"{q},{j}".encode())
            images.append({"id": k, "sid": q, "fid": j, "name": f"{j:06d}.jpg", "width": 1920, "height": 1200})
            k += 1
    ann = tmp_path / "val.json"
    ann.write_text(json.dumps({"sequences": [f"s{q}" for q in range(len(seqs))],
                               "seq_dirs": [f"dir{q}" for q in range(len(seqs))], "images": images}))
    return root, ann


def _args(root, ann, out, runtime, *extra):
    return ["--data-root", str(root), "--annot-path", str(ann), "--config", "c.py", "--weights", "w.pth",
            "--runtime", str(runtime), "--out-dir", str(out), "--overwrite", *extra]


def _runtime_pickle(tmp_path, samples):
    p = tmp_path / "rt.pkl"
    with open(p, "wb") as f:
        pickle.dump({"type": "empirical", "samples": list(samples)}, f)
    return p


def _load(p):
    with open(p, "rb") as f:
        return pickle.load(f)


@pytest.mark.parametrize("name,streams", [("r75_eta0p3", 1), ("r45_dyn_etam0p5", 3), ("r20_eta0", 2)])
def test_simulated_run_equals_the_oracle_streamer(tmp_path, name, streams, capsys):
    g, seqs, _, _ = golden(name)
    seqs = seqs + seqs[:2]                                 # five sequences: streams take a second one
    root, ann = _jpeg_free_dataset(tmp_path, seqs)
    rt = _runtime_pickle(tmp_path, g["samples"])
    eta = str(float(g["eta"]))
    extra = ["--clock", "simulated", "--runtime-ms", str(float(g["runtime"]) * 1000), "--streams", str(streams),
             "--eta", eta] + (["--dynamic-schedule"] if g["dynamic"] else [])
    opts = streamer.parse_args(_args(root, ann, tmp_path / "out", rt, *extra))
    EmulatedDetector.DETS, EmulatedDetector.made = seqs, []
    info = streamer.run(opts, None, detector=EmulatedDetector)
    assert EmulatedDetector.made[0].streams == streams
    rtf = np.asarray(g["samples"]).mean() * 30.0 if g["dynamic"] else None
    n_det = n_fc = 0
    for q, d in enumerate(seqs):
        want, c = so.sequence(lambda f: d[f], len(d), 1920, 1200, eta=float(eta), runtime=opts.runtime_ms / 1000.0,
                              dynamic_schedule=bool(g["dynamic"]), mean_rtf=rtf)
        got = _load(tmp_path / "out" / f"s{q}.pkl")
        assert_pickle_equal(got, want, f"{name} s{q}")
        n_det, n_fc = n_det + c["t_det"], n_fc + c["t_forecast"]
    ti = _load(tmp_path / "out" / "time_info.pkl")
    assert set(ti) == {"n_total", "t_det", "t_send_frame", "t_recv_res", "t_assoc", "t_forecast"}
    assert ti["n_total"] == sum(len(d) for d in seqs) and len(ti["t_forecast"]) == n_fc
    assert ti["t_det"] == [opts.runtime_ms / 1000.0] * n_det and ti["t_assoc"] == [0.0] * n_det
    assert "Runtime forecasting (ms)" in capsys.readouterr().out
    assert info["n_total"] == ti["n_total"]


def test_arguments(tmp_path):
    base = ["--data-root", "d", "--annot-path", "a.json", "--config", "c.py", "--weights", "w.pth", "--runtime", "r.pkl",
            "--out-dir", "o"]
    o = streamer.parse_args(base)
    assert (o.fps, o.eta, o.in_scale, o.dynamic_schedule, o.perf_factor, o.match_iou_th, o.forecast_rt_ub,
            o.overwrite, o.clock, o.runtime_ms, o.streams, o.max_tracks) == \
        (30, 0, 0.5, False, 1, 0.3, 0.003, False, "wall", None, 1, 1024)
    o = streamer.parse_args(base + ["--fps", "10", "--eta", "-0.5", "--in-scale", "0.25", "--no-mask", "--cpu-pre",
                                    "--dynamic-schedule", "--perf-factor", "2", "--match-iou-th", "0.5",
                                    "--forecast-rt-ub", "0.002", "--overwrite", "--max-tracks", "64"])
    assert (o.fps, o.eta, o.in_scale, o.dynamic_schedule, o.perf_factor, o.match_iou_th, o.forecast_rt_ub,
            o.max_tracks) == (10, -0.5, 0.25, True, 2, 0.5, 0.002, 64)
    o = streamer.parse_args(base + ["--clock", "simulated", "--runtime-ms", "33", "--streams", "8"])
    assert (o.clock, o.runtime_ms, o.streams) == ("simulated", 33.0, 8)
    for bad in (["--runtime-ms", "33"], ["--streams", "2"], ["--clock", "simulated"],
                ["--clock", "simulated", "--runtime-ms", "0"], ["--clock", "simulated", "--runtime-ms", "5", "--streams",
                                                                "0"], ["--max-tracks", "0"], ["--in_scale", "0.5"]):
        with pytest.raises(SystemExit):
            streamer.parse_args(base + bad)
    with pytest.raises(SystemExit):
        streamer.parse_args(base[:-2])                                  # --out-dir is required
    assert streamer.mean_rtf(_runtime_pickle(tmp_path, [0.05, 0.07]), 2, 30.0) == pytest.approx(0.9)


# ================================================================================================ GPU
def _queries(st, dts, wh):
    """sy_forecast_extrap_queries of one stream -> list of (ltwh, scores, labels, tracks)"""
    q = len(dts)
    out = ops.forecast_extrap_queries(st, torch.tensor([dts], dtype=torch.float32, device="cuda"),
                                      torch.tensor([q], dtype=torch.int32, device="cuda"),
                                      torch.tensor([wh], dtype=torch.int32, device="cuda"))
    box, score, label, track, count = (t.cpu().numpy() for t in out)
    return [(box[0, k, :n], score[0, k, :n], label[0, k, :n], track[0, k, :n]) for k, n in enumerate(count[0])]


@pytest.mark.gpu
@pytest.mark.parametrize("clear", [True, False])
def test_update_modes_match_the_oracle(clear):
    """sequence 0 of a fixture (phases: tracks, empty, the same tracks fresh, far away) through sy_forecast_update, one
    detection every other frame, then queried at integer and fractional offsets"""
    from test_forecast import det_rows
    _, seqs, wh, _ = golden("r75_eta0p3")
    d = seqs[0]
    st = ops.ForecastState(1, 64, "cuda")
    ref = so.StreamerTracks() if clear else fo.Tracks()
    last = None
    saw_clear = False
    for f in range(0, len(d), 2):
        b, s, lab = d[f]
        rows = torch.from_numpy(det_rows(b, s, lab, 16)[None]).cuda()
        dt = 0 if last is None else f - last
        had = len(ref.x) > 0
        ops.forecast_update(st, rows, torch.tensor([len(b)], dtype=torch.int32, device="cuda"),
                            torch.tensor([dt], dtype=torch.int32, device="cuda"),
                            torch.tensor([int(last is None)], dtype=torch.int32, device="cuda"), None, 0.3,
                            clear_on_empty=clear)
        ref.update(b, s * np.float32(1.0), lab, dt)
        last = f
        meta = st.meta[0].tolist()
        assert meta[0] == len(ref.x) and meta[1] == ref.n_matched and meta[2] == ref.tkidx, (f, meta)
        saw_clear |= had and len(b) == 0 and meta[0] == 0
        for dq, got in zip((1.0, 2.0, 0.3, 1.7), _queries(st, [1.0, 2.0, 0.3, 1.7], wh)):
            want = ref.query(dq, *wh)
            if want is None:
                assert len(got[0]) == 0
                continue
            assert len(got[0]) == len(want[0]), (f, dq)
            np.testing.assert_allclose(got[0], want[0], rtol=0, atol=BOX_ATOL)
            for a, b_ in zip(got[1:], want[1:]):
                np.testing.assert_array_equal(a, b_)
    assert saw_clear == clear


@pytest.mark.gpu
def test_extrap_queries_equal_single_extrapolations_and_fp32_arithmetic():
    from test_forecast import oracle_tracks, random_tracks, set_state
    rng = np.random.default_rng(3)
    S, T, Q = 4, 300, 5
    st = ops.ForecastState(S, T, "cuda")
    ms = [300, 1, 0, 77]
    refs, whs = [], []
    for s in range(S):
        m = ms[s]
        x, P = random_tracks(rng, m)
        lab, sc, tr = rng.integers(0, 8, m), rng.random(m).astype(np.float32), rng.permutation(1000)[:m]
        nm = int(rng.integers(0, m + 1))
        wh = (640 + s, 480 - s)
        set_state(st, s, x, P, lab, sc, tr, nm, m)
        refs.append(oracle_tracks(x, P, lab, sc, tr, nm, m)), whs.append(wh)
    ints = rng.integers(-2, 7, (S, Q))
    nq = torch.tensor([5, 3, 2, 0], dtype=torch.int32, device="cuda")
    wh_t = torch.tensor(whs, dtype=torch.int32, device="cuda")
    box, score, label, track, count = (t.cpu().numpy() for t in ops.forecast_extrap_queries(
        st, torch.from_numpy(ints.astype(np.float32)).cuda(), nq, wh_t))
    for k in range(Q):                                     # integer offsets: sy_forecast_extrap, bit for bit
        one = [t.cpu().numpy() for t in ops.forecast_extrap(st, torch.from_numpy(ints[:, k].astype(np.int32)).cuda(), wh_t)]
        for s in range(S):
            if k >= nq[s]:
                assert count[s, k] == 0
                continue
            n = one[4][s]
            assert count[s, k] == n
            np.testing.assert_array_equal(box[s, k, :n].view(np.int32), one[0][s, :n].view(np.int32))
            for a, b in ((score, one[1]), (label, one[2]), (track, one[3])):
                np.testing.assert_array_equal(a[s, k, :n], b[s, :n])
    fr = [[0.3, 1.0 / 3.0, 2.5, -0.7, 1e-3], [0.1, 7.25, 0.9], [1.5, 2.2], []]
    dt = np.zeros((S, Q), np.float64)
    for s, f in enumerate(fr):
        dt[s, :len(f)] = f
    box, score, label, track, count = (t.cpu().numpy() for t in ops.forecast_extrap_queries(
        st, torch.from_numpy(dt.astype(np.float32)).cuda(), nq, wh_t))
    for s, f in enumerate(fr):                             # fractional offsets: numpy's fp32 arithmetic, bit for bit
        for k, d in enumerate(f):
            want = refs[s].query(d, *whs[s])
            n = count[s, k]
            if want is None:                               # a stream without tracks
                assert n == 0
                continue
            assert n == len(want[0]) and n > 0
            np.testing.assert_array_equal(box[s, k, :n].view(np.int32), want[0].view(np.int32))
            np.testing.assert_array_equal(score[s, k, :n], want[1])
            np.testing.assert_array_equal(label[s, k, :n], want[2])
            np.testing.assert_array_equal(track[s, k, :n], want[3].astype(np.int32))


def _sequences_of_jpegs(tmp_path, lengths):
    from test_sap_driver import _jpeg_dataset
    return _jpeg_dataset(tmp_path, lengths)


@pytest.mark.gpu
@pytest.mark.parametrize("streams", [1, 3])
def test_simulated_run_on_the_device(tmp_path, streams):
    """StreamYOLO-s on JPEG files: each stream's detections equal a forecast=False detector's fed the same ticks, and each
    sequence's pickle equals the oracle streamer fed that stream's own detections"""
    from streamyolo_b200 import stream
    from test_sap_driver import _model
    m = _model("s")
    lengths = [9, 5, 12, 7]
    root, ann = _sequences_of_jpegs(tmp_path, lengths)
    rt = _runtime_pickle(tmp_path, [0.05])
    made, log = [], []

    class Recorder(stream.StreamDetector):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.plain = stream.StreamDetector(*a, **{key: v for key, v in k.items()
                                                      if key not in ("forecast", "clear_on_empty", "queries",
                                                                     "match_iou_th", "max_tracks")})
            made.append(self)

        def reset(self, stream=None):
            super().reset(stream)
            if hasattr(self, "plain"):                     # the constructor's capture resets before plain exists
                self.plain.reset(stream)

        def step_jpeg(self, files, fidx=None, query_dt=None):
            got = super().step_jpeg(files, fidx, query_dt)
            want = self.plain.step_jpeg(files)
            for a, b in zip(got, want):
                for x, y in zip(a, b):
                    assert x.dtype == y.dtype and np.array_equal(x, y)
            log.append((files, got))
            return got

    out = tmp_path / "out"
    opts = streamer.parse_args(_args(root, ann, out, rt, "--clock", "simulated", "--runtime-ms", "50", "--streams",
                                     str(streams), "--eta", "0.5", "--max-tracks", "11850"))
    streamer.run(opts, m, detector=Recorder)
    assert made[0].streams == streams
    # each detection as the device gave it: the ticks of pack_ticks over the schedules (a file's detection depends on
    # the frame before it on its stream, so the same file in two sequences can differ)
    with open(ann) as fh:
        _, paths = streamer.sap.frame_paths(opts, json.load(fh))
    schedules = [streamer.simulated_schedule(len(p), 30.0, 0.05, 0.003) for p in paths]
    ticks = streamer.sap.pack_ticks([len(sch["det_fidx"]) for sch in schedules], streams)
    assert len(ticks) == len(log)
    got_det = {}
    for row, (files, got) in zip(ticks, log):
        for e, dets in zip(row, got):
            if e is not None:
                got_det[(e[0], schedules[e[0]]["det_fidx"][e[1]])] = dets
    n_rows = 0
    for q, p in enumerate(paths):
        want, _ = so.sequence(lambda f, q=q: got_det[(q, f)], len(p), 1920, 1200, eta=0.5, runtime=0.05)
        got = _load(out / f"s{q}.pkl")
        assert_pickle_equal(got, want, f"s{q}", atol=BOX_ATOL)
        n_rows += sum(len(r[0]) for r in got["results_parsed"])
    assert n_rows > 0


@pytest.mark.gpu
def test_wall_clock_run(tmp_path):
    """one short run on the wall clock (tiny model): timestamps increase, each output's input_fidx is the last received
    detection, and each output is the oracle's extrapolation of that detection's tracks to the query asked"""
    from streamyolo_b200 import stream
    from test_sap_driver import _model
    m = _model("tiny")
    root, ann = _sequences_of_jpegs(tmp_path, [12])
    rt = _runtime_pickle(tmp_path, [0.05])
    made = []

    class Recorder(stream.StreamDetector):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.received, self.queries_asked, self.fidx = [], [], None
            made.append(self)

        def submit(self, frames, fidx=None):
            self.fidx = fidx
            return super().submit(frames, fidx)

        def receive(self):
            got = super().receive()
            self.received.append((self.fidx, got[0]))
            return got

        def query(self, dt):
            got = super().query(dt)
            self.queries_asked.append((len(self.received), dt, got[0]))
            return got

    out = tmp_path / "out"
    streamer.run(streamer.parse_args(_args(root, ann, out, rt, "--eta", "0.5", "--max-tracks", "11850")), m,
                 detector=Recorder)
    det, = made
    got = _load(out / "s0.pkl")
    ts = got["timestamps"]
    assert ts and all(a < b for a, b in zip(ts, ts[1:]))
    ref, states, last = so.StreamerTracks(), [], None
    for fidx, dets in det.received:
        ref.update(dets[0], dets[1], dets[2], 0 if last is None else fidx - last)
        last = fidx
        states.append((fidx, copy.deepcopy(ref)))
    asked = [a for a in det.queries_asked]
    assert len(asked) >= len(got["results_parsed"])
    for (n_recv, dt, q), fi, rows in zip(asked, got["input_fidx"], got["results_parsed"]):
        fidx, st = states[n_recv - 1]
        assert fi == fidx
        want = st.query(dt, 1920, 1200)
        assert_rows_equal([rows], [streamer.output_rows(q)], "wall")
        if want is None:
            assert q is None
        else:
            assert len(q[0]) == len(want[0])
            np.testing.assert_allclose(q[0], want[0], rtol=0, atol=BOX_ATOL)
            np.testing.assert_array_equal(q[3], want[3].astype(np.int32))
    ti = _load(out / "time_info.pkl")
    assert len(ti["t_det"]) == len(det.received) and max(ti["t_forecast"]) < 0.1
