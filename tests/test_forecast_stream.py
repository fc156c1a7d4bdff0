"""The forecast inside the streaming detector (StreamDetector(forecast=True), step(..., fidx=...), forecast(fidx)).

CPU: float64 scores in the offline pass come out rounded to fp32, in the input's dtype.

GPU (H100, StreamYOLO-s with calibrated BatchNorm, fp16 storage, the driver's conf 0.01):
  * step() returns the same detections, bit for bit, with forecast=True as with forecast=False;
  * forecast() equals the oracle (oracle/forecast_oracle.py) fed with step()'s own detections and the frame gaps:
    counts, labels, scores and track ids exactly, boxes within the Kalman filter's fp32 rounding;
  * a stream's forecasts do not depend on the frames the other streams see;
  * reset(i) restarts stream i's tracks (ids from 0) and leaves the others; a JPEG frame that does not decode, or no
    frame, leaves the stream's state bit for bit, and a pending reset starts at the next decoded frame;
  * a detection with more rows than max_tracks raises RuntimeError naming the stream.
"""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import forecast_oracle as fo  # noqa: E402
from streamyolo_b200 import forecast, stream  # noqa: E402

BOX_ATOL = 1e-2          # pixels: the Kalman state is fp32 in both, summed in a different order (see test_forecast.py)


def test_float64_scores_round_to_fp32():
    from test_forecast import emulate
    b = np.array([[10, 10, 60, 50], [100, 100, 150, 160]], np.float32)
    s = np.array([0.1 + 1e-12, 0.7], np.float64)
    seq = {"images": [{"id": 5, "width": 640, "height": 480}], "results_parsed": [(b, s, np.array([1, 2]), None)],
           "timestamps": [0.0], "input_fidx": [0]}
    plan = forecast.Plan([seq], 0.0, 30.0)
    rows = forecast.results_ccf(plan, emulate(plan, 0.3))
    assert [type(r["score"]) for r in rows] == [np.float64, np.float64]
    assert sorted(r["score"] for r in rows) == sorted(float(np.float32(v)) for v in s)
    assert [type(r["category_id"]) for r in rows] == [np.int64, np.int64]


# ================================================================================================ GPU


def _model():
    from test_stream import _model_s
    return _model_s(torch.float16)


FRAME_HW, IN_SCALE, CONF, NMS, T = (1200, 1920), 0.5, 0.01, 0.65, 11850


def _frames(n, seed):
    from test_stream import uint8_frames
    return uint8_frames(n, *FRAME_HW, seed=seed)


class Ref:
    """one stream through the oracle: restarted at a reset, updated with what step() returned"""

    def __init__(self, wh):
        self.wh, self.t, self.last = wh, None, None

    def update(self, got, fidx, start):
        if start or self.t is None:
            self.t, self.last = fo.Tracks(), None
        dt = 0 if self.last is None else fidx - self.last
        self.t.update(got[0], got[1], got[2], dt)
        self.last = fidx

    def query(self, fidx):
        q = None if self.t is None else self.t.query(fidx - self.last, *self.wh)
        return q if q is not None else (np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros(0, np.int32),
                                        np.zeros(0, np.uint32))


def same_forecast(got, want, what):
    b, s, l, t = got
    assert len(b) == len(want[0]), f"{what}: {len(b)} rows, want {len(want[0])}"
    np.testing.assert_array_equal(s, want[1], err_msg=what)
    np.testing.assert_array_equal(l, want[2].astype(np.int64), err_msg=what)
    np.testing.assert_array_equal(t, want[3].astype(np.int64), err_msg=what)
    np.testing.assert_allclose(b, want[0], rtol=0, atol=BOX_ATOL, err_msg=what)


def _same_dets(a, b):
    return all(x.dtype == y.dtype and np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_step_unchanged_and_forecast_follows_oracle():
    """S = 2 over six ticks: stream 0 every frame, stream 1 every other frame (dt = 2); stream 1 restarts at tick 3.  A
    frame index shows image fidx // 4, so consecutive detections repeat and tracks match.  A third detector whose stream
    1 sees other images gives stream 0 the same forecasts bit for bit."""
    m = _model()
    plain = stream.StreamDetector(m, FRAME_HW, IN_SCALE, streams=2, conf_thre=CONF, nms_thre=NMS)
    det = stream.StreamDetector(m, FRAME_HW, IN_SCALE, streams=2, conf_thre=CONF, nms_thre=NMS, forecast=True,
                                max_tracks=T)
    other = stream.StreamDetector(m, FRAME_HW, IN_SCALE, streams=2, conf_thre=CONF, nms_thre=NMS, forecast=True,
                                  max_tracks=T)
    assert all(len(r[0]) == 0 for r in det.forecast([0, 0]))                # no tracks before the first step
    seq = _frames(12, seed=41)
    alt = _frames(12, seed=42)
    refs = [Ref((FRAME_HW[1], FRAME_HW[0])) for _ in range(2)]
    n_rows, n_matched = [], []
    for k in range(6):
        fidx = [k, 2 * k]
        start = [k == 0, k in (0, 3)]
        if k == 3:
            for d in (plain, det, other):
                d.reset(1)
        frames = np.stack([seq[fidx[0] // 4], seq[fidx[1] // 4]])
        a = plain.step(frames)
        b = det.step(frames, fidx=fidx)
        other.step(np.stack([seq[fidx[0] // 4], alt[fidx[1] // 4]]), fidx=fidx)
        for i in range(2):
            assert _same_dets(a[i], b[i]), f"tick {k} stream {i}: step() changed"
            refs[i].update(b[i], fidx[i], start[i])
        q = [fidx[0] + 1, fidx[1] + 3]
        got = det.forecast(q)
        for i in range(2):
            same_forecast(got[i], refs[i].query(q[i]), f"tick {k} stream {i}")
        o = other.forecast(q)[0]
        assert all(np.array_equal(x, y) for x, y in zip(o, got[0])), f"tick {k}: stream 0 depends on stream 1"
        if k == 3:                                                              # ids restart at 0
            assert (got[1][3] < len(b[1][0])).all()
        n_rows.append([len(g[0]) for g in got])
        n_matched.append([r.t.n_matched for r in refs])
    assert all(n > 0 for r in n_rows for n in r), n_rows
    assert any(n > 0 for r in n_matched for n in r), n_matched
    print(f"\nforecast rows per tick {n_rows}, matched tracks {n_matched}")


@pytest.mark.gpu
def test_jpeg_gating_keeps_tracks():
    """the JPEG rig of test_stream_jpeg.py over its ticks (a damaged file, a missing frame, a reset issued while the stream
    has no frame, a reset of a decoded stream): a gated stream's tracks stay bit for bit; a decoded stream with a pending
    reset restarts its ids at 0; a decoded stream without one keeps counting"""
    from test_stream_jpeg import NAMES, TICKS, _files, hw
    m = _model()
    sizes = [hw(n) for n in NAMES]
    det = stream.StreamDetector(m, in_scale=IN_SCALE, frame_sizes=sizes, input_size=(600, 960), jpeg_max_bytes=1 << 19,
                                conf_thre=CONF, nms_thre=NMS, forecast=True, max_tracks=T)
    fc = det._tick.fc
    pending = [True] * 3
    gated = 0
    for k, (feed, resets) in enumerate(TICKS):
        for i in resets:
            det.reset(i)
            pending[i] = True
        before = [t.clone() for t in (fc.x, fc.P, fc.label, fc.score, fc.track, fc.meta)]
        got = det.step_jpeg([_files(feed, i) for i in range(3)], fidx=[3 * k] * 3)
        status = det.last_status().tolist()
        for i in range(3):
            meta = fc.meta[i].tolist()
            if status[i] != 0:
                assert feed.get(i) in (None, "bad")
                for a, b in zip(before, (fc.x, fc.P, fc.label, fc.score, fc.track, fc.meta)):
                    assert torch.equal(a[i], b[i]), f"tick {k} stream {i}: a gated stream's state changed"
                gated += 1
                continue
            n = len(got[i][0])
            if pending[i]:
                assert meta[:3] == [n, 0, n] and fc.track[i, :n].tolist() == list(range(n)), (k, i, meta)
                pending[i] = False
            else:
                assert meta[2] >= before[5][i, 2].item() and meta[0] == (n or before[5][i, 0].item()), (k, i, meta)
        out = det.forecast([3 * k + 2] * 3)
        assert all(len(o[0]) <= fc.meta[i, 0].item() for i, o in enumerate(out))
    assert gated == 2


@pytest.mark.gpu
def test_overflow_names_the_stream():
    m = _model()
    det = stream.StreamDetector(m, FRAME_HW, IN_SCALE, streams=2, conf_thre=CONF, nms_thre=NMS, forecast=True,
                                max_tracks=1)
    with pytest.raises(RuntimeError, match="stream 0"):
        det.step(_frames(2, seed=43), fidx=[0, 0])
    with pytest.raises(ValueError, match="fidx"):
        det.step(_frames(2, seed=43))
    plain = stream.StreamDetector(m, FRAME_HW, IN_SCALE, streams=1, conf_thre=CONF, nms_thre=NMS)
    with pytest.raises(ValueError, match="forecast=True"):
        plain.step(_frames(1, seed=43)[0], fidx=0)
    with pytest.raises(RuntimeError, match="forecast=True"):
        plain.forecast(0)
