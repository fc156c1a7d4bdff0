"""The streaming detector on raw camera frames: StreamDetector(frame_format="nv12" | "nv21" | "i420" | "yv12" | "yuyv" |
"uyvy") and the conversion kernel sy_yuv_to_bgr_sized (ops.yuv_to_bgr_sized).

CPU (no GPU needed):
  * the numpy oracle (oracle/yuv_oracle.py) is cv2.cvtColor for all six formats over a sweep of even sizes, widths that
    are no multiple of 8, 16 or 32 included, and equals every fixture (tests/golden/yuv_frames.npz);
  * argument checks: an unknown format, frame_format with jpeg_max_bytes, odd sizes, frames of the wrong shape or dtype;
  * the host staging on a tick built on the CPU: only each frame's bytes reach the stage and the tick's buffer, from a
    list of mixed sizes or one array, and a stream given no frame is refused by name;
  * yuv.cu compiles without spills.

GPU (H100):
  * the kernel is bit-exact on every fixture, all sizes of a format in one launch with a no-frame row, which is left
    untouched as is the rest of every slot; a graph replay equals the eager launch;
  * canary bytes after each frame are never read: filling them differently changes nothing, with rows at misaligned
    pitches as well;
  * StreamYOLO-s (synthetic weights, fp16 storage): step(yuv) gives last_raw() and the detections of step(bgr) on the
    oracle's BGR frames, bit for bit -- one stream, three streams of different sizes, forecast with queries, and
    submit / receive; the default "bgr" tick runs the same ops as before, with no conversion.
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

from oracle.make_yuv_golden import CASES, frames as golden_frames, synth_frame
from oracle.yuv_oracle import CV2_CODES, FORMATS, frame_shape, yuv_to_bgr
from streamyolo_b200 import data, feed, ops, stream

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "yuv_frames.npz"))
ALL_CASES = tuple(CASES) + ("edges",)
IN_SCALE, CONF, NMS = 0.5, 0.01, 0.65


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


def fixture(fmt, case):
    """-> (h, w, the frame, cv2's BGR digest, cv2's BGR frame or a centre crop of it)"""
    k = f"{fmt}.{case}"
    h, w = (int(v) for v in G[f"{k}.hw"])
    if f"{k}.yuv" in G:
        return h, w, G[f"{k}.yuv"], bytes(G[f"{k}.sha256"]), G[f"{k}.bgr"]
    f = synth_frame(fmt, h, w, int(G[f"{k}.seed"]))
    assert sha(f) == bytes(G[f"{k}.yuv_sha256"]), k
    return h, w, f, bytes(G[f"{k}.sha256"]), G[f"{k}.crop"]


def _crop(bgr, h, w):
    return bgr[h // 2 - 16:h // 2 + 16, w // 2 - 16:w // 2 + 16]


# ================================================================================================ CPU
def test_oracle_is_cv2():
    """cv2.cvtColor(COLOR_YUV2BGR_*) on seeded frames of every even size up to 10 x 70, and wider ones whose widths are no
    multiple of 8, 16 or 32 (cv2's SIMD loops leave a tail there)"""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    sizes = [(h, w) for h in (2, 4, 6, 10) for w in range(2, 72, 2)] + [(38, 62), (24, 98), (8, 130), (6, 1918), (36, 66)]
    for fmt in FORMATS:
        for h, w in sizes:
            f = rng.integers(0, 256, frame_shape(fmt, h, w), dtype=np.uint8)
            want = cv2.cvtColor(f, getattr(cv2, CV2_CODES[fmt]))
            assert np.array_equal(yuv_to_bgr(fmt, f), want), (fmt, h, w)


@pytest.mark.parametrize("fmt", FORMATS)
def test_oracle_equals_fixtures(fmt):
    """the oracle gives cv2's stored frame (or digest) of every case; the fixture generator still makes the stored frames"""
    made = golden_frames(fmt)
    for case in ALL_CASES:
        h, w, f, digest, ref = fixture(fmt, case)
        assert np.array_equal(made[case][2], f), case
        got = yuv_to_bgr(fmt, f)
        assert got.shape == (h, w, 3) and sha(got) == digest, case
        assert np.array_equal(got if ref.shape == got.shape else _crop(got, h, w), ref), case
    edges = yuv_to_bgr(fmt, fixture(fmt, "edges")[2])
    assert all((edges[..., c] == 0).any() and (edges[..., c] == 255).any() for c in range(3))


def test_argument_checks():
    """refused before any launch: an unknown format, a YUV format with jpeg_max_bytes, odd sizes (4:2:0: h or w; 4:2:2:
    w); step_frames refuses arrays of the wrong shape or dtype for the format"""
    from test_fp16_storage import _tiny_model
    m = _tiny_model().eval()
    with pytest.raises(ValueError, match="unknown frame_format 'rgb'"):
        stream.StreamDetector(m, frame_hw=(120, 160), frame_format="rgb")
    with pytest.raises(ValueError, match="jpeg_max_bytes"):
        stream.StreamDetector(m, frame_sizes=[(120, 160)], jpeg_max_bytes=1 << 16, frame_format="nv12")
    for fmt, sizes in (("nv12", [(120, 160), (121, 160)]), ("i420", [(120, 161)]), ("yv12", [(119, 160)]),
                       ("yuyv", [(120, 161)]), ("uyvy", [(120, 160), (60, 81)])):
        with pytest.raises(ValueError, match=f"{fmt} frames need an even width"):
            stream.StreamDetector(m, frame_sizes=sizes, input_size=(64, 96), frame_format=fmt)
    assert stream.FRAME_FORMATS == ("bgr",) + FORMATS
    for fmt in FORMATS:
        assert stream.frame_shape(fmt, 12, 16) == frame_shape(fmt, 12, 16)
        ok = np.zeros(frame_shape(fmt, 12, 16), np.uint8)
        assert tuple(stream.step_frames(ok, 1, (12, 16), fmt).shape) == (1,) + ok.shape
        assert tuple(stream.step_frames(np.stack([ok] * 3), 3, (12, 16), fmt).shape) == (3,) + ok.shape
        for bad, s in ((ok, 2), (ok.astype(np.int16), 1), (np.zeros((12, 16, 3), np.uint8), 1), (ok[:-2], 1)):
            with pytest.raises(RuntimeError, match="frames must be uint8"):
                stream.step_frames(bad, s, (12, 16), fmt)


def _stand_in(monkeypatch, sizes, fmt):
    """a detector around a tick built on the CPU (no capture), with plain host memory as its stage"""
    from test_fp16_storage import _tiny_model
    monkeypatch.setattr(feed, "pinned", lambda shape, dtype: torch.zeros(shape, dtype=dtype))
    size = (64, 96)
    table, ratios = data.sized_table(sizes, size, None)
    det = stream.StreamDetector.__new__(stream.StreamDetector)
    det.streams, det.frame_sizes, det.frame_format, det.jpeg_max_bytes = len(sizes), sizes, fmt, None
    det._tick = stream.StreamTick(_tiny_model().eval(), table, ratios, size, len(sizes), CONF, NMS, "cpu",
                                  frame_format=fmt)
    det.frame_hw = tuple(det._tick.frames.shape[1:3])
    det._inputs()
    return det


@pytest.mark.parametrize("fmt", ["nv12", "yuyv", "bgr"])
def test_host_staging(monkeypatch, fmt):
    """mixed sizes from a list (numpy and CPU tensors): row i of the tick's input holds frame i's bytes and nothing past
    them is written; one size from a list and from one array stage the same bytes; a stream without a frame, or with a
    frame of the wrong shape or dtype, is refused by name"""
    sizes = [(12, 16), (6, 10), (8, 14)]
    det = _stand_in(monkeypatch, sizes, fmt)
    t = det._tick
    n_in = [int(np.prod(stream.frame_shape(fmt, h, w))) for h, w in sizes]
    if fmt == "bgr":
        assert t.yuv is None and det._in is t.frames
    else:
        assert det._in is t.yuv and tuple(t.yuv.shape) == (3, max(n_in)) and t.yuv_sizes.tolist() == [list(s) for s in sizes]
    det._in.fill_(0xCD)
    rng = np.random.default_rng(1)
    fr = [rng.integers(0, 256, stream.frame_shape(fmt, h, w), dtype=np.uint8) for h, w in sizes]
    det._stage_frames([fr[0], torch.from_numpy(fr[1]), fr[2]], "step")
    for i, ((h, w), n) in enumerate(zip(sizes, n_in)):
        row = det._in[i]
        got = row[:h, :w] if fmt == "bgr" else row[:n].view(fr[i].shape)
        assert np.array_equal(got.numpy(), fr[i]), i
        rest = row.clone()
        if fmt == "bgr":
            rest[:h, :w] = 0xCD
        else:
            rest[:n] = 0xCD
        assert bool((rest == 0xCD).all()), f"stream {i}: bytes past the frame were written"
        assert bool((det._stage[i].view(-1)[n:] == 0).all()), f"stream {i}: the stage took more than the frame's bytes"
    for bad, match in ((None, "frame 1 is None"), (fr[2], "frame 1 must be uint8"), (fr[1].astype(np.int32), "frame 1 must")):
        with pytest.raises(RuntimeError, match=match):
            det._stage_frames([fr[0], bad, fr[2]], "step")
    with pytest.raises(RuntimeError, match="give a list of 3 frames"):
        det._stage_frames(np.stack([fr[0]] * 3), "step")
    one = _stand_in(monkeypatch, [(6, 10)] * 3, fmt)
    a = np.stack([rng.integers(0, 256, stream.frame_shape(fmt, 6, 10), dtype=np.uint8) for _ in range(3)])
    one._stage_frames(a, "step")
    by_array = one._in.clone()
    one._in.zero_()
    one._stage_frames(list(a), "step")
    assert torch.equal(one._in, by_array) and np.array_equal(by_array.view(a.shape).numpy(), a)


def test_yuv_kernel_compiles_without_spills(tmp_path):
    """every format's instance of yuv_to_bgr_sized_kernel: 0 spill bytes and no stack frame"""
    import re
    import shutil
    import subprocess
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc] + build.COMMON + build.SOURCES["yuv.cu"] + ["-c", os.path.join(build.CSRC, "yuv.cu"), "-o",
                       str(tmp_path / "k.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout
    found = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stdout)
    hits = [f for f in found if "yuv_to_bgr_sized_kernel" in f[0]]
    assert len(hits) == len(FORMATS) and all(f[1:] == ("0", "0", "0") for f in hits), hits


# ================================================================================================ GPU
DEV = "cuda"


def _rows(frames, pitch=None):
    """frames -> uint8 [n, pitch] rows on the device (frame i at the start of row i; None: an empty row), sizes int32 [n, 2]"""
    nb = [0 if f is None else f.size for f in frames]
    pitch = max(nb) if pitch is None else pitch
    rows = np.zeros((len(frames), pitch), np.uint8)
    for i, f in enumerate(frames):
        if f is not None:
            rows[i, :f.size] = f.reshape(-1)
    return torch.from_numpy(rows).to(DEV)


def _sizes(hw):
    return torch.tensor(hw, dtype=torch.int32, device=DEV).reshape(-1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_kernel_is_cv2_on_every_fixture(fmt):
    """one launch of every case of the format (2x2 .. 1200x1920, the edges) and a no-frame row (h = 0, its bytes a valid
    frame): each frame is cv2's bit for bit, and every byte of a slot outside its frame, and the no-frame slot, keep
    their value; a graph replay of the launch writes the same bytes"""
    fx = [fixture(fmt, c) for c in ALL_CASES]
    frames = [f[2] for f in fx] + [fx[1][2]]
    hw = [(f[0], f[1]) for f in fx] + [(0, fx[1][1])]
    src, sizes = _rows(frames), _sizes(hw)
    out = torch.full((len(frames), 1200, 1920, 3), 0x5A, dtype=torch.uint8, device=DEV)
    ops.yuv_to_bgr_sized(src, sizes, fmt, out)
    got = out.cpu().numpy()
    for i, (case, (h, w, f, digest, ref)) in enumerate(zip(ALL_CASES, fx)):
        img = got[i, :h, :w]
        assert sha(img) == digest, (fmt, case, np.argwhere(img != yuv_to_bgr(fmt, f))[:4])
        assert np.array_equal(img if ref.shape == img.shape else _crop(img, h, w), ref)
        rest = got[i].copy()
        rest[:h, :w] = 0x5A
        assert (rest == 0x5A).all(), (fmt, case, "bytes outside the frame were written")
    assert (got[-1] == 0x5A).all(), "the no-frame slot was written"
    eager = out.clone()
    out.fill_(0x5A)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.yuv_to_bgr_sized(src, sizes, fmt, out)
    out.fill_(0x5A)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_kernel_reads_no_byte_past_a_frame(fmt):
    """rows with 1 .. 37 bytes after each frame, at pitches that leave the frames misaligned: with those bytes 0x00 and
    then 0xFF (values that change any pixel they would reach), every frame converts to the oracle's BGR"""
    rng = np.random.default_rng(11)
    hw = [(38, 62), (2, 2), (120, 162), (16, 48), (6, 34), (4, 16)]
    frames = [rng.integers(0, 256, frame_shape(fmt, h, w), dtype=np.uint8) for h, w in hw]
    for pad in (1, 7, 16, 37):
        pitch = max(f.size for f in frames) + pad
        outs = []
        for fill in (0x00, 0xFF):
            rows = np.full((len(frames), pitch), fill, np.uint8)
            for i, f in enumerate(frames):
                rows[i, :f.size] = f.reshape(-1)
            out = torch.zeros((len(frames), 120, 162, 3), dtype=torch.uint8, device=DEV)
            ops.yuv_to_bgr_sized(torch.from_numpy(rows).to(DEV), _sizes(hw), fmt, out)
            outs.append(out.cpu().numpy())
        for i, ((h, w), f) in enumerate(zip(hw, frames)):
            want = yuv_to_bgr(fmt, f)
            assert np.array_equal(outs[0][i, :h, :w], want) and np.array_equal(outs[1][i, :h, :w], want), (fmt, pad, i)


def _model_s():
    from test_stream import _model_s as model_s
    return model_s(torch.float16)


def _yuv_frames(fmt, sizes, t):
    return [synth_frame(fmt, h, w, 1000 * t + i) for i, (h, w) in enumerate(sizes)]


def _same(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


def _pair(m, fmt, sizes, **kw):
    kw = dict(in_scale=IN_SCALE, frame_sizes=sizes, input_size=(600, 960), conf_thre=CONF, nms_thre=NMS, **kw)
    return stream.StreamDetector(m, frame_format=fmt, **kw), stream.StreamDetector(m, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["nv12", "yuyv"])
def test_one_stream_equals_bgr_detector(fmt):
    """one 1200x1920 camera over four ticks (a reset before the third): step(yuv) -- numpy, a CPU tensor, a CUDA tensor,
    an [1, ...] array -- gives the head outputs and detections of step(bgr) on the oracle's frames, bit for bit"""
    m = _model_s()
    dy, db = _pair(m, fmt, [(1200, 1920)])
    n_dets = []
    for t in range(4):
        if t == 2:
            dy.reset(), db.reset()
        f = _yuv_frames(fmt, [(1200, 1920)], t)[0]
        arg = [f, [torch.from_numpy(f)], [torch.from_numpy(f).to(DEV)], f[None]][t]
        got = dy.step(arg)
        want = db.step([yuv_to_bgr(fmt, f)])
        assert torch.equal(dy.last_raw(), db.last_raw()), f"tick {t}: raw head outputs"
        assert _same(got[0], want[0]), f"tick {t}: detections"
        n_dets.append(len(got[0][2]))
    print(f"\n{fmt}: detections per tick {n_dets}")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["i420", "uyvy"])
def test_three_streams_of_different_sizes_equal_bgr_detector(fmt):
    """a rig of 1200x1920, 2048x1550 and 1550x2048 cameras over three ticks with a reset of stream 1: equal to the BGR
    detector on the oracle's frames, stream by stream"""
    m = _model_s()
    sizes = [(1200, 1920), (2048, 1550), (1550, 2048)]
    dy, db = _pair(m, fmt, sizes)
    for t in range(3):
        if t == 1:
            dy.reset(1), db.reset(1)
        fr = _yuv_frames(fmt, sizes, t)
        got = dy.step(fr)
        want = db.step([yuv_to_bgr(fmt, f) for f in fr])
        assert torch.equal(dy.last_raw(), db.last_raw()), f"tick {t}"
        for i in range(3):
            assert _same(got[i], want[i]), (t, i)


@pytest.mark.gpu
def test_forecast_queries_and_submit_equal_bgr_detector():
    """nv21 with forecast=True and queries: detections, per-query extrapolations and forecast(); yv12 through submit /
    poll / receive and publish / query: all as the BGR detector gives them"""
    m = _model_s()
    sizes = [(1200, 1920), (1080, 1920)]
    dy, db = _pair(m, "nv21", sizes, forecast=True, queries=2)
    for t in range(3):
        fr = _yuv_frames("nv21", sizes, t)
        q = [[0.5, 1.0], [2.0]]
        got = dy.step(fr, fidx=[t, t], query_dt=q)
        want = db.step([yuv_to_bgr("nv21", f) for f in fr], fidx=[t, t], query_dt=q)
        assert all(_same(a, b) for a, b in zip(got, want)), t
        for qa, qb in zip(dy.last_queries(), db.last_queries()):
            assert len(qa) == len(qb) and all((a is None and b is None) or _same(a, b) for a, b in zip(qa, qb)), t
    assert all(_same(a, b) for a, b in zip(dy.forecast([5, 5]), db.forecast([5, 5])))
    dy, db = _pair(m, "yv12", [(1200, 1920)], forecast=True, clear_on_empty=True)
    for t in range(3):
        f = _yuv_frames("yv12", [(1200, 1920)], t)[0]
        dy.submit([f], fidx=t)
        db.submit([yuv_to_bgr("yv12", f)], fidx=t)
        assert dy.poll(60.0) and db.poll(60.0)
        got, want = dy.receive(), db.receive()
        assert _same(got[0], want[0]) and torch.equal(dy.last_raw(), db.last_raw()), t
        dy.publish(), db.publish()
        qa, qb = dy.query(1.5)[0], db.query(1.5)[0]
        assert (qa is None and qb is None) or _same(qa, qb), t


@pytest.mark.gpu
def test_default_tick_runs_no_conversion(monkeypatch):
    """the ops calls of one tick: the default detector's have no conversion, and an nv12 detector's are the conversion
    followed by exactly the default's"""
    import inspect
    m = _model_s()
    dy, db = _pair(m, "nv12", [(1200, 1920)])
    calls = []
    for name, fn in inspect.getmembers(ops, inspect.isfunction):
        if fn.__module__ == ops.__name__ and not name.startswith("_") and name not in ("lib", "load_library"):
            monkeypatch.setattr(ops, name, (lambda n, f: lambda *a, **k: (calls.append(n), f(*a, **k))[1])(name, fn))
    db._tick.run()
    default, calls[:] = list(calls), []
    dy._tick.run()
    torch.cuda.synchronize()
    assert default and "yuv_to_bgr_sized" not in default and "letterbox_sized" in default
    assert calls == ["yuv_to_bgr_sized"] + default
