"""The streaming detector on raw sensor frames: StreamDetector(frame_format="bayer_rggb" | "bayer_bggr" | "bayer_gbrg" |
"bayer_grbg", demosaic="bilinear" | "ea") and the demosaicing kernel sy_bayer_to_bgr_sized (ops.bayer_to_bgr_sized).

CPU (no GPU needed):
  * the numpy oracle (oracle/bayer_oracle.py) is cv2.cvtColor for the four patterns and both algorithms on every size
    from 2x2 to 16x16 and on widths that are no multiple of 8, 16 or 32, with the frame inside differently filled
    buffers; it equals every fixture (tests/golden/bayer_frames.npz), which the generator still makes;
  * argument checks, all before any launch: an unknown format (the message lists the YUV and Bayer ones), a Bayer format
    with jpeg_max_bytes, an unknown demosaic, demosaic="ea" without a Bayer format, frames below 2x2, frames of the
    wrong shape or dtype; stream.FRAME_FORMATS is unchanged;
  * the host staging on a tick built on the CPU: only each frame's h * w bytes reach the stage and the tick's buffer;
  * bayer.cu compiles without spills.

GPU (H100):
  * the kernel is bit-exact on every fixture, all sizes of a pattern and algorithm in one launch with a no-frame row;
    nothing outside each frame's h x w is written; a graph replay equals the eager launch;
  * canary bytes after each frame are never read, with rows at misaligned pitches as well;
  * StreamYOLO-s (synthetic weights, fp16 storage): step(bayer) gives last_raw() and the detections of step(bgr) on the
    oracle's BGR frames, bit for bit -- one stream, three streams of different (odd) sizes, forecast with queries,
    submit / receive, and record_quality (the same JPEG files); a Bayer tick runs the BGR tick's ops after exactly one
    bayer_to_bgr_sized, and the BGR and YUV ticks run none.
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

from oracle.bayer_oracle import ALGOS, CV2_CODES, PATTERNS, bayer_to_bgr
from oracle.make_bayer_golden import CASES, frames as golden_frames, synth_frame
from streamyolo_b200 import data, feed, ops, stream

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "bayer_frames.npz"))
ALL_CASES = tuple(CASES) + ("edges",)
IN_SCALE, CONF, NMS = 0.5, 0.01, 0.65
COMBOS = [(p, a) for p in PATTERNS for a in ALGOS]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


def fixture(pattern, algo, case):
    """-> (h, w, the mosaic, cv2's BGR digest, cv2's BGR frame or a centre crop of it)"""
    h, w = (int(v) for v in G[f"{case}.hw"])
    k = f"{pattern}.{algo}.{case}"
    if f"{case}.raw" in G:
        return h, w, G[f"{case}.raw"], bytes(G[f"{k}.sha256"]), G[f"{k}.bgr"]
    f = synth_frame(h, w, int(G[f"{case}.seed"]))
    assert sha(f) == bytes(G[f"{case}.raw_sha256"]), case
    return h, w, f, bytes(G[f"{k}.sha256"]), G[f"{k}.crop"]


def _crop(bgr, h, w):
    return bgr[h // 2 - 16:h // 2 + 16, w // 2 - 16:w // 2 + 16]


# ================================================================================================ CPU
def test_oracle_is_cv2():
    """cv2.cvtColor(COLOR_Bayer*2BGR[_EA]) on seeded frames of every size from 2x2 to 16x16, and on wider ones whose widths
    are no multiple of 8, 16 or 32 (cv2's SIMD loops leave a tail there), each frame contiguous inside a buffer filled
    with 0x00 and then 0xFF around it: cv2's result is the oracle's, whatever the buffer holds"""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    sizes = [(h, w) for h in range(2, 17) for w in range(2, 17)] + [(6, 1918), (37, 131), (8, 130), (33, 517)]
    for (p, a), code in CV2_CODES.items():
        for h, w in sizes:
            f = rng.integers(0, 256, (h, w), dtype=np.uint8)
            want = bayer_to_bgr(p, a, f)
            for fill in (0x00, 0xFF):
                buf = np.full(h * w + 48, fill, np.uint8)
                buf[16:16 + h * w] = f.reshape(-1)
                got = cv2.cvtColor(buf[16:16 + h * w].reshape(h, w), getattr(cv2, code))
                assert np.array_equal(got, want), (p, a, h, w, fill)


@pytest.mark.parametrize("pattern", PATTERNS)
def test_oracle_equals_fixtures(pattern):
    """the oracle gives cv2's stored frame (or digest) of every case and algorithm; the fixture generator still makes the
    stored frames; the edges case reaches 0 and 255 in every channel"""
    made = golden_frames()
    for algo in ALGOS:
        for case in ALL_CASES:
            h, w, f, digest, ref = fixture(pattern, algo, case)
            assert np.array_equal(made[case][2], f), case
            got = bayer_to_bgr(pattern, algo, f)
            assert got.shape == (h, w, 3) and sha(got) == digest, (algo, case)
            assert np.array_equal(got if ref.shape == got.shape else _crop(got, h, w), ref), (algo, case)
        edges = bayer_to_bgr(pattern, algo, fixture(pattern, algo, "edges")[2])
        assert all((edges[..., c] == 0).any() and (edges[..., c] == 255).any() for c in range(3)), algo


def test_argument_checks():
    """refused with ValueError when the detector is built, before any launch: an unknown format (the message names the
    YUV and the Bayer formats), a Bayer format with jpeg_max_bytes, an unknown demosaic, a demosaic other than the
    default without a Bayer format, a frame below 2x2; step_frames refuses arrays of the wrong shape or dtype"""
    from test_fp16_storage import _tiny_model
    m = _tiny_model().eval()
    with pytest.raises(ValueError, match="unknown frame_format 'bayer_rgbg'.*nv12.*bayer_rggb, bayer_bggr, bayer_gbrg, "
                                         "bayer_grbg"):
        stream.StreamDetector(m, frame_hw=(120, 160), frame_format="bayer_rgbg")
    with pytest.raises(ValueError, match="jpeg_max_bytes"):
        stream.StreamDetector(m, frame_sizes=[(120, 160)], jpeg_max_bytes=1 << 16, frame_format="bayer_rggb")
    with pytest.raises(ValueError, match="unknown demosaic 'ahd'"):
        stream.StreamDetector(m, frame_hw=(120, 160), frame_format="bayer_rggb", demosaic="ahd")
    for fmt in ("bgr", "nv12", "yuyv"):
        with pytest.raises(ValueError, match="demosaic='ea' takes a Bayer frame_format"):
            stream.StreamDetector(m, frame_hw=(120, 160), frame_format=fmt, demosaic="ea")
    for sizes in ([(120, 160), (1, 160)], [(120, 1)], [(1, 1)]):
        with pytest.raises(ValueError, match="bayer_gbrg frames need at least 2 rows and 2 columns"):
            stream.StreamDetector(m, frame_sizes=sizes, input_size=(64, 96), frame_format="bayer_gbrg")
    assert stream.FRAME_FORMATS == ("bgr",) + tuple(ops.YUV_FORMATS)
    assert stream.BAYER_FORMATS == tuple("bayer_" + p for p in PATTERNS) == ("bayer_rggb", "bayer_bggr", "bayer_gbrg",
                                                                             "bayer_grbg")
    assert list(ops.BAYER_PATTERNS) == list(PATTERNS) and ops.DEMOSAIC == {"bilinear": 0, "ea": 1}
    for fmt in stream.BAYER_FORMATS:
        assert stream.frame_shape(fmt, 13, 17) == (13, 17)
        ok = np.zeros((13, 17), np.uint8)
        assert tuple(stream.step_frames(ok, 1, (13, 17), fmt).shape) == (1, 13, 17)
        assert tuple(stream.step_frames(np.stack([ok] * 3), 3, (13, 17), fmt).shape) == (3, 13, 17)
        for bad, s in ((ok, 2), (ok.astype(np.int16), 1), (np.zeros((13, 17, 3), np.uint8), 1), (ok[:-1], 1)):
            with pytest.raises(RuntimeError, match="frames must be uint8"):
                stream.step_frames(bad, s, (13, 17), fmt)


def _stand_in(monkeypatch, sizes, fmt, demosaic="bilinear"):
    """a detector around a tick built on the CPU (no capture), with plain host memory as its stage"""
    from test_fp16_storage import _tiny_model
    monkeypatch.setattr(feed, "pinned", lambda shape, dtype: torch.zeros(shape, dtype=dtype))
    size = (64, 96)
    table, ratios = data.sized_table(sizes, size, None)
    det = stream.StreamDetector.__new__(stream.StreamDetector)
    det.streams, det.frame_sizes, det.frame_format, det.jpeg_max_bytes = len(sizes), sizes, fmt, None
    det._tick = stream.StreamTick(_tiny_model().eval(), table, ratios, size, len(sizes), CONF, NMS, "cpu",
                                  frame_format=fmt, demosaic=demosaic)
    det.frame_hw = tuple(det._tick.frames.shape[1:3])
    det._inputs()
    return det


@pytest.mark.parametrize("fmt,demosaic", [("bayer_rggb", "bilinear"), ("bayer_grbg", "ea")])
def test_host_staging(monkeypatch, fmt, demosaic):
    """mixed (odd) sizes from a list (numpy and CPU tensors): row i of the tick's ``bayer`` holds frame i's h * w bytes and
    nothing past them is written, nor staged; one size from a list and from one array stage the same bytes; a stream
    without a frame, or with a frame of the wrong shape or dtype, is refused by name"""
    sizes = [(12, 16), (7, 11), (9, 14)]
    det = _stand_in(monkeypatch, sizes, fmt, demosaic)
    t = det._tick
    assert t.yuv is None and det._in is t.bayer and tuple(t.bayer.shape) == (3, 12 * 16)
    assert t.bayer_sizes.tolist() == [list(s) for s in sizes]
    assert t.bayer_pattern == fmt[len("bayer_"):] and t.demosaic == demosaic
    t.bayer.fill_(0xCD)
    rng = np.random.default_rng(1)
    fr = [rng.integers(0, 256, (h, w), dtype=np.uint8) for h, w in sizes]
    det._stage_frames([fr[0], torch.from_numpy(fr[1]), fr[2]], "step")
    for i, (h, w) in enumerate(sizes):
        n = h * w
        row = t.bayer[i]
        assert np.array_equal(row[:n].view(h, w).numpy(), fr[i]), i
        assert bool((row[n:] == 0xCD).all()), f"stream {i}: bytes past the frame were written"
        assert bool((det._stage[i].view(-1)[n:] == 0).all()), f"stream {i}: the stage took more than the frame's bytes"
    for bad, match in ((None, "frame 1 is None"), (fr[2], "frame 1 must be uint8"), (fr[1].astype(np.int32), "frame 1 must"),
                       (np.zeros((7, 11, 3), np.uint8), "frame 1 must be uint8 \\[7, 11\\]")):
        with pytest.raises(RuntimeError, match=match):
            det._stage_frames([fr[0], bad, fr[2]], "step")
    with pytest.raises(RuntimeError, match="give a list of 3 frames"):
        det._stage_frames(np.stack([fr[0]] * 3), "step")
    one = _stand_in(monkeypatch, [(7, 11)] * 3, fmt, demosaic)
    a = np.stack([rng.integers(0, 256, (7, 11), dtype=np.uint8) for _ in range(3)])
    one._stage_frames(a, "step")
    by_array = one._in.clone()
    one._in.zero_()
    one._stage_frames(list(a), "step")
    assert torch.equal(one._in, by_array) and np.array_equal(by_array.view(a.shape).numpy(), a)


def test_bayer_kernel_compiles_without_spills(tmp_path):
    """both algorithms' instances of bayer_to_bgr_sized_kernel: 0 spill bytes and no stack frame"""
    import re
    import shutil
    import subprocess
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc] + build.COMMON + build.SOURCES["bayer.cu"] + ["-c", os.path.join(build.CSRC, "bayer.cu"),
                       "-o", str(tmp_path / "k.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout
    found = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stdout)
    hits = [f for f in found if "bayer_to_bgr_sized_kernel" in f[0]]
    assert len(hits) == len(ALGOS) and all(f[1:] == ("0", "0", "0") for f in hits), hits


# ================================================================================================ GPU
DEV = "cuda"


def _rows(frames, pitch=None, fill=0):
    """frames -> uint8 [n, pitch] rows on the device (frame i at the start of row i; None: an empty row)"""
    nb = [0 if f is None else f.size for f in frames]
    pitch = max(nb) if pitch is None else pitch
    rows = np.full((len(frames), pitch), fill, np.uint8)
    for i, f in enumerate(frames):
        if f is not None:
            rows[i, :f.size] = f.reshape(-1)
    return torch.from_numpy(rows).to(DEV)


def _sizes(hw):
    return torch.tensor(hw, dtype=torch.int32, device=DEV).reshape(-1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern,algo", COMBOS)
def test_kernel_is_cv2_on_every_fixture(pattern, algo):
    """one launch of every case (2x2 .. 1200x1920, the edges) and a no-frame row (h = 0, its bytes a valid frame): each
    frame is cv2's bit for bit, every byte of a slot outside its frame and the no-frame slot keep their value; a graph
    replay of the launch writes the same bytes"""
    fx = [fixture(pattern, algo, c) for c in ALL_CASES]
    frames = [f[2] for f in fx] + [fx[4][2]]
    hw = [(f[0], f[1]) for f in fx] + [(0, fx[4][1])]
    src, sizes = _rows(frames), _sizes(hw)
    out = torch.full((len(frames), 1200, 1920, 3), 0x5A, dtype=torch.uint8, device=DEV)
    ops.bayer_to_bgr_sized(src, sizes, pattern, algo, out)
    got = out.cpu().numpy()
    for i, (case, (h, w, f, digest, ref)) in enumerate(zip(ALL_CASES, fx)):
        img = got[i, :h, :w]
        assert sha(img) == digest, (pattern, algo, case, np.argwhere(img != bayer_to_bgr(pattern, algo, f))[:4])
        assert np.array_equal(img if ref.shape == img.shape else _crop(img, h, w), ref)
        rest = got[i].copy()
        rest[:h, :w] = 0x5A
        assert (rest == 0x5A).all(), (pattern, algo, case, "bytes outside the frame were written")
    assert (got[-1] == 0x5A).all(), "the no-frame slot was written"
    eager = out.clone()
    out.fill_(0x5A)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.bayer_to_bgr_sized(src, sizes, pattern, algo, out)
    out.fill_(0x5A)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern,algo", COMBOS)
def test_kernel_reads_no_byte_past_a_frame(pattern, algo):
    """rows with 1 .. 37 bytes after each frame, at pitches that leave the frames misaligned: with those bytes 0x00 and
    then 0xFF (values that change any pixel they would reach), every frame demosaics to the oracle's BGR"""
    rng = np.random.default_rng(11)
    hw = [(37, 131), (2, 2), (120, 162), (16, 128), (7, 33), (3, 3), (17, 257)]
    frames = [rng.integers(0, 256, s, dtype=np.uint8) for s in hw]
    for pad in (1, 7, 16, 37):
        pitch = max(f.size for f in frames) + pad
        outs = [torch.zeros((len(frames), 120, 257, 3), dtype=torch.uint8, device=DEV) for _ in range(2)]
        for out, fill in zip(outs, (0x00, 0xFF)):
            ops.bayer_to_bgr_sized(_rows(frames, pitch, fill), _sizes(hw), pattern, algo, out)
        outs = [o.cpu().numpy() for o in outs]
        for i, ((h, w), f) in enumerate(zip(hw, frames)):
            want = bayer_to_bgr(pattern, algo, f)
            assert np.array_equal(outs[0][i, :h, :w], want) and np.array_equal(outs[1][i, :h, :w], want), (pad, i)


def _model_s():
    from test_stream import _model_s as model_s
    return model_s(torch.float16)


def _raw_frames(sizes, t):
    return [synth_frame(h, w, 1000 * t + i) for i, (h, w) in enumerate(sizes)]


def _same(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


def _pair(m, fmt, demosaic, sizes, **kw):
    kw = dict(in_scale=IN_SCALE, frame_sizes=sizes, input_size=(600, 960), conf_thre=CONF, nms_thre=NMS, **kw)
    return stream.StreamDetector(m, frame_format=fmt, demosaic=demosaic, **kw), stream.StreamDetector(m, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,demosaic", [("bayer_rggb", "bilinear"), ("bayer_bggr", "ea")])
def test_one_stream_equals_bgr_detector(fmt, demosaic):
    """one 1200x1920 camera over four ticks (a reset before the third): step(bayer) -- numpy, a CPU tensor, a CUDA tensor,
    an [1, h, w] array -- gives the head outputs and detections of step(bgr) on the oracle's frames, bit for bit"""
    m = _model_s()
    p = fmt[len("bayer_"):]
    dr, db = _pair(m, fmt, demosaic, [(1200, 1920)])
    n_dets = []
    for t in range(4):
        if t == 2:
            dr.reset(), db.reset()
        f = _raw_frames([(1200, 1920)], t)[0]
        arg = [f, [torch.from_numpy(f)], [torch.from_numpy(f).to(DEV)], f[None]][t]
        got = dr.step(arg)
        want = db.step([bayer_to_bgr(p, demosaic, f)])
        assert torch.equal(dr.last_raw(), db.last_raw()), f"tick {t}: raw head outputs"
        assert _same(got[0], want[0]), f"tick {t}: detections"
        n_dets.append(len(got[0][2]))
    print(f"\n{fmt} {demosaic}: detections per tick {n_dets}")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,demosaic", [("bayer_gbrg", "bilinear"), ("bayer_grbg", "ea")])
def test_three_streams_of_different_sizes_equal_bgr_detector(fmt, demosaic):
    """a rig of 1200x1920, 1199x1917 and 1551x2047 cameras (odd heights and widths) over three ticks with a reset of
    stream 1: equal to the BGR detector on the oracle's frames, stream by stream"""
    m = _model_s()
    p = fmt[len("bayer_"):]
    sizes = [(1200, 1920), (1199, 1917), (1551, 2047)]
    dr, db = _pair(m, fmt, demosaic, sizes)
    for t in range(3):
        if t == 1:
            dr.reset(1), db.reset(1)
        fr = _raw_frames(sizes, t)
        got = dr.step(fr)
        want = db.step([bayer_to_bgr(p, demosaic, f) for f in fr])
        assert torch.equal(dr.last_raw(), db.last_raw()), f"tick {t}"
        for i in range(3):
            assert _same(got[i], want[i]), (t, i)


@pytest.mark.gpu
def test_forecast_queries_and_submit_equal_bgr_detector():
    """bayer_rggb / ea with forecast=True and queries: detections, per-query extrapolations and forecast(); bayer_gbrg /
    bilinear through submit / poll / receive and publish / query: all as the BGR detector gives them"""
    m = _model_s()
    sizes = [(1200, 1920), (1081, 1919)]
    dr, db = _pair(m, "bayer_rggb", "ea", sizes, forecast=True, queries=2)
    for t in range(3):
        fr = _raw_frames(sizes, t)
        q = [[0.5, 1.0], [2.0]]
        got = dr.step(fr, fidx=[t, t], query_dt=q)
        want = db.step([bayer_to_bgr("rggb", "ea", f) for f in fr], fidx=[t, t], query_dt=q)
        assert all(_same(a, b) for a, b in zip(got, want)), t
        for qa, qb in zip(dr.last_queries(), db.last_queries()):
            assert len(qa) == len(qb) and all((a is None and b is None) or _same(a, b) for a, b in zip(qa, qb)), t
    assert all(_same(a, b) for a, b in zip(dr.forecast([5, 5]), db.forecast([5, 5])))
    dr, db = _pair(m, "bayer_gbrg", "bilinear", [(1200, 1920)], forecast=True, clear_on_empty=True)
    for t in range(3):
        f = _raw_frames([(1200, 1920)], t)[0]
        dr.submit([f], fidx=t)
        db.submit([bayer_to_bgr("gbrg", "bilinear", f)], fidx=t)
        assert dr.poll(60.0) and db.poll(60.0)
        got, want = dr.receive(), db.receive()
        assert _same(got[0], want[0]) and torch.equal(dr.last_raw(), db.last_raw()), t
        dr.publish(), db.publish()
        qa, qb = dr.query(1.5)[0], db.query(1.5)[0]
        assert (qa is None and qb is None) or _same(qa, qb), t


@pytest.mark.gpu
def test_recorded_frames_equal_bgr_detector():
    """record_quality on two cameras of different sizes: the JPEG files of the demosaiced frames are the BGR detector's,
    byte for byte, and so are the detections; with record_boxes too"""
    m = _model_s()
    sizes = [(1200, 1920), (1081, 1919)]
    palette = [(255, 0, 0), (0, 255, 0), (0, 0, 255)] * 3
    for kw in (dict(record_quality=90), dict(record_quality=75, record_boxes=(0.05, palette))):
        dr, db = _pair(m, "bayer_bggr", "ea", sizes, **kw)
        for t in range(2):
            fr = _raw_frames(sizes, t)
            got = dr.step(fr)
            want = db.step([bayer_to_bgr("bggr", "ea", f) for f in fr])
            assert all(_same(a, b) for a, b in zip(got, want)), (kw, t)
            files = dr.last_jpeg()
            assert files == db.last_jpeg() and all(f is not None and len(f) > 0 for f in files), (kw, t)


@pytest.mark.gpu
def test_bayer_tick_runs_one_demosaic(monkeypatch):
    """the ops calls of one tick: a Bayer detector's are bayer_to_bgr_sized followed by exactly the BGR detector's; the
    BGR and YUV ticks call no demosaicing"""
    import inspect
    m = _model_s()
    dr, db = _pair(m, "bayer_rggb", "ea", [(1200, 1920)])
    dy = stream.StreamDetector(m, frame_format="nv12", in_scale=IN_SCALE, frame_sizes=[(1200, 1920)],
                               input_size=(600, 960), conf_thre=CONF, nms_thre=NMS)
    calls = []
    for name, fn in inspect.getmembers(ops, inspect.isfunction):
        if fn.__module__ == ops.__name__ and not name.startswith("_") and name not in ("lib", "load_library"):
            monkeypatch.setattr(ops, name, (lambda n, f: lambda *a, **k: (calls.append(n), f(*a, **k))[1])(name, fn))
    db._tick.run()
    default, calls[:] = list(calls), []
    dy._tick.run()
    yuv, calls[:] = list(calls), []
    dr._tick.run()
    torch.cuda.synchronize()
    assert default and "bayer_to_bgr_sized" not in default and "letterbox_sized" in default
    assert yuv == ["yuv_to_bgr_sized"] + default
    assert calls == ["bayer_to_bgr_sized"] + default
