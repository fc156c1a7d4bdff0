"""Device JPEG encode (sy_jpeg_encode, streamyolo_b200.data.encode_jpeg, StreamDetector(record_quality=...)).

CPU: the numpy oracle (oracle/jpeg_encode_oracle.py) equals every committed cv2.imencode fixture byte for byte, the
     1200 x 1920 and 600 x 960 frames included, and its files decode (oracle/jpeg_oracle.py) to what cv2's do; it stays
     within sy_jpeg_encode_max_bytes on adversarial content; argument refusals; jpeg_encode.cu compiles for sm_90a without
     spills.
GPU: the kernels equal every fixture (one launch per quality holding every size) and the oracle on seeded random sizes
     and qualities; device decode of their files; overflow and size statuses leave other rows and a guard untouched; a
     CUDA-graph replay follows new frames and sizes; a StreamDetector recording its NV12 or JPEG streams detects exactly
     what one without recording does, and its last_jpeg() is encode_jpeg of the tick's frames.
"""
import ctypes as C
import hashlib
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import jpeg_encode_oracle as eo
from oracle import jpeg_oracle as jo
from oracle import make_jpeg_encode_golden as mk
from streamyolo_b200 import data, ops, stream

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_encode_small.npz"))
FULL = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_encode_full.npz"))
SMALL_NAMES = sorted(k[:-4] for k in SMALL if k.endswith(".jpg"))
FULL_NAMES = sorted(k[:-7] for k in FULL if k.endswith(".sha256"))


def _check_full(name, b):
    """file ``b`` against full fixture ``name`` by its SHA-256, naming the first MCU row band that differs otherwise"""
    if hashlib.sha256(b).digest() == FULL[name + ".sha256"].tobytes():
        return
    crcs, bits = mk.band_crcs(b)
    want_c, want_b = FULL[name + ".bands"], FULL[name + ".band_bits"]
    bad = [k for k in range(min(len(crcs), len(want_c))) if crcs[k] != want_c[k] or bits[k] != want_b[k]]
    raise AssertionError(f"{name}: {len(b)} bytes (want {int(FULL[name + '.length'])}), first wrong MCU row band "
                         f"{bad[0] if bad else 'none'} of {len(want_c)}")


def _full_case(name):
    """(input file, (h, w), quality) of full fixture ``name``"""
    base, q = name.rsplit("_q", 1)
    jpg, hw = mk.full_input(base)
    return jpg, hw, int(q)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_fixtures_record_their_encoder():
    assert "libjpeg-turbo" in str(SMALL["libjpeg_turbo"]) and "libjpeg-turbo" in str(FULL["libjpeg_turbo"])
    assert SMALL_NAMES == sorted(mk.small_cases())
    assert len(FULL_NAMES) == len(mk.FULL) * len(mk.FULL_QUALITIES)


def test_oracle_equals_small_fixtures():
    for name in SMALL_NAMES:
        got = eo.encode(SMALL[name + ".bgr"], int(SMALL[name + ".q"]))
        assert got == SMALL[name + ".jpg"].tobytes(), name


@pytest.mark.parametrize("name", FULL_NAMES)
def test_oracle_equals_full_fixture(name):
    jpg, hw, q = _full_case(name)
    img, st = jo.decode(jpg, hw)
    assert st == jo.OK
    _check_full(name, eo.encode(img, q))


def test_oracle_files_decode_as_cv2s():
    for name in SMALL_NAMES:
        img = SMALL[name + ".bgr"]
        mine, _ = jo.decode(eo.encode(img, int(SMALL[name + ".q"])), img.shape[:2])
        theirs, _ = jo.decode(SMALL[name + ".jpg"], img.shape[:2])
        assert mine is not None and np.array_equal(mine, theirs), name


def test_oracle_within_max_bytes_on_adversarial_content():
    ops.load_library()
    rng = np.random.default_rng(5)
    for h, w in mk.SIZES + [(64, 64), (17, 100)]:
        assert ops.jpeg_encode_max_bytes(h, w) == eo.max_bytes(h, w)
        yy, xx = np.mgrid[0:h, 0:w]
        board = np.repeat((((yy + xx) & 1) * 255).astype(np.uint8)[..., None], 3, axis=2)
        stripes = np.repeat(((xx & 1) * 255).astype(np.uint8)[..., None], 3, axis=2)
        for img in (board, stripes, rng.integers(0, 256, (h, w, 3), dtype=np.uint8), 255 - board):
            for q in (90, 100):
                n = len(eo.encode(img, q))
                assert n <= eo.max_bytes(h, w), (h, w, q, n)
    assert ops.jpeg_encode_max_bytes(1200, 1920) == eo.max_bytes(1200, 1920)


def test_argument_refusals_without_a_device():
    lib = ops.load_library()
    with pytest.raises(RuntimeError, match="quality"):
        ops.jpeg_encode(torch.zeros((1, 8, 8, 3), dtype=torch.uint8), None, 0, None, None, None, None)
    with pytest.raises(RuntimeError, match="quality"):
        ops.jpeg_encode(torch.zeros((1, 8, 8, 3), dtype=torch.uint8), None, 101, None, None, None, None)
    for n, mh, mw, mb in ((0, 8, 8, 1000), (1, 0, 8, 1000), (1, 8, 70000, 1000), (1, 8, 8, 0), (1, 8, 8, 1 << 32)):
        assert lib.sy_jpeg_encode_workspace_bytes(n, mh, mw, mb) == 0
        with pytest.raises(RuntimeError, match="bad sizes"):
            ops.jpeg_encode_workspace_bytes(n, mh, mw, mb)
    assert lib.sy_jpeg_encode_max_bytes(0, 5) == 0 and lib.sy_jpeg_encode_max_bytes(5, 65536) == 0
    # the C entry refuses before it launches anything: fake device addresses are never touched
    ws = lib.sy_jpeg_encode_workspace_bytes(2, 16, 24, 5000)
    good = dict(src=0x1000, sizes=0x2000, n=2, max_h=16, max_w=24, quality=90, out=0x3000, max_bytes=5000,
                lengths=0x4000, status=0x5000, workspace=0x10000, workspace_bytes=ws)
    bad = [dict(quality=0), dict(quality=101), dict(n=0), dict(max_h=0), dict(max_w=70000), dict(max_bytes=0),
           dict(lengths=0x4004), dict(status=0x5002), dict(sizes=0x2001), dict(workspace=0x10010),
           dict(workspace_bytes=ws - 1), dict(src=None), dict(out=None)]
    for kw in bad:
        d = ops.SyJpegEncodeDesc(**dict(good, **kw))
        assert lib.sy_jpeg_encode(C.byref(d), None) == 1, kw           # SY_EINVAL


def test_jpeg_encode_cu_compiles_without_spills():
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc not available")
    cmd = [build.NVCC] + build.COMMON + build.SOURCES["jpeg_encode.cu"] + [
        "-c", os.path.join(build.CSRC, "jpeg_encode.cu"), "-o", os.devnull]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == 8, r.stderr
    assert all(p == ("0", "0", "0") for p in props), r.stderr


# ---------------------------------------------------------------------------------------------------------------- GPU
DEV = "cuda"


def _slots(imgs):
    """uint8 CUDA [n, max_h, max_w, 3] slots holding ``imgs`` at their top-left (the rest 0x77) and their sizes"""
    mh, mw = max(i.shape[0] for i in imgs), max(i.shape[1] for i in imgs)
    s = np.full((len(imgs), mh, mw, 3), 0x77, np.uint8)
    for k, i in enumerate(imgs):
        s[k, :i.shape[0], :i.shape[1]] = i
    return torch.from_numpy(s).to(DEV), [i.shape[:2] for i in imgs]


@pytest.mark.gpu
def test_gpu_small_fixtures_one_launch_per_quality():
    by_q = {}
    for name in SMALL_NAMES:
        by_q.setdefault(int(SMALL[name + ".q"]), []).append(name)
    for q, names in by_q.items():
        slots, sizes = _slots([SMALL[n + ".bgr"] for n in names])
        got = data.encode_jpeg(slots, q, sizes)
        for n, b in zip(names, got):
            assert b == SMALL[n + ".jpg"].tobytes(), n


@pytest.mark.gpu
def test_gpu_full_fixtures():
    for name in FULL_NAMES:
        jpg, hw, q = _full_case(name)
        s, l = data.pack_jpeg([jpg], len(jpg) + 64)
        frames, status = data.decode_jpeg(torch.from_numpy(s).to(DEV), torch.from_numpy(l).to(DEV), hw)
        data.check_jpeg_status(status)
        _check_full(name, data.encode_jpeg(frames, q)[0])


@pytest.mark.gpu
def test_gpu_equals_oracle_on_random_sizes_and_qualities():
    rng = np.random.default_rng(2024)
    kinds = ("smooth", "noise", "flat", "checker")
    for case in range(30):
        h, w, q = int(rng.integers(1, 301)), int(rng.integers(1, 501)), int(rng.integers(1, 101))
        img = mk.content(kinds[case % 4], h, w, case)
        slot = (h + int(rng.integers(0, 20)), w + int(rng.integers(0, 20)))
        other = mk.content("noise", *slot, case + 100)
        slots, _ = _slots([img, other])
        got = data.encode_jpeg(slots, q, [(h, w), slot])
        assert got[0] == eo.encode(img, q), (h, w, q)
        assert got[1] == eo.encode(other, q), (slot, q)


@pytest.mark.gpu
def test_gpu_round_trip_through_the_device_decoder():
    """the device decoder reads the device's files back as the oracle decoder reads cv2's"""
    for q in (10, 75, 95, 100):
        names = [n for n in SMALL_NAMES if int(SMALL[n + ".q"]) == q]
        slots, sizes = _slots([SMALL[n + ".bgr"] for n in names])
        files = data.encode_jpeg(slots, q, sizes)
        s, l = data.pack_jpeg(files, max(len(f) for f in files) + 64)
        out, status = data.decode_jpeg_sized(torch.from_numpy(s).to(DEV), torch.from_numpy(l).to(DEV), sizes,
                                             slots.shape[1:3])
        data.check_jpeg_status(status)
        for k, (h, w) in enumerate(sizes):
            want, st = jo.decode(SMALL[names[k] + ".jpg"], (h, w))
            assert st == jo.OK and np.array_equal(out[k, :h, :w].cpu().numpy(), want), names[k]


@pytest.mark.gpu
def test_gpu_overflow_and_bad_sizes_leave_the_rest_untouched():
    rng = np.random.default_rng(7)
    imgs = [mk.content("smooth", 40, 60, 1), rng.integers(0, 256, (48, 64, 3), dtype=np.uint8),
            mk.content("flat", 33, 65, 2), mk.content("smooth", 16, 16, 3)]
    want = [eo.encode(i, 100) for i in imgs]
    slots, sizes = _slots(imgs)
    sizes_t = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    sizes_t[3] = torch.tensor([0, 16])                                  # no image in row 3
    guard = 4096
    for mb in (len(want[1]) - 1, len(want[1])):                         # image 1 one byte too long, then exactly fits
        n = len(imgs)
        flat = torch.full((n * mb + guard,), 0x5A, dtype=torch.uint8, device=DEV)
        buf = flat[:n * mb].view(n, mb)
        lengths = torch.full((n,), -7, dtype=torch.int64, device=DEV)
        status = torch.full((n,), -7, dtype=torch.int32, device=DEV)
        data.encode_jpeg(slots, 100, sizes_t, out=(buf, lengths, status))
        st, ln = status.cpu().tolist(), lengths.cpu().tolist()
        over = mb < len(want[1])
        assert st == [0, 1 if over else 0, 0, 2] and ln[3] == 0 and ln[1] == (0 if over else len(want[1])), (st, ln)
        host = buf.cpu().numpy()
        for k in (0, 2) + (() if over else (1,)):
            assert host[k, :ln[k]].tobytes() == want[k] and ln[k] == len(want[k]), k
            assert (host[k, ln[k]:] == 0x5A).all(), k
        for k in (1, 3) if over else (3,):
            assert (host[k] == 0x5A).all(), k
        assert (flat[n * mb:] == 0x5A).all()
        with pytest.raises(ValueError, match="frame 1" if over else "frame 3"):
            data.jpeg_files(buf, lengths, status)


@pytest.mark.gpu
def test_gpu_argument_refusals():
    f = torch.zeros((2, 16, 16, 3), dtype=torch.uint8, device=DEV)
    for q in (0, 101, 2.5):
        with pytest.raises(RuntimeError, match="quality"):
            data.encode_jpeg(f, q)
    with pytest.raises(RuntimeError, match="larger than"):
        data.encode_jpeg(f, 90, [(16, 16), (17, 16)])
    with pytest.raises(RuntimeError, match="frames must be"):
        data.encode_jpeg(f.float(), 90)
    with pytest.raises(RuntimeError, match="frames must be"):
        data.encode_jpeg(f.permute(0, 2, 1, 3), 90)
    with pytest.raises(RuntimeError, match="frames must be"):
        data.encode_jpeg(torch.zeros((2, 16, 16, 4), dtype=torch.uint8, device=DEV), 90)
    buf = torch.zeros((2, 4096), dtype=torch.uint8, device=DEV)
    ln, st = torch.zeros(2, dtype=torch.int64, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="lengths"):
        data.encode_jpeg(f, 90, out=(buf, ln.int(), st))


@pytest.mark.gpu
def test_gpu_graph_replay_follows_new_frames_and_sizes():
    n, mh, mw, q = 3, 70, 90, 85
    mb = ops.jpeg_encode_max_bytes(mh, mw)
    src = torch.zeros((n, mh, mw, 3), dtype=torch.uint8, device=DEV)
    sizes = torch.tensor([[mh, mw]] * n, dtype=torch.int32, device=DEV)
    out = (torch.zeros((n, mb), dtype=torch.uint8, device=DEV), torch.zeros(n, dtype=torch.int64, device=DEV),
           torch.zeros(n, dtype=torch.int32, device=DEV))
    ws = torch.empty(ops.jpeg_encode_workspace_bytes(n, mh, mw, mb), dtype=torch.uint8, device=DEV)
    data.encode_jpeg(src, q, sizes, out=out, workspace=ws)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        data.encode_jpeg(src, q, sizes, out=out, workspace=ws)
    rng = np.random.default_rng(11)
    for t in range(3):
        hw = [(int(rng.integers(1, mh + 1)), int(rng.integers(1, mw + 1))) for _ in range(n)]
        imgs = [mk.content(("smooth", "noise", "checker")[(t + k) % 3], h, w, 10 * t + k) for k, (h, w) in enumerate(hw)]
        slots, _ = _slots(imgs)
        src.zero_()
        src[:, :slots.shape[1], :slots.shape[2]] = slots
        sizes.copy_(torch.tensor(hw, dtype=torch.int32))
        g.replay()
        got = data.jpeg_files(*out)
        eager = data.encode_jpeg(src, q, hw)
        assert got == eager, t
        assert got == [eo.encode(i, q) for i in imgs], t


IN_SCALE, CONF, NMS = 0.5, 0.01, 0.65


def _model_s():
    from test_stream import _model_s as model_s
    return model_s(torch.float16)


def _same(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


def _slot_files(det, sizes):
    """encode_jpeg of the BGR frames the detector's last tick detected on"""
    return data.encode_jpeg(det._tick.frames, det.record_quality, sizes)


@pytest.mark.gpu
def test_gpu_stream_detector_records_nv12_streams():
    """three NV12 cameras of mixed sizes with forecast: detections, queries and forecasts equal a detector that does not
    record, and last_jpeg() is encode_jpeg of the frames the tick converted"""
    from oracle.make_yuv_golden import synth_frame
    from oracle.yuv_oracle import yuv_to_bgr
    m = _model_s()
    sizes = [(1200, 1920), (1080, 1920), (720, 1280)]
    kw = dict(in_scale=IN_SCALE, frame_sizes=sizes, input_size=(600, 960), conf_thre=CONF, nms_thre=NMS,
              frame_format="nv12", forecast=True)
    rec = stream.StreamDetector(m, record_quality=95, **kw)
    plain = stream.StreamDetector(m, **kw)
    assert rec.last_jpeg() is None
    for t in range(3):
        fr = [synth_frame("nv12", h, w, 50 * t + i) for i, (h, w) in enumerate(sizes)]
        got, want = rec.step(fr, fidx=[t] * 3), plain.step(fr, fidx=[t] * 3)
        assert torch.equal(rec.last_raw(), plain.last_raw()), t
        assert all(_same(a, b) for a, b in zip(got, want)), t
        files = rec.last_jpeg()
        assert files == _slot_files(rec, sizes), t
        if t == 0:                                                      # the file of cv2.cvtColor's frame
            assert files == [eo.encode(yuv_to_bgr("nv12", x), 95) for x in fr]
    assert all(_same(a, b) for a, b in zip(rec.forecast([4] * 3), plain.forecast([4] * 3)))


@pytest.mark.gpu
def test_gpu_stream_detector_records_jpeg_streams_with_absent_ones():
    """step_jpeg with a stream absent on some ticks and one file that does not decode: detections equal the plain
    detector's, last_jpeg() is None exactly where the tick had no frame and encode_jpeg of the decoded frame elsewhere"""
    m = _model_s()
    sizes = [(600, 960), (480, 640)]
    imgs = [[mk.content("smooth", h, w, 10 * t + i) for i, (h, w) in enumerate(sizes)] for t in range(4)]
    files = [[eo.encode(i, 90) for i in row] for row in imgs]
    files[1][1] = None
    files[2][0] = None
    files[3][1] = files[3][1][:200]                                   # truncated: does not decode
    mb = max(len(f) for row in files for f in row if f is not None) + 64
    kw = dict(in_scale=IN_SCALE, frame_sizes=sizes, input_size=(480, 768), conf_thre=CONF, nms_thre=NMS,
              jpeg_max_bytes=mb, forecast=True)
    rec = stream.StreamDetector(m, record_quality=75, **kw)
    plain = stream.StreamDetector(m, **kw)
    for t, row in enumerate(files):
        got, want = rec.step_jpeg(row, fidx=[t, t]), plain.step_jpeg(row, fidx=[t, t])
        assert all(_same(a, b) for a, b in zip(got, want)), t
        assert np.array_equal(rec.last_status(), plain.last_status()), t
        out = rec.last_jpeg()
        ok = (rec.last_status() == 0).tolist()
        assert [f is None for f in out] == [not o for o in ok], (t, rec.last_status())
        enc = _slot_files(rec, sizes)
        for i, f in enumerate(out):
            if f is not None:
                assert f == enc[i] == eo.encode(jo.decode(files[t][i], sizes[i])[0], 75), (t, i)


@pytest.mark.gpu
def test_gpu_default_tick_is_unchanged_and_recording_adds_one_encode(monkeypatch):
    import inspect
    m = _model_s()
    kw = dict(in_scale=IN_SCALE, frame_sizes=[(1200, 1920)], input_size=(600, 960), frame_format="nv12")
    rec, plain = stream.StreamDetector(m, record_quality=90, **kw), stream.StreamDetector(m, **kw)
    calls = []
    for name, fn in inspect.getmembers(ops, inspect.isfunction):
        if fn.__module__ == ops.__name__ and not name.startswith("_") and name not in ("lib", "load_library"):
            monkeypatch.setattr(ops, name, (lambda n, f: lambda *a, **k: (calls.append(n), f(*a, **k))[1])(name, fn))
    plain._tick.run()
    default, calls[:] = list(calls), []
    rec._tick.run()
    torch.cuda.synchronize()
    assert default and "jpeg_encode" not in default and default[0] == "yuv_to_bgr_sized"
    assert [c for c in calls if c != "jpeg_encode_workspace_bytes"] == default + ["jpeg_encode"]
    with pytest.raises(ValueError, match="record_quality"):
        stream.StreamDetector(m, record_quality=0, **kw)
    with pytest.raises(RuntimeError, match="record_quality"):
        plain.last_jpeg()
