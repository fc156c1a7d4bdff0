"""The streaming detector on JPEG bytes from cameras of different sizes (StreamDetector(frame_sizes=..., jpeg_max_bytes=...),
data.decode_jpeg_sized, data.stream_frames_sized).

CPU (no GPU needed):
  * the host logic: the input size from the frame sizes and in_scale, each stream's transform and ratio (the fixtures' r),
    the routing of the per-stream status to last_status() and the next tick's start flags;
  * argument checks: a file longer than jpeg_max_bytes, a frame larger than its slot, wrong dtypes, wrong counts;
  * the new kernels compile without spills.

GPU (H100):
  * decode_jpeg_sized: 1200x1920 4:2:0, 2048x1550 4:4:4 and 1550x2048 4:2:0 with restart markers in one batch are cv2.imread's
    frames bit for bit; a damaged file and a file of the wrong size get their status and leave their slot untouched;
  * stream_frames_sized: the driver's preproc and the evaluation preproc of every fixture, bit for bit, with r;
  * with every size equal, both equal decode_jpeg / stream_frame;
  * stream_rescale divides the boxes as numpy divides the driver's float32 rows by a Python float, bit for bit;
  * StreamYOLO-s (synthetic weights, fp16 storage) over a sequence with a damaged file, a stream without a frame and resets:
    one stream of each size is bit-identical to its own eager driver loop (transform, model(x, buffer, mode='on_pipe'), the
    driver's inference() with that stream's ratio); the three sizes in one detector are bit-identical, stream by stream,
    to eager calls at batch 3; a gated stream returns nothing and keeps its buffer; step() on the decoded frames gives the
    same detections as step_jpeg on their files.
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

from oracle.make_stream_jpeg_golden import SEQ, requant
from streamyolo_b200 import data, ops, stream

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "stream_jpeg_files.npz"))
NAMES = ("a420", "b444", "c420_r16")
SIZE, IN_SCALE = (600, 960), 0.5
CONF, NMS = 0.01, 0.65


def jpg(name):
    return bytes(G[f"{name}.jpg"])


def hw(name):
    return tuple(int(v) for v in G[f"{name}.hw"])


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


# ================================================================================================ CPU
def test_input_size_and_ratios():
    """the input size is the driver's size of the largest frame unless given; a frame of driver size = the input size
    takes the plain resize and in_scale, every other frame the evaluation letterbox and its r (the fixtures' r)"""
    sizes = [hw(n) for n in NAMES]
    assert stream.input_size_for(sizes, 0.5) == (1024, 775)             # 2048 x 1550: the largest area, listed first
    assert stream.input_size_for([(1200, 1920)], 0.5) == SIZE
    assert stream.input_size_for(sizes, 0.5, (608, 960)) == (608, 960)
    table, ratios = data.sized_table(sizes, SIZE, IN_SCALE)
    assert table.dtype == np.int32 and table.tolist() == [[1200, 1920, 600, 960], [2048, 1550, 600, 454],
                                                          [1550, 2048, 600, 792]]
    assert ratios[0] == IN_SCALE and ratios[1:] == [float(G[f"{n}.r"]) for n in NAMES[1:]]
    table, ratios = data.sized_table(sizes, SIZE)                      # no in_scale: the letterbox everywhere
    assert table[0].tolist() == [1200, 1920, 600, 960] and ratios == [float(G[f"{n}.r"]) for n in NAMES]
    table, ratios = data.sized_table([(1000, 1920)], SIZE, IN_SCALE)   # driver size 500 x 960: letterboxed
    assert table.tolist() == [[1000, 1920, 500, 960]] and ratios == [0.5]
    table, _ = data.sized_table([(1199, 1920)], SIZE, IN_SCALE)
    assert table.tolist() == [[1199, 1920, 599, 960]]                  # r = 0.5: int(599.5) rows
    with pytest.raises(RuntimeError, match="empty"):
        data.sized_table([(5000, 2)], SIZE)


def test_status_routing():
    """decoded: the flag clears; damaged or absent: no detections (on the device) and the flag stays for the next tick"""
    st, nxt = stream.route_status([0, 5, 1, 0], [True, True, False, True], [1, 1, 1, 0])
    assert st.dtype == np.int32 and st.tolist() == [0, 5, stream.NO_FRAME, 0]
    assert nxt.dtype == np.int32 and nxt.tolist() == [0, 1, 1, 0]
    st, nxt = stream.route_status([0, 0], [True, True], [0, 0])
    assert st.tolist() == [0, 0] and nxt.tolist() == [0, 0]


def test_argument_checks():
    files = stream.jpeg_files([b"\xff\xd8abc", np.zeros(5, np.uint8), None, torch.zeros(3, dtype=torch.uint8)], 4, 8)
    assert [a.size for a in files] == [5, 5, 0, 3] and all(a.dtype == np.uint8 for a in files)
    with pytest.raises(ValueError, match="more than jpeg_max_bytes"):
        stream.jpeg_files([b"x" * 9], 1, 8)
    with pytest.raises(TypeError, match="uint8"):
        stream.jpeg_files([np.zeros(4, np.float32)], 1, 8)
    with pytest.raises(ValueError, match="list of 2"):
        stream.jpeg_files([b"x"], 2, 8)
    with pytest.raises(RuntimeError, match="larger than the 1200x1920 slot"):
        data.decode_jpeg_sized(torch.zeros((2, 16), dtype=torch.uint8), torch.zeros(2, dtype=torch.int32),
                               [(1200, 1920), (1550, 2048)], (1200, 1920))
    with pytest.raises(RuntimeError, match="sizes must be int32"):
        data.decode_jpeg_sized(torch.zeros((1, 16), dtype=torch.uint8), torch.zeros(1, dtype=torch.int32),
                               torch.zeros((1, 2), dtype=torch.int64), (8, 8))
    with pytest.raises(RuntimeError, match="larger than the 8x8 slot"):
        data.stream_frames_sized(torch.zeros((1, 8, 8, 3), dtype=torch.uint8), [(9, 8)], (4, 4))
    with pytest.raises(RuntimeError, match="frames must be contiguous uint8"):
        data.stream_frames_sized(torch.zeros((1, 8, 8, 3), dtype=torch.float32), [(8, 8)], (4, 4))
    from test_fp16_storage import _tiny_model
    m = _tiny_model().eval()
    with pytest.raises(ValueError, match="frame_sizes must hold 2"):
        stream.StreamDetector(m, streams=2, frame_sizes=[(120, 160)] * 3)
    with pytest.raises(ValueError, match="jpeg_max_bytes"):
        stream.StreamDetector(m, frame_sizes=[(120, 160)], jpeg_max_bytes=0)
    with pytest.raises(ValueError, match="empty"):
        stream.StreamDetector(m, frame_sizes=[(120, 160), (4000, 2)], input_size=(64, 64))
    with pytest.raises(ValueError, match="input_size takes frame_sizes or jpeg_max_bytes"):
        stream.StreamDetector(m, frame_hw=(120, 160), input_size=(64, 64))


def test_new_kernels_compile_without_spills(tmp_path):
    """letterbox_sized_kernel, the refactored letterbox and JPEG kernels, stream_gate_kernel and stream_rescale_kernel: 0 spill
    bytes and no stack frame"""
    import re
    import shutil
    import subprocess
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    want = {"input.cu": ("letterbox_sized_kernel", "letterbox_kernel"), "jpeg.cu": ("jpeg_parse_kernel", "jpeg_color_kernel"),
            "postprocess.cu": ("stream_gate_kernel", "stream_rescale_kernel")}
    for src, kernels in want.items():
        r = subprocess.run([nvcc] + build.COMMON + build.SOURCES[src] + ["-c", os.path.join(build.CSRC, src), "-o",
                           str(tmp_path / "k.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
        assert r.returncode == 0, r.stdout
        found = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                           r"(\d+) bytes spill loads", r.stdout)
        for k in kernels:
            hits = [f for f in found if k in f[0]]
            assert hits and all(f[1:] == ("0", "0", "0") for f in hits), (k, hits)


def test_fixtures_are_cv2s():
    """the stored digests are cv2's (where cv2 is installed), and requant gives a valid, different frame"""
    cv2 = pytest.importorskip("cv2")
    for n in NAMES:
        img = cv2.imdecode(np.frombuffer(jpg(n), np.uint8), cv2.IMREAD_COLOR)
        assert img.shape[:2] == hw(n) and sha(img) == bytes(G[f"{n}.sha256"])
        img2 = cv2.imdecode(np.frombuffer(requant(jpg(n), 2), np.uint8), cv2.IMREAD_COLOR)
        assert sha(img2) == bytes(G[f"{n}.seq"][2])


# ================================================================================================ GPU
DEV = "cuda"


def _rows(files):
    rows, lengths = data.pack_jpeg(files, max(len(f) for f in files))
    return torch.from_numpy(rows).to(DEV), torch.from_numpy(lengths).to(DEV)


@pytest.mark.gpu
def test_decode_sized_is_cv2_with_mixed_sizes():
    """one batch of the three sizes, a requantised copy, the damaged file and a file given the wrong size: the decoded
    frames are cv2's, the refused slots and every pixel outside a frame keep their poison"""
    files = [jpg(n) for n in NAMES] + [requant(jpg("a420"), 3), jpg("bad"), jpg("b444")]
    sizes = [hw(n) for n in NAMES] + [hw("a420"), hw("bad"), (1550, 2048)]
    slot = (2048, 2048)
    rows, lengths = _rows(files)
    out = torch.full((len(files), *slot, 3), 7, dtype=torch.uint8, device=DEV)
    frames, status = data.decode_jpeg_sized(rows, lengths, sizes, slot, out=out)
    torch.cuda.synchronize()
    assert status.tolist() == [0, 0, 0, 0, 5, 4]
    f = frames.cpu().numpy()
    for i, n in enumerate(NAMES):
        h, w = hw(n)
        assert sha(f[i, :h, :w]) == bytes(G[f"{n}.sha256"]), n
        assert (f[i, h:] == 7).all() and (f[i, :, w:] == 7).all(), n
    assert sha(f[3, :1200, :1920]) == bytes(G["a420.seq"][3])
    assert (f[4] == 7).all() and (f[5] == 7).all()
    # the sizes as a device tensor (the captured form), one larger than the slot: status 4, slot untouched
    out.fill_(7)
    dev_sizes = torch.tensor([[1200, 1920], [2049, 1550]], dtype=torch.int32, device=DEV)
    rows2, len2 = _rows([jpg("a420"), jpg("b444")])
    _, st = data.decode_jpeg_sized(rows2, len2, dev_sizes, slot, out=out[:2])
    assert st.tolist() == [0, 4] and (out[1] == 7).all()


@pytest.mark.gpu
def test_stream_frames_sized_is_preproc():
    """each fixture's evaluation preproc at 600x960 and its r; the driver's plain resize through a table row of (h, w,
    600, 960); with in_scale, the 1200x1920 frame takes the plain resize"""
    files = [jpg(n) for n in NAMES]
    sizes = [hw(n) for n in NAMES]
    rows, lengths = _rows(files)
    frames, status = data.decode_jpeg_sized(rows, lengths, sizes, (2048, 2048))
    assert status.tolist() == [0, 0, 0]
    x, ratios = data.stream_frames_sized(frames, sizes, SIZE)
    xs = x.cpu().numpy()
    for i, n in enumerate(NAMES):
        assert xs[i].dtype == np.float32 and sha(xs[i]) == bytes(G[f"{n}.eval"]), n
        assert ratios[i] == float(G[f"{n}.r"])
    plain = torch.empty_like(x)
    table = torch.tensor([[h, w, SIZE[0], SIZE[1]] for h, w in sizes], dtype=torch.int32, device=DEV)
    ops.letterbox_sized(frames, table, plain)
    for i, n in enumerate(NAMES):
        assert sha(plain[i].cpu().numpy()) == bytes(G[f"{n}.plain"]), n
    x2, ratios2 = data.stream_frames_sized(frames, sizes, SIZE, in_scale=IN_SCALE)
    assert sha(x2[0].cpu().numpy()) == bytes(G["a420.plain"]) and ratios2[0] == IN_SCALE
    assert torch.equal(x2[1:], x[1:])


@pytest.mark.gpu
def test_equal_sizes_match_the_single_size_paths():
    """every frame 1200x1920: decode_jpeg_sized (slot of the frame's size, and a larger slot) equals decode_jpeg, and
    stream_frames_sized equals stream_frame, bit for bit"""
    files = [requant(jpg("a420"), k) for k in range(SEQ)]
    rows, lengths = _rows(files)
    ref, st = data.decode_jpeg(rows, lengths, (1200, 1920))
    got, st2 = data.decode_jpeg_sized(rows, lengths, [(1200, 1920)] * SEQ, (1200, 1920))
    big, st3 = data.decode_jpeg_sized(rows, lengths, [(1200, 1920)] * SEQ, (1216, 2048))
    assert st.tolist() == st2.tolist() == st3.tolist() == [0] * SEQ
    assert torch.equal(got, ref) and torch.equal(big[:, :1200, :1920], ref)
    for k in range(SEQ):
        assert sha(ref[k].cpu().numpy()) == bytes(G["a420.seq"][k])
    x, ratios = data.stream_frames_sized(got, [(1200, 1920)] * SEQ, SIZE)
    xb, _ = data.stream_frames_sized(big, [(1200, 1920)] * SEQ, SIZE)
    want = torch.cat([data.stream_frame(ref[k], SIZE) for k in range(SEQ)])
    assert torch.equal(x, want) and torch.equal(xb, want) and ratios == [0.5] * SEQ


@pytest.mark.gpu
def test_stream_rescale_is_numpys_division():
    """the boxes of each stream's count rows equal numpy's ``rows[:, :4] / ratio`` (the driver's ``det[:, :4] / in_scale``:
    float32 rows divided by a Python float) bit for bit, for ratios that are powers of two and ratios that are not; the
    other columns and the rows past the count keep their bits; a stream whose status is not 0 gets count 0"""
    rng = np.random.default_rng(3)
    ratios = [0.5, 0.3, 1 / 3, float(G["b444.r"]), float(G["c420_r16.r"])]
    n, max_det = len(ratios), 64
    rows = (rng.random((n, max_det, 7)) * rng.choice([1.0, 100.0, 2000.0], (n, max_det, 7))).astype(np.float32)
    counts = np.array([64, 37, 50, 1, 0], np.int32)
    assert (rows[0, :, :4] / 0.3).dtype == np.float32
    for status in (None, np.array([0, 0, 4, 0, 5], np.int32)):
        det, count = torch.from_numpy(rows).to(DEV), torch.from_numpy(counts).to(DEV)
        ops.stream_rescale(det, count, None if status is None else torch.from_numpy(status).to(DEV),
                           torch.tensor(ratios, dtype=torch.float32, device=DEV))
        got, got_n = det.cpu().numpy(), count.cpu().numpy()
        for i, r in enumerate(ratios):
            ok = status is None or status[i] == 0
            want = rows[i].copy()
            if ok:
                want[:counts[i], :4] = rows[i, :counts[i], :4] / r
            assert got_n[i] == (counts[i] if ok else 0), (i, status)
            assert np.array_equal(got[i].view(np.int32), want.view(np.int32)), (i, r, status)


def _model_s():
    from test_stream import _model_s as model_s
    return model_s(torch.float16)


def _driver_inference(result0, nc, r):
    from test_stream import driver_inference
    return driver_inference(result0, nc, r)


# (stream -> requant step of its file) per tick; "bad" = the damaged file, None = no frame; resets before the tick
TICKS = [
    ({0: 0, 1: 0, 2: 0}, ()),
    ({0: 1, 1: 1, 2: "bad"}, ()),
    ({0: 2, 1: None, 2: 1}, (1,)),
    ({0: 3, 1: 2, 2: 2}, (0,)),
    ({0: 0, 1: 3, 2: 3}, ()),
]


def _files(feed, i):
    f = feed.get(i)
    return None if f is None else jpg("bad") if f == "bad" else requant(jpg(NAMES[i]), f)


def _eager_x(i, f):
    """stream i's eager transform of the cv2 frame of file ``f`` (checked against the fixture's digest) and its ratio"""
    rows, lengths = _rows([_files({i: f}, i)])
    frame, s = data.decode_jpeg(rows, lengths, hw(NAMES[i]))
    assert s.tolist() == [0] and sha(frame[0].cpu().numpy()) == bytes(G[f"{NAMES[i]}.seq"][f])
    if i == 0:
        return data.stream_frame(frame[0], SIZE), IN_SCALE
    return data.frame_transform(frame, None, None, None, SIZE)[0], float(G[f"{NAMES[i]}.r"])


def _same(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
@pytest.mark.parametrize("i", [0, 1, 2], ids=list(NAMES))
def test_one_stream_of_each_size_bit_identical_to_eager_loop(i):
    """one stream of each size (1200x1920: the driver's plain resize; 2048x1550, 1550x2048: the evaluation letterbox) over
    the five ticks of TICKS: every decoded frame's head outputs and detections equal the driver's eager loop on cv2's frame
    (transform, model(x, buffer, mode='on_pipe'), inference() with the stream's ratio); the damaged file and the missing
    frame return nothing and leave the loop's buffer where it was, and the graph is never re-captured"""
    m = _model_s()
    nc = m.head.num_classes
    det = stream.StreamDetector(m, in_scale=IN_SCALE, frame_sizes=[hw(NAMES[i])], input_size=SIZE, jpeg_max_bytes=1 << 19,
                                conf_thre=CONF, nms_thre=NMS)
    graph, buffer, n_dets = det._graph, None, []
    for t, (feed, resets) in enumerate(TICKS):
        if i in resets:
            det.reset(0)
            buffer = None
        got = det.step_jpeg([_files(feed, i)])[0]
        assert det._graph is graph
        st = det.last_status().tolist()[0]
        if feed[i] is None or feed[i] == "bad":
            assert st == (stream.NO_FRAME if feed[i] is None else 5) and all(len(a) == 0 for a in got), (t, st)
            continue
        assert st == 0
        x, r = _eager_x(i, feed[i])
        with torch.no_grad():
            result, buffer = m(x, buffer=buffer, mode="on_pipe")
        assert torch.equal(det.last_raw()[0], result[0]), f"tick {t}: raw head outputs"
        assert _same(got, _driver_inference(result[0].cpu(), nc, r)), f"tick {t}: detections"
        n_dets.append(len(got[2]))
    assert all(n > 0 for n in n_dets), n_dets
    print(f"\n{NAMES[i]}: detections per decoded frame {n_dets}")


@pytest.mark.gpu
def test_three_mixed_streams_bit_identical_to_eager_batch():
    """the three sizes in one detector over TICKS (a damaged file, a missing frame, a reset issued while its stream has no
    frame, a reset of a decoded stream): each decoded stream's input is its own eager transform of cv2's frame, and the
    head outputs and detections equal two eager calls at batch 3 (the convs' summation order depends on the batch, so a
    batch-3 tick is compared with batch-3 calls, as tests/test_stream.py does): model(x, mode='on_pipe') for the current
    features, then model(x, buffer=mix) with mix[i] the current features of a stream that starts a sequence and the
    stream's carried features otherwise.  A gated stream returns nothing, keeps its carried features bit for bit and keeps
    its pending start; the graph is never re-captured.  A stream's results do not depend on the other streams: a second
    detector whose other two streams get other frames, and never miss one, gives stream 0 the same results bit for bit."""
    m = _model_s()
    nc = m.head.num_classes
    det = stream.StreamDetector(m, in_scale=IN_SCALE, frame_sizes=[hw(n) for n in NAMES], input_size=SIZE,
                                jpeg_max_bytes=1 << 19, conf_thre=CONF, nms_thre=NMS)
    assert det.streams == 3 and det.size == SIZE and det.frame_hw == (2048, 2048)
    assert det.ratios == [IN_SCALE] + [float(G[f"{n}.r"]) for n in NAMES[1:]]
    graph = det._graph
    carried = None                      # each stream's carried features, eager
    start = [True] * 3
    # a second detector whose streams 1 and 2 see other frames and never miss one: stream 0's results must not change
    other = stream.StreamDetector(m, in_scale=IN_SCALE, frame_sizes=[hw(n) for n in NAMES], input_size=SIZE,
                                  jpeg_max_bytes=1 << 19, conf_thre=CONF, nms_thre=NMS)
    for t, (feed, resets) in enumerate(TICKS):
        for i in resets:
            det.reset(i)
            start[i] = True
            if i == 0:
                other.reset(0)
        keep = [v.torch().clone() for v in det._tick.buffer]
        got = det.step_jpeg([_files(feed, i) for i in range(3)])
        assert det._graph is graph
        got_other = other.step_jpeg([_files(feed, 0)] + [requant(jpg(NAMES[i]), (t + i) % SEQ) for i in (1, 2)])
        assert torch.equal(other.last_raw()[0], det.last_raw()[0]) and _same(got_other[0], got[0]), f"tick {t}: stream 0"
        st = det.last_status().tolist()
        ok = [feed[i] is not None and feed[i] != "bad" for i in range(3)]
        assert st == [0 if ok[i] else stream.NO_FRAME if feed[i] is None else 5 for i in range(3)], (t, st)
        x = det._tick.x.clone()
        ratios = []
        for i in range(3):
            if ok[i]:
                xi, r = _eager_x(i, feed[i])
                assert torch.equal(x[i], xi[0]), f"tick {t} stream {i}: input"
                ratios.append(r)
            else:
                assert all(len(a) == 0 for a in got[i]), (t, i)
                assert all(torch.equal(v.torch()[i], k[i]) for v, k in zip(det._tick.buffer, keep)), f"tick {t} {i}: buffer"
                ratios.append(None)
        with torch.no_grad():
            _, cur = m(x, mode="on_pipe")
            cur = tuple(c.clone() for c in cur)
            mix = tuple(torch.stack([c[i] if (ok[i] and start[i]) or carried is None else p[i] for i in range(3)]).contiguous(
                memory_format=torch.channels_last) for c, p in zip(cur, carried or cur))
            result, _ = m(x, buffer=mix, mode="on_pipe")
        raw = det.last_raw()
        for i in range(3):
            if ok[i]:
                assert torch.equal(raw[i], result[i]), f"tick {t} stream {i}: raw head outputs"
                assert _same(got[i], _driver_inference(result[i].cpu(), nc, ratios[i])), f"tick {t} stream {i}"

        carried = tuple(torch.stack([c[i] if ok[i] else p[i] for i in range(3)]).contiguous(memory_format=torch.channels_last)
                        for c, p in zip(cur, carried or cur))
        start = [s and not o for s, o in zip(start, ok)]


@pytest.mark.gpu
def test_step_on_decoded_frames_equals_step_jpeg():
    """step() with frame_sizes takes the decoded frames of each stream's size (numpy and CUDA) and gives what step_jpeg
    gives for their files; on the detector built with jpeg_max_bytes, step() raises and leaves its state as it was"""
    m = _model_s()
    sizes = [hw(n) for n in NAMES]
    kw = dict(in_scale=IN_SCALE, frame_sizes=sizes, input_size=SIZE, conf_thre=CONF, nms_thre=NMS)
    dj = stream.StreamDetector(m, jpeg_max_bytes=1 << 19, **kw)
    df = stream.StreamDetector(m, **kw)
    for t in range(3):
        files = [requant(jpg(n), t) for n in NAMES]
        got = dj.step_jpeg(files)
        frames = []
        for i, f in enumerate(files):
            rows, lengths = _rows([f])
            fr = data.decode_jpeg(rows, lengths, sizes[i])[0][0]
            frames.append(fr if i % 2 else fr.cpu().numpy())
        want = df.step(frames)
        for i in range(3):
            assert all(np.array_equal(a, b) for a, b in zip(got[i], want[i])), (t, i)
        # the JPEG detector's replay decodes its files: it refuses decoded frames, and the refusal changes nothing (the
        # next step_jpeg still equals the frame detector's next step)
        with pytest.raises(RuntimeError, match="feed it with step_jpeg"):
            dj.step(frames)
    with pytest.raises(RuntimeError, match="frame 1 must be uint8"):
        df.step([frames[0], np.zeros((10, 10, 3), np.uint8), frames[2]])
    with pytest.raises(RuntimeError, match="jpeg_max_bytes"):
        df.step_jpeg(files)
