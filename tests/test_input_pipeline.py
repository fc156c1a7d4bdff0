"""The input transforms on the device (streamyolo_b200.data: sy_pair_labels, sy_letterbox).

CPU: the numpy oracle's 8-bit bilinear resize equals cv2.resize bit for bit on many shapes; the oracle's train / validation
     / streaming transforms equal tests/golden/input_pairs.npz (written from the unmodified reference); argument checks.
GPU: the kernels equal the oracle bit for bit (torch.equal): Argoverse-sized pairs, every fixture case, the streaming frame,
     a CUDA-graph replay, and the six losses of the model fed either input.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import input_oracle as io
from streamyolo_b200 import data, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "input_pairs.npz"))
CASES = sorted({k[:-len("_meta")] for k in GOLD if k.endswith("_meta")})
STREAM = sorted({k[:-len("_frame")] for k in GOLD if k.endswith("_frame")})

# (src h, w) -> (dst h, w): 2x / 4x down, non-integer down and up, tiny, and the Argoverse sizes
FIXED = [((1200, 1920), (600, 960)), ((1200, 1920), (599, 959)), ((1200, 1920), (496, 800)), ((8, 8), (4, 4)),
         ((16, 12), (4, 3)), ((1, 1), (4, 5)), ((750, 1333), (540, 959)), ((540, 959), (540, 960)), ((20, 94), (20, 95)),
         ((20, 95), (20, 96)), ((37, 53), (101, 77)), ((5, 7), (13, 3)), ((64, 64), (48, 80)), ((3, 3), (3, 3)),
         ((100, 1), (7, 9))]
_g = np.random.default_rng(7)
RANDOM = [((int(a), int(b)), (int(c), int(d))) for a, b, c, d in _g.integers(1, 260, (20, 4))]
EDGES = [((1, 37), (1, 12)), ((29, 1), (3, 1)), ((2, 2), (1, 1)), ((1, 1), (1, 1)), ((7, 11), (1, 40))]


def _case(name):
    return {k[len(name) + 1:]: GOLD[k] for k in GOLD if k.startswith(name + "_")}


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("src,dst", FIXED + RANDOM + EDGES)
def test_oracle_resize_equals_cv2(src, dst):
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(src[0] * 7919 + dst[1]).integers(0, 256, (src[0], src[1], 3), dtype=np.uint8)
    want = cv2.resize(img, (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR)
    assert np.array_equal(io.resize_linear_u8(img, (dst[1], dst[0])), want)


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_reference_fixture(name):
    c = _case(name)
    H, W, max_labels, mirror, raw, train = (int(v) for v in c["meta"])
    imgs = list(c["frames"])
    if train:
        tg = [c["ann"][i, :c["counts"][i]] for i in range(2)]
        x, fut, cur, _ = io.pair_transform(imgs, tg, (H, W), max_labels, mirror, raw=bool(raw))
        assert np.array_equal(fut, c["labels"][0]) and np.array_equal(cur, c["labels"][1])
    else:
        x = io.val_pair(imgs, (H, W), raw=bool(raw))
    assert np.array_equal(x, c["x"].astype(np.float32))


@pytest.mark.parametrize("name", STREAM)
def test_oracle_stream_frame_equals_fixture(name):
    out = GOLD[name + "_out"]
    got = io.stream_frame(GOLD[name + "_frame"], out.shape[1:])
    assert np.array_equal(got[0], out.astype(np.float32))


def test_argument_checks():
    frames = torch.zeros((1, 2, 8, 8, 3), dtype=torch.uint8)
    ann = torch.zeros((1, 2, 3, 5), dtype=torch.float64)
    counts = torch.zeros((1, 2), dtype=torch.int32)
    mirror = torch.zeros((1,), dtype=torch.int32)
    with pytest.raises(NotImplementedError):
        data.pair_transform(frames, ann, counts, mirror, (8, 8), hsv=True)
    with pytest.raises(RuntimeError, match="uint8"):
        data.pair_transform(frames.float(), ann, counts, mirror, (8, 8))
    with pytest.raises(RuntimeError, match="uint8"):
        data.pair_transform(frames[:, :1], ann, counts, mirror, (8, 8))
    with pytest.raises(RuntimeError, match="float64"):
        data.pair_transform(frames, ann.float(), counts, mirror, (8, 8))
    with pytest.raises(RuntimeError, match="counts"):
        data.pair_transform(frames, ann, counts.long(), mirror, (8, 8))
    with pytest.raises(RuntimeError, match="mirror"):
        data.pair_transform(frames, ann, counts, torch.zeros((2,), dtype=torch.int32), (8, 8))
    with pytest.raises(RuntimeError, match="out"):
        data.pair_transform(frames, ann, counts, mirror, (8, 8), out=(torch.zeros((1, 6, 8, 9)), None))
    with pytest.raises(RuntimeError, match="uint8"):
        data.stream_frame(torch.zeros((8, 8, 4), dtype=torch.uint8))


def test_entry_points_reject_bad_descriptors():
    """Host-side validation of sy_letterbox / sy_pair_labels: SY_EINVAL before anything reaches the device."""
    lib = ops.load_library()
    buf = (C.c_uint8 * 64)()
    out = (C.c_float * 64)()
    d = ops.SyLetterboxDesc(C.addressof(buf), 1, 2, 2, 2, 2, 3, 2, 2, 2, None, C.addressof(out))    # dst taller than canvas
    assert lib.sy_letterbox(C.byref(d), None) == 1
    d.dst_h, d.mid_w = 2, 0                                                                           # empty first stage
    assert lib.sy_letterbox(C.byref(d), None) == 1
    d.mid_w, d.src = 2, None
    assert lib.sy_letterbox(C.byref(d), None) == 1
    p = ops.SyPairLabelsDesc(C.addressof(out), C.addressof(buf), C.addressof(buf), 1, 2, 0, 1, 8, 1.0,
                             C.addressof(out), C.addressof(out), C.addressof(buf))                 # max_labels 0
    assert lib.sy_pair_labels(C.byref(p), None) == 1
    p.max_labels, p.mirror = 4, None                                                                  # flip without bits
    assert lib.sy_pair_labels(C.byref(p), None) == 1
    assert b"mirror" in lib.sy_last_error_string()


# ---------------------------------------------------------------------------------------------------------------- GPU
def _argoverse_batch(b, h, w, seed):
    """b frame pairs of h x w uint8 and annotations in 600 x 960 coordinates (what pull_item hands the transform), with an
    empty frame, an all-filtered frame and a frame with more rows than max_labels among them"""
    g = np.random.default_rng(seed)
    lo = g.integers(0, 256, (b, 2, h // 16 + 1, w // 16 + 1, 3)).astype(np.uint8)
    frames = np.repeat(np.repeat(lo, 16, 2), 16, 3)[:, :, :h, :w] ^ g.integers(0, 64, (b, 2, h, w, 3), dtype=np.uint8)
    m = 60
    ann = np.zeros((b, 2, m, 5))
    counts = g.integers(1, 30, (b, 2)).astype(np.int32)
    counts[1, 0] = 0
    counts[2, 1] = m
    for i in range(b):
        for f in range(2):
            n = counts[i, f]
            x1, y1 = g.uniform(0, 900, n), g.uniform(0, 560, n)
            bw = g.uniform(0.2, 0.9, n) if (i, f) == (3, 0) else g.uniform(0.5, 200, n)
            bh = g.uniform(0.5, 150, n)
            ann[i, f, :n] = np.stack([x1, y1, np.minimum(x1 + bw, 959), np.minimum(y1 + bh, 599), g.integers(0, 8, n)], 1)
    mirror = np.array([1, 1, 0, 1, 0, 1, 1, 0], np.int32)[:b]
    return frames, ann, counts, mirror


def _oracle_batch(frames, ann, counts, mirror, size, max_labels, raw):
    xs, fut, cur = [], [], []
    for i in range(len(frames)):
        tg = [ann[i, f, :counts[i, f]] for f in range(2)]
        x, a, c, _ = io.pair_transform(list(frames[i]), tg, size, max_labels, mirror[i], raw=raw)
        xs.append(x), fut.append(a), cur.append(c)
    return torch.from_numpy(np.stack(xs)), torch.from_numpy(np.stack(fut)), torch.from_numpy(np.stack(cur))


def _dev(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


@pytest.mark.gpu
@pytest.mark.parametrize("raw", [True, False], ids=["raw_1200x1920", "resized_600x960"])
def test_argoverse_pairs_bit_exact(raw):
    h, w = (1200, 1920) if raw else (600, 960)
    frames, ann, counts, mirror = _argoverse_batch(8, h, w, seed=11 + raw)
    x, (fut, cur) = data.pair_transform(*_dev(frames, ann, counts, mirror), (600, 960), max_labels=50, raw=raw)
    wx, wf, wc = _oracle_batch(frames, ann, counts, mirror, (600, 960), 50, raw)
    assert torch.equal(x.cpu(), wx)
    assert torch.equal(fut.cpu(), wf) and torch.equal(cur.cpu(), wc)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_fixture_case_on_device(name):
    c = _case(name)
    H, W, max_labels, mirror, raw, train = (int(v) for v in c["meta"])
    frames = torch.from_numpy(c["frames"][None]).cuda()
    if train:
        ann, counts, mir = _dev(c["ann"][None], c["counts"][None], np.array([mirror], np.int32))
        x, (fut, cur) = data.pair_transform(frames, ann, counts, mir, (H, W), max_labels, raw=bool(raw))
        assert torch.equal(fut[0].cpu(), torch.from_numpy(c["labels"][0]))
        assert torch.equal(cur[0].cpu(), torch.from_numpy(c["labels"][1]))
    else:
        x, labels = data.pair_transform(frames, None, None, None, (H, W), flip=False, raw=bool(raw))
        assert labels is None
    assert torch.equal(x[0].cpu(), torch.from_numpy(c["x"]).float())


@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", [((1200, 1920), (600, 960)), ((720, 1280), (600, 960))], ids=["1200x1920", "720x1280"])
def test_stream_frame_bit_exact(src, dst):
    frame = np.random.default_rng(src[0]).integers(0, 256, (src[0], src[1], 3), dtype=np.uint8)
    got = data.stream_frame(torch.from_numpy(frame).cuda(), dst)
    assert got.shape == (1, 3) + dst
    assert torch.equal(got.cpu(), torch.from_numpy(io.stream_frame(frame, dst)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", STREAM)
def test_stream_fixture_on_device(name):
    out = torch.from_numpy(GOLD[name + "_out"]).float()[None]
    got = data.stream_frame(torch.from_numpy(GOLD[name + "_frame"]).cuda(), tuple(out.shape[2:]))
    assert torch.equal(got.cpu(), out)


@pytest.mark.gpu
def test_graph_capture_replays_new_inputs():
    """Capture once on static inputs, copy another batch's frames, annotations and mirror bits in, replay: the eager result."""
    size, ml = (600, 960), 50
    batches = [_argoverse_batch(8, 1200, 1920, seed=s) for s in (21, 22)]
    static = _dev(*batches[0])
    out = data.pair_transform(*static, size, ml, raw=True)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        data.pair_transform(*static, size, ml, raw=True, out=out)
    for t, a in zip(static, batches[1]):
        t.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    g.replay()
    torch.cuda.synchronize()
    x, (fut, cur) = data.pair_transform(*_dev(*batches[1]), size, ml, raw=True)
    assert torch.equal(out[0], x) and torch.equal(out[1][0], fut) and torch.equal(out[1][1], cur)


@pytest.mark.gpu
def test_model_losses_match_oracle_input():
    """One training forward: the six losses of the model fed the device transform equal those of the model fed the oracle's
    fp32 tensor (the inputs are bit-identical, so are the losses)."""
    from streamyolo_b200.model import engine
    from test_gpu_model import build_product
    size = (192, 320)
    frames, ann, counts, mirror = _argoverse_batch(4, 384, 640, seed=5)
    ann[..., :4] *= 320 / 960                       # annotations of the 192 x 320 pull_item image
    model = build_product(0.33, 0.25).train()
    engine.name_modules(model)
    x, (fut, cur) = data.pair_transform(*_dev(frames, ann, counts, mirror), size, max_labels=50, raw=True)
    wx, wf, wc = _oracle_batch(frames, ann, counts, mirror, size, 50, True)
    order = ["total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss", "num_fg"]
    with torch.no_grad():
        got = model(x, (fut, cur))
        got = torch.stack([torch.as_tensor(got[k], dtype=torch.float32, device="cuda").reshape(()) for k in order])
        want = model(wx.cuda(), (wf.cuda(), wc.cuda()))
        want = torch.stack([torch.as_tensor(want[k], dtype=torch.float32, device="cuda").reshape(()) for k in order])
    assert torch.isfinite(got).all()
    assert torch.equal(got, want), (got, want)
