"""The single-frame input transform on the device (streamyolo_b200.data.frame_transform: sy_frame_labels, sy_letterbox): the
dataset transform of the still-image baseline, TrainTransform(max_labels, hsv=False, flip) / ValTransform.

CPU: the numpy oracle's ``train_frame`` / letterbox equal tests/golden/input_frames.npz (written from the unmodified reference
by oracle/make_input_frames_golden.py); argument checks.
GPU: the kernels equal the oracle bit for bit (torch.equal): every fixture case, Argoverse-sized frames (raw 1200 x 1920 and
the 600 x 960 pull_item image) with empty, all-filtered and overfull frames among them, and a CUDA-graph replay.
"""
import os

import numpy as np
import pytest
import torch

from oracle import input_oracle as io
from streamyolo_b200 import data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "input_frames.npz"))
CASES = sorted({k[:-len("_meta")] for k in GOLD if k.endswith("_meta")})


def _case(name):
    return {k[len(name) + 1:]: GOLD[k] for k in GOLD if k.startswith(name + "_")}


def _oracle_frame(img, tg, size, max_labels, mirror, raw, train=True):
    if raw:
        img = io.load_resized(img, size)
    if not train:
        return io.letterbox(img, size)[0], None
    x, labels, _ = io.train_frame(img, tg, size, max_labels, mirror)
    return x, labels


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_reference_fixture(name):
    c = _case(name)
    H, W, max_labels, mirror, raw, train = (int(v) for v in c["meta"])
    x, labels = _oracle_frame(c["frame"], c["ann"][:int(c["count"][0])], (H, W), max_labels, mirror, bool(raw), bool(train))
    if train:
        assert np.array_equal(labels, c["labels"])
    assert np.array_equal(x, c["x"].astype(np.float32))


def test_fixture_covers_the_label_rules():
    """the cases the fixture is named for: an empty frame, the all-filtered fallback, more rows than max_labels, raw frames"""
    assert {"no_annotations", "all_filtered", "too_many_rows", "raw", "two_resizes", "val", "val_raw"} <= set(CASES)
    c = _case("too_many_rows")
    assert int(c["count"][0]) > int(c["meta"][2]) and (c["labels"][:, 3:] > 1).all()


def test_argument_checks():
    frames = torch.zeros((1, 8, 8, 3), dtype=torch.uint8)
    ann = torch.zeros((1, 3, 5), dtype=torch.float64)
    counts = torch.zeros((1,), dtype=torch.int32)
    mirror = torch.zeros((1,), dtype=torch.int32)
    with pytest.raises(RuntimeError, match="uint8"):
        data.frame_transform(frames.float(), ann, counts, mirror, (8, 8))
    with pytest.raises(RuntimeError, match="uint8"):
        data.frame_transform(frames[None], ann, counts, mirror, (8, 8))
    with pytest.raises(RuntimeError, match="out image"):
        data.frame_transform(frames, ann, counts, mirror, (8, 8), out=(torch.zeros((1, 6, 8, 8)), None))
    with pytest.raises(RuntimeError, match="out labels"):
        data.frame_transform(frames, ann, counts, mirror, (8, 8), out=(torch.zeros((1, 3, 8, 8)), None))
    with pytest.raises(RuntimeError, match="float64"):
        data.frame_transform(frames, ann.float(), counts, mirror, (8, 8))
    with pytest.raises(RuntimeError, match="counts"):
        data.frame_transform(frames, ann, counts.long(), mirror, (8, 8))
    with pytest.raises(RuntimeError, match="mirror"):
        data.frame_transform(frames, ann, counts, torch.zeros((2,), dtype=torch.int32), (8, 8))


# ---------------------------------------------------------------------------------------------------------------- GPU
def _argoverse_frames(b, h, w, seed):
    """b frames of h x w uint8 and annotations in 600 x 960 coordinates, with an empty frame, an all-filtered frame and a
    frame with more rows than max_labels among them"""
    g = np.random.default_rng(seed)
    lo = g.integers(0, 256, (b, h // 16 + 1, w // 16 + 1, 3)).astype(np.uint8)
    frames = np.repeat(np.repeat(lo, 16, 1), 16, 2)[:, :h, :w] ^ g.integers(0, 64, (b, h, w, 3), dtype=np.uint8)
    m = 60
    ann = np.zeros((b, m, 5))
    counts = g.integers(1, 30, b).astype(np.int32)
    counts[1] = 0
    counts[2] = m
    for i in range(b):
        n = counts[i]
        x1, y1 = g.uniform(0, 900, n), g.uniform(0, 560, n)
        bw = g.uniform(0.2, 0.9, n) if i == 3 else g.uniform(0.5, 200, n)
        bh = g.uniform(0.5, 150, n)
        ann[i, :n] = np.stack([x1, y1, np.minimum(x1 + bw, 959), np.minimum(y1 + bh, 599), g.integers(0, 8, n)], 1)
    mirror = np.array([1, 1, 0, 1, 0, 1, 1, 0], np.int32)[:b]
    return frames, ann, counts, mirror


def _oracle_batch(frames, ann, counts, mirror, size, max_labels, raw):
    xs, ls = [], []
    for i in range(len(frames)):
        x, lab = _oracle_frame(frames[i], ann[i, :counts[i]], size, max_labels, mirror[i], raw)
        xs.append(x), ls.append(lab)
    return torch.from_numpy(np.stack(xs)), torch.from_numpy(np.stack(ls))


def _dev(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


@pytest.mark.gpu
@pytest.mark.parametrize("raw", [True, False], ids=["raw_1200x1920", "resized_600x960"])
def test_argoverse_frames_bit_exact(raw):
    h, w = (1200, 1920) if raw else (600, 960)
    frames, ann, counts, mirror = _argoverse_frames(8, h, w, seed=31 + raw)
    x, labels = data.frame_transform(*_dev(frames, ann, counts, mirror), (600, 960), max_labels=50, raw=raw)
    wx, wl = _oracle_batch(frames, ann, counts, mirror, (600, 960), 50, raw)
    assert x.shape == (8, 3, 600, 960) and labels.shape == (8, 50, 5)
    assert torch.equal(x.cpu(), wx)
    assert torch.equal(labels.cpu(), wl)
    xv, none = data.frame_transform(_dev(frames)[0], None, None, None, (600, 960), raw=raw)      # ValTransform
    assert none is None
    wv = torch.from_numpy(np.stack([_oracle_frame(f, None, (600, 960), 50, 0, raw, train=False)[0] for f in frames]))
    assert torch.equal(xv.cpu(), wv)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_fixture_case_on_device(name):
    c = _case(name)
    H, W, max_labels, mirror, raw, train = (int(v) for v in c["meta"])
    frames = torch.from_numpy(c["frame"][None]).cuda()
    if train:
        ann, counts, mir = _dev(c["ann"][None], c["count"], np.array([mirror], np.int32))
        x, labels = data.frame_transform(frames, ann, counts, mir, (H, W), max_labels, raw=bool(raw))
        assert torch.equal(labels[0].cpu(), torch.from_numpy(c["labels"]))
    else:
        x, labels = data.frame_transform(frames, None, None, None, (H, W), flip=False, raw=bool(raw))
        assert labels is None
    assert torch.equal(x[0].cpu(), torch.from_numpy(c["x"]).float())


@pytest.mark.gpu
def test_graph_capture_replays_new_inputs():
    """Capture once on static inputs, copy another batch's frames, annotations and mirror bits in, replay: the eager result."""
    size, ml = (600, 960), 50
    batches = [_argoverse_frames(8, 1200, 1920, seed=s) for s in (41, 42)]
    static = _dev(*batches[0])
    out = data.frame_transform(*static, size, ml, raw=True)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        data.frame_transform(*static, size, ml, raw=True, out=out)
    for t, a in zip(static, batches[1]):
        t.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    g.replay()
    torch.cuda.synchronize()
    x, labels = data.frame_transform(*_dev(*batches[1]), size, ml, raw=True)
    assert torch.equal(out[0], x) and torch.equal(out[1], labels)
    wx, wl = _oracle_batch(*batches[1], size, ml, True)
    assert torch.equal(x.cpu(), wx) and torch.equal(labels.cpu(), wl)
