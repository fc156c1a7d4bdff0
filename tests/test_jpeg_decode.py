"""Device JPEG decode (sy_jpeg_decode, streamyolo_b200.data.decode_jpeg).

CPU: the numpy oracle (oracle/jpeg_oracle.py) equals cv2.imdecode bit for bit over qualities, samplings, restart intervals,
     standard and optimised tables and sizes; it equals every committed fixture; it gives each unsupported or damaged
     stream its status; argument checks; jpeg.cu compiles for sm_90a without spills.
GPU: every fixture decodes bit-exact (restart-interval and self-synchronising paths, full 1200 x 1920 frames), mixed
     batches with bad streams, determinism, a CUDA-graph replay, decode -> pair_transform(raw=True), and a Trainer whose
     captured prologue decodes the bytes against eager steps on cv2's frames.
"""
import hashlib
import os
import re
import subprocess
import zlib

import numpy as np
import pytest
import torch

from oracle import jpeg_oracle as jo
from oracle import make_jpeg_golden as mk
from streamyolo_b200 import data, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_small.npz"))
FULL = mk.load_full()
BAD = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_bad.npz"))
SMALL_NAMES = sorted(k[:-4] for k in SMALL if k.endswith(".jpg"))
FULL_NAMES = sorted(k[:-4] for k in FULL if k.endswith(".jpg"))
BAD_NAMES = sorted(k[:-4] for k in BAD if k.endswith(".jpg"))

SIZES = [(1, 1), (8, 8), (17, 23), (15, 31), (33, 65)]
MATRIX = [(hw, q, s, r, o) for hw in SIZES for q in (50, 75, 95, 100) for s in ("420", "422", "444") for r in (0, 1, 7)
          for o in (0, 1)]
LARGE = [((600, 960), 75, "420", 0, 0), ((600, 960), 95, "422", 7, 1), ((600, 960), 50, "444", 1, 0),
         ((600, 960), 100, "420", 0, 1)]


def _band(name):
    return 16 if "420" in name else 8


def _check_full(name, img):
    """cv2's output of fixture ``name`` by its SHA-256, naming the first differing MCU row otherwise"""
    rows = FULL[name + ".rows"]
    band = _band(name)
    got = np.array([zlib.crc32(img[y:y + band].tobytes()) for y in range(0, img.shape[0], band)], np.int64)
    bad = np.nonzero(got != rows)[0]
    assert bad.size == 0, f"{name}: first wrong MCU row {bad[0]} (pixel rows {bad[0] * band}..)"
    assert hashlib.sha256(np.ascontiguousarray(img).tobytes()).digest() == FULL[name + ".sha256"].tobytes()


def _full_hw(name):
    return (600, 960) if name.startswith("m") else (1200, 1920)


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("hw,q,samp,rst,opt", MATRIX + LARGE)
def test_oracle_equals_cv2(hw, q, samp, rst, opt):
    cv2 = pytest.importorskip("cv2")
    b = mk.encode(mk.synth_frame(hw[0], hw[1], q + rst), q, samp, rst, opt)
    got, st = jo.decode(b, hw)
    assert st == jo.OK
    assert np.array_equal(got, cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR))


@pytest.mark.parametrize("name", SMALL_NAMES)
def test_oracle_equals_small_fixture(name):
    want = SMALL[name + ".bgr"]
    got, st = jo.decode(SMALL[name + ".jpg"], want.shape[:2])
    assert st == jo.OK and np.array_equal(got, want)


@pytest.mark.parametrize("name", FULL_NAMES)
def test_oracle_equals_full_fixture(name):
    got, st = jo.decode(FULL[name + ".jpg"], _full_hw(name))
    assert st == jo.OK
    _check_full(name, got)


def test_oracle_status_of_bad_streams():
    pytest.importorskip("cv2")
    want = {"progressive": jo.EUNSUPPORTED, "arithmetic_sof9": jo.EUNSUPPORTED, "precision_12": jo.EUNSUPPORTED,
            "sampling_411": jo.EUNSUPPORTED, "grayscale": jo.EUNSUPPORTED, "exif_orientation_6": jo.EORIENTATION,
            "size_mismatch": jo.ESIZE}
    streams = mk.bad_streams()
    for name, st in want.items():
        assert jo.decode(streams[name], (33, 65))[1] == st, name
    cuts = [k for k in streams if k.startswith("cut_")]
    assert len(cuts) == 5
    for k in cuts:
        assert jo.decode(streams[k], (33, 65))[1] in (jo.EHEADER, jo.EDATA), k
    # the stream with orientation 1 decodes like the plain one
    plain = mk.encode(mk.synth_frame(33, 65, 7), 90, "420", 0, 0)
    assert np.array_equal(jo.decode(plain[:2] + mk.exif_app1(1) + plain[2:])[0], jo.decode(plain)[0])


def test_bad_fixture_status_is_the_oracles():
    for name in BAD_NAMES:
        assert jo.decode(BAD[name + ".jpg"], (33, 65))[1] == int(BAD[name + ".status"]), name
        assert int(BAD[name + ".status"]) != jo.OK


def test_pack_jpeg():
    files = [b"\xff\xd8abc", np.arange(7, dtype=np.uint8), bytearray(b"")]
    rows, lengths = data.pack_jpeg(files, 8)
    assert rows.dtype == np.uint8 and rows.shape == (3, 8) and lengths.dtype == np.int32
    assert lengths.tolist() == [5, 7, 0]
    assert rows[0, :5].tobytes() == b"\xff\xd8abc" and not rows[0, 5:].any()
    assert np.array_equal(rows[1, :7], np.arange(7))
    with pytest.raises(ValueError, match="file 1"):
        data.pack_jpeg([b"ab", b"abcdefghi"], 8)


def test_argument_checks():
    ops.load_library()
    u8 = lambda *s: torch.zeros(s, dtype=torch.uint8)
    i32 = lambda *s: torch.zeros(s, dtype=torch.int32)
    ws = u8(ops.jpeg_decode_workspace_bytes(2, 64, 8, 8))
    good = dict(streams=u8(2, 64), lengths=i32(2), out=u8(2, 8, 8, 3), status=i32(2), workspace=ws)
    bad = [("streams", torch.zeros((2, 64), dtype=torch.int32)), ("streams", u8(2, 64, 1)), ("lengths", i32(3)),
           ("lengths", torch.zeros(2, dtype=torch.int64)), ("out", u8(2, 8, 8, 4)), ("out", u8(3, 8, 8, 3)),
           ("status", i32(1)), ("workspace", u8(16))]
    for key, val in bad:
        args = dict(good, **{key: val})
        with pytest.raises(RuntimeError, match="jpeg_decode"):
            ops.jpeg_decode(**args)
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.jpeg_decode(**good)                  # CPU tensors
    for n, mb, h, w in ((0, 64, 8, 8), (1, 0, 8, 8), (1, 64, 0, 8), (1, 64, 8, 70000), (1, 1 << 29, 8, 8)):
        with pytest.raises(RuntimeError, match="bad sizes"):
            ops.jpeg_decode_workspace_bytes(n, mb, h, w)


def test_jpeg_cu_compiles_without_spills():
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc not available")
    cmd = [build.NVCC] + build.COMMON + build.SOURCES["jpeg.cu"] + ["-c", os.path.join(build.CSRC, "jpeg.cu"), "-o",
                                                                    os.devnull]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == 5, r.stderr
    assert all(p == ("0", "0", "0") for p in props), r.stderr


# ---------------------------------------------------------------------------------------------------------------- GPU
def _pack_cuda(files, max_bytes=None):
    max_bytes = max_bytes or max(len(f) for f in files) + 64
    rows, lengths = data.pack_jpeg([np.asarray(f, np.uint8) for f in files], max_bytes)
    return torch.from_numpy(rows).cuda(), torch.from_numpy(lengths).cuda()


@pytest.mark.gpu
def test_gpu_small_fixtures_bit_exact():
    by_size = {}
    for name in SMALL_NAMES:
        by_size.setdefault(SMALL[name + ".bgr"].shape[:2], []).append(name)
    for hw, names in by_size.items():
        s, l = _pack_cuda([SMALL[n + ".jpg"] for n in names])
        frames, status = data.decode_jpeg(s, l, hw)
        data.check_jpeg_status(status)
        for k, n in enumerate(names):
            assert np.array_equal(frames[k].cpu().numpy(), SMALL[n + ".bgr"]), n


@pytest.mark.gpu
def test_gpu_full_fixtures_bit_exact_with_truncated():
    big = [n for n in FULL_NAMES if _full_hw(n) == (1200, 1920)]
    files = [FULL[n + ".jpg"] for n in big]
    files.append(files[0][: len(files[0]) * 3 // 5])                  # cut inside the entropy-coded segment
    s, l = _pack_cuda(files)
    frames, status = data.decode_jpeg(s, l, (1200, 1920))
    st = status.cpu().tolist()
    assert st == [0] * len(big) + [jo.EDATA], st
    for k, n in enumerate(big):
        _check_full(n, frames[k].cpu().numpy())
    med = [n for n in FULL_NAMES if _full_hw(n) == (600, 960)]
    s, l = _pack_cuda([FULL[n + ".jpg"] for n in med])
    frames, status = data.decode_jpeg(s, l, (600, 960))
    data.check_jpeg_status(status)
    for k, n in enumerate(med):
        _check_full(n, frames[k].cpu().numpy())


@pytest.mark.gpu
def test_gpu_mixed_batch_with_bad_streams():
    good = [n for n in SMALL_NAMES if SMALL[n + ".bgr"].shape[:2] == (33, 65)]
    files = []
    for k in range(len(BAD_NAMES)):                                     # interleave good and bad streams
        files.append(("good", good[k % len(good)]))
        files.append(("bad", BAD_NAMES[k]))
    s, l = _pack_cuda([(SMALL if kind == "good" else BAD)[n + ".jpg"] for kind, n in files])
    out = torch.full((len(files), 33, 65, 3), 0x5A, dtype=torch.uint8, device="cuda")
    frames, status = data.decode_jpeg(s, l, (33, 65), out=out)
    st = status.cpu().tolist()
    for k, (kind, n) in enumerate(files):
        if kind == "good":
            assert st[k] == 0, n
            assert np.array_equal(frames[k].cpu().numpy(), SMALL[n + ".bgr"]), n
        else:
            assert st[k] == int(BAD[n + ".status"]), (n, st[k])
            assert bool((frames[k] == 0x5A).all()), n                  # a refused image is left untouched
    with pytest.raises(RuntimeError, match="frame 1 did not decode"):
        data.check_jpeg_status(status)
    # lengths outside [4, max_bytes] are refused per image
    l2 = l.clone()
    l2[0], l2[2] = s.shape[1] + 1, -5
    _, status = data.decode_jpeg(s, l2, (33, 65))
    st = status.cpu().tolist()
    assert st[0] == jo.EHEADER and st[2] == jo.EHEADER


@pytest.mark.gpu
def test_gpu_decode_is_deterministic():
    files = [FULL[n + ".jpg"] for n in FULL_NAMES if _full_hw(n) == (1200, 1920)]
    s, l = _pack_cuda(files)
    a, sa = data.decode_jpeg(s, l, (1200, 1920))
    a = a.clone()
    b, sb = data.decode_jpeg(s, l, (1200, 1920))
    assert torch.equal(a, b) and torch.equal(sa, sb)


@pytest.mark.gpu
def test_gpu_graph_replay_follows_new_bytes():
    names = [n for n in SMALL_NAMES if SMALL[n + ".bgr"].shape[:2] == (33, 65)]
    max_bytes = max(SMALL[n + ".jpg"].size for n in names) + 64
    s, l = _pack_cuda([SMALL[n + ".jpg"] for n in names], max_bytes)
    out = torch.empty((len(names), 33, 65, 3), dtype=torch.uint8, device="cuda")
    status = torch.empty((len(names),), dtype=torch.int32, device="cuda")
    ws = torch.empty(ops.jpeg_decode_workspace_bytes(len(names), max_bytes, 33, 65), dtype=torch.uint8, device="cuda")
    data.decode_jpeg(s, l, (33, 65), out=out, status=status, workspace=ws)      # warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        data.decode_jpeg(s, l, (33, 65), out=out, status=status, workspace=ws)
    rev = names[::-1]
    s2, l2 = _pack_cuda([SMALL[n + ".jpg"] for n in rev], max_bytes)
    s.copy_(s2)
    l.copy_(l2)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    eager, est = data.decode_jpeg(s2, l2, (33, 65))
    assert torch.equal(status, est) and status.abs().sum().item() == 0
    assert torch.equal(out, eager)
    for k, n in enumerate(rev):
        assert np.array_equal(out[k].cpu().numpy(), SMALL[n + ".bgr"])


@pytest.mark.gpu
def test_gpu_decode_then_pair_transform():
    names = [n for n in SMALL_NAMES if SMALL[n + ".bgr"].shape[:2] == (33, 65)]
    assert len(names) % 2 == 0
    s, l = _pack_cuda([SMALL[n + ".jpg"] for n in names])
    frames, status = data.decode_jpeg(s, l, (33, 65))
    data.check_jpeg_status(status)
    b = len(names) // 2
    ref = torch.from_numpy(np.stack([SMALL[n + ".bgr"] for n in names])).cuda()
    ann = torch.zeros((b, 2, 3, 5), dtype=torch.float64, device="cuda")
    ann[..., 0:2] = 2.0
    ann[..., 2] = 30.0
    ann[..., 3] = 20.0
    counts = torch.full((b, 2), 3, dtype=torch.int32, device="cuda")
    mirror = torch.tensor([1, 0] * (b // 2) + [1] * (b % 2), dtype=torch.int32, device="cuda")
    for raw_size in ((32, 64), (24, 40)):
        x1, l1 = data.pair_transform(frames.view(b, 2, 33, 65, 3), ann, counts, mirror, raw_size, raw=True)
        x2, l2 = data.pair_transform(ref.view(b, 2, 33, 65, 3), ann, counts, mirror, raw_size, raw=True)
        assert torch.equal(x1, x2) and torch.equal(l1[0], l2[0]) and torch.equal(l1[1], l2[1])


@pytest.mark.gpu
def test_gpu_trainer_prologue_decode_equals_eager_on_cv2_frames():
    """A Trainer step graph whose prologue is decode_jpeg + pair_transform(raw=True) on static file bytes: each replay, fed
    new bytes, gives the losses and the training state of an eager step fed cv2's decoded frames, bit for bit"""
    from oracle.make_golden import CASES
    from streamyolo_b200 import train
    from test_gpu_model import build_product
    from test_multiscale_train import _assert_same, _snapshot
    c = CASES["tiny_120x160"]
    names = [n for n in SMALL_NAMES if SMALL[n + ".bgr"].shape[:2] == (33, 65)]
    b, hw, size, max_labels = len(names) // 2, (33, 65), (96, 160), 50
    orders = [names, names[::-1], names[1:] + names[:1]]
    max_bytes = max(SMALL[n + ".jpg"].size for n in names) + 64
    ann = torch.zeros((b, 2, 4, 5), dtype=torch.float64, device="cuda")
    ann[..., 0], ann[..., 1], ann[..., 2], ann[..., 3] = 10.0, 8.0, 90.0, 60.0
    ann[:, :, 1, :4] = torch.tensor([70.0, 20.0, 150.0, 78.0], dtype=torch.float64)
    ann[..., 4] = torch.tensor([0.0, 3.0, 5.0, 7.0], dtype=torch.float64)
    counts = torch.tensor([[2, 2], [2, 1]], dtype=torch.int32, device="cuda")[:b]
    mirror = torch.tensor([1, 0], dtype=torch.int32, device="cuda")[:b]
    lrs = [1e-4, 2e-4, 1.5e-4]

    ta = train.Trainer(build_product(c["depth"], c["width"]).train(), lr=1e-4)
    want = []
    for order, lr in zip(orders, lrs):
        ref = torch.from_numpy(np.stack([SMALL[n + ".bgr"] for n in order])).cuda()
        x, tg = data.pair_transform(ref.view(b, 2, *hw, 3), ann, counts, mirror, size, max_labels, raw=True)
        want.append({k: float(v) for k, v in ta.step(x, tg, lr=lr).items()})
    torch.cuda.synchronize()

    streams = torch.zeros((2 * b, max_bytes), dtype=torch.uint8, device="cuda")
    lengths = torch.zeros((2 * b,), dtype=torch.int32, device="cuda")
    frames = torch.empty((2 * b, *hw, 3), dtype=torch.uint8, device="cuda")
    status = torch.empty((2 * b,), dtype=torch.int32, device="cuda")
    ws = torch.empty(ops.jpeg_decode_workspace_bytes(2 * b, max_bytes, *hw), dtype=torch.uint8, device="cuda")
    inputs = (torch.empty((b, 6) + size, dtype=torch.float32, device="cuda"),
              tuple(torch.empty((b, max_labels, 5), dtype=torch.float32, device="cuda") for _ in range(2)))

    def load(order):
        s, l = _pack_cuda([SMALL[n + ".jpg"] for n in order], max_bytes)
        streams.copy_(s)
        lengths.copy_(l)

    def prologue(sz, x, targets):
        data.decode_jpeg(streams, lengths, hw, out=frames, status=status, workspace=ws)
        data.pair_transform(frames.view(b, 2, *hw, 3), ann, counts, mirror, size, max_labels, raw=True, out=(x, targets))

    tb = train.Trainer(build_product(c["depth"], c["width"]).train(), lr=1e-4)
    load(orders[0])
    tb.capture_sizes([size], lambda sz: inputs, prologue)
    for order, lr, w in zip(orders, lrs, want):
        load(order)
        got = tb.replay_size(size, lr=lr)
        assert {k: float(v) for k, v in got.items()} == w
        assert status.abs().sum().item() == 0
    torch.cuda.synchronize()
    _assert_same(_snapshot(tb), _snapshot(ta), "after the steps")
