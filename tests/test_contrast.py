"""Split-screen comparison frames on the device (sy_splice_frames, data.splice_frames, python -m
streamyolo_b200.contrast).

CPU: the fixture's inputs decode alike in cv2 and PIL; the numpy oracle (oracle/contrast_oracle.py), on those decodes
     and encoded as the script's PIL does, equals every file the unmodified vis_contrast.py wrote
     (tests/golden/contrast_script.npz), and the fixture reaches every case of the split; the CLI's split arithmetic
     equals the oracle's; the CLI's host logic with the device pass emulated writes the script's files, directories and
     printed lines for every run, keeps skipped files, and runs make_videos_numbered's ffmpeg argv once; the SOF reader;
     the refusals, in the CLI and in the C entry without a device; contrast.cu compiles for sm_90a without spills.
GPU: sy_splice_frames equals the oracle on mixed sizes in larger slots, vertical and horizontal, with B aligned as A or
     at an odd offset, and every slot pixel outside the frames keeping its poison value; two replays of a captured graph
     repeat bit for bit and follow rewritten splits; the CLI writes the script's files byte for byte and names a file the
     decoder refuses.
"""
import ctypes as C
import io
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import contrast_oracle as co
from streamyolo_b200 import contrast, data, ops, vis

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "contrast_script.npz"))
RUNS = [str(r) for r in GOLD["runs"]]
BGR = data.CONTRAST_BAND_BGR


def _cv2():
    return pytest.importorskip("cv2")


def inputs():
    """{relative path under the fixture root: bytes}"""
    return {k[3:]: GOLD[k].tobytes() for k in GOLD.files if k.startswith("in/")}


def setup_fixture(tmp_path):
    """the fixture's directories A and B under tmp_path -> (dir A, dir B)"""
    for rel, b in inputs().items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(b)
    return str(tmp_path / "A"), str(tmp_path / "B")


def run_opts(a, b, out, run):
    return contrast.parse_args(["--dir-A", a, "--dir-B", b, "--out-dir", out] + [str(v) for v in GOLD[run + ".argv"]])


def decode(b):
    cv2 = _cv2()
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def encode(img):
    cv2 = _cv2()
    return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 75])[1].tobytes()


def emulated_pass(files_a, files_b, frames, opts):
    """the device half of contrast.run on the host: the SOF sizes, cv2.imdecode, the splice rule of sy_splice_frames
    on the CLI's clamped (split, band_start, band_end), cv2.imencode at quality 75"""
    sizes = contrast.pair_sizes(frames, files_a, files_b)
    out = []
    for fa, fb, f, (h, w) in zip(files_a, files_b, frames, sizes):
        a, b = decode(fa), decode(fb)
        assert a.shape[:2] == b.shape[:2] == (h, w)
        out.append(encode(splice_rule(a, b, contrast.frame_split(opts, f.ii, h if opts.horizontal else w),
                                      opts.horizontal)))
    return out


def splice_rule(a, b, triple, horizontal, color=BGR):
    """sy_splice_frames's per-pixel rule (the C header) on one pair"""
    split, start, end = triple
    c = (np.arange(a.shape[0])[:, None] if horizontal else np.arange(a.shape[1])[None, :]) + np.zeros(a.shape[:2], int)
    out = np.where((c >= split)[..., None], b, a)
    out[(c >= start) & (c < end)] = color
    return out


def check_written(out, run):
    """the files and directories under ``out`` against the script's run ``run``"""
    names = [str(v) for v in GOLD[run + ".files"]]
    got = sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs)
    assert got == names, run
    assert sorted(os.path.relpath(d, out) for d, _, _ in os.walk(out) if d != out) == [str(v) for v in GOLD[run + ".dirs"]]
    for rel in names:
        assert open(os.path.join(out, rel), "rb").read() == GOLD[f"{run}/{rel}"].tobytes(), (run, rel)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_inputs_decode_alike_in_cv2_and_pil():
    from PIL import Image
    n = 0
    for rel, b in inputs().items():
        if rel.endswith(".jpg"):
            assert np.array_equal(decode(b)[..., ::-1], np.array(Image.open(io.BytesIO(b)).convert("RGB"))), rel
            assert contrast.sof_size(b) == decode(b).shape[:2], rel
            n += 1
    assert n == 70


def _expected_frames(run):
    """(relative path, oracle file, split, l) of every frame the script's run ``run`` composed"""
    opts = contrast.parse_args(["--out-dir", "x"] + [str(v) for v in GOLD[run + ".argv"]])
    src = inputs()
    pre = {str(v) for v in GOLD[run + ".pre"]}
    out = []
    for rel in (str(v) for v in GOLD[run + ".files"]):
        if rel in pre:
            assert GOLD[f"{run}/{rel}"].tobytes() == b"kept"
            continue
        seq, name = rel.split("/")
        ii = sorted(k for k in src if k.startswith(f"A/{seq}/") and k.endswith(".jpg")).index(f"A/{seq}/{name}")
        a, b = decode(src[f"A/{rel}"]), decode(src[f"B/{rel}"])
        l = a.shape[0] if opts.horizontal else a.shape[1]
        split = co.split_at(ii, l, opts.split_pos, opts.split_animation, opts.fps)
        out.append((rel, encode(co.compose(a, b, split, opts.horizontal, BGR)), split, l))
    return out


def test_oracle_equals_the_script_files():
    splits = []
    for run in RUNS:
        for rel, want, split, l in _expected_frames(run):
            assert want == GOLD[f"{run}/{rel}"].tobytes(), (run, rel)
            splits.append((run, split, l))
    # every case of :148-165 is among them
    assert any(s <= 0 for _, s, _ in splits), "B alone"
    assert any(s >= l + 7 for _, s, l in splits), "A alone, no band"
    assert any(l <= s < l + 7 for _, s, l in splits), "A alone, part of the band"
    assert any(0 < s < 7 for _, s, l in splits) and any(l - 7 < s < l for _, s, l in splits), "band cut by an edge"
    assert any(-7 < s <= 0 for _, s, _ in splits), "B alone with the band's right part"
    assert any(7 <= s <= l - 7 for _, s, l in splits)
    assert ("default", 26, 53) in splits                     # 26.5 rounds half to even
    assert any(r == "swing_horizontal" and 0 < s < l for r, s, l in splits)


def test_swing_and_split_match_the_oracle():
    t = np.concatenate([np.linspace(-0.5, 16, 3301), [0, 4, 5, 8, 10, 13, 14, 4.5, 9.0, 13.5]])
    for l, pos in ((64, 32.0), (53, 26.5), (37, 20.0), (40, 40.0), (48, 55.0), (1, 0.5)):
        want = co.swing(t, pos, l)
        got = np.array([contrast.split_anime_swing(float(v), pos, l, contrast.LINE_WIDTH) for v in t], np.float64)
        assert np.array_equal(got, want), (l, pos)
    for argv in ([], ["--horizontal"], ["--split-pos", "1"], ["--split-pos", "20"], ["--split-pos", "0.05"],
                 ["--split-animation", "swing", "--fps", "3"], ["--split-animation", "swing", "--fps", "1.5"],
                 ["--split-pos", "1e12"], ["--split-pos", "-3"]):
        opts = contrast.parse_args(["--out-dir", "x"] + argv)
        for l in (1, 14, 37, 53, 64):
            for ii in range(0, 60, 1):
                s = co.split_at(ii, l, opts.split_pos, opts.split_animation, opts.fps)
                triple = contrast.frame_split(opts, ii, l)
                assert triple == contrast.splice_args(s, l)
                a = np.random.default_rng(ii).integers(0, 256, (3, l, 3), dtype=np.uint8)
                b = np.random.default_rng(ii + 99).integers(0, 256, (3, l, 3), dtype=np.uint8)
                assert np.array_equal(splice_rule(a, b, triple, False), co.compose(a, b, s, False, BGR)), (argv, l, ii)
                assert all(0 <= v <= l for v in triple)


def test_cli_emulated_writes_the_script_files(tmp_path, monkeypatch, capsys):
    a, b = setup_fixture(tmp_path)
    for run in RUNS:
        out = str(tmp_path / f"out_{run}")
        for rel in GOLD[run + ".pre"]:
            os.makedirs(os.path.dirname(os.path.join(out, str(rel))), exist_ok=True)
            open(os.path.join(out, str(rel)), "wb").write(b"kept")
        videos = []
        monkeypatch.setattr(contrast, "make_video", lambda d, fps: videos.append((os.path.relpath(d, out), str(fps))))
        n = contrast.run(run_opts(a, b, out, run), device_pass=emulated_pass)
        assert n == len(GOLD[run + ".files"]) - len(GOLD[run + ".pre"])
        check_written(out, run)
        assert capsys.readouterr().out == str(GOLD[run + ".printed"]).replace("<out-dir>", out), run
        assert videos == [tuple(str(x) for x in v) for v in GOLD[run + ".videos"]], run


def test_cli_overwrite_and_one_ffmpeg_argv(tmp_path, monkeypatch, capsys):
    a, b = setup_fixture(tmp_path)
    out = str(tmp_path / "out")
    calls = []
    never = lambda *x: calls.append(x)                      # noqa: E731
    contrast.run(run_opts(a, b, out, "swing"), device_pass=emulated_pass)
    p = os.path.join(out, "s1", "000004.jpg")
    open(p, "wb").write(b"kept")
    assert contrast.run(run_opts(a, b, out, "swing"), device_pass=never) == 0   # every frame exists: none is composed
    assert not calls and open(p, "rb").read() == b"kept"
    opts = run_opts(a, b, out, "swing")
    opts.overwrite = True
    assert contrast.run(opts, device_pass=emulated_pass) == 35
    check_written(out, "swing")
    capsys.readouterr()
    runs = []
    monkeypatch.setattr(vis.subprocess, "run", lambda argv, **kw: runs.append((argv, kw)))
    opts.make_video, opts.fps = True, 25.0
    contrast.run(opts, device_pass=emulated_pass)
    assert capsys.readouterr().out.splitlines()[-1] == "Making the video"
    d = os.path.join(out, "s2")                              # the last sequence only, as the script's indentation does
    assert runs == [(["ffmpeg", "-loglevel", "panic", "-y", "-framerate", "25.0", "-i", os.path.join(d, "%06d.jpg"),
                      "-c:v", "libx264", "-pix_fmt", "yuv420p", "-vf", "pad=width=ceil(iw/2)*2:height=ceil(ih/2)*2",
                      d + ".mp4"], {"check": True})]
    open(d + ".mp4", "wb").close()                           # an existing video is kept without --overwrite
    opts.overwrite = False
    contrast.run(opts, device_pass=emulated_pass)
    assert len(runs) == 1 and "Making the video" not in capsys.readouterr().out


def test_cli_refusals(tmp_path):
    a, b = setup_fixture(tmp_path)
    out = str(tmp_path / "out")
    never = lambda *x: pytest.fail("the device pass ran")   # noqa: E731
    opts = run_opts(a, b, out, "default")
    opts.split_animation = "zoom"
    with pytest.raises(KeyError, match="split_anime_zoom"):
        contrast.run(opts, device_pass=never)
    assert not os.path.exists(out)
    missing = os.path.join(b, "s1", "000005.jpg")
    os.rename(missing, missing + ".bak")
    with pytest.raises(FileNotFoundError, match=re.escape(missing)):
        contrast.run(run_opts(a, b, out, "edge_seq_name"), device_pass=emulated_pass)
    assert os.listdir(os.path.join(out, "s1")) == []         # refused before the sequence's first file
    os.rename(missing + ".bak", missing)
    other = os.path.join(b, "s1", "000003.jpg")
    open(other, "wb").write(GOLD["in/B/s1/000002.jpg"].tobytes())      # 24 x 40 where A's is 37 x 53
    with pytest.raises(ValueError, match=re.escape(os.path.join(a, "s1", "000003.jpg")) + ".*37x53.*" +
                       re.escape(other) + ".*24x40"):
        contrast.run(run_opts(a, b, out, "edge_seq_name"), device_pass=emulated_pass)
    open(other, "wb").write(b"\xff\xd8\xff\xe0\x00")        # no SOF header
    with pytest.raises(RuntimeError, match=re.escape(other) + ".*did not decode"):
        contrast.run(run_opts(a, b, out, "edge_seq_name"), device_pass=emulated_pass)


def test_sof_size():
    src = inputs()
    b = src["A/s1/000002.jpg"]
    assert contrast.sof_size(b) == (24, 40)
    # APPn and COM segments and fill bytes before the SOF, and progressive SOF2
    extra = b"\xff\xe1\x00\x06Exif\xff\xfe\x00\x04hi\xff\xff"
    assert contrast.sof_size(b[:2] + extra + b[2:]) == (24, 40)
    k = b.index(b"\xff\xc0")
    assert contrast.sof_size(b[:k + 1] + b"\xc2" + b[k + 2:]) == (24, 40)
    for bad in (b"", b"\xff\xd8", b"\x00\xd8\xff\xc0", b[:k + 6], b[:k], b"GIF89a" + b[6:]):
        assert contrast.sof_size(bad) is None


def test_refusals_without_a_device():
    lib = ops.load_library()
    good = dict(a=0x1000, b=0x9000, sizes=0x2000, splits=0x3000, n=2, max_h=16, max_w=24, horizontal=0)
    for kw in (dict(a=None), dict(b=None), dict(sizes=None), dict(splits=None), dict(b=0x1000), dict(n=0),
               dict(n=65536), dict(max_h=0), dict(max_w=70000), dict(horizontal=2), dict(horizontal=-1)):
        d = ops.SySpliceFramesDesc(**dict(good, **kw))
        assert lib.sy_splice_frames(C.byref(d), None) == 1, kw              # SY_EINVAL, before any launch


def test_contrast_cu_compiles_without_spills():
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc not available")
    cmd = [build.NVCC] + build.COMMON + build.SOURCES["contrast.cu"] + ["-c", os.path.join(build.CSRC, "contrast.cu"),
                                                                        "-o", os.devnull]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == 1 and props[0] == ("0", "0", "0"), r.stderr


# ---------------------------------------------------------------------------------------------------------------- GPU
DEV = "cuda"
POISON = 0xA7


def _pairs(rng):
    """mixed sizes: widths on and off 16-pixel runs, a 1 x 1 frame, one of slot size"""
    sizes = [(37, 53), (48, 64), (1, 1), (70, 130), (24, 40), (33, 97), (70, 130), (5, 200)]
    a = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    b = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    return sizes, a, b


def _slots(imgs, mh, mw):
    s = np.full((len(imgs), mh, mw, 3), POISON, np.uint8)
    for k, i in enumerate(imgs):
        s[k, :i.shape[0], :i.shape[1]] = i
    return torch.from_numpy(s).to(DEV)


@pytest.mark.gpu
def test_gpu_splice_equals_the_oracle():
    rng = np.random.default_rng(5)
    sizes, a, b = _pairs(rng)
    for mh, mw in ((80, 208), (71, 201)):                   # 16-byte aligned rows, and rows that are not
        for horizontal in (False, True):
            for trial in range(6):
                splits, raw = [], []
                for h, w in sizes:
                    l = h if horizontal else w
                    s = int(rng.choice([-20, -8, -7, -1, 0, 1, 3, l // 2, l - 3, l, l + 6, l + 7, l + 30,
                                        int(rng.integers(-10, l + 10))]))
                    raw.append(s)
                    splits.append(contrast.splice_args(s, l))
                ta, tb = _slots(a, mh, mw), _slots(b, mh, mw)
                if trial % 2:                                # B at an odd offset in a larger buffer, as the CLI's
                    buf = torch.empty(tb.numel() + 2 * trial + 1, dtype=torch.uint8, device=DEV)   # decode output
                    tb = buf[2 * trial + 1:].view(tb.shape).copy_(tb)
                keep_b = tb.clone()
                got = data.splice_frames(ta, tb, splits, sizes, horizontal)
                assert got.data_ptr() == ta.data_ptr() and torch.equal(tb, keep_b)
                host = got.cpu().numpy()
                for k, (h, w) in enumerate(sizes):
                    want = co.compose(a[k], b[k], raw[k], horizontal, BGR)
                    assert np.array_equal(host[k, :h, :w], want), (mh, mw, horizontal, trial, k, raw[k])
                    assert (host[k, h:] == POISON).all() and (host[k, :, w:] == POISON).all(), (k, "poison")


@pytest.mark.gpu
def test_gpu_graph_replays_repeat_and_follow_splits():
    rng = np.random.default_rng(6)
    sizes, a, b = _pairs(rng)
    mh, mw = 80, 208
    src_a, tb = _slots(a, mh, mw), _slots(b, mh, mw)
    ta = src_a.clone()
    s_t = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    sp_t = torch.zeros((len(sizes), 3), dtype=torch.int32, device=DEV)
    data.splice_frames(ta, tb, sp_t, s_t)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ta.copy_(src_a)
        data.splice_frames(ta, tb, sp_t, s_t)
    for t in range(3):
        raw = [int(rng.integers(-10, w + 10)) for _, w in sizes]
        sp_t.copy_(torch.tensor([contrast.splice_args(s, w) for s, (_, w) in zip(raw, sizes)], dtype=torch.int32))
        g.replay()
        first = ta.cpu().numpy()
        g.replay()
        assert np.array_equal(ta.cpu().numpy(), first), t
        for k, (h, w) in enumerate(sizes):
            assert np.array_equal(first[k, :h, :w], co.compose(a[k], b[k], raw[k], False, BGR)), (t, k)
            assert (first[k, h:] == POISON).all() and (first[k, :, w:] == POISON).all()


@pytest.mark.gpu
def test_gpu_cli_writes_the_script_files(tmp_path, monkeypatch, capsys):
    a, b = setup_fixture(tmp_path)
    monkeypatch.setattr(contrast, "make_video", lambda d, fps: None)
    for run in RUNS:
        out = str(tmp_path / f"out_{run}")
        for rel in GOLD[run + ".pre"]:
            os.makedirs(os.path.dirname(os.path.join(out, str(rel))), exist_ok=True)
            open(os.path.join(out, str(rel)), "wb").write(b"kept")
        assert contrast.run(run_opts(a, b, out, run)) == len(GOLD[run + ".files"]) - len(GOLD[run + ".pre"])
        check_written(out, run)
        assert capsys.readouterr().out == str(GOLD[run + ".printed"]).replace("<out-dir>", out), run


@pytest.mark.gpu
def test_gpu_cli_names_a_file_that_does_not_decode(tmp_path):
    a, b = setup_fixture(tmp_path)
    p = os.path.join(b, "s0", "000011.jpg")
    f = open(p, "rb").read()
    open(p, "wb").write(f[:f.index(b"\xff\xda")])           # headers only: the size is read, the scan is missing
    with pytest.raises(RuntimeError, match=re.escape(p) + ".*did not decode"):
        contrast.run(run_opts(a, b, str(tmp_path / "out"), "default"))
