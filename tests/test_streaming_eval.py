"""``python -m streamyolo_b200.streaming_eval`` against the unmodified sAP/det/streaming_eval.py
(tests/golden/streaming_eval_script.npz, oracle/make_streaming_eval_golden.py), and its kernels sy_draw_outlines and
sy_resize_sized against numpy and cv2.

CPU: the command's host half with the device pass emulated (tests/emul_streaming_eval.py) writes the script's pickles,
frames and printed lines byte for byte; the boxes and label pixels it sends to the device equal what cv2.rectangle and
cv2.putText draw in vis_det; the label-pixel scan equals a scan of the whole canvas; arguments, --overwrite, the
out-dir default, the refusals and the call of the toolkit's eval_ccf.
GPU: the kernels against the numpy restatement and cv2 over mixed sizes in sentinel-filled slots, inside a CUDA graph
too; the emulation against the kernels; and the command itself, byte for byte, at --vis-scale 1 and 0.5."""
import hashlib
import importlib
import io
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from streamyolo_b200 import data, ops
from streamyolo_b200 import streaming_eval as se

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_streaming_eval as emul                                  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "streaming_eval_script.npz"))
FULL_JPG = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_full_f420_q90.npz"))["jpg"].tobytes()
DATASET = json.loads(GOLD["annot"].tobytes().decode())
RUNS = ("raw", "parsed", "nomap")
FULL_SEQ = "s2"


def _cv2():
    return pytest.importorskip("cv2")


def setup_fixture(tmp_path):
    """the fixture's frames, annotation file and pickles under tmp_path -> (data root, annotation path, result dir)"""
    root = tmp_path / "data"
    for k in GOLD.files:
        if k.startswith("in/"):
            p = root / k[3:]
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_bytes(GOLD[k].tobytes())
    (root / "d2").mkdir(parents=True, exist_ok=True)
    (root / "d2" / "000000.jpg").write_bytes(FULL_JPG)
    annot, res = tmp_path / "annot.json", tmp_path / "res"
    annot.write_text(json.dumps(DATASET))
    res.mkdir()
    for k in GOLD.files:
        if k.startswith("pkl/"):
            (res / (k[4:] + ".pkl")).write_bytes(GOLD[k].tobytes())
    return str(root), str(annot), str(res)


def run_argv(run, root, annot, res, vis_dir, out_dir):
    extra = [str(v) for v in GOLD[run + ".argv"]]
    if extra and extra[-1] == "--out-dir":
        extra = extra[:-1] + ["--out-dir", out_dir]
    return ["--data-root", root, "--annot-path", annot, "--fps", str(int(GOLD["fps"])), "--result-dir", res,
            "--vis-dir", vis_dir, "--no-eval"] + extra


def out_of(run, res, out_dir):
    return out_dir if "--out-dir" in [str(v) for v in GOLD[run + ".argv"]] else res


def check_outputs(run, res, vis_dir, out_dir, full=True):
    """the pickles and the files under vis_dir against the script's run ``run``"""
    d = out_of(run, res, out_dir)
    for name in ("results_ccf.pkl", "eval_assoc.pkl"):
        assert open(os.path.join(d, name), "rb").read() == GOLD[f"{run}.{name}"].tobytes(), (run, name)
    names = [str(v) for v in GOLD[run + ".files"]]
    for rel in names:
        if rel.startswith(FULL_SEQ) and not full:
            continue
        b = open(os.path.join(vis_dir, rel), "rb").read()
        if rel.startswith(FULL_SEQ):
            assert len(b) == int(GOLD[f"{run}/{rel}.len"]) and hashlib.sha256(b).digest() == \
                GOLD[f"{run}/{rel}.sha256"].tobytes(), (run, rel)
        else:
            assert b == GOLD[f"{run}/{rel}"].tobytes(), (run, rel)
    got = sorted(os.path.relpath(os.path.join(p, f), vis_dir) for p, _, fs in os.walk(vis_dir) for f in fs)
    assert got == sorted(names)


def printed_of(run, vis_dir, text):
    return text.replace(vis_dir, "<vis-dir>") == str(GOLD[run + ".printed"])


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("run", RUNS)
def test_emulated_pass_writes_the_script_files(tmp_path, capsys, run):
    _cv2()
    pytest.importorskip("PIL")
    root, annot, res = setup_fixture(tmp_path)
    vis_dir, out_dir = str(tmp_path / "vis"), str(tmp_path / "out")
    se.run(se.parse_args(run_argv(run, root, annot, res, vis_dir, out_dir)), device_pass=emul.device_pass)
    check_outputs(run, res, vis_dir, out_dir)
    assert printed_of(run, vis_dir, capsys.readouterr().out)


def _decoded(run, rel):
    from PIL import Image
    seq = rel.split("/")[0]
    sid = DATASET["sequences"].index(seq)
    src = FULL_JPG if seq == FULL_SEQ else GOLD[f"in/{DATASET['seq_dirs'][sid]}/{rel.split('/')[1]}"].tobytes()
    return np.array(Image.open(io.BytesIO(src)))


@pytest.mark.parametrize("run", RUNS)
def test_boxes_and_label_pixels_equal_what_vis_det_draws(tmp_path, run):
    """every frame: the green pixels of the host's boxes and label pixels, drawn by the numpy restatement, equal those
    of cv2.rectangle and cv2.putText as vis_det calls them on the rows the pairing gave the frame"""
    cv2 = _cv2()
    pytest.importorskip("PIL")
    root, annot, res = setup_fixture(tmp_path)
    opts = se.parse_args(run_argv(run, root, annot, res, str(tmp_path / "vis"), str(tmp_path / "out")))
    imgs = {img["id"]: img for img in DATASET["images"]}
    p = se.pair(opts, DATASET, imgs)
    assert len(p.frames) == len(GOLD[run + ".files"])
    drawn = 0
    for f in p.frames:
        rel = os.path.relpath(f.out, opts.vis_dir)
        img = _decoded(run, rel)
        if opts.vis_scale != 1:
            h, w = data.imrescale_size(img.shape[0], img.shape[1], opts.vis_scale)
            img = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)
        se.render(f, opts.vis_scale)
        assert f.out_hw == img.shape[:2]
        ref = img.copy()
        for (x1, y1, x2, y2), (text, org) in zip(f.boxes, f.texts):
            cv2.rectangle(ref, (x1, y1), (x2, y2), (0, 255, 0), thickness=1)
            cv2.putText(ref, text, org, cv2.FONT_HERSHEY_COMPLEX, 0.5, (0, 255, 0))
        got = img.copy()
        m = emul.outline_mask(*img.shape[:2], f.boxes)
        m.reshape(-1)[f.points] = True
        got[m] = (0, 255, 0)
        assert np.array_equal(got, ref), rel
        drawn += len(f.boxes)
    assert drawn > 30


def test_fixture_covers_the_cases(tmp_path):
    """misses, empty frames, every border crossed, labels clipped at the top and left, both scales"""
    root, annot, res = setup_fixture(tmp_path)
    seen = set()
    for run in RUNS:
        opts = se.parse_args(run_argv(run, root, annot, res, str(tmp_path / "vis"), str(tmp_path / "out")))
        p = se.pair(opts, DATASET, {img["id"]: img for img in DATASET["images"]})
        assert p.miss > 0
        seen.add(("scale", opts.vis_scale))
        for f in p.frames:
            se.render(f, opts.vis_scale)
            h, w = f.out_hw
            if not len(f.boxes):
                seen.add("empty")
                continue
            b = np.asarray(f.boxes, np.int64)
            lo, hi = b[:, [0, 2]].min(1), b[:, [0, 2]].max(1)
            seen |= {k for k, c in (("left", (lo < 0) & (hi >= 0)), ("right", (lo < w) & (hi >= w))) if c.any()}
            lo, hi = b[:, [1, 3]].min(1), b[:, [1, 3]].max(1)
            seen |= {k for k, c in (("top", (lo < 0) & (hi >= 0)), ("bottom", (lo < h) & (hi >= h))) if c.any()}
            seen |= {"text_top" for _, (x, y) in f.texts if 0 <= y < 11}
            seen |= {"text_left" for _, (x, y) in f.texts if -40 < x < 0}
            seen |= {"zero_size" for x1, y1, x2, y2 in b if x1 == x2 and y1 == y2}
            seen |= {"reversed" for x1, y1, x2, y2 in b if x1 > x2 or y1 > y2}
    assert seen >= {("scale", 1.0), ("scale", 0.5), "empty", "left", "right", "top", "bottom", "text_top", "text_left",
                    "zero_size", "reversed"}, seen


def test_text_scan_equals_the_whole_canvas():
    """the label pixels found in the text boxes equal a scan of a whole fresh canvas, and the canvas is left clear"""
    cv2 = _cv2()
    rng = np.random.default_rng(3)
    alphabet = [chr(c) for c in range(32, 127)]
    for trial in range(200):
        h, w = int(rng.integers(8, 90)), int(rng.integers(8, 160))
        texts = []
        for _ in range(int(rng.integers(1, 6))):
            s = "".join(rng.choice(alphabet, int(rng.integers(1, 12))))
            texts.append((s, (np.int32(rng.integers(-60, w + 5)), np.int32(rng.integers(-10, h + 15)))))
        got = se.text_points(texts, (h, w))
        ref = np.zeros((h, w), np.uint8)
        for s, org in texts:
            cv2.putText(ref, s, org, cv2.FONT_HERSHEY_COMPLEX, 0.5, 255)
        assert np.array_equal(got, np.flatnonzero(ref).astype(np.int32)), (trial, texts)
        assert not se._canvases.__dict__[(h, w)].any()


def test_imrescale_size_is_mmcv_rescale_size():
    for h, w, s in ((120, 192, 0.5), (75, 131, 0.5), (1200, 1920, 0.5), (75, 131, 0.37), (7, 9, 1.7), (1, 1, 0.6)):
        assert data.imrescale_size(h, w, s) == (int(h * s + 0.5), int(w * s + 0.5))
    for s in (0, -0.5):
        with pytest.raises(ValueError, match="must be positive"):
            data.imrescale_size(10, 10, s)
    with pytest.raises(ValueError, match="empty"):
        data.imrescale_size(3, 300, 0.1)


def test_arguments_are_the_scripts():
    o = se.parse_args(["--data-root", "d", "--annot-path", "a", "--result-dir", "r"])
    assert (o.fps, o.eta, o.out_dir, o.vis_dir, o.vis_scale) == (30, 0, None, None, 1)
    assert not (o.no_class_mapping or o.no_eval or o.use_parsed or o.eval_mask or o.overwrite)
    with pytest.raises(SystemExit):
        se.parse_args(["--data-root", "d", "--annot-path", "a"])


def test_existing_files_are_kept_without_overwrite(tmp_path, capsys):
    _cv2()
    pytest.importorskip("PIL")
    root, annot, res = setup_fixture(tmp_path)
    vis_dir, out_dir = str(tmp_path / "vis"), str(tmp_path / "out")
    argv = run_argv("nomap", root, annot, res, vis_dir, out_dir)
    se.run(se.parse_args(argv), device_pass=emul.device_pass)
    keep = [os.path.join(vis_dir, "s0", "000003.jpg"), os.path.join(out_dir, "eval_assoc.pkl")]
    for k in keep:
        with open(k, "wb") as f:
            f.write(b"kept")
    calls = []

    def counting(files, frames, scale):
        calls.extend(f.out for f in frames)
        return emul.device_pass(files, frames, scale)
    se.run(se.parse_args(argv), device_pass=counting)
    assert calls == [] and all(open(k, "rb").read() == b"kept" for k in keep)
    os.remove(keep[0])
    se.run(se.parse_args(argv), device_pass=counting)
    assert calls == [keep[0]] and open(keep[1], "rb").read() == b"kept"
    se.run(se.parse_args(argv + ["--overwrite"]), device_pass=counting)
    assert len(calls) == 1 + len(GOLD["nomap.files"])
    check_outputs("nomap", res, vis_dir, out_dir)


def test_without_vis_dir_no_device_and_no_cv2(tmp_path, capsys, monkeypatch):
    root, annot, res = setup_fixture(tmp_path)
    monkeypatch.setitem(sys.modules, "cv2", None)                  # the pairing needs no cv2

    def no_device(*a):
        raise AssertionError("no frame is drawn without --vis-dir")
    se.run(se.parse_args(["--data-root", root, "--annot-path", annot, "--fps", "30", "--result-dir", res, "--no-eval"]),
           device_pass=no_device)
    assert open(os.path.join(res, "results_ccf.pkl"), "rb").read() == GOLD["raw.results_ccf.pkl"].tobytes()
    assert capsys.readouterr().out == "Pairing the output with the ground truth\n"
    with pytest.raises(RuntimeError, match="cv2"):
        se.run(se.parse_args(["--data-root", root, "--annot-path", annot, "--result-dir", res, "--no-eval",
                              "--vis-dir", str(tmp_path / "v")]), device_pass=no_device)


def _rewrite_pickle(res, seq, fn):
    path = os.path.join(res, seq + ".pkl")
    d = pickle.load(open(path, "rb"))
    fn(d)
    pickle.dump(d, open(path, "wb"))


def _nothing_written(tmp_path, out_dir):
    assert not os.path.exists(tmp_path / "vis") and not os.path.exists(out_dir)


def test_refusals_before_anything_is_written(tmp_path):
    root, annot, res = setup_fixture(tmp_path)
    vis_dir, out_dir = str(tmp_path / "vis"), str(tmp_path / "out")

    def no_device(*a):
        raise AssertionError("refused before the device")
    argv = run_argv("parsed", root, annot, res, vis_dir, out_dir)
    pytest.importorskip("cv2")
    for scale in ("0", "-0.5"):
        with pytest.raises(ValueError, match="must be positive"):
            se.run(se.parse_args(argv + ["--vis-scale", scale]), device_pass=no_device)
        _nothing_written(tmp_path, out_dir)

    def masks(d):
        b, s, lab, _ = d["results_parsed"][-1]
        d["results_parsed"][-1] = (b, s, lab, [{"size": [1, 1], "counts": b"0"}] * len(b))
    _rewrite_pickle(res, "s1", masks)
    with pytest.raises(NotImplementedError, match="masks"):
        se.run(se.parse_args(argv), device_pass=no_device)
    _nothing_written(tmp_path, out_dir)

    root, annot, res = setup_fixture(tmp_path / "t")

    def tracks(d):
        d["results_parsed"][0] = (*d["results_parsed"][0], np.arange(len(d["results_parsed"][0][0]), dtype=np.uint32))
    _rewrite_pickle(res, "s0", tracks)
    with pytest.raises(NotImplementedError, match="tracks"):
        se.run(se.parse_args(run_argv("parsed", root, annot, res, vis_dir, out_dir)), device_pass=no_device)
    _nothing_written(tmp_path, out_dir)

    root, annot, res = setup_fixture(tmp_path / "l")

    def bad_label(d):
        b, lab = d["results_raw"][0]
        d["results_raw"][0] = (b, np.full_like(lab, 8))
    _rewrite_pickle(res, "s0", bad_label)
    with pytest.raises(IndexError):                                # class_names[label], as vis_det raises
        se.run(se.parse_args(run_argv("nomap", root, annot, res, vis_dir, out_dir)), device_pass=no_device)
    _nothing_written(tmp_path, out_dir)

    root, annot, res = setup_fixture(tmp_path / "f")
    os.remove(os.path.join(root, "d1", "000004.jpg"))
    with pytest.raises(FileNotFoundError, match="000004.jpg"):
        se.run(se.parse_args(run_argv("raw", root, annot, res, vis_dir, out_dir)), device_pass=no_device)
    _nothing_written(tmp_path, out_dir)

    open(os.path.join(root, "d1", "000004.jpg"), "wb").write(GOLD["in/d1/000004.jpg"].tobytes())
    os.remove(os.path.join(res, "s3.pkl"))
    with pytest.raises(FileNotFoundError, match="s3.pkl"):
        se.run(se.parse_args(run_argv("raw", root, annot, res, vis_dir, out_dir)), device_pass=no_device)


def test_tracks_and_masks_pass_through_without_vis_dir(tmp_path):
    """without --vis-dir the script pairs such rows; masks go into 'segmentation'"""
    root, annot, res = setup_fixture(tmp_path)

    def both(d):
        b, s, lab, _ = d["results_parsed"][0]
        d["results_parsed"][0] = (b, s, lab, [f"m{i}" for i in range(len(b))], np.arange(len(b), dtype=np.uint32))
    _rewrite_pickle(res, "s0", both)
    p = se.run(se.parse_args(["--data-root", root, "--annot-path", annot, "--result-dir", res, "--no-eval",
                              "--use-parsed", "--eta", "-1"]))
    assert any(r.get("segmentation") == "m0" for r in p.results_ccf)


def test_eval_ccf_gets_the_scripts_results(tmp_path, monkeypatch, capsys):
    root, annot, res = setup_fixture(tmp_path)
    seen = []

    class FakeCOCO:
        def __init__(self, path):
            with open(path) as f:
                self.dataset = json.load(f)
            self.imgs = {img["id"]: img for img in self.dataset["images"]}

    def eval_ccf(db, results, class_subset=None, iou_type="bbox"):
        assert isinstance(db, FakeCOCO)
        seen.append((iou_type, pickle.dumps(results)))
        return {"stats": np.arange(12, dtype=np.float64) + len(seen), "iou_type": iou_type}
    monkeypatch.setattr(se, "toolkit", lambda: (eval_ccf, FakeCOCO))
    out_dir = str(tmp_path / "out")
    argv = ["--data-root", root, "--annot-path", annot, "--fps", "30", "--result-dir", res, "--out-dir", out_dir]
    se.run(se.parse_args(argv))
    assert seen == [("bbox", GOLD["raw.results_ccf.pkl"].tobytes())]
    s = pickle.load(open(os.path.join(out_dir, "eval_summary.pkl"), "rb"))
    assert s["iou_type"] == "bbox" and s["stats"][0] == 1
    assert not os.path.exists(os.path.join(out_dir, "eval_summary_mask.pkl"))
    capsys.readouterr()
    se.run(se.parse_args(argv + ["--eval-mask"]))
    assert [t for t, _ in seen] == ["bbox", "bbox", "segm"]
    assert pickle.load(open(os.path.join(out_dir, "eval_summary.pkl"), "rb"))["stats"][0] == 1    # kept
    assert pickle.load(open(os.path.join(out_dir, "eval_summary_mask.pkl"), "rb"))["iou_type"] == "segm"
    assert capsys.readouterr().out == "Pairing the output with the ground truth\nEvaluating instance segmentation\n"


def test_toolkit_is_found_from_the_sap_directory(tmp_path, monkeypatch):
    sap = tmp_path / "sAP"
    (sap / "det").mkdir(parents=True)
    (sap / "det" / "__init__.py").write_text("def eval_ccf(db, results, class_subset=None, iou_type='bbox'):\n"
                                             "    return 'toolkit'\n")
    pc = tmp_path / "site" / "pycocotools"
    pc.mkdir(parents=True)
    (pc / "__init__.py").write_text("")
    (pc / "coco.py").write_text("class COCO:\n    pass\n")
    monkeypatch.chdir(sap)
    monkeypatch.setattr(sys, "path", [str(tmp_path / "site")] + sys.path)
    for m in ("det", "pycocotools", "pycocotools.coco"):
        monkeypatch.delitem(sys.modules, m, raising=False)
    eval_ccf, COCO = se.toolkit()
    assert eval_ccf(None, []) == "toolkit" and COCO.__module__ == "pycocotools.coco"
    for m in ("det", "pycocotools", "pycocotools.coco"):
        monkeypatch.delitem(sys.modules, m, raising=False)
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(sys, "path", [p for p in sys.path if p not in ("..", ".")])
    importlib.invalidate_caches()                                   # "." named the sAP directory a moment ago
    with pytest.raises(RuntimeError, match="--no-eval"):
        se.toolkit()


def test_new_kernels_compile_without_spills():
    import re
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc not available")
    for src, kernel in (("vis_det.cu", "draw_outlines_kernel"), ("input.cu", "resize_sized_kernel")):
        cmd = [build.NVCC] + build.COMMON + build.SOURCES[src] + ["-c", os.path.join(build.CSRC, src), "-o", os.devnull]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        m = re.search(kernel + r".*?\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                      r.stderr)
        assert m and m.groups() == ("0", "0", "0"), r.stderr


def test_c_entries_refuse_bad_descriptors():
    lib = ops.load_library()
    d = ops.SyDrawOutlinesDesc()
    assert lib.sy_draw_outlines(C_byref(d), None) != 0
    r = ops.SyResizeSizedDesc()
    assert lib.sy_resize_sized(C_byref(r), None) != 0


def C_byref(d):
    import ctypes
    return ctypes.byref(d)


# ---------------------------------------------------------------------------------------------------------------- GPU
DEV = "cuda"
SENTINEL = 0x5A


def _random_frames(rng, sizes):
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]


def _slots(imgs, hw=None):
    mh = max(i.shape[0] for i in imgs) if hw is None else hw[0]
    mw = max(i.shape[1] for i in imgs) if hw is None else hw[1]
    s = np.full((len(imgs), mh, mw, 3), SENTINEL, np.uint8)
    for k, i in enumerate(imgs):
        s[k, :i.shape[0], :i.shape[1]] = i
    return s


def _boxes(rng, h, w, n):
    big = np.iinfo(np.int32)
    b = np.stack([rng.integers(-w // 2, w + w // 2, n), rng.integers(-h // 2, h + h // 2, n),
                  rng.integers(-w // 2, w + w // 2, n), rng.integers(-h // 2, h + h // 2, n)], 1)
    extra = [(5, 5, 5, 5), (w - 1, h - 1, w - 1, h - 1), (-3, -3, -1, -1), (w, 0, w + 3, h), (10, 20, 2, 3),
             (big.min, big.min, big.max, big.max), (-5, h - 1, w + 5, h - 1), (0, -7, 0, h + 7)]
    return np.concatenate([b, np.asarray(extra)]).astype(np.int32)


def _expected(imgs, boxes, points, hw=None, color=(0, 255, 0)):
    want = _slots(imgs, hw)
    for k, (img, b, p) in enumerate(zip(imgs, boxes, points)):
        h, w = img.shape[:2]
        m = emul.outline_mask(h, w, b)
        q = np.asarray(p, np.int64)
        m.reshape(-1)[q[(q >= 0) & (q < h * w)]] = True
        want[k, :h, :w][m] = color
    return want


@pytest.mark.gpu
def test_gpu_draw_outlines_equals_the_restatement():
    rng = np.random.default_rng(5)
    sizes = [(120, 192), (75, 131), (1, 1), (33, 7), (600, 960)]
    imgs = _random_frames(rng, sizes)
    boxes = [_boxes(rng, h, w, int(rng.integers(0, 40))) for h, w in sizes]
    boxes[2] = boxes[2][:0]                                         # a frame without boxes
    points = [np.concatenate([rng.integers(0, h * w, int(rng.integers(0, 500))), [-1, h * w, h * w + 7]]).astype(np.int32)
              for h, w in sizes]
    slots = torch.from_numpy(_slots(imgs)).to(DEV)
    data.draw_outlines(slots, boxes, points, sizes)
    assert np.array_equal(slots.cpu().numpy(), _expected(imgs, boxes, points))
    # BGR order, another colour, frames filling the slot
    one = torch.from_numpy(_slots(imgs[:1])).to(DEV)
    data.draw_outlines(one, boxes[:1], points[:1], color=(7, 8, 9))
    assert np.array_equal(one.cpu().numpy(), _expected(imgs[:1], boxes[:1], points[:1], color=(7, 8, 9)))


@pytest.mark.gpu
def test_gpu_draw_outlines_graph_follows_rewritten_boxes():
    rng = np.random.default_rng(9)
    sizes = [(120, 192), (75, 131)]
    imgs = _random_frames(rng, sizes)
    K, M = 48, 600
    base = torch.from_numpy(_slots(imgs)).to(DEV)
    frames = base.clone()
    t_boxes = torch.zeros((2, K, 4), dtype=torch.int32, device=DEV)
    t_counts = torch.zeros(2, dtype=torch.int32, device=DEV)
    t_points = torch.zeros((2, M), dtype=torch.int32, device=DEV)
    t_np = torch.zeros(2, dtype=torch.int32, device=DEV)
    t_sizes = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    data.draw_outlines(frames, t_boxes, t_points, t_sizes, t_counts, t_np)          # warm up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        data.draw_outlines(frames, t_boxes, t_points, t_sizes, t_counts, t_np)
    for trial in range(3):
        boxes = [_boxes(rng, h, w, int(rng.integers(1, K - 8)))[:K] for h, w in sizes]
        points = [rng.integers(-5, h * w + 5, int(rng.integers(0, M))).astype(np.int32) for h, w in sizes]
        frames.copy_(base)
        t_boxes.zero_()
        t_points.zero_()
        for k in range(2):
            t_boxes[k, :len(boxes[k])] = torch.from_numpy(boxes[k])
            t_points[k, :len(points[k])] = torch.from_numpy(points[k])
        t_counts.copy_(torch.tensor([len(b) for b in boxes], dtype=torch.int32))
        t_np.copy_(torch.tensor([len(p) for p in points], dtype=torch.int32))
        g.replay()
        assert np.array_equal(frames.cpu().numpy(), _expected(imgs, boxes, points)), trial


@pytest.mark.gpu
def test_gpu_resize_sized_equals_cv2():
    cv2 = _cv2()
    rng = np.random.default_rng(13)
    sizes = [(120, 192), (75, 131), (1200, 1920), (9, 5), (31, 47)]
    imgs = _random_frames(rng, sizes)
    for scale in (0.5, 0.37, 1.3, 1):
        dst = [data.imrescale_size(h, w, scale) for h, w in sizes]
        src = torch.from_numpy(_slots(imgs)).to(DEV)
        oh, ow = max(h for h, _ in dst) + 3, max(w for _, w in dst) + 5
        out = torch.full((len(imgs), oh, ow, 3), SENTINEL, dtype=torch.uint8, device=DEV)
        data.resize_sized(src, sizes, dst, out=out)
        want = _slots([cv2.resize(i, (w, h), interpolation=cv2.INTER_LINEAR) for i, (h, w) in zip(imgs, dst)], (oh, ow))
        assert np.array_equal(out.cpu().numpy(), want), scale


@pytest.mark.gpu
def test_gpu_emulation_conforms_to_the_kernels():
    """emul_streaming_eval's draw_outlines and resize_sized write what the kernels write, element for element"""
    rng = np.random.default_rng(21)
    sizes = [(120, 192), (75, 131), (40, 40)]
    imgs = _random_frames(rng, sizes)
    sl = _slots(imgs, (130, 200))
    boxes = np.zeros((3, 20, 4), np.int32)
    points = rng.integers(-10, 130 * 200, (3, 300)).astype(np.int32)
    for k, (h, w) in enumerate(sizes):
        boxes[k] = _boxes(rng, h, w, 12)[:20]
    counts = np.array([20, 0, 25], np.int32)                        # clamped to [0, K]
    n_points = np.array([300, -1, 150], np.int32)
    tsz = np.array(sizes + [], np.int32)
    args = [torch.from_numpy(v) for v in (tsz, boxes, counts, points, n_points)]
    lib_img = torch.from_numpy(sl.copy()).to(DEV)
    ops.draw_outlines(lib_img, *[a.to(DEV) for a in args], (0, 255, 0))
    em_img = torch.from_numpy(sl.copy())
    emul.draw_outlines(em_img, *args, (0, 255, 0))
    assert torch.equal(lib_img.cpu(), em_img)
    table = torch.tensor([[120, 192, 60, 96], [75, 131, 38, 66], [40, 40, 90, 77]], dtype=torch.int32)
    out_lib = torch.full((3, 100, 110, 3), SENTINEL, dtype=torch.uint8, device=DEV)
    ops.resize_sized(torch.from_numpy(sl).to(DEV), table.to(DEV), out_lib)
    out_em = torch.full((3, 100, 110, 3), SENTINEL, dtype=torch.uint8)
    emul.resize_sized(torch.from_numpy(sl), table, out_em)
    assert torch.equal(out_lib.cpu(), out_em)


@pytest.mark.gpu
@pytest.mark.parametrize("run", RUNS)
def test_gpu_command_writes_the_script_files(tmp_path, run):
    _cv2()
    root, annot, res = setup_fixture(tmp_path)
    vis_dir, out_dir = str(tmp_path / "vis"), str(tmp_path / "out")
    r = subprocess.run([sys.executable, "-m", "streamyolo_b200.streaming_eval"]
                       + run_argv(run, root, annot, res, vis_dir, out_dir), cwd=ROOT, capture_output=True, text=True,
                       env={**os.environ, "PYTHONPATH": ROOT})
    assert r.returncode == 0, r.stderr
    check_outputs(run, res, vis_dir, out_dir)
    assert printed_of(run, vis_dir, r.stdout)


@pytest.mark.gpu
def test_gpu_command_names_a_frame_that_does_not_decode(tmp_path):
    _cv2()
    root, annot, res = setup_fixture(tmp_path)
    path = os.path.join(root, "d1", "000002.jpg")
    b = open(path, "rb").read()
    open(path, "wb").write(b[:len(b) * 2 // 3])                    # headers whole, the scan cut short
    with pytest.raises(RuntimeError, match="000002.jpg.*did not decode"):
        se.run(se.parse_args(run_argv("raw", root, annot, res, str(tmp_path / "vis"), str(tmp_path / "out"))))
