"""Detection drawing on the device (sy_draw_boxes, sy_vis_det_boxes, data.draw_boxes, python -m streamyolo_b200.vis,
StreamDetector(record_boxes=...)).

CPU: the numpy oracle (oracle/vis_oracle.py) equals cv2's drawing on thousands of random boxes, and its drawing of the
     fixture rows, encoded as the script's PIL does, equals every file the unmodified vis_det_th.py wrote
     (tests/golden/vis_script.npz) and every record_boxes fixture (vis_record.npz); the fp32 blend equals
     cv2.addWeighted on all 256 x 256 pairs; the CLI's host logic with the device pass emulated writes the script's files,
     names and directories, honours --seq, --gt and --overwrite, prints the script's line and runs make_videos_numbered's
     ffmpeg argv; the palette comes from a vis/vis_det_th.py and a missing one is refused; the refusals; vis.cu compiles
     for sm_90a without spills.
GPU: sy_draw_boxes equals the fixtures in place and out of place over mixed sizes, leaves pixels outside each image and
     untouched pixels alone, follows rewritten boxes and counts in a graph replay and repeats bit for bit;
     sy_vis_det_boxes equals the host path; the CLI writes the script's files byte for byte; record_boxes equals its
     fixtures and the oracle on a detector's own detections, which it leaves bit-identical.
"""
import ctypes as C
import json
import os
import pickle
import re
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import vis_oracle as vo
from streamyolo_b200 import data, ops, stream, vis

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "vis_script.npz"))
REC = np.load(os.path.join(ROOT, "tests", "golden", "vis_record.npz"))
FULL_JPG = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_full_f420_q90.npz"))["jpg"].tobytes()
DATASET = json.loads(GOLD["annot"].tobytes().decode())
RESULTS = pickle.loads(GOLD["results"].tobytes())
PALETTE_RGB = GOLD["palette_rgb"]
CLASS_PALETTE = {int(k): tuple(int(c) for c in v) for k, v in zip(GOLD["palette_keys"], PALETTE_RGB)}


def _cv2():
    return pytest.importorskip("cv2")


def setup_toolkit(tmp_path, palette=True):
    """the fixture dataset (frames, annotation file, result pickle) under tmp_path, and a sAP directory whose
    vis/vis_det_th.py holds the fixture's class_palette -> (data root, annotation path, result path, sAP dir)"""
    root = tmp_path / "data"
    for k in GOLD.files:
        if k.startswith("in/"):
            p = root / k[3:]
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_bytes(GOLD[k].tobytes())
    (root / "dF").mkdir(parents=True, exist_ok=True)
    (root / "dF" / "000000.jpg").write_bytes(FULL_JPG)
    annot, res = tmp_path / "annot.json", tmp_path / "res.pkl"
    annot.write_text(json.dumps(DATASET))
    res.write_bytes(GOLD["results"].tobytes())
    sap = tmp_path / "sAP"
    (sap / "vis").mkdir(parents=True)
    if palette:
        (sap / "vis" / "vis_det_th.py").write_text("import numpy as np\n\nclass_palette = " + repr(CLASS_PALETTE) + "\n")
    return str(root), str(annot), str(res), str(sap)


def emulated_pass(files, frames, palette_bgr):
    """the device half of vis.run on the host: cv2.imdecode, the oracle's drawing, cv2.imencode at quality 75"""
    cv2 = _cv2()
    out = []
    for b, f in zip(files, frames):
        img = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        assert img.shape[:2] == f.hw
        out.append(cv2.imencode(".jpg", vo.draw(img, f.boxes, f.labels, palette_bgr), [cv2.IMWRITE_JPEG_QUALITY, 75])[1]
                   .tobytes())
    return out


def check_written(vis_dir, run, only=None):
    """the files under vis_dir against the script's run ``run`` of the fixture"""
    import hashlib
    names = [str(v) for v in GOLD[run + ".files"]]
    for rel in names:
        if only is not None and not rel.startswith(only):
            continue
        b = open(os.path.join(vis_dir, rel), "rb").read()
        if rel.startswith("seqF"):
            assert len(b) == int(GOLD[f"{run}/{rel}.len"]) and hashlib.sha256(b).digest() == \
                GOLD[f"{run}/{rel}.sha256"].tobytes(), rel
        else:
            assert b == GOLD[f"{run}/{rel}"].tobytes(), rel
    got = sorted(os.path.relpath(os.path.join(d, f), vis_dir) for d, _, fs in os.walk(vis_dir) for f in fs)
    assert got == sorted(n for n in names if only is None or n.startswith(only))


def opts(root, annot, res, out, *extra):
    return vis.parse_args(["--data-root", root, "--annot-path", annot, "--result-path", res, "--vis-dir", out, *extra])


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_blend_equals_cv2_add_weighted_on_every_pair():
    cv2 = _cv2()
    a = np.arange(256, dtype=np.uint8)
    orig, paint = (v.copy() for v in np.meshgrid(a, a, indexing="ij"))
    assert np.array_equal(vo.blend(orig, paint), cv2.addWeighted(orig, 0.8, paint, 0.2, 0))
    assert np.array_equal(vo.blend(orig, orig), orig)


def _cv2_draw(cv2, img, boxes, labels, palette):
    """vis_obj_fancy's box branch in cv2 calls, as the script makes them"""
    img = img.copy()
    filled = img.copy()
    for b, l in zip(boxes, labels):
        cv2.rectangle(img, (int(b[0]), int(b[1])), (int(b[2]), int(b[3])), [int(c) for c in palette[l]], thickness=-1)
    img = cv2.addWeighted(filled, 0.8, img, 0.2, 0)
    for b, l in zip(boxes, labels):
        cv2.rectangle(img, (int(b[0]), int(b[1])), (int(b[2]), int(b[3])), [int(c) for c in palette[l]], thickness=2)
    return img


def test_oracle_equals_cv2_on_random_boxes():
    cv2 = _cv2()
    rng = np.random.default_rng(3)
    palette = rng.integers(0, 256, (7, 3)).astype(np.uint8)
    n_boxes = 0
    for case in range(300):
        h, w = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        k = int(rng.integers(0, 20))
        span = int(rng.choice([3, 80, 5000, 100000]))
        boxes = rng.integers(-span, span, (k, 4), dtype=np.int64)
        small = rng.random(k) < 0.5                          # boxes near the image, degenerate ones among them
        boxes[small, :2] = rng.integers(-3, max(h, w) + 3, (int(small.sum()), 2))
        boxes[small, 2:] = boxes[small, :2] + rng.integers(-3, 25, (int(small.sum()), 2))
        boxes = boxes.astype(np.int32)
        labels = rng.integers(0, len(palette), k)
        assert np.array_equal(vo.draw(img, boxes, labels, palette), _cv2_draw(cv2, img, boxes, labels, palette)), case
        n_boxes += k
    assert n_boxes > 2500


def test_oracle_equals_the_script_files():
    """the oracle's drawing of the fixture rows, encoded as PIL saves them, is every file the script wrote"""
    cv2 = _cv2()
    import hashlib
    pal_bgr = PALETTE_RGB[:, ::-1]
    for run in ("res", "gt"):
        by_image = {}
        for r in (DATASET["annotations"] if run == "gt" else RESULTS):
            by_image.setdefault(r["image_id"], []).append(r)
        seqs = DATASET["sequences"]
        for sid, seq in enumerate(seqs):
            for ii, img in enumerate(v for v in DATASET["images"] if v["sid"] == sid):
                rel = f"{seq}/{ii + 1:06d}.jpg"
                src = FULL_JPG if seq == "seqF" else GOLD[f"in/{DATASET['seq_dirs'][sid]}/{img['name']}"].tobytes()
                frame = cv2.imdecode(np.frombuffer(src, np.uint8), cv2.IMREAD_COLOR)
                boxes, labels = vo.script_rows(by_image.get(img["id"], []), 0.3, gt=run == "gt")
                b = cv2.imencode(".jpg", vo.draw(frame, boxes, labels, pal_bgr), [cv2.IMWRITE_JPEG_QUALITY, 75])[1].tobytes()
                if seq == "seqF":
                    assert hashlib.sha256(b).digest() == GOLD[f"{run}/{rel}.sha256"].tobytes(), (run, rel)
                else:
                    assert b == GOLD[f"{run}/{rel}"].tobytes(), (run, rel)


def test_fixture_rows_cover_the_cases():
    res = {}
    for r in RESULTS:
        res.setdefault(r["image_id"], []).append(r)
    assert RESULTS[0]["bbox"].dtype == np.float32 and RESULTS[0]["score"].dtype == np.float32
    assert isinstance(DATASET["annotations"][0]["bbox"][0], float)
    assert any(r["score"] == np.float32(0.3) for r in RESULTS)
    assert any(r["bbox"][2] < 0 for r in RESULTS) and any(r["bbox"][2] == 0 and r["bbox"][3] == 0 for r in RESULTS)
    assert {int(r["category_id"]) for r in RESULTS} == set(range(len(PALETTE_RGB)))
    ids = {img["id"] for img in DATASET["images"]}
    assert ids - set(res), "a frame without rows"
    assert any(all(r["score"] < np.float32(0.3) for r in rows) for rows in res.values())
    for i in range(len(REC["count"])):                      # ties at the threshold and at .5 in the record fixture
        det = REC["det"][i, :REC["count"][i]]
        assert (det[:, 4] * det[:, 5] == np.float32(0.3)).any() and (det[:, :4] % 1 == 0.5).any()


def test_record_fixtures_equal_the_oracle():
    cv2 = _cv2()
    pal_bgr = REC["palette_rgb"][:, ::-1]
    for s in range(len(REC["count"])):
        boxes, labels = vo.tick_rows(REC["det"][s], int(REC["count"][s]), float(REC["score_th"]))
        drawn = vo.draw(REC[f"frame{s}"], boxes, labels, pal_bgr)
        assert cv2.imencode(".jpg", drawn, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() == REC[f"jpg{s}"].tobytes(), s


def test_cli_emulated_writes_the_script_files(tmp_path, monkeypatch, capsys):
    root, annot, res, sap = setup_toolkit(tmp_path)
    monkeypatch.chdir(os.path.join(sap, "vis"))                 # found through ../vis, as the script's sys.path does
    for run, extra in (("res", []), ("gt", ["--gt"])):
        out = str(tmp_path / f"out_{run}")
        assert vis.run(opts(root, annot, res, out, *extra), device_pass=emulated_pass) == 8
        check_written(out, run)
        assert capsys.readouterr().out == str(GOLD[run + ".printed"]).replace("<vis-dir>", out)


def test_cli_seq_overwrite_and_make_video(tmp_path, monkeypatch, capsys):
    root, annot, res, sap = setup_toolkit(tmp_path)
    monkeypatch.chdir(sap)
    out = str(tmp_path / "out")
    for seq in ("1", "seqB"):
        assert vis.run(opts(root, annot, res, out, "--seq", seq), device_pass=emulated_pass) in (3, 0)
        check_written(out, "res", only="seqB")
    # without --overwrite an existing file is kept and not drawn again
    p = os.path.join(out, "seqB", "000002.jpg")
    open(p, "wb").write(b"kept")
    calls = []
    assert vis.run(opts(root, annot, res, out, "--seq", "seqB"), device_pass=lambda *a: calls.append(a)) == 0
    assert not calls and open(p, "rb").read() == b"kept"
    assert vis.run(opts(root, annot, res, out, "--seq", "seqB", "--overwrite"), device_pass=emulated_pass) == 3
    check_written(out, "res", only="seqB")
    capsys.readouterr()
    runs = []
    monkeypatch.setattr(vis.subprocess, "run", lambda argv, **kw: runs.append((argv, kw)))
    vis.run(opts(root, annot, res, out, "--make-video", "--fps", "25", "--seq", "0"), device_pass=emulated_pass)
    assert capsys.readouterr().out == ""                         # the closing line only without --make-video
    d = os.path.join(out, "seqA")
    assert runs == [(["ffmpeg", "-loglevel", "panic", "-y", "-framerate", "25.0", "-i", os.path.join(d, "%06d.jpg"),
                      "-c:v", "libx264", "-pix_fmt", "yuv420p", "-vf", "pad=width=ceil(iw/2)*2:height=ceil(ih/2)*2",
                      d + ".mp4"], {"check": True})]
    open(d + ".mp4", "wb").close()                               # an existing video is kept without --overwrite
    vis.run(opts(root, annot, res, out, "--make-video", "--seq", "0"), device_pass=emulated_pass)
    assert len(runs) == 1


def test_palette_from_the_toolkit(tmp_path, monkeypatch):
    _, _, _, sap = setup_toolkit(tmp_path)
    monkeypatch.chdir(sap)
    assert vis.read_class_palette() == CLASS_PALETTE
    assert vis.color_palette(CLASS_PALETTE, DATASET) == [tuple(int(c) for c in v) for v in PALETTE_RGB]
    monkeypatch.chdir(tmp_path)
    with pytest.raises(RuntimeError, match="toolkit's sAP directory"):
        vis.read_class_palette()
    root, annot, res, _ = setup_toolkit(tmp_path / "b", palette=False)
    monkeypatch.chdir(tmp_path / "b" / "sAP")
    with pytest.raises(RuntimeError, match="toolkit's sAP directory"):
        vis.run(opts(root, annot, res, str(tmp_path / "o")), device_pass=emulated_pass)
    assert not os.path.exists(tmp_path / "o")


def test_cli_refusals_before_any_work(tmp_path, monkeypatch):
    root, annot, res, sap = setup_toolkit(tmp_path)
    monkeypatch.chdir(sap)
    out = str(tmp_path / "out")
    never = lambda *a: pytest.fail("the device pass ran")            # noqa: E731
    with pytest.raises(ValueError, match="vis-scale"):
        vis.run(opts(root, annot, res, out, "--vis-scale", "0.5"), device_pass=never)
    cv2 = _cv2()
    with pytest.raises(cv2.error, match="dsize"):               # why: the script's own call cannot run in cv2 4.x
        cv2.resize(np.zeros((4, 4, 3), np.uint8), fx=0.5, fy=0.5, interpolation=cv2.INTER_LINEAR)
    for rows, err in (([dict(RESULTS[0], segmentation={"counts": "", "size": [1, 1]})], NotImplementedError),
                      ([dict(RESULTS[0], category_id=np.int32(len(PALETTE_RGB)))], IndexError),
                      ([dict(RESULTS[0], category_id=np.int32(-1))], IndexError)):
        bad = tmp_path / "bad.pkl"
        bad.write_bytes(pickle.dumps(RESULTS[1:] + rows))
        with pytest.raises(err):
            vis.run(opts(root, annot, str(bad), out), device_pass=never)
    # a label outside the palette on a row below the threshold is never indexed by the script either
    bad.write_bytes(pickle.dumps(RESULTS + [dict(RESULTS[0], category_id=np.int32(99), score=np.float32(0.1))]))
    assert vis.run(opts(root, annot, str(bad), out), device_pass=emulated_pass) == 8
    assert not os.path.exists(os.path.join(out, "never"))


def test_refusals_without_a_device():
    lib = ops.load_library()
    good = dict(src=0x1000, sizes=0x2000, n=2, max_h=16, max_w=24, boxes=0x3000, labels=0x4000, counts=0x5000, K=4,
                palette=0x6000, P=3, dst=0x1000, dst_h=16, dst_w=24)
    for kw in (dict(src=None), dict(dst=None), dict(boxes=None), dict(palette=None), dict(n=0), dict(max_h=0),
               dict(max_w=70000), dict(K=0), dict(K=(1 << 24) + 1), dict(P=0), dict(P=65537), dict(dst_h=15),
               dict(dst_w=25), dict(boxes=0x3004)):
        d = ops.SyDrawBoxesDesc(**dict(good, **kw))
        assert lib.sy_draw_boxes(C.byref(d), None) == 1, kw            # SY_EINVAL, before any launch
    good = dict(det=0x1000, count=0x2000, S=2, A=10, score_th=0.3, boxes=0x3000, labels=0x4000, counts=0x5000)
    for kw in (dict(det=None), dict(count=None), dict(labels=None), dict(S=0), dict(A=0), dict(boxes=0x3008)):
        d = ops.SyVisDetBoxesDesc(**dict(good, **kw))
        assert lib.sy_vis_det_boxes(C.byref(d), None) == 1, kw


def test_record_boxes_refusals():
    m = types.SimpleNamespace(head=types.SimpleNamespace(num_classes=3))
    ok = stream.record_boxes_args((0.3, [(1, 2, 3)] * 3), 95, 3)
    assert ok[0] == float(np.float32(0.3)) and ok[1].tolist() == [[3, 2, 1]] * 3
    assert stream.record_boxes_args((0, [(1, 2, 3)] * 3), 95, 3)[0] == -np.inf
    for rb, q, match in (((0.3, [(1, 2, 3)] * 3), None, "record_quality"), ((0.3, [(1, 2, 3)] * 2), 95, "3 classes"),
                         ((0.3, [(1, 2, 300)] * 3), 95, "palette"), ((0.3, [(1, 2)] * 3), 95, "palette"),
                         ((float("nan"), [(1, 2, 3)] * 3), 95, "score_th"), ((0.3,), 95, "record_boxes"),
                         (("0.3", [(1, 2, 3)] * 3), 95, "score_th")):
        with pytest.raises(ValueError, match=match):
            stream.record_boxes_args(rb, q, m.head.num_classes)


def test_vis_cu_compiles_without_spills():
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc not available")
    cmd = [build.NVCC] + build.COMMON + build.SOURCES["vis.cu"] + ["-c", os.path.join(build.CSRC, "vis.cu"), "-o",
                                                                   os.devnull]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == 2 and all(p == ("0", "0", "0") for p in props), r.stderr


# ---------------------------------------------------------------------------------------------------------------- GPU
DEV = "cuda"
SENTINEL = 0x5A


def _fixture_frames():
    """the small fixture frames of the result run: (BGR images, int32 boxes, labels) by the host path"""
    cv2 = _cv2()
    by_image = {}
    for r in RESULTS:
        by_image.setdefault(r["image_id"], []).append(r)
    out = []
    for img in DATASET["images"]:
        if img["height"] > 1000:
            continue
        src = GOLD[f"in/{DATASET['seq_dirs'][img['sid']]}/{img['name']}"].tobytes()
        frame = cv2.imdecode(np.frombuffer(src, np.uint8), cv2.IMREAD_COLOR)
        boxes, labels = vo.script_rows(by_image.get(img["id"], []), 0.3)
        out.append((frame, boxes, labels))
    return out


def _slots(imgs):
    mh, mw = max(i.shape[0] for i in imgs), max(i.shape[1] for i in imgs)
    s = np.full((len(imgs), mh, mw, 3), SENTINEL, np.uint8)
    for k, i in enumerate(imgs):
        s[k, :i.shape[0], :i.shape[1]] = i
    return torch.from_numpy(s).to(DEV), [i.shape[:2] for i in imgs]


@pytest.mark.gpu
def test_gpu_draw_boxes_equals_the_oracle_in_and_out_of_place():
    fx = _fixture_frames()
    pal = PALETTE_RGB[:, ::-1].copy()
    want = [vo.draw(f, b, l, pal) for f, b, l in fx]
    slots, sizes = _slots([f for f, _, _ in fx])
    boxes, labels = [b for _, b, _ in fx], [l for _, _, l in fx]
    runs = []
    for place in ("in", "out", "in"):
        src = slots.clone()
        if place == "in":
            got = data.draw_boxes(src, boxes, labels, None, pal, sizes)
            assert got.data_ptr() == src.data_ptr()
        else:
            out = torch.full_like(src, SENTINEL)
            b_t, l_t, c_t = _packed(boxes, labels)
            got = data.draw_boxes(src, b_t, l_t, c_t, torch.from_numpy(pal).to(DEV),
                                  torch.tensor(sizes, dtype=torch.int32, device=DEV), out=out)
            assert torch.equal(src, slots)                        # the source is not written
        host = got.cpu().numpy()
        for k, ((h, w), wnt, (f, _, _)) in enumerate(zip(sizes, want, fx)):
            if place == "in":
                assert np.array_equal(host[k, :h, :w], wnt), k
            else:                                             # only the pixels a box touches are written
                touched = (wnt != f).any(axis=2) | _covered(h, w, boxes[k])
                assert np.array_equal(host[k, :h, :w][touched], wnt[touched]), k
                assert (host[k, :h, :w][~touched] == SENTINEL).all(), k
            assert (host[k, h:] == SENTINEL).all() and (host[k, :, w:] == SENTINEL).all(), k
        runs.append(host)
    assert np.array_equal(runs[0], runs[2])


def _covered(h, w, boxes):
    """pixels of an h x w image some box's fill or outline covers"""
    fill, line = vo._owner_maps(h, w, np.asarray(boxes).reshape(-1, 4))
    return (fill >= 0) | (line >= 0)


def _packed(boxes, labels, k=None):
    n = len(boxes)
    k = k or max([1] + [len(b) for b in boxes])
    b = np.zeros((n, k, 4), np.int32)
    l = np.zeros((n, k), np.int32)
    for i, (bb, ll) in enumerate(zip(boxes, labels)):
        b[i, :len(bb)], l[i, :len(ll)] = bb, ll
    c = np.asarray([len(bb) for bb in boxes], np.int32)
    return (torch.from_numpy(b).to(DEV), torch.from_numpy(l).to(DEV), torch.from_numpy(c).to(DEV))


@pytest.mark.gpu
def test_gpu_draw_boxes_many_boxes_and_tiles():
    """more boxes than one compaction chunk, on frames of several tiles, against the oracle"""
    rng = np.random.default_rng(9)
    pal = rng.integers(0, 256, (5, 3)).astype(np.uint8)
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((130, 300), (64, 64), (33, 129))]
    boxes, labels = [], []
    for i, img in enumerate(imgs):
        h, w = img.shape[:2]
        k = (600, 0, 300)[i]
        b = np.stack([rng.integers(-10, w + 10, k), rng.integers(-10, h + 10, k), rng.integers(-10, w + 10, k),
                      rng.integers(-10, h + 10, k)], 1).astype(np.int32)
        boxes.append(b)
        labels.append(rng.integers(0, len(pal), k))
    slots, sizes = _slots(imgs)
    got = data.draw_boxes(slots, boxes, labels, None, pal, sizes).cpu().numpy()
    for k, img in enumerate(imgs):
        h, w = img.shape[:2]
        assert np.array_equal(got[k, :h, :w], vo.draw(img, boxes[k], labels[k], pal)), k
        assert (got[k, h:] == SENTINEL).all() and (got[k, :, w:] == SENTINEL).all()


@pytest.mark.gpu
def test_gpu_draw_boxes_graph_follows_rewritten_boxes():
    rng = np.random.default_rng(4)
    pal = rng.integers(0, 256, (4, 3)).astype(np.uint8)
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((70, 90), (40, 100))]
    src, sizes = _slots(imgs)
    out = torch.empty_like(src)
    K = 32
    b_t = torch.zeros((2, K, 4), dtype=torch.int32, device=DEV)
    l_t = torch.zeros((2, K), dtype=torch.int32, device=DEV)
    c_t = torch.zeros((2,), dtype=torch.int32, device=DEV)
    p_t, s_t = torch.from_numpy(pal).to(DEV), torch.tensor(sizes, dtype=torch.int32, device=DEV)
    data.draw_boxes(src, b_t, l_t, c_t, p_t, s_t, out=out)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out.copy_(src)
        data.draw_boxes(src, b_t, l_t, c_t, p_t, s_t, out=out)
    for t in range(4):
        boxes = [rng.integers(-5, 100, (int(rng.integers(0, K + 1)), 4)).astype(np.int32) for _ in imgs]
        labels = [rng.integers(0, len(pal), len(b)) for b in boxes]
        b2, l2, c2 = _packed(boxes, labels, K)
        b_t.copy_(b2), l_t.copy_(l2), c_t.copy_(c2)
        g.replay()
        host = out.cpu().numpy()
        for k, img in enumerate(imgs):
            h, w = img.shape[:2]
            assert np.array_equal(host[k, :h, :w], vo.draw(img, boxes[k], labels[k], pal)), (t, k)


@pytest.mark.gpu
def test_gpu_vis_det_boxes_equals_the_host_path():
    det = torch.from_numpy(REC["det"]).to(DEV)
    count = torch.from_numpy(REC["count"]).to(DEV)
    th = float(REC["score_th"])
    rng = np.random.default_rng(1)
    extra = np.zeros((1, det.shape[1], 7), np.float32)                 # many rows at .5 and at the threshold
    n = det.shape[1]
    extra[0, :, :4] = np.sort(rng.integers(-40, 400, (n, 4)), axis=1) + 0.5
    extra[0, :, 4], extra[0, :, 5] = np.float32(0.5), np.float32(0.6)
    extra[0, ::3, 5] = np.nextafter(np.float32(0.6), np.float32(0))
    extra[0, :, 6] = np.arange(n) % 9
    extra[0, 1:9, :4] = [[np.inf, 1, 2, 3], [-np.inf, 1, 2, 3], [np.nan, 1, 2, 3], [1, 2, np.inf, 3], [1, 2, 3e9, 4],
                         [-3e9, 1, 5, 6], [2147483520, 0, 2147483647, 1], [-2147483904, 0, 1, 1]]   # numpy's int32 cast
    det = torch.cat([det, torch.from_numpy(extra).to(DEV)])
    count = torch.cat([count, torch.tensor([n], dtype=torch.int32, device=DEV)])
    for t in (th, 0.0, 0.95):
        boxes, labels, counts = ops.vis_det_boxes(det, count, t if t > 0 else -np.inf)
        b, l, c = boxes.cpu().numpy(), labels.cpu().numpy(), counts.cpu().numpy()
        dh, ch = det.cpu().numpy(), count.cpu().numpy()
        for s in range(det.shape[0]):
            with np.errstate(invalid="ignore"):
                wb, wl = vo.tick_rows(dh[s], int(ch[s]), t)
            assert c[s] == len(wb), (t, s)
            assert np.array_equal(b[s, :c[s]], wb) and np.array_equal(l[s, :c[s]], wl), (t, s)


def _vis_cli(tmp_path, monkeypatch, run, extra):
    root, annot, res, sap = setup_toolkit(tmp_path)
    monkeypatch.chdir(sap)
    out = str(tmp_path / f"out_{run}")
    assert vis.run(opts(root, annot, res, out, *extra)) == 8
    check_written(out, run)


@pytest.mark.gpu
def test_gpu_cli_writes_the_script_files(tmp_path, monkeypatch, capsys):
    _vis_cli(tmp_path / "a", monkeypatch, "res", [])
    _vis_cli(tmp_path / "b", monkeypatch, "gt", ["--gt"])


@pytest.mark.gpu
def test_gpu_cli_names_a_frame_that_does_not_decode(tmp_path, monkeypatch):
    root, annot, res, sap = setup_toolkit(tmp_path)
    monkeypatch.chdir(sap)
    p = os.path.join(root, "dB", "000001.jpg")
    open(p, "wb").write(open(p, "rb").read()[:100])
    with pytest.raises(RuntimeError, match=re.escape(p) + ".*did not decode"):
        vis.run(opts(root, annot, res, str(tmp_path / "out"), "--seq", "seqB"))


@pytest.mark.gpu
def test_gpu_record_path_equals_its_fixtures():
    """sy_vis_det_boxes -> sy_draw_boxes onto a copy -> sy_jpeg_encode, as the tick runs them, on the fixture rows"""
    s = len(REC["count"])
    imgs = [REC[f"frame{i}"] for i in range(s)]
    frames, sizes = _slots(imgs)
    keep = frames.clone()
    th, pal = stream.record_boxes_args((float(REC["score_th"]), REC["palette_rgb"].tolist()), 95, 9)
    boxes, labels, counts = ops.vis_det_boxes(torch.from_numpy(REC["det"]).to(DEV),
                                              torch.from_numpy(REC["count"]).to(DEV), th)
    rec = frames.clone()
    s_t = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    ops.draw_boxes(rec, s_t, boxes, labels, counts, torch.from_numpy(pal).to(DEV), rec)
    files = data.encode_jpeg(rec, 95, sizes)
    assert files == [REC[f"jpg{i}"].tobytes() for i in range(s)]
    assert torch.equal(frames, keep)


IN_SCALE, CONF, NMS = 0.5, 0.01, 0.65


def _model_s():
    from test_stream import _model_s as model_s
    return model_s(torch.float16)


def _same(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


def _expected(frames_bgr, dets, th, palette_rgb, q):
    """cv2.imencode of vis_obj_fancy's drawing of each stream's detections (the driver's (bboxes, scores, labels))"""
    cv2 = _cv2()
    out = []
    for f, (bb, sc, lb) in zip(frames_bgr, dets):
        ltwh = bb.copy()
        ltwh[:, 2:] -= ltwh[:, :2]
        rows = [{"bbox": ltwh[i], "score": sc[i], "category_id": lb[i]} for i in range(len(bb))]
        boxes, labels = vo.script_rows(rows, th)
        drawn = vo.draw(f, boxes, labels, np.asarray(palette_rgb, np.uint8)[:, ::-1])
        out.append(cv2.imencode(".jpg", drawn, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes())
    return out


@pytest.mark.gpu
def test_gpu_stream_detector_record_boxes_nv12_and_submit():
    """three NV12 cameras with forecast: detections, raw outputs and forecasts equal a detector that records without
    boxes and one that does not record; last_jpeg() is the oracle's drawing of the tick's own detections; the tick's
    frames are not drawn on; submit / receive give the same"""
    from oracle.make_yuv_golden import synth_frame
    from oracle.yuv_oracle import yuv_to_bgr
    m = _model_s()
    nc = m.head.num_classes
    rng = np.random.default_rng(0)
    palette = [tuple(int(v) for v in rng.integers(0, 256, 3)) for _ in range(nc)]
    sizes = [(1200, 1920), (1080, 1920), (720, 1280)]
    kw = dict(in_scale=IN_SCALE, frame_sizes=sizes, input_size=(600, 960), conf_thre=CONF, nms_thre=NMS,
              frame_format="nv12", forecast=True)
    boxes = stream.StreamDetector(m, record_quality=90, record_boxes=(0.05, palette), **kw)
    frames_only = stream.StreamDetector(m, record_quality=90, **kw)
    plain = stream.StreamDetector(m, **kw)
    for t in range(3):
        fr = [synth_frame("nv12", h, w, 70 * t + i) for i, (h, w) in enumerate(sizes)]
        got = boxes.step(fr, fidx=[t] * 3)
        assert all(_same(a, b) for a, b in zip(got, frames_only.step(fr, fidx=[t] * 3))), t
        assert all(_same(a, b) for a, b in zip(got, plain.step(fr, fidx=[t] * 3))), t
        assert torch.equal(boxes.last_raw(), plain.last_raw()), t
        bgr = [yuv_to_bgr("nv12", x) for x in fr]
        for i, (h, w) in enumerate(sizes):
            assert np.array_equal(boxes._tick.frames[i, :h, :w].cpu().numpy(), bgr[i]), (t, i)
        assert sum(len(g[0]) for g in got) > 0
        assert boxes.last_jpeg() == _expected(bgr, got, 0.05, palette, 90), t
        assert frames_only.last_jpeg() == [data.encode_jpeg(torch.from_numpy(b).to(DEV)[None], 90)[0] for b in bgr], t
    assert all(_same(a, b) for a, b in zip(boxes.forecast([4] * 3), plain.forecast([4] * 3)))
    fr = [synth_frame("nv12", h, w, 999 + i) for i, (h, w) in enumerate(sizes)]
    boxes.submit(fr, fidx=[5] * 3)
    got = boxes.receive()
    assert boxes.last_jpeg() == _expected([yuv_to_bgr("nv12", x) for x in fr], got, 0.05, palette, 90)


@pytest.mark.gpu
def test_gpu_stream_detector_record_boxes_jpeg_with_absent_streams():
    """step_jpeg with a stream absent on a tick: its slot keeps the previous frame undrawn; a stream without a frame
    records nothing; the others get their own detections drawn"""
    from oracle import jpeg_encode_oracle as eo
    from oracle import jpeg_oracle as jo
    from oracle.make_jpeg_encode_golden import content
    m = _model_s()
    nc = m.head.num_classes
    palette = [((37 * c) % 256, (91 * c) % 256, (151 * c) % 256) for c in range(nc)]
    sizes = [(600, 960), (480, 640)]
    imgs = [[content("smooth", h, w, 10 * t + i) for i, (h, w) in enumerate(sizes)] for t in range(3)]
    files = [[eo.encode(i, 90) for i in row] for row in imgs]
    files[1][1] = None
    mb = max(len(f) for row in files for f in row if f is not None) + 64
    kw = dict(in_scale=IN_SCALE, frame_sizes=sizes, input_size=(480, 768), conf_thre=CONF, nms_thre=NMS,
              jpeg_max_bytes=mb)
    rec = stream.StreamDetector(m, record_quality=95, record_boxes=(0.0, palette), **kw)
    plain = stream.StreamDetector(m, **kw)
    for t, row in enumerate(files):
        got = rec.step_jpeg(row, fidx=None)
        assert all(_same(a, b) for a, b in zip(got, plain.step_jpeg(row))), t
        dec = [None if f is None else jo.decode(f, s)[0] for f, s in zip(row, sizes)]
        for i, (h, w) in enumerate(sizes):                   # a slot holds its last decoded frame, undrawn
            last = next(jo.decode(files[u][i], sizes[i])[0] for u in range(t, -1, -1) if files[u][i] is not None)
            assert np.array_equal(rec._tick.frames[i, :h, :w].cpu().numpy(), last), (t, i)
        out = rec.last_jpeg()
        want = _expected([d if d is not None else np.zeros((1, 1, 3), np.uint8) for d in dec], got, 0.0, palette, 95)
        for i, f in enumerate(out):
            assert (f is None) == (row[i] is None), (t, i)
            if f is not None:
                assert f == want[i], (t, i)


@pytest.mark.gpu
def test_gpu_default_tick_unchanged_and_record_boxes_launches(monkeypatch):
    import inspect
    m = _model_s()
    kw = dict(in_scale=IN_SCALE, frame_sizes=[(1200, 1920)], input_size=(600, 960), frame_format="nv12")
    nc = m.head.num_classes
    rec = stream.StreamDetector(m, record_quality=90, **kw)
    boxed = stream.StreamDetector(m, record_quality=90, record_boxes=(0.3, [(1, 2, 3)] * nc), **kw)
    calls = []
    for name, fn in inspect.getmembers(ops, inspect.isfunction):
        if fn.__module__ == ops.__name__ and not name.startswith("_") and name not in ("lib", "load_library"):
            monkeypatch.setattr(ops, name, (lambda n, f: lambda *a, **k: (calls.append(n), f(*a, **k))[1])(name, fn))
    rec._tick.run()
    default, calls[:] = list(calls), []
    boxed._tick.run()
    torch.cuda.synchronize()
    assert "draw_boxes" not in default and "vis_det_boxes" not in default
    default = [c for c in default if c != "jpeg_encode_workspace_bytes"]
    assert default[-1] == "jpeg_encode"
    assert [c for c in calls if c != "jpeg_encode_workspace_bytes"] == default[:-1] + ["vis_det_boxes", "draw_boxes",
                                                                                        "jpeg_encode"]
    for bad in ((0.3, [(1, 2, 3)] * (nc - 1)), (0.3, [(1, 2, 3, 4)] * nc)):
        with pytest.raises(ValueError, match="record_boxes"):
            stream.StreamDetector(m, record_quality=90, record_boxes=bad, **kw)
    with pytest.raises(ValueError, match="record_quality"):
        stream.StreamDetector(m, record_boxes=(0.3, [(1, 2, 3)] * nc), **kw)
