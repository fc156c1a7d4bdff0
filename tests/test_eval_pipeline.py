"""The validation evaluators' batch loop on the device (streamyolo_b200/evaluate.py, sy_coco_rows).

CPU (no GPU needed):
  * the oracle's convert_to_coco_format equals the data_lists the unmodified reference methods wrote
    (tests/golden/eval_coco_{onex,twox,still}.npz): ids, categories, every bbox and score float;
  * the frame-id table equals the reference's kept / dropped images and output ids;
  * the batches come from the loader's own sampler, DistributedSampler padding included (world sizes 2 and 3);
  * rows of several ranks merge rank-major, as gather + itertools.chain;
  * argument checks: max_bytes, the class table size, one frame size;
  * coco_rows_kernel compiles without spills.

GPU (H100):
  * sy_coco_rows is bit-identical to torch-CPU convert_to_coco_format on the same NMS outputs;
  * DeviceEvaluator (as the drop-in subclass of a stand-in for the reference evaluator) hands evaluate_prediction the
    data_list of the eager composition, bit for bit, for the pair model (onex / twox rules) and the still model, bf16 and
    fp16 storage, with a partial last batch; a second evaluate after a weight change gives the new weights' rows;
  * a damaged file or a file of another size raises with its dataset index.
"""
import itertools
import os
import sys

import numpy as np
import pytest
import torch

from oracle import eval_oracle
from oracle.make_stream_jpeg_golden import damaged, requant
from streamyolo_b200 import evaluate

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
RULES = ("onex", "twox", "still")


def golden(rule):
    return np.load(os.path.join(GOLD, f"eval_coco_{rule}.npz"))


def images_of(fid):
    return [{"id": i, "fid": int(f)} for i, f in enumerate(fid)]


def as_arrays(data_list):
    return (np.array([d["image_id"] for d in data_list], np.int64), np.array([d["category_id"] for d in data_list], np.int64),
            np.array([d["bbox"] for d in data_list], np.float64).reshape(-1, 4),
            np.array([d["score"] for d in data_list], np.float64))


# ================================================================================================ CPU
@pytest.mark.parametrize("rule", RULES)
def test_oracle_equals_reference_data_list(rule):
    g = golden(rule)
    det, count, hw, ids = g["det"], g["count"], g["hw"], g["ids"]
    outputs = [torch.from_numpy(det[i, :count[i]].copy()) if count[i] else None for i in range(len(ids))]
    got = eval_oracle.convert_to_coco_format(outputs, (hw[:, 0].tolist(), hw[:, 1].tolist()), ids.tolist(),
                                             tuple(g["img_size"].tolist()), g["class_ids"].tolist(), images_of(g["fid"]), rule)
    assert all(d["segmentation"] == [] for d in got)
    gi, gc, gb, gs = as_arrays(got)
    assert len(gi) == len(g["image_id"]) > 0
    assert np.array_equal(gi, g["image_id"]) and np.array_equal(gc, g["category_id"])
    assert np.array_equal(gb.view(np.int64), g["bbox"].view(np.int64)) and np.array_equal(gs.view(np.int64),
                                                                                          g["score"].view(np.int64))
    # rows as the device returns them (fp32 arrays) -> coco_dicts: the same data_list, the same Python values
    rows = {"bbox": gb.astype(np.float32), "score": gs.astype(np.float32), "image_id": gi, "category_id": gc}
    assert evaluate.coco_dicts(rows) == got


@pytest.mark.parametrize("rule", RULES)
def test_frame_id_table_equals_reference(rule):
    g = golden(rule)
    table = evaluate.image_id_table(images_of(g["fid"]), g["ids"].tolist(), rule)
    has = g["count"] > 0
    assert table.dtype == np.int32 and np.array_equal(table[has], g["table"][has])
    if rule != "still":                      # the cases the fixture covers
        fid = g["fid"][g["ids"]]
        assert {15060, 15061} <= set(g["ids"].tolist()) and (table[np.isin(g["ids"], [15060, 15061])] == -1).all()
        assert (fid == 0).any() and (fid == 1).any() and (table >= 0).any() and (table[has] == -1).any()
    assert [eval_oracle.output_id(images_of(g["fid"]), i, rule) for i in g["ids"]] == [None if t < 0 else t for t in table]


def test_frame_id_table_past_the_end():
    images = images_of([0, 1, 2, 3])
    assert evaluate.image_id_table(images, [1, 2], "onex").tolist() == [2, 3]
    with pytest.raises(ValueError, match="reads images\\[4\\]"):
        evaluate.image_id_table(images, [3], "onex")
    with pytest.raises(ValueError, match="reads images\\[4\\]"):
        evaluate.image_id_table(images, [2], "twox")
    with pytest.raises(ValueError, match="rule"):
        evaluate.image_id_table(images, [1], "threex")


class FakeDataset(torch.utils.data.Dataset):
    """what DeviceEvaluator reads of the reference's val datasets: annotations, ids, class_ids, coco.dataset['images']"""

    def __init__(self, files, hw, rule, fid, ids, class_ids=tuple(range(8))):
        self.ids, self.class_ids = list(ids), list(class_ids)
        if rule == "still":                       # (res, img_info, resized_info, file_name)
            self.annotations = [(None, hw, None, f[0]) for f in files]
        else:                                     # (res, support_res, img_info, resized_info, file_name, support_file_name)
            self.annotations = [(None, None, hw, None, f[0], f[1]) for f in files]
        self.coco = type("Coco", (), {"dataset": {"images": images_of(fid)}})()

    def __len__(self):
        return len(self.ids)

    def __getitem__(self, i):
        return i


def loader(ds, batch, sampler=None):
    return torch.utils.data.DataLoader(ds, batch_size=batch, sampler=sampler or torch.utils.data.SequentialSampler(ds))


@pytest.mark.parametrize("world", [2, 3])
def test_sampler_batches_with_distributed_padding(world):
    n, batch = 11, 2
    ds = FakeDataset([("a", "b")] * n, (1200, 1920), "onex", [1] * 40, range(n))
    total = -(-n // world) * world
    padded = list(range(n)) + list(range(total - n))       # DistributedSampler(shuffle=False) repeats from the start
    for rank in range(world):
        s = torch.utils.data.distributed.DistributedSampler(ds, num_replicas=world, rank=rank, shuffle=False)
        got = evaluate.sampler_batches(loader(ds, batch, s))
        mine = padded[rank:total:world]
        assert got == [mine[k:k + batch] for k in range(0, len(mine), batch)], (world, rank)
    assert sum(len(b) for r in range(world) for b in evaluate.sampler_batches(
        loader(ds, batch, torch.utils.data.distributed.DistributedSampler(ds, world, r, shuffle=False)))) == total


def test_rank_order_merge():
    rng = np.random.default_rng(1)
    parts = []
    for r, n in enumerate([3, 0, 5]):
        parts.append({"bbox": rng.random((n, 4)).astype(np.float32), "score": rng.random(n).astype(np.float32),
                      "image_id": np.full(n, r, np.int64), "category_id": rng.integers(0, 8, n)})
    merged = evaluate.merge_ranks(parts)
    assert merged["image_id"].tolist() == [0, 0, 0, 2, 2, 2, 2, 2]
    assert evaluate.coco_dicts(merged) == list(itertools.chain(*[evaluate.coco_dicts(p) for p in parts]))
    assert evaluate.coco_dicts(evaluate.empty_rows()) == []


def test_argument_checks():
    files = [("a.jpg", "b.jpg")] * 5
    ds = FakeDataset(files, (1200, 1920), "onex", [0, 1, 2, 3, 4, 5, 6, 0], range(1, 6))
    ok = evaluate.DeviceEvaluator(loader(ds, 2), (600, 960), 0.01, 0.65, 8, rule="onex")
    assert ok.frame_hw == (1200, 1920) and ok.ratio == 0.5 and [ok.table[i] for i in range(5)] == [2, 3, 4, 5, 6]
    assert ok.batches == [[0, 1], [2, 3], [4]] and ok.detections() is None
    for bad in (0, 3, 2.5, (1 << 28) + 1):
        with pytest.raises(ValueError, match="max_bytes"):
            evaluate.DeviceEvaluator(loader(ds, 2), (600, 960), 0.01, 0.65, 8, rule="onex", max_bytes=bad)
    with pytest.raises(ValueError, match="class table has 8 entries for 80 classes"):
        evaluate.DeviceEvaluator(loader(ds, 2), (600, 960), 0.01, 0.65, 80, rule="onex")
    ds.annotations[3] = (None, None, (1080, 1920), None, "a.jpg", "b.jpg")
    with pytest.raises(ValueError, match="one frame size"):
        evaluate.DeviceEvaluator(loader(ds, 2), (600, 960), 0.01, 0.65, 8, rule="onex")
    with pytest.raises(ValueError, match="rule"):
        evaluate.DeviceEvaluator(loader(ds, 2), (600, 960), 0.01, 0.65, 8)


def test_dropin_evaluators_without_yolox():
    """install(evaluators=True) does nothing where the reference's evaluators cannot be imported"""
    import subprocess
    code = ("import streamyolo_b200.dropin as d; d.install(evaluators=True); d.install(postprocess=False, evaluators=True);"
            "import sys; print('ok')")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr


def test_coco_rows_kernel_compiles_without_spills(tmp_path):
    import re
    import shutil
    import subprocess
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    assert "-fmad=false" in build.SOURCES["postprocess.cu"]
    r = subprocess.run([nvcc] + build.COMMON + build.SOURCES["postprocess.cu"] + ["-c", os.path.join(build.CSRC, "postprocess.cu"),
                       "-o", str(tmp_path / "k.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout
    found = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stdout)
    hits = [f for f in found if "coco_rows_kernel" in f[0]]
    assert hits and all(f[1:] == ("0", "0", "0") for f in hits), hits


# ================================================================================================ GPU
DEV = "cuda"
SIZE = (600, 960)
CONF, NMS = 0.01, 0.65


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, 8])
def test_coco_rows_bit_identical_to_torch_cpu(b):
    """random NMS outputs with 80 classes, counts 0 and max_det among them, ratios 0.5 and 600 / 1080, dropped images and
    an undecoded frame: the rows equal torch-CPU convert_to_coco_format bit for bit; torch's in-place division of the fp32
    boxes by the Python float is the IEEE division by the float-rounded scale on this torch (checked live)"""
    from streamyolo_b200 import ops
    rng = np.random.default_rng(b)
    a, nc = 300, 80
    det = np.zeros((b, a, 7), np.float32)
    det[..., :4] = rng.uniform(-30, 1000, (b, a, 4))
    det[..., 2:4] += det[..., 0:2]
    det[..., 4:6] = rng.uniform(0, 1, (b, a, 2))
    det[..., 6] = rng.integers(0, nc, (b, a))
    count = rng.integers(1, a, b).astype(np.int32)
    count[0] = a
    if b > 1:
        count[1] = 0
    hw = [(1200, 1920) if i % 2 == 0 else (1080, 1440) for i in range(b)]
    scales = [min(SIZE[0] / h, SIZE[1] / w) for h, w in hw]
    assert scales[0] == 0.5 and (b == 1 or scales[1] == 600 / 1080)
    class_ids = [int(v) for v in rng.permutation(1000)[:nc]]
    image_id = np.arange(100, 100 + b, dtype=np.int32)
    status = np.zeros(2 * b, np.int32)
    if b > 2:
        image_id[2] = -1
        status[7] = 5                             # image 3's second frame did not decode
    # the division the reference relies on, live: torch CPU fp32 /= Python float == IEEE fp32 division by float(scale)
    t = torch.from_numpy(det[0, :, :4].copy())
    t /= 600 / 1080
    assert np.array_equal(t.numpy().view(np.int32), (det[0, :, :4] / np.float32(600 / 1080)).view(np.int32))
    d = torch.from_numpy(det).to(DEV)
    out = ops.coco_rows(d, torch.from_numpy(count).to(DEV), torch.tensor(scales, dtype=torch.float32, device=DEV),
                        torch.from_numpy(image_id).to(DEV), torch.tensor(class_ids, dtype=torch.int32, device=DEV),
                        status=torch.from_numpy(status).to(DEV))
    bbox, score, ids, cat, total = (x.cpu().numpy() for x in out)
    keep = [i for i in range(b) if image_id[i] >= 0 and (status[2 * i:2 * i + 2] == 0).all()]
    outputs = [torch.from_numpy(det[i, :count[i]].copy()) if count[i] else None for i in keep]
    want = eval_oracle.convert_to_coco_format(outputs, ([hw[i][0] for i in keep], [hw[i][1] for i in keep]),
                                              [int(image_id[i]) for i in keep], SIZE, class_ids, None, "still")
    n = int(total[0])
    assert n == len(want) == sum(int(count[i]) for i in keep) > 0
    rows = {"bbox": bbox[:n], "score": score[:n], "image_id": ids[:n].astype(np.int64), "category_id": cat[:n].astype(np.int64)}
    assert evaluate.coco_dicts(rows) == want


def _fixture_files(tmp_path):
    from test_stream_jpeg import jpg
    paths = []
    for k in range(4):
        p = tmp_path / f"f{k}.jpg"
        p.write_bytes(requant(jpg("a420"), k))
        paths.append(str(p))
    return paths


def _dataset(paths, rule, n=11):
    fid = [i % 5 for i in range(200)]              # sequences of 5 frames: starts, second frames and ends among the ids
    files = [(paths[i % 4], paths[(i + 1) % 4]) if rule != "still" else (paths[i % 4],) for i in range(n)]
    return FakeDataset(files, (1200, 1920), rule, fid, range(100, 100 + n))


class StandIn:
    """the reference evaluators' constructor and attributes; evaluate_prediction keeps what it is given"""

    def __init__(self, dataloader, img_size, confthre, nmsthre, num_classes, testdev=False, per_class_mAP=True):
        self.dataloader, self.img_size, self.confthre, self.nmsthre = dataloader, img_size, confthre, nmsthre
        self.num_classes, self.testdev, self.per_class_mAP = num_classes, testdev, per_class_mAP
        self.got = []

    def evaluate_prediction(self, data_dict, statistics):
        self.got.append((data_dict, statistics.cpu().tolist()))
        return 0.0, 0.0, f"{len(data_dict)} detections"


def _eager(model, ds, rule, batches):
    """decode_jpeg, the val transform, model(x), postprocess, then the oracle's conversion, batch by batch"""
    from streamyolo_b200 import data
    from streamyolo_b200.postprocess import postprocess
    fpi = evaluate.RULES[rule]
    out = []
    for batch in batches:
        files = [np.fromfile(p, np.uint8) for i in batch for p in evaluate._sample(ds, i, fpi)[0]]
        rows, lengths = data.pack_jpeg(files, max(f.size for f in files))
        frames, status = data.decode_jpeg(torch.from_numpy(rows).to(DEV), torch.from_numpy(lengths).to(DEV), (1200, 1920))
        assert status.tolist() == [0] * len(files)
        if fpi == 2:
            x, _ = data.pair_transform(frames.view(len(batch), 2, 1200, 1920, 3), None, None, None, SIZE, flip=False, raw=True)
        else:
            x, _ = data.frame_transform(frames, None, None, None, SIZE, flip=False, raw=True)
        with torch.no_grad():
            outputs = postprocess(model(x), model.head.num_classes, CONF, NMS)
        out += eval_oracle.convert_to_coco_format([None if o is None else o.cpu() for o in outputs],
                                                  ([1200] * len(batch), [1920] * len(batch)), [ds.ids[i] for i in batch],
                                                  SIZE, ds.class_ids, ds.coco.dataset["images"], rule)
    return out


def _still_model(dtype):
    from streamyolo_b200 import synth
    from test_gpu_still import build_still
    m = build_still(0.33, 0.50, momentum=1.0)
    x = synth.synth_frames(8, 600, 960, seed=99)[:, :3].contiguous().cuda()
    with torch.no_grad():
        m(x, synth.synth_labels(8, 600, 960, seed=11)[0].cuda())
    m.eval()
    m.activation_dtype = dtype
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("rule,dtype", [("onex", torch.bfloat16), ("twox", torch.float16), ("still", torch.float16),
                                        ("still", torch.bfloat16)], ids=["onex-bf16", "twox-fp16", "still-fp16", "still-bf16"])
def test_evaluate_bit_identical_to_eager(rule, dtype, tmp_path):
    """11 samples in batches of 4 (the last one partial, with its own graph): the data_list evaluate_prediction gets equals
    the eager composition's; detections() holds the same rows.  onex-bf16 also changes the weights and evaluates again."""
    from test_stream import _model_s
    m = _still_model(dtype) if rule == "still" else _model_s(dtype)
    ds = _dataset(_fixture_files(tmp_path), rule)
    cls = evaluate.device_evaluator(StandIn, rule)
    ev = cls(loader(ds, 4), SIZE, CONF, NMS, 8)
    assert isinstance(ev, StandIn) and ev.rule == rule and ev.batches == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9, 10]]
    assert ev.evaluate(m) == (0.0, 0.0, f"{len(ev.got[0][0])} detections")
    got, stats = ev.got[-1]
    want = _eager(m, ds, rule, ev.batches)
    assert len(want) > 0 and got == want
    assert stats[1] == 0.0 and stats[2] == 2 and stats[0] > 0
    rows = ev.detections()
    assert evaluate.coco_dicts(rows) == want and rows["bbox"].dtype == np.float32
    kept = {i for i, v in ev.table.items() if v >= 0}
    assert 0 < len(kept) and (rule == "still") == (len(kept) == len(ds))
    print(f"\n{rule} {dtype}: {len(want)} rows; capture {ev.capture_seconds:.2f} s")
    if rule == "onex":
        with torch.no_grad():
            m.head.cls_preds[0].bias.add_(0.7)
        ev.evaluate(m)
        again = _eager(m, ds, rule, ev.batches)
        assert ev.got[-1][0] == again and again != want


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["damaged", "size"])
def test_undecodable_file_raises_with_its_index(case, tmp_path):
    from test_stream import _model_s
    from test_stream_jpeg import jpg
    paths = _fixture_files(tmp_path)
    bad = tmp_path / "bad.jpg"
    bad.write_bytes(damaged(jpg("a420")) if case == "damaged" else jpg("b444"))
    ds = _dataset(paths, "onex", n=6)
    ds.annotations[5] = ds.annotations[5][:5] + (str(bad),)
    ev = evaluate.device_evaluator(StandIn, "onex")(loader(ds, 4), SIZE, CONF, NMS, 8)
    reason = "corrupt or truncated" if case == "damaged" else "image size differs"
    with pytest.raises(RuntimeError, match=f"dataset index 5 \\(file .*bad.jpg\\) did not decode: {reason}"):
        ev.evaluate(_model_s(torch.bfloat16))
    assert ev.got == [] and ev.detections() is None
