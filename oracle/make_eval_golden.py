"""Write tests/golden/eval_coco_{onex,twox,still}.npz FROM THE UNMODIFIED REFERENCE (test infrastructure).

Runs only where /root/reference is present:

    python -m oracle.make_eval_golden

It imports /root/reference/exps/evaluators/{onex,twox,still}_stream_evaluator.py untouched, on top of the yolox==0.3.0
stand-in of oracle/ref_shim (the evaluators' extra yolox.utils names are added here: ``xyxy2xywh`` restated from yolox
0.3.0's utils/boxes.py, the distributed helpers as single-process no-ops; none of them is the code under test), and runs
their ``convert_to_coco_format`` on

  * seeded NMS outputs of a batch of images: empty images (None), images at max_det rows, and everything between;
  * per-image frame sizes giving the ratio 0.5 and non-dyadic ratios (600 / 1080, 600 / 1201);
  * a synthetic ``images`` list of 15062 frames in sequences, whose evaluated ids include sequence starts (fid 0), second
    frames (fid 1), sequence ends and the ids 15060 / 15061.

Each file holds the inputs (``det`` [B, MAX_DET, 7], ``count`` [B], ``hw`` [B, 2], ``ids`` [B], ``fid`` [15062],
``class_ids``, ``img_size``), the reference's data_list as arrays (``image_id``, ``category_id``, ``bbox`` float64 [N, 4],
``score`` float64 [N]: the Python floats it holds) and ``table`` [B]: the id each image's detections are emitted under
when the method is run on that image alone, -1 when they are dropped (and for images without detections).
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(ROOT, "tests", "golden")
N_IMAGES = 15062
MAX_DET = 40
IMG_SIZE = (600, 960)
CLASS_IDS = [0, 1, 2, 3, 4, 5, 6, 7]
RULES = {"onex": ("onex_stream_evaluator", "ONEX_COCOEvaluator"), "twox": ("twox_stream_evaluator", "TWOX_COCOEvaluator"),
         "still": ("still_stream_evaluator", "STILL_COCOEvaluator")}


def fids():
    """sequence frame ids of N_IMAGES frames: sequences of 5 to 40 frames (seeded), the last one ending at the list's end"""
    g = np.random.default_rng(5)
    out, n = [], 0
    while n < N_IMAGES:
        k = min(int(g.integers(5, 41)), N_IMAGES - n)
        out += list(range(k))
        n += k
    return np.array(out, np.int32)


def eval_ids(fid):
    """the ids evaluated: the first 48 frames, frames around sequence boundaries, and the last 8 (15054 .. 15061)"""
    starts = np.nonzero(fid == 0)[0]
    near = [s + d for s in starts[5:9] for d in (-2, -1, 0, 1, 2)]
    return np.array(sorted(set(list(range(48)) + near + list(range(N_IMAGES - 8, N_IMAGES)))), np.int64)


def batch(n, seed=7):
    """seeded NMS outputs of n images: count 0 for every 7th image, MAX_DET for every 5th, else random"""
    g = np.random.default_rng(seed)
    det = np.zeros((n, MAX_DET, 7), np.float32)
    count = g.integers(1, MAX_DET, n).astype(np.int32)
    count[::7] = 0
    count[3::5] = MAX_DET
    x1 = g.uniform(-20, 900, (n, MAX_DET))
    y1 = g.uniform(-20, 560, (n, MAX_DET))
    det[..., 0], det[..., 1] = x1, y1
    det[..., 2] = x1 + g.uniform(0.5, 300, (n, MAX_DET))
    det[..., 3] = y1 + g.uniform(0.5, 200, (n, MAX_DET))
    det[..., 4] = g.uniform(0.01, 1, (n, MAX_DET))
    det[..., 5] = g.uniform(0.01, 1, (n, MAX_DET))
    det[..., 6] = g.integers(0, len(CLASS_IDS), (n, MAX_DET))
    sizes = np.array([(1200, 1920), (1080, 1440), (1201, 1920), (1200, 1920)], np.int32)
    hw = sizes[g.integers(0, len(sizes), n)]
    return det, count, hw


def install_stubs():
    sys.path.insert(0, os.path.join(HERE, "ref_shim"))
    sys.path.insert(0, "/root/reference")
    import yolox.utils as yu

    def xyxy2xywh(bboxes):                        # yolox 0.3.0 yolox/utils/boxes.py
        bboxes[:, 2] = bboxes[:, 2] - bboxes[:, 0]
        bboxes[:, 3] = bboxes[:, 3] - bboxes[:, 1]
        return bboxes

    yu.xyxy2xywh = xyxy2xywh
    yu.gather = lambda data, dst=0: [data]
    yu.is_main_process = lambda: True
    yu.synchronize = lambda: None
    yu.time_synchronized = lambda: 0.0
    yu.postprocess = None                         # not called: convert_to_coco_format is given NMS outputs
    for name in ("loguru", "tqdm", "tabulate"):
        try:
            __import__(name)
        except ImportError:
            m = types.ModuleType(name)
            m.logger, m.tqdm, m.tabulate = None, None, None
            sys.modules[name] = m


def reference(rule, fid, class_ids):
    """an instance of the reference evaluator with only what convert_to_coco_format reads"""
    import importlib
    mod, cls = RULES[rule]
    ev = object.__new__(getattr(importlib.import_module(f"exps.evaluators.{mod}"), cls))
    images = [{"id": i, "fid": int(f)} for i, f in enumerate(fid)]
    ds = types.SimpleNamespace(class_ids=class_ids, coco=types.SimpleNamespace(dataset={"images": images}))
    ev.dataloader = types.SimpleNamespace(dataset=ds)
    ev.img_size = IMG_SIZE
    return ev


def run(ev, det, count, hw, ids):
    outputs = [torch.from_numpy(det[i, :count[i]].copy()) if count[i] else None for i in range(len(ids))]
    info = (torch.from_numpy(hw[:, 0].copy()), torch.from_numpy(hw[:, 1].copy()))
    return ev.convert_to_coco_format(outputs, info, torch.from_numpy(ids.reshape(-1, 1).copy()))


def arrays(data_list):
    return dict(image_id=np.array([d["image_id"] for d in data_list], np.int64),
                category_id=np.array([d["category_id"] for d in data_list], np.int64),
                bbox=np.array([d["bbox"] for d in data_list], np.float64).reshape(-1, 4),
                score=np.array([d["score"] for d in data_list], np.float64))


def main():
    install_stubs()
    fid = fids()
    ids = eval_ids(fid)
    det, count, hw = batch(len(ids))
    for rule in RULES:
        ev = reference(rule, fid, CLASS_IDS)
        data_list = run(ev, det, count, hw, ids)
        assert all(d["segmentation"] == [] for d in data_list)
        table = np.full(len(ids), -1, np.int64)
        for i in range(len(ids)):
            one = run(ev, det[i:i + 1], count[i:i + 1], hw[i:i + 1], ids[i:i + 1])
            if one:
                assert len({d["image_id"] for d in one}) == 1 and len(one) == count[i]
                table[i] = one[0]["image_id"]
        path = os.path.join(GOLDEN, f"eval_coco_{rule}.npz")
        np.savez_compressed(path, det=det, count=count, hw=hw, ids=ids, fid=fid, class_ids=np.array(CLASS_IDS, np.int64),
                            img_size=np.array(IMG_SIZE, np.int64), table=table, **arrays(data_list))
        print(f"{rule}: {len(data_list)} rows from {int((count > 0).sum())} images with detections, "
              f"{int((table >= 0).sum())} kept; {path} {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
