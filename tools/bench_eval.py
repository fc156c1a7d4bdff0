"""Samples per second of a full validation pass (StreamYOLO-l, fp16 activation storage, synthetic weights with
BatchNorm calibrated as in tools/bench_stream.py, 600x960 input, test_conf 0.01, NMS 0.65, 8 pairs per batch) over the
1200x1920 JPEG fixtures of tests/golden/jpeg_full_*.npz cycled into a synthetic onex dataset of N samples (two files
each, written to a temporary directory).

  device  DeviceEvaluator.evaluate (streamyolo_b200/evaluate.py): files read by one host thread, decode, transform,
          forward, NMS and COCO rows in one graph replay per batch, the data_list built from the rows at the end; the
          capture at the start of the call is included (and printed on its own)
  host    the reference's loop: a DataLoader with 6 workers whose samples are cv2.imread + load_resized_img's cv2.resize
          + DoubleValTransform's preproc (pad 114, cv2.resize, HWC -> CHW fp32), pinned; model(imgs), postprocess (the
          device NMS) and convert_to_coco_format's per-detection loop (oracle/eval_oracle.py)

Both legs are timed by the host clock around the whole pass, ending in a device synchronise.  Legs alternate within
each round; every round is printed, with the median and spread, the card's name and power limit.  The two legs'
data_lists are compared in the first round.

usage: python tools/bench_eval.py [samples] [rounds] [out path]"""
import os
import statistics
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

from bench_stream import calibrated_l, card
from oracle import eval_oracle
from oracle.make_jpeg_golden import load_full
from streamyolo_b200 import evaluate
from streamyolo_b200.postprocess import postprocess

SIZE, CONF, NMS, BATCH, WORKERS = (600, 960), 0.01, 0.65, 8, 6


class Dataset(torch.utils.data.Dataset):
    """the onex val dataset's table (annotations, ids, class_ids, coco.dataset['images']); a sample is what
    DoubleValTransform returns for its two frames"""

    def __init__(self, paths, n):
        self.ids, self.class_ids = list(range(n)), list(range(8))
        self.annotations = [(None, None, (1200, 1920), None, paths[i % len(paths)], paths[(i + 1) % len(paths)])
                            for i in range(n)]
        images = [{"id": i, "fid": i % 30} for i in range(n + 2)]       # sequences of 30 frames
        self.coco = type("Coco", (), {"dataset": {"images": images}})()

    def __len__(self):
        return len(self.ids)

    def __getitem__(self, i):
        import cv2
        x = []
        for path in self.annotations[i][4:6]:
            img = cv2.imread(path)
            r = min(SIZE[0] / img.shape[0], SIZE[1] / img.shape[1])       # load_resized_img
            img = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR)
            padded = np.full((SIZE[0], SIZE[1], 3), 114, np.uint8)        # preproc
            r = min(SIZE[0] / img.shape[0], SIZE[1] / img.shape[1])
            resized = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR)
            padded[:resized.shape[0], :resized.shape[1]] = resized
            x.append(np.ascontiguousarray(padded.transpose(2, 0, 1), dtype=np.float32))
        return np.concatenate(x, 0), 0, (1200, 1920), np.array([self.ids[i]])


class Sink:
    """stand-in for the reference evaluator: keeps the data_list instead of running COCOeval"""

    def __init__(self, dataloader, img_size, confthre, nmsthre, num_classes, testdev=False, per_class_mAP=True):
        self.dataloader = dataloader

    def evaluate_prediction(self, data_dict, statistics):
        self.data_list = data_dict
        return 0, 0, ""


def host_pass(model, ds):
    loader = torch.utils.data.DataLoader(ds, batch_size=BATCH, num_workers=WORKERS, pin_memory=True)
    images = ds.coco.dataset["images"]
    data_list = []
    for imgs, _, info, ids in loader:
        with torch.no_grad():
            outputs = postprocess(model(imgs.cuda(non_blocking=True)), 8, CONF, NMS)
        data_list += eval_oracle.convert_to_coco_format(outputs, info, ids, SIZE, ds.class_ids, images, "onex")
    torch.cuda.synchronize()
    return data_list


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    out = sys.argv[3] if len(sys.argv) > 3 else None
    dev = torch.device("cuda", 0)
    model = calibrated_l(dev)
    fixtures = load_full()
    lines = [f"card: {card()}", f"torch {torch.__version__}, CUDA {torch.version.cuda}, host cores {os.cpu_count()}"]
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for name in sorted(k for k in fixtures if k.endswith(".jpg") and k.startswith("f")):     # the 1200x1920 ones
            p = os.path.join(tmp, name)
            fixtures[name].tofile(p)
            paths.append(p)
        ds = Dataset(paths, n)
        ev = evaluate.device_evaluator(Sink, "onex")(torch.utils.data.DataLoader(ds, batch_size=BATCH), SIZE, CONF, NMS, 8)
        lines.append(f"{n} samples (2 files each: {', '.join(os.path.basename(p) for p in paths)} cycled), {BATCH} pairs "
                     f"per batch, StreamYOLO-l fp16 storage, conf {CONF}, NMS {NMS}")
        for line in lines:
            print(line, flush=True)
        ev.evaluate(model)                            # warm-up: module load, first capture
        host_pass(model, Dataset(paths, 2 * BATCH))
        t = {"device": [], "host": []}
        captures = []
        for r in range(rounds):
            for leg in (("device", "host") if r % 2 == 0 else ("host", "device")):
                t0 = time.perf_counter()
                if leg == "device":
                    ev.evaluate(model)
                    torch.cuda.synchronize()
                    captures.append(ev.capture_seconds)
                else:
                    host_list = host_pass(model, ds)
                t[leg].append(time.perf_counter() - t0)
                print(f"round {r} {leg}: {t[leg][-1]:.2f} s", flush=True)
            if r == 0:
                same = ev.data_list == host_list
                lines.append(f"round 0: {len(ev.data_list)} detections; device data_list == host data_list: {same}")
                print(lines[-1], flush=True)
            host_list = None
    for leg in ("device", "host"):
        sps = [n / s for s in t[leg]]
        lines.append(f"{leg:7s} pass seconds per round {' '.join(f'{s:.2f}' for s in t[leg])}; samples/s median "
                     f"{statistics.median(sps):.1f} (min {min(sps):.1f}, max {max(sps):.1f})")
    lines.append(f"device capture at the start of each evaluate (two batch sizes when N % {BATCH} != 0): "
                 f"{' '.join(f'{c:.2f}' for c in captures)} s")
    ratio = statistics.median(t["host"]) / statistics.median(t["device"])
    lines.append(f"host / device pass time (medians): {ratio:.2f}x")
    for line in lines[-4:]:
        print(line, flush=True)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
