"""The drop-in training loop (streamyolo_b200/train_loop.py) against the same graphs with feeding taken out, and the
non-finite gradient guard on against off.  StreamYOLO-l, 4 pairs, a fixed 600x960 input, over the 1200x1920 JPEG
fixtures of tests/golden/jpeg_full_f*.npz cycled into a synthetic onex dataset (two files per sample, written to a
temporary directory; labels: 6 boxes per frame).

  loop      DeviceTrainer.train_one_iter: the reader thread's np.fromfile into the pinned slot, the copy-stream H2D, the
            replay (decode, transform, step), the lr schedule; iterations as the drop-in runs them
  replay    the same DeviceStep.replay on a batch already in its device slot: the loop with feeding taken out
  guard     ``replay`` on a second Trainer built with skip_nonfinite=True (sy_nonfinite_flag + the skip-with-EMA step)
  host      the loop the reference's tools/train.py runs with install() alone: a DataLoader with 6 workers whose samples
            are cv2.imread + load_resized_img's cv2.resize + DoubleTrainTransform (mirror, preproc's pad 114 and
            cv2.resize, HWC -> CHW fp32, padded cxcywh labels), pinned and copied to the device, then the autograd step
            (``model(inps, targets)``, ``backward``), train.build_optimizer's torch SGD and train.ModelEMA

Each leg runs ``steps`` iterations, timed by the host clock from a device synchronise to a device synchronise; legs
alternate within a round, rounds alternate their order.  Prints every round, then medians and spread, with the card's
name and power limit.

usage: python tools/bench_train_loop.py [steps] [rounds] [out path]"""
import gc
import os
import statistics
import sys
import tempfile
import time
import types

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

import bench
from bench_still import card
from oracle.make_jpeg_golden import load_full
from streamyolo_b200 import train, train_loop

INPUT, PAIRS, SAMPLES, WORKERS, MAX_LABELS = (600, 960), 4, 256, 6, 50


def _boxes(n):
    rng = np.random.default_rng(0)
    out = []
    for _ in range(n):
        x1, y1 = rng.uniform(0, 700, 6), rng.uniform(0, 400, 6)
        out.append(np.stack([x1, y1, x1 + rng.uniform(20, 200, 6), y1 + rng.uniform(20, 150, 6),
                             rng.integers(0, 8, 6).astype(np.float64)], 1))
    return out


class HostDataset(torch.utils.data.Dataset):
    """what the onex dataset + DoubleTrainTransform hand the reference's DataLoader, with cv2 as the reference runs it"""

    def __init__(self, paths, boxes):
        self.paths, self.boxes = paths, boxes

    def __len__(self):
        return 10 ** 6

    def _frame(self, path, boxes, mirror):
        import cv2
        img = cv2.imread(path)
        r = min(INPUT[0] / img.shape[0], INPUT[1] / img.shape[1])                 # load_resized_img
        img = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR)
        b = boxes[:, :4].copy()
        if mirror:                                                                  # _mirror
            img = img[:, ::-1]
            b[:, 0::2] = img.shape[1] - b[:, 2::-2]
        padded = np.full((INPUT[0], INPUT[1], 3), 114, np.uint8)                   # preproc
        r = min(INPUT[0] / img.shape[0], INPUT[1] / img.shape[1])
        resized = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR)
        padded[:resized.shape[0], :resized.shape[1]] = resized
        x = np.ascontiguousarray(padded.transpose(2, 0, 1), dtype=np.float32)
        lab = np.zeros((MAX_LABELS, 5), np.float32)
        cxcywh = np.stack([(b[:, 0] + b[:, 2]) / 2, (b[:, 1] + b[:, 3]) / 2, b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]], 1) * r
        lab[:len(b), 0], lab[:len(b), 1:] = boxes[:, 4], cxcywh
        return x, lab

    def __getitem__(self, i):
        import random
        a = random.randrange(2)
        k = i % SAMPLES
        x0, l0 = self._frame(self.paths[k % len(self.paths)], self.boxes[(2 * k) % len(self.boxes)], a)
        x1, l1 = self._frame(self.paths[(k + 1) % len(self.paths)], self.boxes[(2 * k + 1) % len(self.boxes)], a)
        return np.concatenate((x0, x1), 0), (l0, l1), (1200, 1920), np.array([k])


def host_leg(paths, dev):
    """one iteration of the reference loop per call: next batch, H2D, autograd step, torch SGD, ModelEMA"""
    model = bench.build_model("l", dev)
    opt = train.build_optimizer(model, 0.01 / 64 * PAIRS)
    ema = train.ModelEMA(model)
    loader = torch.utils.data.DataLoader(HostDataset(paths, _boxes(2 * len(paths))), batch_size=PAIRS,
                                         num_workers=WORKERS, pin_memory=True)
    batches = iter(loader)

    def step():
        inps, (fut, cur), _, _ = next(batches)
        inps = inps.to(dev, non_blocking=True)
        targets = (fut.to(dev, non_blocking=True), cur.to(dev, non_blocking=True))
        loss = model(inps, targets)["total_loss"]
        opt.zero_grad()
        loss.backward()
        opt.step()
        ema.update(model)

    return step


class Sampler:
    batch_size = PAIRS

    def __iter__(self):
        k = 0
        while True:
            yield [(False, (k + j) % SAMPLES) for j in range(PAIRS)]
            k += PAIRS


def loop_for(tr, paths, dev):
    """a DeviceTrainer driven without the reference class: only the attributes train_one_iter reads"""
    boxes = _boxes(2 * len(paths))
    ann = [(boxes[(2 * i) % len(boxes)], boxes[(2 * i + 1) % len(boxes)], (1200, 1920), (600, 960),
            paths[i % len(paths)], paths[(i + 1) % len(paths)]) for i in range(SAMPLES)]
    pre = types.SimpleNamespace(max_labels=50, trasform1=types.SimpleNamespace(flip=True, hsv=False))
    loader = types.SimpleNamespace(dataset=types.SimpleNamespace(_dataset=types.SimpleNamespace(annotations=ann),
                                                                 preproc=pre), batch_sampler=Sampler())
    t = train_loop.DeviceTrainer()
    t.train_loader, t.table, t.tr, t.device, t.rank = loader, train_loop.BatchTable(loader), tr, dev, 0
    t.exp = types.SimpleNamespace(seed=0, input_size=INPUT, random_size=(60, 60))        # sizes: 592x960, 600x960
    t.max_epoch, t.start_epoch, t.max_iter, t.epoch, t.iter = 1, 0, 10 ** 9, 0, 0
    t.input_size, t._lr = INPUT, tr.lr
    t.lr_scheduler = types.SimpleNamespace(update_lr=lambda it: 0.01 / 64 * PAIRS)
    t._start_feed()
    return t


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    out = sys.argv[3] if len(sys.argv) > 3 else None
    dev = torch.device("cuda", 0)
    fixtures = load_full()
    lines = [f"card: {card()}", f"torch {torch.__version__}, CUDA {torch.version.cuda}, host cores {os.cpu_count()}"]
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for name in sorted(k for k in fixtures if k.endswith(".jpg") and k.startswith("f")):     # the 1200x1920 ones
            p = os.path.join(tmp, name)
            fixtures[name].tofile(p)
            paths.append(p)
        lines.append(f"StreamYOLO-l, {PAIRS} pairs, {INPUT[0]}x{INPUT[1]}, {SAMPLES} samples cycling "
                     f"{', '.join(os.path.basename(p) for p in paths)}; {steps} iterations per leg")
        for line in lines:
            print(line, flush=True)
        legs = {}
        for guard in (False, True):
            tr = train.Trainer(bench.build_model("l", dev), lr=0.01 / 64 * PAIRS, skip_nonfinite=guard)
            t = loop_for(tr, paths, dev)
            if guard:
                legs["guard"] = lambda t=t: t.step.replay(0, INPUT, 1e-4)
            else:
                legs["loop"] = t.train_one_iter
                legs["replay"] = lambda t=t: t.step.replay(0, INPUT, 1e-4)
            if guard:
                skipper = tr
        legs["host"] = host_leg(paths, dev)
        for fn in legs.values():
            timed(fn, 10)                                           # warm-up
        ms = {k: [] for k in legs}
        for r in range(rounds):
            order = list(legs) if r % 2 == 0 else list(reversed(list(legs)))
            for k in order:
                ms[k].append(timed(legs[k], steps))
                print(f"round {r} {k}: {ms[k][-1]:.3f} ms/iteration", flush=True)
        assert skipper.skipped_steps() == 0
        del legs                                                    # the host leg's workers stop before the files go
        gc.collect()
    med = {k: statistics.median(v) for k, v in ms.items()}
    for k, v in ms.items():
        lines.append(f"{k:7s} ms/iteration per round {' '.join(f'{x:.3f}' for x in v)}; median {med[k]:.3f} "
                     f"(min {min(v):.3f}, max {max(v):.3f})")
    lines.append(f"loop / replay (medians): {med['loop'] / med['replay']:.4f}; guard / replay: "
                 f"{med['guard'] / med['replay']:.4f}; host / loop: {med['host'] / med['loop']:.3f}")
    for line in lines[-5:]:
        print(line, flush=True)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
