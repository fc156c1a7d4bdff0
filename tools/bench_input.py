"""Input-transform measurement: the device pair transform (streamyolo_b200.data.pair_transform) against the host path it
replaces, and its cost inside the captured training step.

    python tools/bench_input.py [--iters 200] [--steps 20] [--rounds 6] [--out report.txt]

1. device time per 8-pair batch, raw 1200x1920 frames (load_resized_img + letterbox) and pre-resized 600x960 frames
   (letterbox only): one CUDA graph of the transform, CUDA events around ``iters`` replays after a warm-up.  Bytes moved
   = uint8 frames read once + fp32 [8, 6, 600, 960] written (+ annotations / labels), over the time, against the H100 SXM
   data-sheet 3.35 TB/s;
2. host time per pair of the same transform on one CPU core: the numpy restatement with cv2.resize (cv2.setNumThreads(1)),
   i.e. the data-loader worker's work; "not measured" without cv2;
3. the train.Trainer StreamYOLO-s 8-pair step captured as one graph, without and with the transform (raw frames) at its
   front (a second Trainer, ``prologue``), and the first Trainer with the transform replayed as a graph of its own before
   each step; ``rounds`` rounds of ``steps`` steps per arm, the order of the arms rotating from round to round.
The card's name and power limit are read in the same run.
"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from oracle import input_oracle as io
from streamyolo_b200 import data, train

SIZE, B, MAX_LABELS, HBM_TBS = (600, 960), 8, 50, 3.35


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60)
        return r.stdout.strip() or "power limit not read"
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not read"


def batch(h, w, seed):
    """8 frame pairs of uint8 h x w BGR and 12-30 annotation rows per frame in 600 x 960 coordinates, mixed mirror bits"""
    g = np.random.default_rng(seed)
    lo = g.integers(0, 256, (B, 2, h // 16 + 1, w // 16 + 1, 3)).astype(np.uint8)
    frames = np.repeat(np.repeat(lo, 16, 2), 16, 3)[:, :, :h, :w] ^ g.integers(0, 64, (B, 2, h, w, 3), dtype=np.uint8)
    m = 30
    ann = np.zeros((B, 2, m, 5))
    counts = g.integers(12, m + 1, (B, 2)).astype(np.int32)
    for i in range(B):
        for f in range(2):
            n = counts[i, f]
            x1, y1 = g.uniform(0, 900, n), g.uniform(0, 560, n)
            ann[i, f, :n] = np.stack([x1, y1, np.minimum(x1 + g.uniform(4, 200, n), 959),
                                      np.minimum(y1 + g.uniform(4, 150, n), 599), g.integers(0, 8, n)], 1)
    return np.ascontiguousarray(frames), ann, counts, (np.arange(B) % 2).astype(np.int32)


def dev(arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def device_time(raw, iters):
    h, w = (1200, 1920) if raw else SIZE
    inputs = dev(batch(h, w, seed=1))
    out = data.pair_transform(*inputs, SIZE, MAX_LABELS, raw=raw)
    g, _ = bench.capture(lambda: data.pair_transform(*inputs, SIZE, MAX_LABELS, raw=raw, out=out))
    ms = min(bench.time_replays(g, iters, warmup=10) for _ in range(3))
    moved = sum(t.numel() * t.element_size() for t in inputs) + out[0].numel() * 4 + 2 * out[1][0].numel() * 4
    return ms, moved


def host_time(raw, pairs=8):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    io.resize_linear_u8 = lambda img, dsize: cv2.resize(img, dsize, interpolation=cv2.INTER_LINEAR)
    h, w = (1200, 1920) if raw else SIZE
    frames, ann, counts, mirror = batch(h, w, seed=2)
    io.pair_transform(list(frames[0]), [ann[0, f, :counts[0, f]] for f in range(2)], SIZE, MAX_LABELS, 1, raw=raw)
    t0 = time.perf_counter()
    for i in range(pairs):
        io.pair_transform(list(frames[i]), [ann[i, f, :counts[i, f]] for f in range(2)], SIZE, MAX_LABELS, mirror[i],
                          raw=raw)
    return (time.perf_counter() - t0) * 1e3 / pairs


def trainer_step(steps, rounds):
    dev_ = torch.device("cuda", torch.cuda.current_device())
    lr = 0.01 / 64 * B
    inputs = dev(batch(1200, 1920, seed=3))
    xb, tgb = data.pair_transform(*inputs, SIZE, MAX_LABELS, raw=True)
    # every arm trains on the same images and labels (the loss's cost grows with the number of boxes)
    xs, tgs = xb.clone(), (tgb[0].clone(), tgb[1].clone())
    plain = train.Trainer(bench.build_model("s", dev_), lr=lr)
    plain.capture(xs, tgs)
    front = train.Trainer(bench.build_model("s", dev_), lr=lr)
    front.capture(xb, tgb, prologue=lambda: data.pair_transform(*inputs, SIZE, MAX_LABELS, raw=True, out=(xb, tgb)))
    # the same transform as a graph of its own writing the first trainer's static inputs, replayed before each step
    g, _ = bench.capture(lambda: data.pair_transform(*inputs, SIZE, MAX_LABELS, raw=True, out=(xs, tgs)))

    def separate():
        g.replay()
        return plain.replay()
    arms = [("without", plain.replay), ("with", front.replay), ("separate", separate)]
    res = {k: [] for k, _ in arms}

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    for i in range(rounds):                        # rotate the order: a power-capped card slows down under sustained load
        for k, fn in arms[i % 3:] + arms[:i % 3]:
            res[k].append(timed(fn))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_input: needs a CUDA device")
    lines = [f"card: {card()}", f"torch {torch.__version__}, CUDA {torch.version.cuda}", ""]
    lines.append(f"1. device pair transform, {B} pairs -> fp32 [{B}, 6, {SIZE[0]}, {SIZE[1]}] + labels [{B}, {MAX_LABELS}, 5] "
                 f"x 2; CUDA graph, best of 3 x {args.iters} replays")
    for raw in (True, False):
        ms, moved = device_time(raw, args.iters)
        gbs = moved / (ms * 1e-3) / 1e9
        tag = "raw 1200x1920 (resized to 600x960 in the kernel)" if raw else "pre-resized 600x960 (letterbox only)"
        lines.append(f"   {tag:48s} {ms * 1e3:8.1f} us/batch  {ms * 1e3 / B:6.1f} us/pair  {moved / 1e6:6.1f} MB  "
                     f"{gbs:7.1f} GB/s = {100 * gbs / (HBM_TBS * 1e3):4.1f} % of {HBM_TBS} TB/s")
    lines.append("")
    lines.append("2. host path per pair, one core (numpy restatement of DoubleTrainTransform with cv2.resize, cv2 1 thread)")
    for raw in (True, False):
        ms = host_time(raw)
        tag = "raw 1200x1920 (load_resized_img + transform)" if raw else "pre-resized 600x960 (transform)"
        lines.append(f"   {tag:48s} " + ("not measured (no cv2)" if ms is None else f"{ms:8.2f} ms/pair"))
    lines.append(f"   host cores: {os.cpu_count()}")
    lines.append("")
    res = trainer_step(args.steps, args.rounds)
    lines.append(f"3. train.Trainer StreamYOLO-s, {B} pairs 600x960; {args.rounds} rounds of {args.steps} replays per arm, "
                 "arm order rotated each round (ms/step)")
    lines.append("   without:  the step graph on static fp32 inputs")
    lines.append("   with:     a second Trainer (same model and data) whose step graph starts with the transform (prologue)")
    lines.append("   separate: the first Trainer, the transform replayed as its own graph into its static inputs before each step")
    for k, v in res.items():
        lines.append(f"   {k:9s} " + " ".join(f"{t:7.3f}" for t in v) + f"   median {sorted(v)[len(v) // 2]:7.3f}")
    for k in ("with", "separate"):
        d = sorted(b - a for a, b in zip(res["without"], res[k]))
        lines.append(f"   {k} - without, each round, sorted: " + " ".join(f"{t:+.3f}" for t in d) + " ms")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
