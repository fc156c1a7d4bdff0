"""Device JPEG decode (data.decode_jpeg) against cv2.imdecode, and its cost inside the captured training step.

    python tools/bench_decode.py [--iters 50] [--rounds 7] [--steps 10] [--out report.txt]

1. decode_jpeg of 16 full-size 1200 x 1920 fixture frames (tests/golden/jpeg_full_f*.npz, cycled; one 8-pair batch) as one
   CUDA graph: CUDA events around ``iters`` replays per round, median and spread over ``rounds`` rounds; compressed MB/s.
2. cv2.imdecode of the same files on one host core (cv2.setNumThreads(1)), or "not measured" without cv2.
3. the graphed train.Trainer step of StreamYOLO-l (4 pairs) and StreamYOLO-s (8 pairs) on static fp32 inputs ("without")
   and a second Trainer whose captured step starts with decode + pair_transform(raw=True) ("with"); ``rounds`` rounds of
   ``steps`` replays per arm, arm order alternating from round to round.
4. host-to-device bytes per pair: decoded uint8 frames against the files' bytes.
The card's name and power limit are read in the same run.
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from streamyolo_b200 import data, train
from oracle.make_jpeg_golden import load_full
from tools.bench_input import batch, card

HW, SIZE, MAX_LABELS = (1200, 1920), (600, 960), 50


def fixture_files(n):
    f = load_full()
    names = sorted(k for k in f if k.endswith(".jpg") and k.startswith("f"))
    return [f[names[i % len(names)]] for i in range(n)], [names[i % len(names)] for i in range(n)]


def packed(n):
    files, _ = fixture_files(n)
    max_bytes = max(x.size for x in files) + 64
    rows, lengths = data.pack_jpeg(files, max_bytes)
    return files, torch.from_numpy(rows).cuda(), torch.from_numpy(lengths).cuda()


def decode_time(iters, rounds, n=16):
    files, s, l = packed(n)
    out, st = data.decode_jpeg(s, l, HW)
    data.check_jpeg_status(st)
    g, _ = bench.capture(lambda: data.decode_jpeg(s, l, HW, out=out, status=st))
    per = sorted(bench.time_replays(g, iters, warmup=5) for _ in range(rounds))
    data.check_jpeg_status(st)
    return per, sum(x.size for x in files)


def host_time(n=16):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    files, _ = fixture_files(n)
    cv2.imdecode(files[0], cv2.IMREAD_COLOR)
    t0 = time.perf_counter()
    for f in files:
        cv2.imdecode(f, cv2.IMREAD_COLOR)
    return (time.perf_counter() - t0) * 1e3 / n


def trainer_step(arch, pairs, steps, rounds):
    dev_ = torch.device("cuda", torch.cuda.current_device())
    lr = 0.01 / 64 * pairs
    _, s, l = packed(2 * pairs)
    frames, st = data.decode_jpeg(s, l, HW)
    data.check_jpeg_status(st)
    _, ann, counts, mirror = batch(8, 8, seed=3)
    ann, counts, mirror = (torch.from_numpy(np.ascontiguousarray(a[:pairs])).cuda() for a in (ann, counts, mirror))
    fv = frames.view(pairs, 2, HW[0], HW[1], 3)
    xb, tgb = data.pair_transform(fv, ann, counts, mirror, SIZE, MAX_LABELS, raw=True)
    xs, tgs = xb.clone(), (tgb[0].clone(), tgb[1].clone())
    plain = train.Trainer(bench.build_model(arch, dev_), lr=lr)
    plain.capture(xs, tgs)
    front = train.Trainer(bench.build_model(arch, dev_), lr=lr)

    def prologue():
        data.decode_jpeg(s, l, HW, out=frames, status=st)
        data.pair_transform(fv, ann, counts, mirror, SIZE, MAX_LABELS, raw=True, out=(xb, tgb))
    front.capture(xb, tgb, prologue=prologue)
    arms = [("without", plain.replay), ("with", front.replay)]
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

    for i in range(rounds):                        # alternate the order: a power-capped card slows down under load
        for k, fn in (arms if i % 2 == 0 else arms[::-1]):
            res[k].append(timed(fn))
    data.check_jpeg_status(st)
    del plain, front
    torch.cuda.empty_cache()
    return res


class _Report(list):
    """report lines, printed and written to ``out`` as they come (the Trainer arms take minutes)"""

    def __init__(self, out):
        super().__init__()
        self.out = out
        if out:
            os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
            open(out, "w").close()

    def append(self, line):
        super().append(line)
        print(line, flush=True)
        if self.out:
            with open(self.out, "a") as fh:
                fh.write(line + "\n")

    def extend(self, lines):
        for line in lines:
            self.append(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode: needs a CUDA device")
    lines = _Report(args.out)
    lines.extend([f"card: {card()}", f"torch {torch.__version__}, CUDA {torch.version.cuda}", ""])
    per, nbytes = decode_time(args.iters, args.rounds)
    med = per[len(per) // 2]
    _, names = fixture_files(16)
    lines.append(f"1. decode_jpeg, 16 frames 1200x1920 (one 8-pair batch; fixtures {sorted(set(names))} cycled), "
                 f"{nbytes / 1e6:.2f} MB of files; CUDA graph, {args.rounds} rounds x {args.iters} replays")
    lines.append("   per round, sorted: " + " ".join(f"{t:.3f}" for t in per) + " ms")
    lines.append(f"   median {med:.3f} ms/batch ({med / 16 * 1e3:.1f} us/frame), spread {per[-1] - per[0]:.3f} ms, "
                 f"{nbytes / 1e6 / (med * 1e-3):.0f} MB/s compressed")
    lines.append("")
    ms = host_time()
    lines.append("2. cv2.imdecode of the same files, one host core (cv2.setNumThreads(1)): " +
                 ("not measured (no cv2)" if ms is None else f"{ms:.2f} ms/frame") + f"; host cores: {os.cpu_count()}")
    lines.append("")
    lines.append(f"3. train.Trainer step graph, 600x960; {args.rounds} rounds of {args.steps} replays per arm, order "
                 "alternating (ms/step)")
    lines.append("   without: static fp32 inputs;  with: a second Trainer whose step graph starts with decode_jpeg + "
                 "pair_transform(raw=True)")
    for arch, pairs in (("l", 4), ("s", 8)):
        res = trainer_step(arch, pairs, args.steps, args.rounds)
        lines.append(f"   StreamYOLO-{arch}, {pairs} pairs ({2 * pairs} frames)")
        for k, v in res.items():
            lines.append(f"     {k:8s} " + " ".join(f"{t:7.3f}" for t in v) + f"   median {sorted(v)[len(v) // 2]:7.3f}")
        d = sorted(b - a for a, b in zip(res["without"], res["with"]))
        lines.append("     with - without, each round, sorted: " + " ".join(f"{t:+.3f}" for t in d) +
                     f" ms; median {d[len(d) // 2]:+.3f} ms")
    lines.append("")
    files, _ = fixture_files(16)
    per_pair = 2 * np.mean([f.size for f in files])
    lines.append(f"4. host-to-device bytes per pair: decoded frames 2 x {HW[0]}x{HW[1]}x3 = {2 * HW[0] * HW[1] * 3 / 1e6:.2f} MB; "
                 f"files {per_pair / 1e6:.2f} MB (mean of the fixtures; the padded rows of pack_jpeg copy max_bytes each)")


if __name__ == "__main__":
    main()
