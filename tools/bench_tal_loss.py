"""sy_tal_loss of two builds of the library, timed alternately at the benchmarked shape (600x960, A = 11 850, B = 16,
120 label rows, 8 classes, 12 synthetic ground truths per image, the outputs of tests/test_gpu_parity_l.py).

    python tools/bench_tal_loss.py LIB_A LIB_B [--rounds 7] [--iters 200] [--out FILE]

Per round, each library in turn: CUDA events around ``--iters`` back-to-back sy_tal_loss calls after a warm-up.  Prints the
median and min-max per-call time over the rounds with the GPU name and power limit, checks that both builds give the
same foreground and matched GT ids on these outputs, and writes the table to ``--out``."""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from streamyolo_b200 import ops
from test_gpu_parity_l import A_TOTAL, HW, STRIDES, _labels, _synthetic_head_outputs


def load(path):
    ops._lib, ops.LIB_PATH = None, os.path.abspath(path)
    return ops.load_library()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs=2)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out")
    a = ap.parse_args()
    libs = [load(p) for p in a.libs]
    b = 16
    fut, cur = _labels(b, 12, 19)
    outputs, origin = _synthetic_head_outputs(b, fut, 23)
    dev = "cuda"
    od, ogd, fd, cd = outputs.to(dev), origin.to(dev), fut.to(dev), cur.to(dev)
    ws = torch.empty(ops.tal_loss_workspace_bytes(b, A_TOTAL, 120, 8), dtype=torch.uint8, device=dev)
    loss = torch.empty(6, device=dev)
    res = []
    for lib in libs:
        ops._lib = lib
        fg = torch.empty((b, A_TOTAL), dtype=torch.int32, device=dev)
        mt = torch.empty((b, A_TOTAL), dtype=torch.int32, device=dev)
        ops.tal_loss(od, ogd, fd, cd, HW, STRIDES, 1.0, 0.5, 1.6, True, ws, loss, fg, mt)
        torch.cuda.synchronize()
        res.append((fg.cpu(), mt.cpu(), loss.cpu()))
    same = torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    times = [[], []]
    for _ in range(a.rounds):
        for i, lib in enumerate(libs):
            ops._lib = lib
            for _ in range(20):
                ops.tal_loss(od, ogd, fd, cd, HW, STRIDES, 1.0, 0.5, 1.6, True, ws, loss)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                ops.tal_loss(od, ogd, fd, cd, HW, STRIDES, 1.0, 0.5, 1.6, True, ws, loss)
            e1.record()
            torch.cuda.synchronize()
            times[i].append(e0.elapsed_time(e1) * 1000.0 / a.iters)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    lines = [f"sy_tal_loss, 600x960, A = {A_TOTAL}, B = {b}, 120 label rows (12 GTs / image), 8 classes; {gpu}",
             f"{a.rounds} alternating rounds x {a.iters} calls, CUDA events; per call [us]: median (min - max)"]
    for p, t in zip(a.libs, times):
        lines.append(f"  {p:50s} {statistics.median(t):8.2f} ({min(t):.2f} - {max(t):.2f})")
    lines.append(f"same foreground and matched ids: {same}; losses {res[0][2].tolist()} / {res[1][2].tolist()}")
    print("\n".join(lines))
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
