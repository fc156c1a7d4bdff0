"""bf16 vs fp16 activation storage (``model.activation_dtype``) of the inference forwards, timed in one process:
eval off_pipe of StreamYOLO-l at 8 frame pairs and on_pipe streaming at batch 1 (one 600x960 frame, the feature buffer
carried over), each as a CUDA graph timed with CUDA events, the two storage types alternating for ``rounds`` rounds so that
clock and neighbour drift hit both alike.  The model's running statistics are calibrated by one train pass (BatchNorm
momentum 1) so that the activations have the scale of a trained network.  Prints the card name and power limit, one line
per (round, mode, storage), and the medians.   usage: python tools/bench_storage.py [rounds] [steps]"""
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from streamyolo_b200 import synth

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
STEPS = int(sys.argv[2]) if len(sys.argv) > 2 else 30
PAIRS = 8
STORAGE = {"bf16": torch.bfloat16, "fp16": torch.float16}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return q


def main():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card (name, power limit, max SM clock):", card())
    model = bench.build_model("l", dev)
    x = synth.synth_frames(PAIRS, 600, 960, seed=99).to(dev)
    xc = torch.cat([x[:, 0:3], x[:, 0:3]], 1)
    tg = tuple(t.to(dev) for t in synth.synth_labels(PAIRS, 600, 960, seed=11))
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    mom = [m.momentum for m in bns]
    with torch.no_grad():
        for m in bns:
            m.momentum = 1.0
        model.train()
        model(xc, tg)                                # running statistics := batch statistics
        for m, v in zip(bns, mom):
            m.momentum = v
    model.eval()
    f = synth.synth_frames(1, 600, 960, seed=98)[:, :3].contiguous().to(dev)
    graphs = {}
    with torch.no_grad():
        for name, dt in STORAGE.items():
            model.activation_dtype = dt
            g_eval, out = bench.capture(lambda: model(xc))
            _, buf = model(f, mode="on_pipe")
            buf_static = tuple(b.clone() for b in buf)

            def frame():
                o, nb = model(f, buffer=buf_static, mode="on_pipe")
                for d_, s_ in zip(buf_static, nb):
                    d_.copy_(s_)
                return o
            g_pipe, o = bench.capture(frame)
            assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(o).all()), name
            graphs[name] = {"eval": g_eval, "on_pipe": g_pipe}
    times = {(mode, name): [] for mode in ("eval", "on_pipe") for name in STORAGE}
    for r in range(ROUNDS):
        for mode in ("eval", "on_pipe"):
            for name in (list(STORAGE) if r % 2 == 0 else list(STORAGE)[::-1]):
                ms = bench.time_replays(graphs[name][mode], STEPS)
                times[(mode, name)].append(ms)
                print(f"round {r} {mode:8s} {name}: {ms:.4f} ms")
    print("medians over", ROUNDS, "rounds x", STEPS, "replays:")
    for mode, unit in (("eval", f"ms per step ({PAIRS} pairs)"), ("on_pipe", "ms per frame (batch 1)")):
        mb, mf = statistics.median(times[(mode, "bf16")]), statistics.median(times[(mode, "fp16")])
        spread = {n: max(times[(mode, n)]) - min(times[(mode, n)]) for n in STORAGE}
        print(f"  {mode:8s} {unit}: bf16 {mb:.4f}, fp16 {mf:.4f}, fp16 / bf16 {mf / mb:.4f} "
              f"(spread bf16 {spread['bf16']:.4f}, fp16 {spread['fp16']:.4f})")


if __name__ == "__main__":
    main()
