"""SiLU against ReLU and LeakyReLU(0.1): the same StreamYOLO-l workloads built with each ``act``, timed alternately.

    python tools/bench_act.py [--rounds 5] [--steps 10] [--out profiles/h100_activations.txt]

Per round, for each activation in turn (silu, relu, lrelu, so that clock and neighbour drift spread over all three):
  * train   the 4-pair training step captured as one CUDA graph (Trainer.capture / replay), 600x960;
  * eval    the 8-pair eval forward (off_pipe, bf16 storage) as one CUDA graph;
  * stream  one StreamDetector tick (one 1200x1920 camera stream: frame copy in, replay, detections out), fp16 storage.
CUDA events around ``--steps`` calls after warm-up (the tick: a host clock around calls that end in a synchronise); medians
and min-max spreads over the rounds.  Each (round, activation) runs in a process of its own (``--one ACT``), which builds
and captures its three workloads and prints one JSON line.  Prints the table with the GPU name and power limit, and
writes it to ``--out``."""
import json
import argparse
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from streamyolo_b200 import stream, synth, train
from streamyolo_b200.model import DFPPAFPN, TALHead, YOLOX

ACTS = ("silu", "relu", "lrelu")
FRAME_HW, IN_SCALE = (1200, 1920), 0.5


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def build(act, dev):
    """bench.build_model("l") with every BaseConv's activation set to ``act``"""
    depth, width = bench.MODELS["l"]
    gamma, thr, val = bench.TAL["l"]
    ch = [256, 512, 1024]
    m = YOLOX(DFPPAFPN(depth, width, in_channels=ch, act=act),
              TALHead(8, width, in_channels=ch, act=act, gamma=gamma, ignore_thr=thr, ignore_value=val))
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, 0.03
    m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}))
    m.head.use_l1 = True
    return m.to(dev).train()


def calibrated(act, dev, x, tg):
    m = build(act, dev)
    bns = [b for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d)]
    with torch.no_grad():
        for b in bns:
            b.momentum = 1.0
        m(x, tg)                                        # running statistics := batch statistics
        for b in bns:
            b.momentum = 0.03
    return m.eval()


def measure(act, steps):
    """the three workloads of one activation, in this process"""
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    x4 = synth.synth_frames(4, 600, 960, seed=1234).to(dev)
    tg4 = tuple(t.to(dev) for t in synth.synth_labels(4, 600, 960, seed=1))
    x8 = synth.synth_frames(8, 600, 960, seed=99).to(dev)
    tg8 = tuple(t.to(dev) for t in synth.synth_labels(8, 600, 960, seed=11))
    frames = synth.synth_frames(4, *FRAME_HW, seed=5)[:, :3].permute(0, 2, 3, 1).round().clamp(0, 255).to(torch.uint8)
    frames = [np.ascontiguousarray(f.numpy()) for f in frames]

    def time_train(tr):
        for _ in range(3):
            tr.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            tr.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    def time_tick(det):
        for i in range(3):
            det.step(frames[i % 4])
        ts = []
        for i in range(steps):
            t0 = time.perf_counter()
            det.step(frames[i % 4])                    # copies in, replay, copies out, one synchronise
            ts.append((time.perf_counter() - t0) * 1e3)
        return statistics.median(ts)

    tr = train.Trainer(build(act, dev), lr=0.01 / 64 * 4)
    tr.capture(x4, tg4)
    out = {"train": time_train(tr)}
    del tr
    ev_model = calibrated(act, dev, x8, tg8)
    g_eval, keep = bench.capture(lambda: ev_model(x8))          # (the output stays referenced while the graph lives)
    out["eval"] = bench.time_replays(g_eval, steps)
    del g_eval, keep
    ev_model.activation_dtype = torch.float16
    out["stream"] = time_tick(stream.StreamDetector(ev_model, FRAME_HW, IN_SCALE, streams=1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--one", choices=ACTS, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.one:
        print(json.dumps(measure(args.one, args.steps)))
        return
    res = {a: {"train": [], "eval": [], "stream": []} for a in ACTS}
    for _ in range(args.rounds):
        for act in ACTS:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", act, "--steps", str(args.steps)],
                               capture_output=True, text=True, check=True)
            for k, v in json.loads(r.stdout.strip().splitlines()[-1]).items():
                res[act][k].append(v)
    lines = [f"card (name, power limit, max SM clock): {card()}",
             f"StreamYOLO-l, synthetic weights and frames; {args.rounds} rounds, activations alternating within each round "
             "(one process per round and activation); "
             f"{args.steps} calls per measurement",
             "train  = 4-pair training step (600x960), one CUDA graph replay (Trainer.replay)",
             "eval   = 8-pair eval forward (off_pipe, bf16 storage), one CUDA graph replay",
             "stream = one StreamDetector tick, 1 stream of 1200x1920 frames, fp16 storage (host clock, median per round)",
             "",
             f"{'act':6s} {'workload':7s} {'median ms':>10s} {'min':>8s} {'max':>8s}  {'vs silu':>8s}"]
    for wl in ("train", "eval", "stream"):
        base = statistics.median(res["silu"][wl])
        for act in ACTS:
            v = res[act][wl]
            med = statistics.median(v)
            lines.append(f"{act:6s} {wl:7s} {med:10.3f} {min(v):8.3f} {max(v):8.3f}  {med / base:8.3f}x")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
