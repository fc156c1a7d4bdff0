"""Training step of the still-image baseline (cfgs/l_s50_still_dfp_flip.py: YOLOX(DFPPAFPN, PIPEHead) on single frames):
one backbone + PAFPN pass per frame against the reference's duplicated pair.

    python tools/bench_still.py [--model l] [--batch 8] [--steps 10] [--rounds 5]

Both arms are train.Trainer replaying one CUDA graph of the whole step on the same model and B frames:
  single  x [B, 3, H, W]: one pass over B images, each BatchNorm's running update applied twice (model/backward.py)
  pair    cat(x, x) [B, 6, H, W]: the reference's arithmetic, two passes batched as 2B images with grouped statistics
Each arm: CUDA events around ``steps`` replays, best of ``rounds``; the arms run single, pair, single (one at a time: two
Trainers of StreamYOLO-l hold two sets of graphs and activations).  The SM clock is sampled during the timed rounds and the
card's name / power limit are printed with the numbers.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from streamyolo_b200 import synth, train


# BASELINE.md's algorithmic table: one backbone + PAFPN pass of StreamYOLO-l is 384.30 - 219.4 = 165 of the 384.30 forward
# conv GFLOP of a pair step, and the backward has the same share
PREDICTION = {"l": "saving ~0.43 of the conv work (FLOP share, not a time)"}


def build_still(tag, device):
    from streamyolo_b200.model import DFPPAFPN, PIPEHead, YOLOX
    depth, width = bench.MODELS[tag]
    ch = [256, 512, 1024]
    model = YOLOX(DFPPAFPN(depth, width, in_channels=ch), PIPEHead(8, width, in_channels=ch))
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eps, m.momentum = 1e-3, 0.03
    model.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}))
    model.head.use_l1 = True
    return model.to(device).train()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # noqa: BLE001
        out = f"nvidia-smi unavailable: {e}"
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": out}


def time_arm(tag, x, labels, steps, rounds, warmup, dev):
    model = build_still(tag, dev)
    tr = train.Trainer(model, lr=0.01 / 64 * x.shape[0])
    tr.capture(x, labels)
    for _ in range(warmup):
        losses = tr.replay()
    torch.cuda.synchronize()
    clk = bench.ClockSampler(0)
    clk.start()
    times = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            losses = tr.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / steps)
    clocks = clk.stop()
    out = {"ms_per_step_best": round(min(times), 3), "ms_per_step_rounds": [round(t, 3) for t in times],
           "loss": float(losses["total_loss"]), "clocks": clocks}
    del tr, model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="l", choices=["s", "m", "l"])
    ap.add_argument("--batch", type=int, default=8, help="frames")
    ap.add_argument("--steps", type=int, default=10, help="graph replays per timed round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_still: needs a CUDA device (there is no CPU timing)")
    dev = torch.device("cuda", 0)
    x = synth.synth_frames(args.batch, 600, 960, seed=1234)[:, :3].contiguous().to(dev)
    labels = synth.synth_labels(args.batch, 600, 960, seed=1)[0].to(dev)
    x6 = torch.cat([x, x], 1)
    arms = []
    for name, inp in (("single", x), ("pair", x6), ("single", x)):
        r = time_arm(args.model, inp, labels, args.steps, args.rounds, args.warmup, dev)
        r["arm"] = name
        arms.append(r)
    single, pair = arms[0]["ms_per_step_best"], arms[1]["ms_per_step_best"]     # arms[2]: the repeat, for the spread
    line = {
        "metric": f"ms per training step, StreamYOLO-{args.model} still model (PIPEHead) 600x960, {args.batch} frames, Trainer graph",
        "single_pass_ms": single, "duplicated_pair_ms": pair, "single_pass_repeat_ms": arms[2]["ms_per_step_best"], "saving": round(1.0 - single / pair, 4),
        "frames_per_s_single": round(args.batch / (single * 1e-3), 1), "frames_per_s_pair": round(args.batch / (pair * 1e-3), 1),
        "flop_share_prediction": PREDICTION.get(args.model),
        "arms": arms, "steps": args.steps, "rounds": args.rounds, "warmup": args.warmup, "card": card(),
        "data": "synthetic frames and labels (streamyolo_b200.synth)"}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
