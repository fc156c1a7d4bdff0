"""Training step at 8 and at 80 classes (COCO's count), and the 80-class prediction-conv backward on its own.

    python tools/bench_classes.py [--model l] [--pairs 4] [--frames 8] [--steps 10] [--rounds 5]

Step arms: train.Trainer replaying one CUDA graph of the whole step of StreamYOLO-<model> at 600x960, synthetic frames and
labels (labels drawn from all of the model's classes): the pair model on ``--pairs`` pairs and the still model
(PIPEHead) on ``--frames`` frames, each at 8 and at 80 classes, one arm at a time.  CUDA events around ``steps`` replays,
best of ``rounds``.  Up to 27 classes the walk runs sy_head_pred_backward; above, sy_head_pred_backward_wide.

Kernel arm: the three head levels of the pair step (``--pairs`` images, 600x960) of sy_head_pred_backward_wide at 80
classes, and of both entry points at 8 classes, captured as one CUDA graph per arm and replayed.  Bytes are the compulsory
traffic of one launch triple: gradient rows read, both tower outputs read, both data gradients written, fp32 partial rows
written and read back, weights read, weight gradients written.  The SM clock is sampled during the timed rounds and the
card's name / power limit are printed with the numbers.  Prints one JSON line."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from streamyolo_b200 import ops, synth, train
from streamyolo_b200.ops import View
from tools.bench_still import card

HBM_BYTES_PER_S = 3.35e12          # H100 SXM5 80GB HBM3, data sheet
HW = [(75, 120), (38, 60), (19, 30)]


def build(tag, nc, still, device):
    from streamyolo_b200.model import DFPPAFPN, PIPEHead, TALHead, YOLOX
    depth, width = bench.MODELS[tag]
    gamma, thr, val = bench.TAL[tag]
    ch = [256, 512, 1024]
    head = PIPEHead(nc, width, in_channels=ch) if still else TALHead(nc, width, in_channels=ch, gamma=gamma,
                                                                       ignore_thr=thr, ignore_value=val)
    model = YOLOX(DFPPAFPN(depth, width, in_channels=ch), head)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eps, m.momentum = 1e-3, 0.03
    model.head.initialize_biases(1e-2)
    model.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}))
    model.head.use_l1 = True
    return model.to(device).train()


def timed(fn, steps, rounds, warmup):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    clk = bench.ClockSampler(0)
    clk.start()
    times = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            out = fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / steps)
    return min(times), times, clk.stop(), out


def step_arm(tag, nc, still, n, args, dev):
    model = build(tag, nc, still, dev)
    x = synth.synth_frames(n, 600, 960, seed=1234).to(dev)
    fut, cur = (t.to(dev) for t in synth.synth_labels(n, 600, 960, seed=1, num_classes=nc))
    if still:
        x, labels = x[:, :3].contiguous(), fut
    else:
        labels = (fut, cur)
    tr = train.Trainer(model, lr=0.01 / 64 * n)
    tr.capture(x, labels)
    best, times, clocks, losses = timed(tr.replay, args.steps, args.rounds, args.warmup)
    out = {"arm": ("still" if still else "pair") + f"_{nc}_classes", "images": n, "ms_per_step_best": round(best, 3),
           "ms_per_step_rounds": [round(t, 3) for t in times], "loss": float(losses["total_loss"]), "clocks": clocks}
    del tr, model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return out


def kernel_arm(fn, nc, b, c, args, dev):
    g = torch.Generator(device=dev).manual_seed(3)
    a_total = sum(h * w for h, w in HW)
    grad_raw = torch.randn((b, a_total, 5 + nc), generator=g, device=dev) * 1e-3
    ws = [torch.randn((o, c), generator=g, device=dev) * 0.05 for o in (4, 1, nc)]
    dws = [torch.empty((o, c), device=dev) for o in (4, 1, nc)]
    dbs = [torch.empty((o,), device=dev) for o in (4, 1, nc)]
    levels, off, nbytes = [], 0, 0
    for h, w in HW:
        feats = [View((torch.randn((b, h, w, c), generator=g, device=dev)).to(torch.bfloat16)) for _ in range(2)]
        grads = [View.empty(b, h, w, c, dev) for _ in range(2)]
        levels.append((feats, grads, off))
        p = b * h * w
        rows = -(-p // 256)
        nbytes += p * (5 + nc) * 4 + 4 * p * c * 2 + 2 * rows * (5 + nc) * (c + 1) * 4 + 2 * (5 + nc) * (c + 1) * 4
        off += h * w

    def launch():
        for (cf, rf), (dcf, drf), o in levels:
            fn(grad_raw, cf, rf, dcf, drf, *ws, a_total, o, *dws, *dbs, accumulate=True)

    graph, _ = bench.capture(launch)
    best, times, clocks, _ = timed(graph.replay, args.steps * 10, args.rounds, args.warmup)
    return {"arm": f"{fn.__name__}_{nc}_classes", "images": b, "channels": c, "us_best": round(best * 1e3, 1),
            "us_rounds": [round(t * 1e3, 1) for t in times], "compulsory_bytes": nbytes,
            "bytes_per_s": round(nbytes / (best * 1e-3) / 1e12, 3), "fraction_of_3.35_TB_s": round(nbytes / (best * 1e-3) / HBM_BYTES_PER_S, 3),
            "clocks": clocks}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="l", choices=["s", "m", "l"])
    ap.add_argument("--pairs", type=int, default=4)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10, help="graph replays per timed round (x10 for the kernel arms)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_classes: needs a CUDA device (there is no CPU timing)")
    dev = torch.device("cuda", 0)
    steps = [step_arm(args.model, nc, still, args.frames if still else args.pairs, args, dev)
             for still in (False, True) for nc in (8, 80)]
    c = int(256 * bench.MODELS[args.model][1])
    kernels = [kernel_arm(ops.head_pred_backward_wide, 80, args.pairs, c, args, dev),
               kernel_arm(ops.head_pred_backward_wide, 8, args.pairs, c, args, dev),
               kernel_arm(ops.head_pred_backward, 8, args.pairs, c, args, dev)]
    ms = {s["arm"]: s["ms_per_step_best"] for s in steps}
    line = {
        "metric": f"ms per training step, StreamYOLO-{args.model} 600x960, 8 vs 80 classes, Trainer graph; "
                  f"prediction-conv backward of the {args.pairs}-pair step",
        "pair_8_ms": ms["pair_8_classes"], "pair_80_ms": ms["pair_80_classes"],
        "still_8_ms": ms["still_8_classes"], "still_80_ms": ms["still_80_classes"],
        "wide_80_us": kernels[0]["us_best"], "wide_80_TB_s": kernels[0]["bytes_per_s"],
        "steps": steps, "kernels": kernels, "rounds": args.rounds, "warmup": args.warmup, "card": card(),
        "data": "synthetic frames and labels (streamyolo_b200.synth)"}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
