"""Multi-scale training with CUDA graphs: one captured step per input size of ``Exp.random_resize`` (train.multiscale_sizes,
22 sizes from 496x800 to 688x1120 plus 600x960), all in one graph memory pool (Trainer.capture_sizes / replay_size).

    python tools/bench_multiscale.py [--model l] [--pairs 4] [--steps 10] [--rounds 3] [--run 200]

Each size's graph starts with the input prologue on the device: data.pair_transform of the static uint8 batch into a
600x960 staging buffer, then data.preprocess (bilinear resize + label rescale) into that size's static input.  Reported:
  * the time to capture all sizes (host clock around capture_sizes, which includes one eager warm-up step per size);
  * torch.cuda.max_memory_reserved after capturing all sizes, against capturing only the largest size (fresh Trainer,
    after empty_cache, so each figure is that configuration's own peak);
  * the replayed step time at every size (CUDA events around ``steps`` replays, best of ``rounds``);
  * ``run`` steps drawing a size every 10 steps (random.Random(seed), Exp.random_resize's formula) against ``run`` steps
    fixed at 600x960, in pairs/s (CUDA events around the whole run; arms alternate fixed, multi-scale, fixed,
    multi-scale).
The SM clock is sampled during the timed regions and the card's name / power limit are printed with the numbers.
Prints one JSON line."""
import argparse
import gc
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import bench
from bench_still import card
from streamyolo_b200 import data, synth, train

INPUT = (600, 960)
MAX_LABELS = 50


def setup(tag, pairs, sizes, dev):
    model = bench.build_model(tag, dev)
    tr = train.Trainer(model, lr=0.01 / 64 * pairs)
    frames, ann, counts, mirror = (t.to(dev) for t in synth.synth_uint8_pairs(pairs, INPUT[0], INPUT[1], seed=1))

    def labels():
        return tuple(torch.empty((pairs, MAX_LABELS, 5), dtype=torch.float32, device=dev) for _ in range(2))

    stage = (torch.empty((pairs, 6) + INPUT, dtype=torch.float32, device=dev), labels())
    # the resized inputs of all sizes are views of one buffer of the largest size (one size graph runs at a time)
    shared = torch.empty(pairs * 6 * max(h * w for h, w in sizes), dtype=torch.float32, device=dev)

    def make_inputs(s):
        return stage if s == INPUT else (shared[:pairs * 6 * s[0] * s[1]].view((pairs, 6) + s), labels())

    def prologue(s, x, targets):
        data.pair_transform(frames, ann, counts, mirror, INPUT, max_labels=MAX_LABELS, out=stage)
        data.preprocess(stage[0], stage[1], s, INPUT, out=(x, targets))

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tr.capture_sizes(sizes, make_inputs, prologue)
    torch.cuda.synchronize()
    return model, tr, time.perf_counter() - t0


def release():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def draw_sizes(n_steps, seed):
    """the size of every step when Exp.random_resize runs every 10 iterations (the first 10 steps at input_size)"""
    rng = random.Random(seed)
    size, out = INPUT, []
    f = INPUT[0] * 1.0 / INPUT[1]
    for it in range(n_steps):
        out.append(size)
        if (it + 1) % 10 == 0:
            s = rng.randint(50, 70)
            size = (16 * int(s * f), int(16 * s))
    return out


def timed_run(tr, seq):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in seq:
        losses = tr.replay_size(s)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), float(losses["total_loss"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="l", choices=["s", "m", "l"])
    ap.add_argument("--pairs", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10, help="replays per timed round at each size")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--run", type=int, default=200, help="steps of the multi-scale / fixed-size runs")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multiscale: needs a CUDA device (there is no CPU timing)")
    dev = torch.device("cuda", 0)
    sizes = train.multiscale_sizes(INPUT)
    largest = max(sizes, key=lambda s: s[0] * s[1])

    release()
    model, tr, t_one = setup(args.model, args.pairs, [largest], dev)
    mem_one = torch.cuda.max_memory_reserved()
    del model, tr
    release()
    model, tr, t_all = setup(args.model, args.pairs, sizes, dev)
    mem_all = torch.cuda.max_memory_reserved()

    clk = bench.ClockSampler(0)
    clk.start()
    per_size = {}
    for s in sizes:
        for _ in range(3):
            tr.replay_size(s)
        best = None
        for _ in range(args.rounds):
            ms, _ = timed_run(tr, [s] * args.steps)
            best = ms / args.steps if best is None else min(best, ms / args.steps)
        per_size[f"{s[0]}x{s[1]}"] = round(best, 3)
    clocks_sizes = clk.stop()

    seq = draw_sizes(args.run, args.seed)
    fixed = [INPUT] * args.run
    clk = bench.ClockSampler(0)
    clk.start()
    arms = []
    for name, sq in (("fixed", fixed), ("multiscale", seq), ("fixed", fixed), ("multiscale", seq)):
        ms, loss = timed_run(tr, sq)
        arms.append({"arm": name, "ms": round(ms, 2), "pairs_per_s": round(args.pairs * len(sq) / (ms * 1e-3), 1),
                     "last_loss": loss})
    clocks_run = clk.stop()
    expected = sum(per_size[f"{s[0]}x{s[1]}"] for s in seq)
    best = {n: max(a["pairs_per_s"] for a in arms if a["arm"] == n) for n in ("fixed", "multiscale")}
    line = {
        "metric": f"multi-scale training, StreamYOLO-{args.model}, {args.pairs} pairs, Trainer.capture_sizes / replay_size",
        "sizes": len(sizes), "capture_all_s": round(t_all, 2), "capture_largest_only_s": round(t_one, 2),
        "max_memory_reserved_all_gib": round(mem_all / 2 ** 30, 3),
        "max_memory_reserved_largest_only_gib": round(mem_one / 2 ** 30, 3),
        "memory_ratio_all_over_largest": round(mem_all / mem_one, 4),
        "step_ms_per_size": per_size, "clocks_per_size": clocks_sizes,
        "run_steps": args.run, "run_seed": args.seed,
        "run_sizes_drawn": sorted({f"{s[0]}x{s[1]}" for s in seq}),
        "pairs_per_s_fixed_600x960": best["fixed"], "pairs_per_s_multiscale": best["multiscale"],
        "multiscale_ms_expected_from_per_size": round(expected, 2), "run_arms": arms, "clocks_run": clocks_run,
        "card": card(), "data": "synthetic uint8 frames and annotations (streamyolo_b200.synth.synth_uint8_pairs)"}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
