"""Virtual ranks (train.Trainer(virtual_ranks=K)): K ranks of a data-parallel run executed one after another in one
process, e.g. the reference's 8-rank recipe (``-d 8 -b 32``: 4 pairs per rank) on one GPU with K = 8.

    python tools/bench_virtual_ranks.py [--models l m] [--pairs 4] [--ks 1 2 8] [--steps 10] [--rounds 5]

For every model and K, one Trainer captures the whole step (K micro-steps + one optimiser step) at 600x960 on K x pairs
synthetic pairs.  Reported:
  * max_memory_reserved of each configuration: the peak while it was built and captured and replayed, minus what was
    reserved before (the earlier configurations stay alive for the alternating rounds);
  * the graphed iteration time: CUDA events around ``steps`` replays; the configurations alternate within every round,
    and the median and min-max over the rounds are given, with the time per virtual rank (iteration / K);
  * the drop-in loop (train_loop.DeviceTrainer.train_one_iter: reader thread, JPEG decode, transform, the K micro-steps,
    one graph per multi-scale size) at ``--loop-k`` virtual ranks of ``--loop-model`` over the 1200x1920 JPEG fixtures
    (tools/bench_train_loop.py's synthetic onex dataset), against DeviceStep.replay alone on a batch already on the
    device; host clock from a device synchronise to a device synchronise, legs alternating, median and min-max.
The card's name and power limit are printed with the numbers.  Prints one JSON line."""
import argparse
import gc
import json
import os
import statistics
import sys
import tempfile
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import bench
from bench_still import card
from bench_train_loop import SAMPLES, _boxes
from oracle.make_jpeg_golden import load_full
from streamyolo_b200 import synth, train, train_loop

INPUT = (600, 960)


def setup(tag, K, pairs, dev):
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    before = torch.cuda.memory_reserved()
    torch.cuda.reset_peak_memory_stats()
    n = K * pairs
    x = synth.synth_frames(n, *INPUT, seed=11).to(dev)
    tg = tuple(t.to(dev) for t in synth.synth_labels(n, *INPUT, seed=12))
    tr = train.Trainer(bench.build_model(tag, dev), lr=0.01 / 64 * pairs * K, virtual_ranks=K)
    tr.capture(x, tg)
    loss = tr.replay()["total_loss"]
    torch.cuda.synchronize()
    assert bool(torch.isfinite(loss)), (tag, K)
    return {"tr": tr, "inputs": (x, tg), "mem": torch.cuda.max_memory_reserved() - before,
            "buffer_copy_bytes": 2 * 4 * (K - 1) * tr.fs.n_buf}


def timed(tr, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        tr.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def loop_leg(tag, K, pairs, steps, rounds, dev):
    """the DeviceTrainer loop with K virtual ranks of ``pairs`` pairs over the JPEG fixtures -> {leg: [ms per round]}"""
    n = K * pairs

    class Sampler:
        batch_size = n

        def __iter__(self):
            k = 0
            while True:
                yield [(False, (k + j) % SAMPLES) for j in range(n)]
                k += n

    fixtures = load_full()
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for name in sorted(k for k in fixtures if k.endswith(".jpg") and k.startswith("f")):
            p = os.path.join(tmp, name)
            fixtures[name].tofile(p)
            paths.append(p)
        boxes = _boxes(2 * len(paths))
        ann = [(boxes[(2 * i) % len(boxes)], boxes[(2 * i + 1) % len(boxes)], (1200, 1920), (600, 960),
                paths[i % len(paths)], paths[(i + 1) % len(paths)]) for i in range(SAMPLES)]
        pre = types.SimpleNamespace(max_labels=50, trasform1=types.SimpleNamespace(flip=True, hsv=False))
        loader = types.SimpleNamespace(dataset=types.SimpleNamespace(_dataset=types.SimpleNamespace(annotations=ann),
                                                                     preproc=pre), batch_sampler=Sampler())
        tr = train.Trainer(bench.build_model(tag, dev), lr=0.01 / 64 * n, virtual_ranks=K)
        t = train_loop.DeviceTrainer()
        t.virtual_ranks, t._virtual = K, None              # the K ranks' batches arrive side by side from one sampler
        t.train_loader, t.table, t.tr, t.device, t.rank = loader, train_loop.BatchTable(loader), tr, dev, 0
        t.exp = types.SimpleNamespace(seed=0, input_size=INPUT, random_size=(60, 60))    # sizes: 592x960, 600x960
        t.max_epoch, t.start_epoch, t.max_iter, t.epoch, t.iter = 1, 0, 10 ** 9, 0, 0
        t.input_size, t._lr = INPUT, tr.lr
        t.lr_scheduler = types.SimpleNamespace(update_lr=lambda it: 0.01 / 64 * n)
        t._start_feed()
        legs = {"loop": t.train_one_iter, "replay": lambda: t.step.replay(0, INPUT, 1e-4)}

        def timed_host(fn, k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(k):
                fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / k * 1e3

        for fn in legs.values():
            timed_host(fn, 3)
        ms = {k: [] for k in legs}
        for r in range(rounds):
            for k in (list(legs) if r % 2 == 0 else list(reversed(list(legs)))):
                ms[k].append(timed_host(legs[k], steps))
        loss = float(t.step.losses["total_loss"])
        assert loss == loss, "non-finite loss"
        t._reader.shutdown(wait=True, cancel_futures=True)
        t.step.close()
        mem = torch.cuda.max_memory_reserved()
        del legs, t, tr
        gc.collect()
    return ms, mem


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["l", "m"])
    ap.add_argument("--pairs", type=int, default=4, help="frame pairs per virtual rank")
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 2, 8])
    ap.add_argument("--steps", type=int, default=10, help="replays per timed round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loop-model", default="m")
    ap.add_argument("--loop-k", type=int, default=8)
    ap.add_argument("--loop-steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_virtual_ranks: needs a CUDA device (there is no CPU timing)")
    dev = torch.device("cuda", 0)
    out = {"metric": f"virtual ranks, graphed step at {INPUT[0]}x{INPUT[1]}, {args.pairs} pairs per virtual rank",
           "card": card(), "models": {}}
    for tag in args.models:
        cfg = {K: setup(tag, K, args.pairs, dev) for K in args.ks}
        for c in cfg.values():
            for _ in range(3):
                c["tr"].replay()
        torch.cuda.synchronize()
        times = {K: [] for K in args.ks}
        clk = bench.ClockSampler(0)
        clk.start()
        for _ in range(args.rounds):
            for K in args.ks:
                times[K].append(timed(cfg[K]["tr"], args.steps))
        clocks = clk.stop()
        res = {}
        for K in args.ks:
            t = times[K]
            res[f"K={K}"] = {"iteration_ms_median": round(statistics.median(t), 3),
                             "iteration_ms_min_max": [round(min(t), 3), round(max(t), 3)],
                             "per_virtual_rank_ms_median": round(statistics.median(t) / K, 3),
                             "max_memory_reserved_gib": round(cfg[K]["mem"] / 2 ** 30, 3),
                             "extra_buffer_copies_mib": round(cfg[K]["buffer_copy_bytes"] / 2 ** 20, 3)}
        res["clocks"] = clocks
        out["models"][tag] = res
        print(json.dumps({tag: res}), flush=True)
        del cfg
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    clk = bench.ClockSampler(0)
    clk.start()
    ms, mem = loop_leg(args.loop_model, args.loop_k, args.pairs, args.loop_steps, args.rounds, dev)
    out["drop_in_loop"] = {"model": args.loop_model, "virtual_ranks": args.loop_k, "pairs_per_rank": args.pairs,
                           "steps_per_round": args.loop_steps, "clocks": clk.stop(),
                           "max_memory_reserved_gib": round(mem / 2 ** 30, 3),
                           **{f"{k}_ms_median": round(statistics.median(v), 3) for k, v in ms.items()},
                           **{f"{k}_ms_min_max": [round(min(v), 3), round(max(v), 3)] for k, v in ms.items()}}
    print(json.dumps({"drop_in_loop": out["drop_in_loop"]}), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
