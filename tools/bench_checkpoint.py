"""Time to save and to load the whole training state of a Trainer (train.Trainer.state_dict / load_state_dict): the
weights with the BatchNorm buffers, the momentum and the EMA copy, three flat fp32 buffers of ~219 MB each for StreamYOLO-l.

    python tools/bench_checkpoint.py [--model l] [--rounds 5]

One eager training step (1 pair, 600x960) runs first, so that the momentum is part of the state.  Each round, on a host
clock with a device synchronise at both ends:
  save         torch.save(tr.state_dict(), file)   the device->host copies happen inside torch.save; the file is in a
                                                   temporary directory, written without fsync (as the reference's
                                                   save_checkpoint does)
  save_memory  the same into an io.BytesIO         (no file system)
  load         tr.load_state_dict(torch.load(file, map_location=device))
Reported: the file size, min and median of each over the rounds, the card's name and power limit.  Prints one JSON
line."""
import argparse
import io
import json
import os
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import bench
from bench_still import card
from streamyolo_b200 import synth, train


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="l")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    tr = train.Trainer(bench.build_model(args.model, dev), lr=0.01 / 64)
    x = synth.synth_frames(1, 600, 960).to(dev)
    tg = tuple(t.to(dev) for t in synth.synth_labels(1, 600, 960))
    tr.step(x, tg)
    times = {"save": [], "save_memory": [], "load": []}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "state.pt")
        for _ in range(args.rounds + 1):                    # the first round warms up and is dropped
            t_save = timed(lambda: torch.save(tr.state_dict(), path))
            t_mem = timed(lambda: torch.save(tr.state_dict(), io.BytesIO()))
            t_load = timed(lambda: tr.load_state_dict(torch.load(path, map_location=dev)))
            for k, t in (("save", t_save), ("save_memory", t_mem), ("load", t_load)):
                times[k].append(t)
        size = os.path.getsize(path)
    fs = tr.fs
    out = {"model": args.model, "file_bytes": size,
           "flat_bytes": 4 * (2 * fs.n_total + fs.n_param),
           "rounds": args.rounds, "card": card()}
    for k, v in times.items():
        v = v[1:]
        out[k + "_ms"] = {"min": round(1e3 * min(v), 1), "median": round(1e3 * statistics.median(v), 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
