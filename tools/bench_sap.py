"""The sAP driver on the device (streamyolo_b200.sap) against the reference driver's host work, StreamYOLO-l with
synthetic weights (BatchNorm calibrated as in tools/bench_stream.py), fp16 activation storage, 1200x1920 frames -> 600x960,
conf 0.01 / NMS 0.65.  Sequences are the 1200x1920 JPEG fixture (tests/golden/stream_jpeg_files.npz, a420) requantised
into SEQ distinct files and cycled to FRAMES frames.

Wall clock (one sequence, the legs alternating over ROUNDS rounds):
  (a) load     the sequence's files -> frames: sap.decode_sequence (device) against the driver's cv2.imread loop (host),
               seconds, and the process's resident host memory they add (VmRSS after the load minus before)
  (b) runtime  the driver's real-time loop (sap.wall_sequence, perf_counter) on 30 fps, once with StreamDetector.step on
               the device-decoded frames and once with the eager driver body (bench_stream.eager_frame: host frame ->
               device, resize, on_pipe forward, NMS, .cpu()) on cv2's frames: the per-frame runtimes (median, p90, max)
               and the share under 1/30 s
Simulated clock: 16 sequences at a constant 40 ms runtime through sap.run_simulated at S = 1, 4, 8, 16 streams, total
seconds (the pickles are built but not written), ROUNDS_SIM rounds alternating S.

usage: python tools/bench_sap.py [rounds] [frames] [out path]"""
import os
import statistics
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

from bench_stream import calibrated_l, card, eager_frame
from oracle.make_stream_jpeg_golden import SEQ, requant
from streamyolo_b200 import sap, stream

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
FRAMES = int(sys.argv[2]) if len(sys.argv) > 2 else 900
OUT = sys.argv[3] if len(sys.argv) > 3 else None
ROUNDS_SIM = 2
N_SEQ, RUNTIME, FPS = 16, 0.040, 30.0
STREAMS = (1, 4, 8, 16)
G = np.load(os.path.join(os.path.dirname(HERE), "tests", "golden", "stream_jpeg_files.npz"))


def rss_bytes():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) * 1024
    return -1


class EagerDriver:
    """the driver's per-frame body (:176-184) eagerly, behind the interface sap.wall_sequence drives"""

    def __init__(self, model):
        self.model, self.buffer, self.raw = model, None, None

    def reset(self):
        self.buffer = None

    def step(self, frame):
        out, self.buffer = eager_frame(self.model, frame, self.buffer)
        return [out]

    def last_raw(self):
        return None


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def main():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lines = [f"card (name, power limit, max SM clock): {card()}", f"host cores: {os.cpu_count()} (affinity "
             f"{len(os.sched_getaffinity(0))})", f"rounds {ROUNDS} (simulated {ROUNDS_SIM}), {FRAMES} frames per sequence"]
    print("\n".join(lines), flush=True)
    try:
        import cv2
    except ImportError:
        cv2 = None
    tmp = os.path.join("/tmp", f"bench_sap_{os.getpid()}")
    os.makedirs(tmp, exist_ok=True)
    files = []
    for k in range(SEQ):
        p = os.path.join(tmp, f"f{k}.jpg")
        with open(p, "wb") as f:
            f.write(requant(bytes(G["a420.jpg"]), k))
        files.append(p)
    seq = [files[j % SEQ] for j in range(FRAMES)]
    mb = sum(os.path.getsize(p) for p in seq) / 1e6
    lines.append(f"sequence: {FRAMES} files, {mb:.1f} MB")
    model = calibrated_l(dev)
    model.activation_dtype = torch.float16
    det = stream.StreamDetector(model, frame_hw=sap.DRIVER_HW, in_scale=0.5)
    eager = EagerDriver(model)
    sap.decode_sequence(seq[:32], sap.DRIVER_HW, dev)                # warm-up: module load, workspace
    torch.cuda.synchronize()
    load = {"device": [], "cv2": []}
    mem = {"device": [], "cv2": []}
    rt = {"step": [], "eager": []}
    for r in range(ROUNDS):
        before = rss_bytes()
        t0 = time.perf_counter()
        frames = sap.decode_sequence(seq, sap.DRIVER_HW, dev)
        torch.cuda.synchronize()
        load["device"].append(time.perf_counter() - t0)
        mem["device"].append(rss_bytes() - before)
        if cv2 is not None:
            before = rss_bytes()
            t0 = time.perf_counter()
            host = [cv2.imread(p) for p in seq]
            load["cv2"].append(time.perf_counter() - t0)
            mem["cv2"].append(rss_bytes() - before)
        else:
            host = [f.numpy() for f in frames.cpu()]
        out = sap.wall_sequence(det, frames, FRAMES, FPS, 1, False)
        rt["step"].append(out["runtime"])
        out = sap.wall_sequence(eager, host, FRAMES, FPS, 1, False)
        rt["eager"].append(out["runtime"])
        del frames, host, out
        print(f"round {r}: load device {load['device'][-1]:.2f} s, RSS +{mem['device'][-1] / 1e9:.3f} GB"
              + (f"; cv2 {load['cv2'][-1]:.2f} s, RSS +{mem['cv2'][-1] / 1e9:.3f} GB" if load["cv2"] else "")
              + "".join(f"; {k} {len(v[-1])} frames, median {pct(v[-1], 50):.2f} ms, under 1/30 s "
                        f"{100 * float(np.mean(np.asarray(v[-1]) < 1 / FPS)):.1f} %" for k, v in rt.items()), flush=True)
    lines.append("wall clock, load of one sequence (median over rounds, min-max):")
    for k in ("device", "cv2"):
        if load[k]:
            lines.append(f"  {k:6s} {statistics.median(load[k]):7.2f} s ({min(load[k]):.2f}-{max(load[k]):.2f}), "
                         f"{FRAMES / statistics.median(load[k]):.0f} frames/s, host RSS added "
                         f"{statistics.median(mem[k]) / 1e9:.3f} GB ({min(mem[k]) / 1e9:.3f}-{max(mem[k]) / 1e9:.3f})")
        else:
            lines.append(f"  {k:6s} not measured (cv2 is not installed; the eager leg ran on device-decoded frames)")
    lines.append("wall clock, per-frame runtime of the real-time loop at 30 fps (per round: frames run, median / p90 / max "
                 "ms, share under 1/30 s):")
    for k in ("step", "eager"):
        for r, v in enumerate(rt[k]):
            small = float(np.mean(np.asarray(v) < 1 / FPS))
            lines.append(f"  {k:5s} round {r}: {len(v)} frames, {pct(v, 50):.2f} / {pct(v, 90):.2f} / {pct(v, 100):.2f} ms, "
                         f"{100 * small:.1f} %")
    # simulated clock
    paths = [seq] * N_SEQ
    schedules = [sap.simulated_schedule(FRAMES, FPS, 1, False, RUNTIME)] * N_SEQ
    used = sum(len(f) for f, _ in schedules)
    dets = {s: stream.StreamDetector(model, frame_sizes=[sap.DRIVER_HW] * s, in_scale=0.5,
                                     jpeg_max_bytes=max(os.path.getsize(p) for p in files) + 4096) for s in STREAMS}
    sim = {s: [] for s in STREAMS}
    for r in range(ROUNDS_SIM):
        for s in STREAMS:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sap.run_simulated(dets[s], paths, schedules, RUNTIME, lambda q, o: None)
            torch.cuda.synchronize()
            sim[s].append(time.perf_counter() - t0)
            print(f"round {r}: simulated S={s} {sim[s][-1]:.2f} s", flush=True)
    lines.append(f"simulated clock, {N_SEQ} sequences at {RUNTIME * 1e3:.0f} ms per frame ({used} frames run), total seconds "
                 "(median, min-max), frames/s:")
    for s in STREAMS:
        m = statistics.median(sim[s])
        lines.append(f"  S={s:2d} {m:7.2f} s ({min(sim[s]):.2f}-{max(sim[s]):.2f}), {used / m:.0f} frames/s")
    text = "\n".join(lines)
    print(text)
    if OUT:
        os.makedirs(os.path.dirname(os.path.abspath(OUT)), exist_ok=True)
        with open(OUT, "w") as f:
            f.write(text + "\n")
    for p in files:
        os.remove(p)
    os.rmdir(tmp)


if __name__ == "__main__":
    main()
