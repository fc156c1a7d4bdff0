"""The streaming detector fed raw Bayer sensor frames (StreamYOLO-l, fp16 activation storage, synthetic weights with
BatchNorm calibrated as in tools/bench_stream.py, eight 1200x1920 RGGB streams at in_scale 0.5, the driver's conf 0.01 /
NMS 0.65), for the bilinear and the edge-aware demosaicing.  Two legs per algorithm, alternating tick by tick:

  (1) cv2     cv2.cvtColor(raw, COLOR_BayerRGGB2BGR[_EA]) on the host for every stream, then StreamDetector().step(bgr)
  (2) device  StreamDetector(frame_format="bayer_rggb", demosaic=...).step(raw): the demosaicing runs inside the replay
              (sy_bayer_to_bgr_sized)

Per tick: median and p90 of the host wall time, the host CPU time of the process (every thread, cv2's and torch's
included; a mean over all ticks), and the bytes each leg copies from host to device.  The demosaicing kernel alone is
also timed (its own graph, CUDA events) with the bytes it must move (the mosaics read once, the BGR frames written), as
a rate and as a share of the H100 SXM's 3.35 TB/s.  Both legs' detections are checked equal first.  The measurement is
repeated ``rounds`` times; the spread is the max - min of the round medians.  The card's name, power limit and clock are
read in the same run.  usage: python tools/bench_stream_bayer.py [rounds] [ticks] [out path]"""
import os
import statistics
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

import bench
from bench_stream import calibrated_l, card
from oracle.bayer_oracle import CV2_CODES
from oracle.make_bayer_golden import synth_frame
from streamyolo_b200 import ops, stream

FRAME_HW, IN_SCALE, CONF, NMS, STREAMS = (1200, 1920), 0.5, 0.01, 0.65, 8
SEQ = 4                      # distinct frames per stream, cycled
HBM_BYTES_PER_S = 3.35e12    # H100 SXM data sheet


def pct(v, q):
    return float(np.percentile(np.asarray(v), q))


def main():
    import cv2
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    ticks = int(sys.argv[2]) if len(sys.argv) > 2 else 100
    out_path = sys.argv[3] if len(sys.argv) > 3 else os.path.join(os.path.dirname(HERE), "profiles",
                                                                  "h100_stream_bayer.txt")
    lines = []

    def say(s):
        print(s, flush=True)
        lines.append(s)

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    say(f"$ python tools/bench_stream_bayer.py {rounds} {ticks}")
    say(f"card (name, power limit, max SM clock): {card()}")
    say(f"host: {os.cpu_count()} cores, cv2 {cv2.__version__} with {cv2.getNumThreads()} threads")
    model = calibrated_l(dev)
    h, w, s = *FRAME_HW, STREAMS
    raws = [[synth_frame(h, w, 100 * k + i) for i in range(s)] for k in range(SEQ)]
    for algo in ("bilinear", "ea"):
        code = getattr(cv2, CV2_CODES["rggb", algo])
        d_cv2 = stream.StreamDetector(model, FRAME_HW, IN_SCALE, streams=s, conf_thre=CONF, nms_thre=NMS)
        d_dev = stream.StreamDetector(model, FRAME_HW, IN_SCALE, streams=s, conf_thre=CONF, nms_thre=NMS,
                                      frame_format="bayer_rggb", demosaic=algo)
        legs = {"cv2": lambda k: d_cv2.step([cv2.cvtColor(f, code) for f in raws[k]]),
                "device": lambda k: d_dev.step(raws[k])}
        n_det = []
        for k in range(SEQ):                     # what is timed computes the same detections
            a, b = legs["cv2"](k), legs["device"](k)
            assert all(np.array_equal(x, y) for u, v in zip(a, b) for x, y in zip(u, v)), (algo, k)
            assert torch.equal(d_cv2.last_raw(), d_dev.last_raw()), (algo, k)
            n_det.append(sum(len(u[2]) for u in a))
        h2d = {"cv2": s * h * w * 3, "device": s * h * w}
        wall = {k: [[] for _ in range(rounds)] for k in legs}
        cpu = {k: [] for k in legs}
        for r in range(rounds):
            for t in range(2 * ticks):
                leg = ("cv2", "device")[(t + t // 2) % 2]      # cv2, device, device, cv2, cv2, device, ...
                c0, t0 = time.process_time(), time.perf_counter()
                legs[leg](t % SEQ)
                wall[leg][r].append((time.perf_counter() - t0) * 1e3)
                cpu[leg].append((time.process_time() - c0) * 1e3)
        tk = d_dev._tick
        g, _ = bench.capture(lambda tk=tk: ops.bayer_to_bgr_sized(tk.bayer, tk.bayer_sizes, "rggb", algo, tk.frames))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        g.replay()
        torch.cuda.synchronize()
        a.record()
        for _ in range(200):
            g.replay()
        b.record()
        torch.cuda.synchronize()
        k_ms = a.elapsed_time(b) / 200
        k_bytes = s * h * w * 4
        say(f"{algo} S={s}: detections per tick (all streams, first {SEQ} ticks, both legs equal): {n_det}")
        for leg in legs:
            every = [v for rw in wall[leg] for v in rw]
            meds = [statistics.median(rw) for rw in wall[leg]]
            say(f"  ({'1' if leg == 'cv2' else '2'}) {leg:6s}  wall median {statistics.median(every):8.3f} ms "
                f"(spread {max(meds) - min(meds):.3f}), p90 {pct(every, 90):8.3f} ms; host CPU mean "
                f"{statistics.fmean(cpu[leg]):8.3f} ms; host->device {h2d[leg] / 1e6:6.2f} MB per tick")
        say(f"  demosaicing kernel alone: {k_ms * 1e3:7.1f} us for {k_bytes / 1e6:.1f} MB moved "
            f"({k_bytes / k_ms / 1e6:.0f} GB/s, {100 * k_bytes / (k_ms * 1e-3) / HBM_BYTES_PER_S:.0f}% of 3.35 TB/s)")
        del d_cv2, d_dev
    say(f"{rounds} rounds of {ticks} ticks per leg, legs alternated; wall = host clock around step (which synchronises once)")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as fh:
        fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
