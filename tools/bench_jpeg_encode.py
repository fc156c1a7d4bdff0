"""The device JPEG encoder (sy_jpeg_encode) on 1200 x 1920 camera-like BGR frames at quality 95, against cv2.imencode on
the host, and what recording costs the streaming detector.

  (1) encode    n = 1, 8, 16 frames per launch: CUDA events around ``iters`` launches after warm-up; the bytes the
                encode must move (the frames read, the files written) over that time, against the 3.35 TB/s HBM3 bound
  (2) stages    the same at n = 8 under torch.profiler: mean time of each kernel (jpeg_enc_*) per launch
  (3) cv2       cv2.imencode of the same frames on one host core, and on a thread pool over every core
  (4) tick      StreamDetector (StreamYOLO-l, calibrated synthetic weights, fp16 storage, in_scale 0.5) on S = 8 NV12
                cameras, with record_quality=None and record_quality=95, alternating tick by tick: median and p90 of the
                host wall time of ``step`` (which synchronises once), and last_jpeg() (one more synchronisation)

Every file is checked equal to cv2's (when cv2 is present) before anything is timed.  The card's name and power limit are
read in the same run.  usage: python tools/bench_jpeg_encode.py [iters] [ticks] [out path]"""
import os
import re
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

from bench_stream import calibrated_l, card
from oracle.make_jpeg_golden import synth_frame
from oracle.make_yuv_golden import synth_frame as synth_yuv
from streamyolo_b200 import data, ops, stream

FRAME_HW, QUALITY, HBM = (1200, 1920), 95, 3.35e12


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    ticks = int(sys.argv[2]) if len(sys.argv) > 2 else 60
    out_path = sys.argv[3] if len(sys.argv) > 3 else os.path.join(os.path.dirname(HERE), "profiles", "h100_jpeg_encode.txt")
    lines = []

    def say(s):
        print(s, flush=True)
        lines.append(s)

    try:
        import cv2
    except ImportError:
        cv2 = None
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    say(f"$ python tools/bench_jpeg_encode.py {iters} {ticks}")
    say(f"card (name, power limit, max SM clock): {card()}")
    say(f"host: {os.cpu_count()} cores, " + (f"cv2 {cv2.__version__}" if cv2 else "no cv2"))
    h, w = FRAME_HW
    host = [synth_frame(h, w, 300 + i) for i in range(16)]
    frames = torch.from_numpy(np.stack(host)).to(dev)
    files = data.encode_jpeg(frames, QUALITY)
    if cv2 is not None:
        want = [cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, QUALITY])[1].tobytes() for f in host]
        assert files == want, "device files differ from cv2's"
    say(f"(1) encode, {h}x{w} at q {QUALITY}; files of {statistics.mean(len(f) for f in files) / 1e3:.0f} kB "
        f"(min {min(len(f) for f in files) / 1e3:.0f}, max {max(len(f) for f in files) / 1e3:.0f})"
        + ("; every file equals cv2.imencode's" if cv2 else ""))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    per_frame = {}
    for n in (1, 8, 16):
        src = frames[:n].contiguous()
        sizes = torch.tensor([FRAME_HW] * n, dtype=torch.int32, device=dev)
        mb = ops.jpeg_encode_max_bytes(h, w)
        out = (torch.empty((n, mb), dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.int64, device=dev),
               torch.empty(n, dtype=torch.int32, device=dev))
        ws = torch.empty(ops.jpeg_encode_workspace_bytes(n, h, w, mb), dtype=torch.uint8, device=dev)
        run = lambda: ops.jpeg_encode(src, sizes, QUALITY, *out, ws)
        for _ in range(5):
            run()
        torch.cuda.synchronize()
        a.record()
        for _ in range(iters):
            run()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / iters
        ok = out[2].tolist() == [0] * n and [out[0][i, :l].cpu().numpy().tobytes() for i, l in
                                             enumerate(out[1].tolist())] == files[:n]
        assert ok, n
        moved = n * h * w * 3 + sum(out[1].tolist())
        per_frame[n] = ms / n
        say(f"  n={n:2d}: {ms * 1e3:8.1f} us per launch, {ms / n * 1e3:7.1f} us per frame; {moved / 1e6:6.1f} MB read + "
            f"written = {moved / ms / 1e6:6.1f} GB/s, {100 * moved / ms * 1e3 / HBM:.1f}% of {HBM / 1e12:.2f} TB/s")
        if n == 8:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    run()
                torch.cuda.synchronize()
            stages = {}
            for e in prof.events():
                m = re.search(r"jpeg_enc_\w+", e.name)
                if m:
                    stages[m.group(0)] = stages.get(m.group(0), 0.0) + e.device_time_total / 10
    say("(2) stages at n=8, mean per launch (torch.profiler):")
    for k, us in stages.items():
        say(f"  {k:24s} {us:8.1f} us")
    if cv2 is not None:
        enc = lambda f: cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, QUALITY])
        t0 = time.perf_counter()
        for f in host:
            enc(f)
        one = (time.perf_counter() - t0) / len(host)
        cores = os.cpu_count() or 1
        with ThreadPoolExecutor(cores) as ex:
            list(ex.map(enc, host))
            t0 = time.perf_counter()
            for _ in range(4):
                list(ex.map(enc, host))
            pool = (time.perf_counter() - t0) / (4 * len(host))
        say(f"(3) cv2.imencode: {one * 1e3:.2f} ms per frame on one core; {pool * 1e3:.2f} ms per frame "
            f"({1 / pool:.0f} frames/s) on a pool of {cores} threads; device at n=16: {per_frame[16]:.3f} ms per "
            f"frame ({1e3 / per_frame[16]:.0f} frames/s)")
    del frames, out, ws
    model = calibrated_l(dev)
    s = 8
    yuv = [[synth_yuv("nv12", h, w, 100 * k + i) for i in range(s)] for k in range(4)]
    kw = dict(frame_hw=FRAME_HW, in_scale=0.5, streams=s, conf_thre=0.01, nms_thre=0.65, frame_format="nv12")
    dets = {"plain": stream.StreamDetector(model, **kw), "record": stream.StreamDetector(model, record_quality=QUALITY, **kw)}
    for k in range(4):
        r, p = dets["record"].step(yuv[k]), dets["plain"].step(yuv[k])
        assert all(np.array_equal(x, y) for u, v in zip(r, p) for x, y in zip(u, v)), k
    wall = {k: [] for k in dets}
    read = []
    for t in range(2 * ticks):
        leg = ("plain", "record")[(t + t // 2) % 2]
        t0 = time.perf_counter()
        dets[leg].step(yuv[t % 4])
        wall[leg].append((time.perf_counter() - t0) * 1e3)
        if leg == "record":
            t0 = time.perf_counter()
            got = dets["record"].last_jpeg()
            read.append((time.perf_counter() - t0) * 1e3)
    kb = statistics.mean(len(f) for f in got) / 1e3
    say(f"(4) StreamDetector tick, S={s} NV12 {h}x{w} cameras, StreamYOLO-l fp16 storage, {ticks} ticks per leg, "
        "alternated; detections equal")
    for leg in dets:
        say(f"  record_quality={'None' if leg == 'plain' else QUALITY}: step median {statistics.median(wall[leg]):7.2f} ms, "
            f"p90 {float(np.percentile(wall[leg], 90)):7.2f} ms")
    say(f"  last_jpeg(): median {statistics.median(read):6.2f} ms for {s} files of {kb:.0f} kB")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as fh:
        fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
