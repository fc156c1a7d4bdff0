"""Time the streamer (streamyolo_b200.streamer) on the device.

    python tools/bench_streamer.py [out_file]

StreamYOLO-l (synthetic weights, BatchNorm calibrated by one train pass at momentum 1, as tools/bench_forecast.py does;
fp16 storage), 1200x1920 JPEG frames (synthetic, encoded at quality 90) at in_scale 0.5, the driver's conf 0.01 / NMS
0.65:
  * the simulated clock: 16 sequences of 30 frames at S = 1, 8, 16 streams and R = 33 / 100 ms, ``run_simulated`` on
    the host clock after the detector is built -> emitted frames/s and sequences/s;
  * the in-graph extrapolation: ``step_jpeg`` of a detector with queries=4 against one without, alternating rounds of 40
    ticks, medians per round;
  * the wall clock: one 90-frame sequence through ``wall_sequence`` on ``time.perf_counter``; each emission's forecast
    time (``t_forecast``: one ``query``, one launch and one synchronisation) p50 / p90 / max against --forecast-rt-ub.
The card's name and power limit are read in the same run."""
import os
import subprocess
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_forecast import calibrated_l  # noqa: E402
from streamyolo_b200 import feed, ops, sap, stream, streamer, synth  # noqa: E402

N_SEQ, N_FRAMES, FPS, UB = 16, 30, 30.0, 0.003


def jpeg_frames(n):
    frames = synth.synth_frames(n, 1200, 1920, seed=5)[:, :3]
    frames = frames.permute(0, 2, 3, 1).round().clamp(0, 255).to(torch.uint8).numpy()
    return [cv2.imencode(".jpg", np.ascontiguousarray(f), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes() for f in frames]


def simulated(model, paths):
    lines = []
    used = [p for ps in paths for p in ps]
    for R in (0.033, 0.100):
        schedules = [streamer.simulated_schedule(len(p), FPS, R, UB) for p in paths]
        n_q = max(int(np.bincount(s["emit_det"]).max()) for s in schedules)
        n_emit = sum(len(s["timestamps"]) for s in schedules)
        for S in (1, 8, 16):
            det = stream.StreamDetector(model, frame_sizes=[(1200, 1920)] * S, in_scale=0.5, forecast=True,
                                        clear_on_empty=True, queries=n_q, max_tracks=11850,
                                        jpeg_max_bytes=feed.default_max_bytes(used))
            streamer.run_simulated(det, paths[:S], schedules[:S], 0.0, R, lambda *a: None)       # warm-up
            t0 = time.perf_counter()
            streamer.run_simulated(det, paths, schedules, 0.0, R, lambda *a: None)
            t = time.perf_counter() - t0
            n_det = sum(len(s["det_fidx"]) for s in schedules)
            lines.append(f"simulated R={1e3 * R:.0f} ms S={S:2d}: {n_emit / t:.1f} emitted frames/s, {len(paths) / t:.2f} "
                         f"sequences/s ({n_det} ticks of up to {n_q} queries, {t:.2f} s)")
            del det
    return lines


def in_graph_cost(model, files):
    dets = {q: stream.StreamDetector(model, frame_sizes=[(1200, 1920)] * 8, in_scale=0.5, forecast=True,
                                     clear_on_empty=True, queries=q, max_tracks=11850, jpeg_max_bytes=1 << 21)
            for q in (0, 4)}
    ms = {0: [], 4: []}
    k = 0
    for r in range(4):
        for q in (0, 4):
            t = []
            for _ in range(40):
                f = [files[(k + s) % len(files)] for s in range(8)]
                t0 = time.perf_counter()
                if q:
                    dets[q].step_jpeg(f, [k] * 8, [[0.5, 1.0, 1.5, 2.0]] * 8)
                else:
                    dets[q].step_jpeg(f, [k] * 8)
                t.append(time.perf_counter() - t0)
                k += 1
            if r:
                ms[q].append(1e3 * np.median(t))
    m0, m4 = float(np.median(ms[0])), float(np.median(ms[4]))
    return [f"in-graph extrapolation, S=8, 4 queries per stream: step_jpeg {m4:.3f} ms "
            f"({min(ms[4]):.3f}-{max(ms[4]):.3f}) against {m0:.3f} ms ({min(ms[0]):.3f}-{max(ms[0]):.3f}) without, "
            f"+{m4 - m0:.3f} ms per tick"]


def wall(model, paths):
    det = stream.StreamDetector(model, frame_hw=(1200, 1920), in_scale=0.5, forecast=True, clear_on_empty=True,
                                max_tracks=11850)
    frames = sap.decode_sequence(paths, (1200, 1920), "cuda")
    streamer.wall_sequence(det, frames, 15, FPS, 0.0, UB)                 # warm-up
    out, times = streamer.wall_sequence(det, frames, len(paths), FPS, 0.0, UB)
    f = 1e3 * np.asarray(times["t_forecast"])
    d = 1e3 * np.asarray(times["t_det"])
    n_rows = [len(r[0]) for r in out["results_parsed"]]
    n_det = np.mean([len(det.step(frames[j], fidx=j)[0][2]) for j in range(8)])
    return [f"wall clock, one {len(paths)}-frame sequence ({n_det:.0f} detections per frame): "
            f"{len(out['timestamps'])} emissions ({np.mean(n_rows):.0f} rows each), forecast per emission p50 "
            f"{np.percentile(f, 50):.3f} ms, p90 {np.percentile(f, 90):.3f} ms, max {f.max():.3f} ms against "
            f"--forecast-rt-ub {1e3 * UB:.0f} ms; detection p50 {np.percentile(d, 50):.1f} ms "
            f"({len(d)} detections)"]


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    ops.lib()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    lines = [f"GPU: {gpu}"]
    model = calibrated_l()
    files = jpeg_frames(16)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for q in range(N_SEQ):
            ps = []
            for j in range(max(N_FRAMES, 90 if q == 0 else 0)):
                p = os.path.join(tmp, f"{q}_{j:04d}.jpg")
                with open(p, "wb") as fh:
                    fh.write(files[(q + j) % len(files)])
                ps.append(p)
            paths.append(ps)
        lines += wall(model, paths[0])
        lines += in_graph_cost(model, [np.frombuffer(f, np.uint8) for f in files])
        lines += simulated(model, [p[:N_FRAMES] for p in paths])
    text = "\n".join(lines)
    print(text)
    if out:
        os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
        with open(out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
