"""Time the offline forecast (streamyolo_b200.forecast) on the device against the fp32 reference loop on the host.

    python tools/bench_forecast.py [out_file]

S synthetic 900-frame sequences (S = 1 and 24) of about 100 detections per frame, one detection per frame (the
detector's input frame ii, out 0.8 frames later), objects moving at constant velocity with noise: the host plan
(forecast.Plan), the device pass (forecast.device_pass: upload, sy_forecast_sequences, read-back) on the host clock,
and the kernel alone on CUDA events, median of 5 after a warm-up; the fp32 oracle loop (oracle/forecast_oracle.py, the
script's arithmetic) on one sequence on the host cores.

Online: StreamYOLO-l (synthetic weights, BatchNorm calibrated by one train pass at momentum 1, fp16 storage), 1200x1920
frames at in_scale 0.5, the driver's conf 0.01 / NMS 0.65, S = 1 and 8 streams: StreamDetector.step with forecast=False
and forecast=True (max_tracks = every anchor) in alternating rounds of 40 ticks, host clock per tick (each step ends in
its one synchronisation), medians per round; and one forecast() call per tick of the forecast=True rounds.  The card's
name and power limit are read in the same run."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import forecast_oracle as fo  # noqa: E402
import bench  # noqa: E402
from streamyolo_b200 import forecast, ops, stream, synth  # noqa: E402

FPS, N_FRAMES, N_OBJ, W, H = 30.0, 900, 100, 1920, 1200


def sequence(rng):
    p0 = rng.uniform([0, 0], [W - 200, H - 150], (N_OBJ, 2))
    v = rng.uniform(-3, 3, (N_OBJ, 2))
    wh = rng.uniform([20, 20], [200, 150], (N_OBJ, 2))
    lab = rng.integers(0, 8, N_OBJ)
    parsed = []
    for f in range(N_FRAMES):
        seen = rng.random(N_OBJ) > 0.05
        p = p0[seen] + v[seen] * f + rng.normal(0, 1.5, (seen.sum(), 2))
        b = np.concatenate((p, p + wh[seen]), 1).astype(np.float32)
        parsed.append((b, rng.permutation(np.linspace(0.01, 0.99, seen.sum())).astype(np.float32),
                       lab[seen].astype(np.int32), None))
    images = [{"id": f, "width": W, "height": H} for f in range(N_FRAMES)]
    return {"images": images, "results_parsed": parsed, "timestamps": [(f + 0.8) / FPS for f in range(N_FRAMES)],
            "input_fidx": list(range(N_FRAMES))}


def kernel_ms(plan):
    s = len(plan.seq_frames) - 1
    state = ops.ForecastState(s, plan.max_tracks, "cuda")
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    args = (up(plan.rows), up(plan.det_start), up(plan.det_n), up(plan.frames), up(plan.seq_frames), plan.n_rows)
    ops.forecast_sequences(state, *args)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = []
    for _ in range(5):
        e0.record()
        ops.forecast_sequences(state, *args)
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1))
    return float(np.median(t))


ROUNDS, TICKS = 3, 40


def calibrated_l():
    model = bench.build_model("l", "cuda")
    x = synth.synth_frames(8, 600, 960, seed=99).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(8, 600, 960, seed=11))
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    mom = [m.momentum for m in bns]
    with torch.no_grad():
        for m in bns:
            m.momentum = 1.0
        model(x, tg)
        for m, v in zip(bns, mom):
            m.momentum = v
    model.eval()
    model.activation_dtype = torch.float16
    return model


def online():
    model = calibrated_l()
    frames = synth.synth_frames(16, 1200, 1920, seed=5)[:, :3]
    frames = np.ascontiguousarray(frames.permute(0, 2, 3, 1).round().clamp(0, 255).to(torch.uint8).numpy())
    lines = []
    for S in (1, 8):
        dets = {on: stream.StreamDetector(model, (1200, 1920), 0.5, streams=S, forecast=on, max_tracks=11850)
                for on in (False, True)}
        ms = {False: [], True: [], "forecast": []}
        n_det, k = [], 0
        for r in range(ROUNDS + 1):                 # round 0 warms up
            for on in (False, True):
                t_step, t_fc = [], []
                for i in range(TICKS):
                    f = np.stack([frames[(k + s) % 16] for s in range(S)])
                    t0 = time.perf_counter()
                    got = dets[on].step(f, fidx=[k] * S) if on else dets[on].step(f)
                    t_step.append(time.perf_counter() - t0)
                    if on:
                        t0 = time.perf_counter()
                        dets[on].forecast([k + 1] * S)
                        t_fc.append(time.perf_counter() - t0)
                        n_det += [len(g[2]) for g in got]
                    k += 1
                if r:
                    ms[on].append(1e3 * np.median(t_step))
                    if on:
                        ms["forecast"].append(1e3 * np.median(t_fc))
        med = {key: float(np.median(v)) for key, v in ms.items()}
        spread = {key: f"{min(v):.3f}-{max(v):.3f}" for key, v in ms.items()}
        lines.append(f"StreamYOLO-l S={S}: step {med[False]:.3f} ms ({spread[False]}) forecast=False, {med[True]:.3f} ms "
                     f"({spread[True]}) forecast=True, +{med[True] - med[False]:.3f} ms per tick; forecast() "
                     f"{med['forecast']:.3f} ms ({spread['forecast']}); {np.mean(n_det):.0f} detections per stream "
                     f"and tick (max {max(n_det)})")
    return lines


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    ops.lib()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    lines = [f"GPU: {gpu}", f"{N_FRAMES}-frame sequences, {N_OBJ} objects, ~{int(N_OBJ * 0.95)} detections per frame, "
             f"one detection per frame"]
    rng = np.random.default_rng(0)
    seqs = [sequence(rng) for _ in range(24)]
    for S in (1, 24):
        t0 = time.perf_counter()
        plan = forecast.Plan(seqs[:S], 0.0, FPS)
        t_plan = time.perf_counter() - t0
        forecast.device_pass(plan, 0.3)
        t = []
        for _ in range(5):
            t0 = time.perf_counter()
            res = forecast.device_pass(plan, 0.3)
            t.append(time.perf_counter() - t0)
        k = kernel_ms(plan)
        lines.append(f"S={S:2d}: host plan {1e3 * t_plan:.0f} ms, device pass {1e3 * np.median(t):.1f} ms "
                     f"(kernel {k:.1f} ms), {int(res[4].sum())} rows, max_tracks {plan.max_tracks}")
    t0 = time.perf_counter()
    ref = fo.run(seqs[:1], eta=0.0, fps=FPS)
    t_host = time.perf_counter() - t0
    lines.append(f"fp32 oracle loop on the host, S=1: {1e3 * t_host:.0f} ms ({sum(len(r[1]) for r in ref)} rows)")
    lines += online()
    text = "\n".join(lines)
    print(text)
    if out:
        os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
        with open(out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
