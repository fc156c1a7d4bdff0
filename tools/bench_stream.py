"""The streaming driver loop, eager vs ``stream.StreamDetector``, in one process (StreamYOLO-l, fp16 activation storage,
synthetic weights with BatchNorm calibrated by one train pass at momentum 1, seeded 1200x1920 uint8 frames, in_scale 0.5
-> 600x960, the driver's conf 0.01 / NMS 0.65):

  (a) eager   the driver's loop body (sAP/streamyolo/streamyolo_det.py:176-184): H2D of the numpy frame, data.stream_frame,
              model(x, buffer=buffer, mode='on_pipe'), postprocess, .cpu(), the driver's conversion, synchronise; host clock
              per frame, plus CUDA events from the H2D to the D2H (the device's span of the frame)
  (b) step    StreamDetector.step(numpy frame) -> host detections; host clock per frame
  (c) replay  the detector's graph alone, back to back, CUDA events
  (d) S       StreamDetector.step on S = 1, 2, 4, 8 streams (one frame each); host clock per tick, and the replay alone; and
              the NMS kernel alone at batch 1 (its own graph, CUDA events)

The legs alternate within each round (``rounds`` rounds of ``frames`` frames / ticks each); medians and the spread of the
per-round medians are printed with the card's name, power limit and max SM clock.
    usage: python tools/bench_stream.py [rounds] [frames]"""
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from streamyolo_b200 import data, ops, stream, synth
from streamyolo_b200.postprocess import postprocess

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
FRAMES = int(sys.argv[2]) if len(sys.argv) > 2 else 300
FRAME_HW, IN_SCALE = (1200, 1920), 0.5
SIZE = (int(FRAME_HW[0] * IN_SCALE), int(FRAME_HW[1] * IN_SCALE))
CONF, NMS = 0.01, 0.65
STREAMS = (1, 2, 4, 8)
N_DISTINCT = 16


def card():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def calibrated_l(dev):
    model = bench.build_model("l", dev)
    x = synth.synth_frames(8, 600, 960, seed=99).to(dev)
    tg = tuple(t.to(dev) for t in synth.synth_labels(8, 600, 960, seed=11))
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    mom = [m.momentum for m in bns]
    with torch.no_grad():
        for m in bns:
            m.momentum = 1.0
        model(x, tg)                                 # running statistics := batch statistics
        for m, v in zip(bns, mom):
            m.momentum = v
    model.eval()
    model.activation_dtype = torch.float16
    return model


def uint8_frames(n, seed):
    f = synth.synth_frames(n, FRAME_HW[0], FRAME_HW[1], seed=seed)[:, :3]
    return np.ascontiguousarray(f.permute(0, 2, 3, 1).round().clamp(0, 255).to(torch.uint8).numpy())


def eager_frame(model, frame, buffer, ev=None):
    """the driver's loop body; -> (detections, buffer)"""
    if ev is not None:
        ev[0].record()
    with torch.no_grad():
        f = torch.from_numpy(frame).cuda()
        x = data.stream_frame(f, SIZE)
        result, buffer = model(x, buffer=buffer, mode="on_pipe")
        d = postprocess(result, model.head.num_classes, CONF, NMS)[0]
        d = np.zeros((0, 7), np.float32) if d is None else d.cpu().numpy()
    if ev is not None:
        ev[1].record()
    out = d[:, :4] / IN_SCALE, d[:, 4] * d[:, 5], d[:, 6].astype(np.int32)     # the driver's inference() conversion
    torch.cuda.synchronize()
    return out, buffer


def host_ms(fn, n):
    ts = []
    for i in range(n):
        t0 = time.perf_counter()
        fn(i)
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def main():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card (name, power limit, max SM clock):", card())
    model = calibrated_l(dev)
    frames = uint8_frames(N_DISTINCT, seed=5)
    dets = {s: stream.StreamDetector(model, FRAME_HW, IN_SCALE, streams=s, conf_thre=CONF, nms_thre=NMS) for s in STREAMS}
    batches = {s: [np.ascontiguousarray(np.roll(frames, -k, 0)[:s]) for k in range(N_DISTINCT)] for s in STREAMS}

    # the NMS alone at batch 1, on the detector's own head outputs
    raw1 = dets[1]._tick.raw
    g_nms, _ = bench.capture(lambda: ops.postprocess_nms(raw1, model.head.num_classes, CONF, NMS, max_det=raw1.shape[1]))

    # correctness of what is timed: the detector's detections equal the eager loop's on the same frames
    buf = None
    dets[1].reset()
    n_det = []
    for i in range(4):
        want, buf = eager_frame(model, frames[i], buf)
        got = dets[1].step(frames[i])[0]
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), f"frame {i}: detector != eager loop"
        n_det.append(len(want[2]))
    raw = dets[1].last_raw()
    print("detections per frame (first 4 frames, eager == detector):", n_det,
          f"; frame 3: head outputs finite {bool(torch.isfinite(raw).all())}, max obj * class score "
          f"{float((raw[0, :, 4] * raw[0, :, 5:].max(1).values).max()):.4f}")

    state = {"buf": None}
    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
    spans = []

    def leg_a(i):
        _, state["buf"] = eager_frame(model, frames[i % N_DISTINCT], state["buf"], ev)
        spans.append(ev[0].elapsed_time(ev[1]))

    legs = {"(a) eager loop": leg_a,
            "(b) step": lambda i: dets[1].step(frames[i % N_DISTINCT])}
    for s in STREAMS[1:]:
        legs[f"(d) step S={s}"] = (lambda s_: lambda i: dets[s_].step(batches[s_][i % N_DISTINCT]))(s)
    for name, fn in legs.items():                    # warm-up
        host_ms(fn, 20)
    times = {k: [] for k in list(legs) + ["(a) device span"] + [f"(c) replay S={s}" for s in STREAMS] + ["(d) NMS alone S=1"]}
    for r in range(ROUNDS):
        order = list(legs) if r % 2 == 0 else list(legs)[::-1]
        for name in order:
            spans.clear()
            ms = host_ms(legs[name], FRAMES)
            times[name].append(ms)
            print(f"round {r} {name:20s} {ms:.4f} ms (host clock, median of {FRAMES})")
            if name.startswith("(a)"):
                times["(a) device span"].append(statistics.median(spans))
        for s in STREAMS:
            ms = bench.time_replays(dets[s]._graph, FRAMES)
            times[f"(c) replay S={s}"].append(ms)
            print(f"round {r} (c) replay S={s:<9d} {ms:.4f} ms (CUDA events, {FRAMES} replays)")
        ms = bench.time_replays(g_nms, FRAMES)
        times["(d) NMS alone S=1"].append(ms)
        print(f"round {r} (d) NMS alone S=1     {ms:.4f} ms (CUDA events, {FRAMES} replays)")
    print(f"medians over {ROUNDS} rounds of {FRAMES} frames / ticks (spread = max - min of the round medians):")
    for k, v in times.items():
        s = int(k.split("S=")[1]) if "S=" in k else 1
        per = f", {statistics.median(v) / s:.4f} ms per frame" if s > 1 else ""
        print(f"  {k:22s} {statistics.median(v):.4f} ms per tick{per} (spread {max(v) - min(v):.4f})")
    a, b = statistics.median(times["(a) eager loop"]), statistics.median(times["(b) step"])
    print(f"  eager / detector at one stream: {a / b:.3f}x")


if __name__ == "__main__":
    main()
