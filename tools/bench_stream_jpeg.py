"""The streaming detector fed JPEG bytes, for one camera and for rigs of mixed frame sizes (StreamYOLO-l, fp16 activation
storage, synthetic weights with BatchNorm calibrated as in tools/bench_stream.py, 600x960 input, the driver's conf 0.01 /
NMS 0.65).  The files are the fixtures of tests/golden/stream_jpeg_files.npz (1200x1920 4:2:0, 2048x1550 4:4:4, 1550x2048
4:2:0 with restart markers), requantised into SEQ distinct frames each.

  (a) step        StreamDetector.step on decoded 1200x1920 numpy frames (cv2.imread's output), host clock per frame
  (b) step_jpeg   StreamDetector(jpeg_max_bytes=...).step_jpeg on the same frames' files, host clock per frame
  (c) replay      the JPEG detector's graph alone, CUDA events
  (d) rigs        step_jpeg and the replay alone for 3 streams (1200x1920, 2048x1550, 1550x2048) and 6 (each twice)
  (e) kernels     decode_jpeg_sized and letterbox_sized alone (each its own graph, CUDA events), with the bytes they must
                  move: the file bytes read and the uint8 frame written by the decode; the uint8 frame read and the fp32
                  [3, 600, 960] image written by the resize

Legs alternate within each round; medians over the rounds and their spread are printed with the card's name and power
limit.  usage: python tools/bench_stream_jpeg.py [rounds] [frames] [out path]"""
import hashlib
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
from oracle.make_stream_jpeg_golden import SEQ, requant
from streamyolo_b200 import data, ops, stream

SIZE, IN_SCALE, CONF, NMS = (600, 960), 0.5, 0.01, 0.65
G = np.load(os.path.join(os.path.dirname(HERE), "tests", "golden", "stream_jpeg_files.npz"))
NAMES = ("a420", "b444", "c420_r16")
MAX_BYTES = 1 << 19
HBM = 3.35e12


def files_of(name):
    return [requant(bytes(G[f"{name}.jpg"]), k) for k in range(SEQ)]


def hw(name):
    return tuple(int(v) for v in G[f"{name}.hw"])


def host_ms(fn, n):
    ts = []
    for i in range(n):
        t0 = time.perf_counter()
        fn(i)
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def graph_ms(g, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g.replay()
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    frames = int(sys.argv[2]) if len(sys.argv) > 2 else 200
    out_path = sys.argv[3] if len(sys.argv) > 3 else os.path.join(os.path.dirname(HERE), "profiles", "h100_stream_jpeg.txt")
    lines = []

    def say(s):
        print(s, flush=True)
        lines.append(s)

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    say(f"$ python tools/bench_stream_jpeg.py {rounds} {frames}")
    say(f"card (name, power limit, max SM clock): {card()}")
    model = calibrated_l(dev)
    a_files = files_of("a420")
    rows, lengths = data.pack_jpeg(a_files, MAX_BYTES)
    a_frames = data.decode_jpeg(torch.from_numpy(rows).cuda(), torch.from_numpy(lengths).cuda(), hw("a420"))[0].cpu().numpy()
    for k in range(SEQ):
        assert bytes(G["a420.seq"][k]) == hashlib.sha256(a_frames[k].tobytes()).digest()

    plain = stream.StreamDetector(model, (1200, 1920), IN_SCALE, conf_thre=CONF, nms_thre=NMS)
    dets = {1: stream.StreamDetector(model, in_scale=IN_SCALE, frame_sizes=[hw("a420")], input_size=SIZE,
                                     jpeg_max_bytes=MAX_BYTES, conf_thre=CONF, nms_thre=NMS)}
    rig = {1: ["a420"], 3: list(NAMES), 6: list(NAMES) * 2}
    for s in (3, 6):
        dets[s] = stream.StreamDetector(model, in_scale=IN_SCALE, frame_sizes=[hw(n) for n in rig[s]], input_size=SIZE,
                                        jpeg_max_bytes=MAX_BYTES, conf_thre=CONF, nms_thre=NMS)
    seqs = {s: [[files_of(n)[(k + i) % SEQ] for i, n in enumerate(rig[s])] for k in range(SEQ)] for s in rig}

    # what is timed computes what the decoded-frame path computes
    plain.reset()
    dets[1].reset()
    n_det = []
    for k in range(SEQ):
        want = plain.step(a_frames[k])[0]
        got = dets[1].step_jpeg([a_files[k]])[0]
        assert all(np.array_equal(x, y) for x, y in zip(got, want)), f"frame {k}: step_jpeg != step"
        n_det.append(len(want[2]))
    say(f"detections per frame (first {SEQ} frames, step_jpeg == step on cv2's frames): {n_det}")
    for s in (3, 6):
        out = dets[s].step_jpeg(seqs[s][0])
        assert dets[s].last_status().tolist() == [0] * s
        say(f"{s} streams: detections per stream at tick 0: {[len(o[2]) for o in out]}")

    # kernels alone, each its own graph
    kern = {}
    for s in (1, 3):
        t = dets[s]._tick
        g_dec, _ = bench.capture(lambda t=t: data.decode_jpeg_sized(t.bytes, t.lengths, t.sizes, t.frames.shape[1:3],
                                                                     out=t.frames, status=t.status, workspace=t.workspace))
        g_res, _ = bench.capture(lambda t=t: ops.letterbox_sized(t.frames, t.table, t.x))
        file_bytes = sum(len(f) for f in seqs[s][0])
        frame_bytes = sum(h * w * 3 for h, w in (hw(n) for n in rig[s]))
        kern[s] = (g_dec, g_res, file_bytes + frame_bytes, frame_bytes + s * 3 * SIZE[0] * SIZE[1] * 4)

    legs = {"(a) step 1x1200x1920": lambda: host_ms(lambda i: plain.step(a_frames[i % SEQ]), frames),
            "(b) step_jpeg 1x1200x1920": lambda: host_ms(lambda i: dets[1].step_jpeg([a_files[i % SEQ]]), frames),
            "(c) replay 1 stream": lambda: graph_ms(dets[1]._graph, frames)}
    for s in (3, 6):
        legs[f"(d) step_jpeg {s} streams"] = (lambda s=s: host_ms(lambda i: dets[s].step_jpeg(seqs[s][i % SEQ]), frames))
        legs[f"(d) replay {s} streams"] = (lambda s=s: graph_ms(dets[s]._graph, frames))
    for s in (1, 3):
        legs[f"(e) decode_jpeg_sized {s}"] = (lambda s=s: graph_ms(kern[s][0], frames))
        legs[f"(e) letterbox_sized {s}"] = (lambda s=s: graph_ms(kern[s][1], frames))
    res = {k: [] for k in legs}
    names = list(legs)
    for r in range(rounds):
        for k in (names if r % 2 == 0 else names[::-1]):
            v = legs[k]()
            res[k].append(v)
            say(f"round {r} {k:32s} {v:9.4f} ms")
    say(f"medians over {rounds} rounds of {frames} frames / ticks / replays (spread = max - min of the round medians):")
    for k in names:
        m = statistics.median(res[k])
        extra = ""
        for s in (3, 6):
            if k.endswith(f"{s} streams"):
                extra = f", {m / s:.4f} ms per frame"
        for s in (1, 3):
            if k.startswith("(e)") and k.endswith(f" {s}"):
                b = kern[s][2] if "decode" in k else kern[s][3]
                extra = f", {b / 1e6:.2f} MB moved at least, {b / (m * 1e-3) / 1e12:.3f} TB/s = {100 * b / (m * 1e-3) / HBM:.1f} % of 3.35 TB/s"
        say(f"  {k:32s} {m:9.4f} ms (spread {max(res[k]) - min(res[k]):.4f}){extra}")
    a, b = statistics.median(res["(a) step 1x1200x1920"]), statistics.median(res["(b) step_jpeg 1x1200x1920"])
    say(f"  step / step_jpeg at one 1200x1920 stream: {a / b:.3f}x")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as fh:
        fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
