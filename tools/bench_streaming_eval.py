"""``python -m streamyolo_b200.streaming_eval --vis-dir`` on a synthetic 900-frame 1200 x 1920 sequence with 30
detections per frame, at --vis-scale 1 and 0.5, against the sAP toolkit's host path.

  (1) command   streaming_eval.run (--no-eval --overwrite) in a temporary directory: wall time per frame, file reads,
                label rendering, the device pass and file writes included
  (2) device    streaming_eval.device_pass alone on batches of 8 frames whose labels are already rendered: host wall time
                per frame (the copies in and out and the synchronisations included)
  (3) labels    the host's label rendering of one frame (cv2.putText into the canvas and the scan), on one core
  (4) script    vis_det's per-frame work on one core: PIL open, cv2.resize at the scale (mmcv.imrescale), cv2.rectangle
                and cv2.putText per detection, PIL save
Before anything is timed, frames written by the command are checked against PIL decode + cv2 drawing + PIL encode.  The
card's name and power limit are read in the same run.
usage: python tools/bench_streaming_eval.py [frames] [out path]"""
import io
import json
import os
import pickle
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

from oracle.make_jpeg_golden import synth_frame
from streamyolo_b200 import data
from streamyolo_b200 import streaming_eval as se

FRAME_HW = (1200, 1920)
DETS = 30
CLASSES = ["person", "bicycle", "car", "motorcycle", "bus", "truck", "traffic_light", "stop_sign"]


def card():
    """the card's name, power limit and max SM clock (nvidia-smi's query, read only)"""
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def fixture(tmp, n_frames, rng):
    """the sequence's files, annotation and pickle under tmp -> (data root, annotation path, result dir)"""
    h, w = FRAME_HW
    uniq = [synth_frame(h, w, 700 + i) for i in range(16)]
    files = data.encode_jpeg(torch.from_numpy(np.stack(uniq)).cuda(), 90)
    root = os.path.join(tmp, "data", "d0")
    os.makedirs(root)
    images = []
    for i in range(n_frames):
        name = f"{i:06d}.jpg"
        with open(os.path.join(root, name), "wb") as f:
            f.write(files[i % len(files)])
        images.append({"id": i, "sid": 0, "fid": i, "name": name, "width": w, "height": h})
    parsed = []
    for i in range(n_frames):
        x, y = rng.uniform(-0.05 * w, w, DETS), rng.uniform(-0.05 * h, h, DETS)
        bw, bh = rng.uniform(8, 0.25 * w, DETS), rng.uniform(8, 0.25 * h, DETS)
        parsed.append((np.stack([x, y, x + bw, y + bh], 1).astype(np.float32), rng.uniform(0, 1, DETS).astype(np.float32),
                       rng.integers(0, len(CLASSES), DETS).astype(np.int32), None))
    res = os.path.join(tmp, "res")
    os.makedirs(res)
    with open(os.path.join(res, "seq0.pkl"), "wb") as f:
        pickle.dump({"results_parsed": parsed, "timestamps": [i / 30 for i in range(n_frames)],
                     "input_fidx": list(range(n_frames))}, f)
    annot = os.path.join(tmp, "annot.json")
    with open(annot, "w") as f:
        json.dump({"images": images, "annotations": [], "sequences": ["seq0"], "seq_dirs": ["d0"],
                   "categories": [{"id": i, "name": c} for i, c in enumerate(CLASSES)]}, f)
    return os.path.join(tmp, "data"), annot, res


def script_frame(cv2, Image, path, boxes, texts, scale, out):
    """vis_det's work on one frame (PIL open, mmcv.imrescale, the cv2 drawing, PIL save)"""
    img = np.array(Image.open(path))
    if scale != 1:
        h, w = data.imrescale_size(img.shape[0], img.shape[1], scale)
        img = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)
    for (x1, y1, x2, y2), (text, org) in zip(boxes, texts):
        cv2.rectangle(img, (x1, y1), (x2, y2), (0, 255, 0), thickness=1)
        cv2.putText(img, text, org, cv2.FONT_HERSHEY_COMPLEX, 0.5, (0, 255, 0))
    Image.fromarray(img).save(out, format="JPEG")
    return img


def main():
    n_frames = int(sys.argv[1]) if len(sys.argv) > 1 else 900
    out_path = sys.argv[2] if len(sys.argv) > 2 else os.path.join(os.path.dirname(HERE), "profiles",
                                                                   "h100_streaming_eval.txt")
    lines = []

    def say(s):
        print(s, flush=True)
        lines.append(s)

    import cv2
    from PIL import Image
    cv2.setNumThreads(1)
    torch.cuda.set_device(0)
    say(f"$ python tools/bench_streaming_eval.py {n_frames}")
    say(f"card (name, power limit, max SM clock): {card()}")
    say(f"host: {os.cpu_count()} cores, cv2 {cv2.__version__}, PIL; {n_frames} frames of {FRAME_HW[0]}x{FRAME_HW[1]}, "
        f"{DETS} detections each")
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as tmp:
        root, annot, res = fixture(tmp, n_frames, rng)
        for scale in (1.0, 0.5):
            vis_dir = os.path.join(tmp, f"vis{scale}")
            argv = ["--data-root", root, "--annot-path", annot, "--result-dir", res, "--out-dir",
                    os.path.join(tmp, "out"), "--vis-dir", vis_dir, "--vis-scale", str(scale), "--no-eval", "--overwrite"]
            opts = se.parse_args(argv)
            se.run(opts)                                           # warm-up and the files to check
            p = se.pair(opts, json.load(open(annot)), {i: img for i, img in enumerate(json.load(open(annot))["images"])})
            for k in (0, 1, n_frames - 1):
                f = p.frames[k]
                want = script_frame(cv2, Image, f.path, f.boxes, f.texts, scale, io.BytesIO())
                buf = io.BytesIO()
                Image.fromarray(want).save(buf, format="JPEG")
                assert open(f.out, "rb").read() == buf.getvalue(), (scale, k)
            t0 = time.perf_counter()
            se.run(opts)
            ms = (time.perf_counter() - t0) * 1e3
            say(f"--vis-scale {scale}")
            say(f"  (1) command: {ms / n_frames:6.2f} ms per frame ({ms / 1e3:.2f} s for {n_frames} frames, "
                f"{n_frames / ms * 1e3:.0f} frames/s), reads, labels, device and writes included")
            frames = p.frames[:64]
            files = []
            for f in frames:
                files.append(se.render(f, scale))
            batches = [(files[k:k + se.BATCH], frames[k:k + se.BATCH]) for k in range(0, len(frames), se.BATCH)]
            for fb, frb in batches[:2]:
                se.device_pass(fb, frb, scale)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(3):
                for fb, frb in batches:
                    se.device_pass(fb, frb, scale)
            ms = (time.perf_counter() - t0) * 1e3 / (3 * len(frames))
            say(f"  (2) device pass alone (decode, {'resize, ' if scale != 1 else ''}draw, encode; batches of "
                f"{se.BATCH}): {ms:6.2f} ms per frame")
            t0 = time.perf_counter()
            for f in frames:
                se.text_points(f.texts, f.out_hw)
            ms = (time.perf_counter() - t0) * 1e3 / len(frames)
            say(f"  (3) host labels alone ({DETS} putText + scan, one core): {ms:6.2f} ms per frame")
            k = 24
            t0 = time.perf_counter()
            for f in frames[:k]:
                script_frame(cv2, Image, f.path, f.boxes, f.texts, scale, os.path.join(tmp, "script.jpg"))
            ms = (time.perf_counter() - t0) * 1e3 / k
            say(f"  (4) script's host path (PIL open, {'imrescale, ' if scale != 1 else ''}cv2 drawing, PIL save; one "
                f"core): {ms:6.2f} ms per frame")
    with open(out_path, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
