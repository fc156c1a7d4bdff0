"""Detection drawing on the device (sy_draw_boxes, python -m streamyolo_b200.vis, StreamDetector(record_boxes=...)) on
1200 x 1920 frames, against the sAP toolkit's host path.

  (1) device    decode (data.decode_jpeg_sized) + draw (data.draw_boxes) + encode at q 75 (data.encode_jpeg) of n = 1, 8,
                16 frames with about 20 and about 200 boxes each: host wall time of ``iters`` batches after warm-up (each
                ends in a synchronisation), per frame; and the draw kernel alone (CUDA events)
  (2) host      vis_det_th.py's per-frame work on one core: PIL open, the cv2 drawing of vis_obj_fancy, PIL save (when
                PIL and cv2 are installed; otherwise reported as not measured)
  (3) CLI       python -m streamyolo_b200.vis on a synthetic 900-frame sequence (20 boxes per frame) in a temporary
                directory: frames/s end to end, and the time of reading every input and writing every output file alone
  (4) tick      StreamDetector (StreamYOLO-l, calibrated synthetic weights, fp16 storage) on S = 8 NV12 cameras with
                record_quality=95, without and with record_boxes=(0.3, palette), alternating tick by tick: median and p90
                of ``step`` and of last_jpeg()

The device's drawn files are checked against the oracle (oracle/vis_oracle.py) and cv2 when present before anything is
timed.  The card's name and power limit are read in the same run.
usage: python tools/bench_vis.py [iters] [ticks] [out path]"""
import json
import os
import pickle
import statistics
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

from bench_stream import calibrated_l, card
from oracle import vis_oracle as vo
from oracle.make_jpeg_golden import synth_frame
from oracle.make_yuv_golden import synth_frame as synth_yuv
from streamyolo_b200 import data, stream, vis

FRAME_HW = (1200, 1920)


def rand_boxes(rng, n, h, w):
    x, y = rng.uniform(-0.05 * w, w, n), rng.uniform(-0.05 * h, h, n)
    bw, bh = rng.uniform(8, 0.25 * w, n), rng.uniform(8, 0.25 * h, n)
    return np.round(np.stack([x, y, x + bw, y + bh], 1)).astype(np.int32), rng.integers(0, 8, n)


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    ticks = int(sys.argv[2]) if len(sys.argv) > 2 else 60
    out_path = sys.argv[3] if len(sys.argv) > 3 else os.path.join(os.path.dirname(HERE), "profiles", "h100_vis.txt")
    lines = []

    def say(s):
        print(s, flush=True)
        lines.append(s)

    try:
        import cv2
        from PIL import Image
    except ImportError:
        cv2 = Image = None
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    say(f"$ python tools/bench_vis.py {iters} {ticks}")
    say(f"card (name, power limit, max SM clock): {card()}")
    say(f"host: {os.cpu_count()} cores, " + (f"cv2 {cv2.__version__}, PIL" if cv2 else "no cv2 / PIL"))
    h, w = FRAME_HW
    rng = np.random.default_rng(0)
    palette_rgb = rng.integers(0, 256, (8, 3)).astype(np.uint8)
    pal_bgr = palette_rgb[:, ::-1].copy()
    host = [synth_frame(h, w, 500 + i) for i in range(16)]
    files = data.encode_jpeg(torch.from_numpy(np.stack(host)).to(dev), 90)
    decoded = [None] * 16
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    say(f"(1) device decode + draw + encode at q {vis.QUALITY}, {h}x{w} frames (input files of "
        f"{statistics.mean(len(f) for f in files) / 1e3:.0f} kB)")
    for nb in (20, 200):
        boxes = [rand_boxes(rng, nb, h, w) for _ in range(16)]
        frames = [vis.Frame("", FRAME_HW, "", bx, lb) for bx, lb in boxes]
        got = vis.device_pass(files, frames, pal_bgr)
        if decoded[0] is None:
            s, l = data.pack_jpeg(files, max(len(f) for f in files))
            img, st = data.decode_jpeg_sized(torch.from_numpy(s).to(dev), torch.from_numpy(l).to(dev), [FRAME_HW] * 16,
                                             FRAME_HW)
            decoded = [img[i].cpu().numpy() for i in range(16)]
        for i in (0, 7, 15):                                 # against the oracle drawing, encoded by the device encoder
            want = data.encode_jpeg(torch.from_numpy(vo.draw(decoded[i], *boxes[i], pal_bgr)).to(dev)[None], vis.QUALITY)[0]
            assert got[i] == want, (nb, i)
            if cv2 is not None:
                assert want == cv2.imencode(".jpg", vo.draw(decoded[i], *boxes[i], pal_bgr),
                                            [cv2.IMWRITE_JPEG_QUALITY, vis.QUALITY])[1].tobytes()
        for n in (1, 8, 16):
            for _ in range(3):
                vis.device_pass(files[:n], frames[:n], pal_bgr)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(iters):
                vis.device_pass(files[:n], frames[:n], pal_bgr)
            ms = (time.perf_counter() - t0) * 1e3 / iters
            say(f"  {nb:3d} boxes, n={n:2d}: {ms:7.2f} ms per batch (host wall, with the copies in and out and two "
                f"synchronisations), {ms / n:6.2f} ms per frame")
        slots = torch.from_numpy(np.stack(decoded)).to(dev)
        work = slots.clone()
        b_t = torch.from_numpy(np.stack([bx for bx, _ in boxes])).to(dev)
        l_t = torch.from_numpy(np.stack([lb for _, lb in boxes]).astype(np.int32)).to(dev)
        c_t = torch.full((16,), nb, dtype=torch.int32, device=dev)
        p_t = torch.from_numpy(pal_bgr).to(dev)
        s_t = torch.tensor([FRAME_HW] * 16, dtype=torch.int32, device=dev)
        for n in (1, 16):
            run = lambda: data.draw_boxes(slots[:n], b_t[:n], l_t[:n], c_t[:n], p_t, s_t[:n], out=work[:n])
            for _ in range(5):
                run()
            torch.cuda.synchronize()
            a.record()
            for _ in range(iters * 5):
                run()
            b.record()
            torch.cuda.synchronize()
            us = a.elapsed_time(b) * 1e3 / (iters * 5)
            say(f"  draw kernel alone, {nb} boxes, n={n:2d}: {us:7.1f} us per launch, {us / n:6.1f} us per frame "
                "(CUDA events)")
    if cv2 is not None:
        with tempfile.TemporaryDirectory() as tmp:
            paths = []
            for i, f in enumerate(files[:8]):
                p = os.path.join(tmp, f"{i}.jpg")
                open(p, "wb").write(f)
                paths.append(p)
            for nb in (20, 200):
                boxes = [rand_boxes(rng, nb, h, w) for _ in range(8)]
                t0 = time.perf_counter()
                for p, (bx, lb) in zip(paths, boxes):
                    img = np.array(Image.open(p))
                    filled = img.copy()
                    for q, l in zip(bx, lb):
                        cv2.rectangle(img, (int(q[0]), int(q[1])), (int(q[2]), int(q[3])),
                                      [int(c) for c in palette_rgb[l]], thickness=-1)
                    img = cv2.addWeighted(filled, 0.8, img, 0.2, 0)
                    for q, l in zip(bx, lb):
                        cv2.rectangle(img, (int(q[0]), int(q[1])), (int(q[2]), int(q[3])),
                                      [int(c) for c in palette_rgb[l]], thickness=2)
                    Image.fromarray(img).save(p + ".out.jpg")
                ms = (time.perf_counter() - t0) * 1e3 / len(paths)
                say(f"(2) host path, {nb} boxes: {ms:.1f} ms per frame on one core (PIL open, cv2 drawing, PIL save)")
    else:
        say("(2) host path: not measured (no PIL / cv2 on this host)")
    n_frames = 900
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "data", "s0"))
        images, results = [], []
        for i in range(n_frames):
            name = f"{i:06d}.jpg"
            open(os.path.join(tmp, "data", "s0", name), "wb").write(files[i % 16])
            images.append({"id": i, "sid": 0, "fid": i, "name": name, "width": w, "height": h})
            bx, lb = rand_boxes(rng, 20, h, w)
            for q, l in zip(bx, lb):
                results.append({"image_id": i, "bbox": np.asarray([q[0], q[1], q[2] - q[0], q[3] - q[1]], np.float32),
                                "score": np.float32(rng.uniform(0.2, 1)), "category_id": np.int32(l)})
        annot = os.path.join(tmp, "annot.json")
        json.dump({"images": images, "annotations": [], "sequences": ["s0"], "seq_dirs": ["s0"],
                   "categories": [{"id": k, "name": str(k)} for k in range(8)], "coco_subset": list(range(8))},
                  open(annot, "w"))
        pickle.dump(results, open(os.path.join(tmp, "res.pkl"), "wb"))
        os.makedirs(os.path.join(tmp, "sAP", "vis"))
        open(os.path.join(tmp, "sAP", "vis", "vis_det_th.py"), "w").write(
            "class_palette = " + repr({k: tuple(int(c) for c in palette_rgb[k]) for k in range(8)}) + "\n")
        argv = ["--data-root", os.path.join(tmp, "data"), "--annot-path", annot, "--result-path",
                os.path.join(tmp, "res.pkl"), "--vis-dir", os.path.join(tmp, "vis"), "--overwrite"]
        vis.run(vis.parse_args(argv), search=(os.path.join(tmp, "sAP"),))     # warm-up: caches, first launches
        walls = []
        for _ in range(2):
            t0 = time.perf_counter()
            with open(os.devnull, "w") as nul:
                old, sys.stdout = sys.stdout, nul
                try:
                    vis.run(vis.parse_args(argv), search=(os.path.join(tmp, "sAP"),))
                finally:
                    sys.stdout = old
            walls.append(time.perf_counter() - t0)
        outs = sorted(os.listdir(os.path.join(tmp, "vis", "s0")))
        sizes = [os.path.getsize(os.path.join(tmp, "vis", "s0", f)) for f in outs]
        t0 = time.perf_counter()
        for i in range(n_frames):
            vis._read(os.path.join(tmp, "data", "s0", f"{i:06d}.jpg"))
            vis._write(os.path.join(tmp, "io", f"{i:06d}.jpg"), bytes(sizes[i]))
        io_s = time.perf_counter() - t0
        wall = min(walls)
        say(f"(3) CLI, {n_frames} frames of {h}x{w}, 20 boxes each: {wall:.2f} s, {n_frames / wall:.0f} frames/s "
            f"(best of {len(walls)}); reading the inputs and writing the {statistics.mean(sizes) / 1e3:.0f} kB outputs "
            f"alone, on one thread: {io_s:.2f} s ({100 * io_s / wall:.0f}% of the run, overlapped with the device there)")
    model = calibrated_l(dev)
    nc = model.head.num_classes
    s = 8
    yuv = [[synth_yuv("nv12", h, w, 100 * k + i) for i in range(s)] for k in range(4)]
    kw = dict(frame_hw=FRAME_HW, in_scale=0.5, streams=s, conf_thre=0.01, nms_thre=0.65, frame_format="nv12",
              record_quality=95)
    pal = [tuple(int(v) for v in rng.integers(0, 256, 3)) for _ in range(nc)]
    dets = {"record": stream.StreamDetector(model, **kw),
            "record+boxes": stream.StreamDetector(model, record_boxes=(0.3, pal), **kw)}
    for k in range(4):
        r, p = dets["record+boxes"].step(yuv[k]), dets["record"].step(yuv[k])
        assert all(np.array_equal(x, y) for u, v in zip(r, p) for x, y in zip(u, v)), k
    n_drawn = sum(int((sc >= np.float32(0.3)).sum()) for _, sc, _ in r)
    wall = {k: [] for k in dets}
    read = {k: [] for k in dets}
    for t in range(2 * ticks):
        leg = ("record", "record+boxes")[(t + t // 2) % 2]
        t0 = time.perf_counter()
        dets[leg].step(yuv[t % 4])
        wall[leg].append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        dets[leg].last_jpeg()
        read[leg].append((time.perf_counter() - t0) * 1e3)
    say(f"(4) StreamDetector tick, S={s} NV12 {h}x{w} cameras, StreamYOLO-l fp16 storage, record_quality=95, {ticks} "
        f"ticks per leg, alternated; detections equal; {n_drawn} boxes drawn over the 8 frames of the last warm-up tick")
    for leg in dets:
        say(f"  {leg:13s}: step median {statistics.median(wall[leg]):7.2f} ms, p90 "
            f"{float(np.percentile(wall[leg], 90)):7.2f} ms; last_jpeg() median {statistics.median(read[leg]):6.2f} ms")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as fh:
        fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
