"""The sAP streaming driver (sAP/streamyolo/streamyolo_det.py) on the device: JPEG files in, the driver's per-sequence
pickles and time_info.pkl out, for the reference's streaming_eval.py to score.

    cd StreamYOLO/sAP/streamyolo
    python -m streamyolo_b200.sap --data-root ... --annot-path .../val.json --fps 30 --in_scale 0.5 --no-mask \\
        --out-dir ... --overwrite --config cfgs/l_s50_onex_dfp_tal_flip.py --weights l_s50_one_x.pth     # wall clock
    python -m streamyolo_b200.sap ... --clock simulated --runtime-ms 33 --streams 8                       # simulated clock
    python -m streamyolo_b200.sap ... --clock simulated --runtime rt.pkl --seed 0 --streams 8           # drawn runtimes
    python -m streamyolo_b200.sap ... --clock infinite --runtime rt.pkl --seed 0 --streams 8            # infinite GPUs

It takes the driver's arguments (``--cpu-pre`` and ``--no-class-mapping`` are ignored, as there) and these:

  --clock wall       (default) the driver's loop (:152-195) on ``time.perf_counter``, one sequence at a time.  Before a
                     sequence starts its files are decoded on the device (``data.decode_jpeg``, bit-exact against
                     cv2.imread) into one device tensor, outside the timed region as the driver's cv2.imread loop is;
                     each tick is one ``StreamDetector.step`` (one CUDA graph replay).
  --clock simulated  the simulated-time scheduler of sAP/det/srt_det.py:102-165 with a constant runtime of
                     ``--runtime-ms`` per frame, or with each frame's runtime drawn from the ``--runtime`` distribution
                     (scaled by ``--perf-factor``, seeded by ``--seed``) as srt_det.py draws it: the schedule no longer
                     depends on the detector, so every sequence's frame list is computed first and up to ``--streams``
                     sequences run at once, one stream each, in one ``StreamDetector(jpeg_max_bytes=...)``.  ``runtime``
                     holds each kept frame's runtime.
  --clock infinite   sAP/det/srt_det_inf.py, the same protocol with infinite GPUs: every frame ii is detected and its
                     result is out at ``ii / fps + draw``; each pickle is then reordered by ``np.argsort(timestamps)``.
                     The script runs single-frame detectors; here frame ii is fused with frame ii - 1 (frame 0 with
                     itself), what the driver's loop gives when it detects every frame.  The frames run as on the
                     simulated clock, a sequence's frames on one stream, up to ``--streams`` sequences at once.

``--runtime`` is a pickled ``{'type': 'empirical', 'samples': [...]}``, what sAP/util/add_to_runtime_zoo.py makes of a
run's time_info.pkl.  The draws are the scripts' bit for bit: ``np.random.RandomState(seed).choice(samples /
perf_factor)``, one per frame that passes the stride / dynamic-schedule checks (the one that ends a sequence included),
the generator carried from one sequence to the next in the annotation file's order.  The global numpy state is left
alone.  ``--cached-res`` (replaying stored single-frame results) raises NotImplementedError: a StreamYOLO detection
depends on the frame processed before it, so cached single-frame results cannot be re-scheduled.

Boxes are in frame pixels: the detector divides by ``--in_scale``, which is what the driver's ``inference()`` divides by
at the default 0.5 (it keeps its own default of 0.5 whatever ``--in_scale`` says).  Frames must be 1200 x 1920, the size
the driver's ``preproc`` assumes when it computes its input size (:177).
"""
import argparse
import json
import os
import pickle
import time
from collections import deque
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import data, feed, ops, stream

DRIVER_HW = (1200, 1920)          # streamyolo_det.py:177: the input size is int(1200 * in_scale) x int(1920 * in_scale)
DECODE_BATCH = 16                 # files per decode_jpeg call when a sequence is loaded


def parse_args(argv=None):
    """The driver's arguments (streamyolo_det.py:30-47) and ``--clock``, ``--runtime-ms``, ``--streams``; srt_det.py's
    ``--runtime``, ``--perf-factor``, ``--seed`` and ``--cached-res``."""
    p = argparse.ArgumentParser(prog="python -m streamyolo_b200.sap")
    p.add_argument("--data-root", type=str, required=True)
    p.add_argument("--annot-path", type=str, required=True)
    p.add_argument("--det-stride", type=float, default=None)
    p.add_argument("--in_scale", type=float, default=0.5)
    p.add_argument("--fps", type=float, default=30)
    p.add_argument("--no-mask", action="store_true", default=False)
    p.add_argument("--no-class-mapping", action="store_true", default=False)
    p.add_argument("--cpu-pre", action="store_true", default=False)
    p.add_argument("--dynamic-schedule", action="store_true", default=False)
    p.add_argument("--out-dir", type=str, required=True)
    p.add_argument("--config", type=str, required=True)
    p.add_argument("--weights", type=str, required=True)
    p.add_argument("--overwrite", action="store_true", default=False)
    p.add_argument("--clock", choices=("wall", "simulated", "infinite"), default="wall")
    p.add_argument("--runtime-ms", type=float, default=None, help="simulated clock: the runtime of every frame")
    p.add_argument("--runtime", type=str, default=None, help="simulated and infinite clocks: a pickled runtime "
                   "distribution ({'type': 'empirical', 'samples': [...]}) to draw each frame's runtime from")
    p.add_argument("--perf-factor", type=float, default=None, help="with --runtime: samples are divided by it (default 1)")
    p.add_argument("--seed", type=int, default=None, help="with --runtime: the draws' seed (default 0)")
    p.add_argument("--cached-res", type=str, default=None, help="not supported (see the module doc)")
    p.add_argument("--streams", type=int, default=1, help="simulated and infinite clocks: sequences run at once")
    opts = p.parse_args(argv)
    if opts.clock == "wall" and (opts.runtime_ms is not None or opts.runtime is not None or opts.streams != 1):
        p.error("--runtime-ms, --runtime and --streams take --clock simulated or infinite; the wall clock runs one "
                "sequence at a time")
    if opts.runtime_ms is not None and opts.runtime is not None:
        p.error("--runtime-ms and --runtime are mutually exclusive")
    if opts.clock == "simulated" and opts.runtime is None and (opts.runtime_ms is None or not opts.runtime_ms > 0):
        p.error("--clock simulated needs a positive --runtime-ms or a --runtime distribution")
    if opts.clock == "infinite":
        if opts.runtime is None:
            p.error("--clock infinite needs a --runtime distribution")
        if opts.det_stride is not None or opts.dynamic_schedule:
            p.error("--clock infinite detects every frame: it takes neither --det-stride nor --dynamic-schedule")
    if opts.runtime is None and (opts.perf_factor is not None or opts.seed is not None):
        p.error("--perf-factor and --seed take --runtime")
    if opts.perf_factor is not None and not opts.perf_factor > 0:
        p.error("--perf-factor must be positive")
    if opts.streams < 1:
        p.error("--streams must be at least 1")
    opts.det_stride = 1 if opts.det_stride is None else opts.det_stride
    opts.perf_factor = 1 if opts.perf_factor is None else opts.perf_factor
    opts.seed = 0 if opts.seed is None else opts.seed
    if opts.cached_res is not None:
        raise NotImplementedError("--cached-res: a StreamYOLO detection depends on the frame processed before it, so "
                                  "stored single-frame results cannot be re-scheduled")
    return opts


class Empirical:
    """srt_det.py's runtime distribution (util/runtime_dist.py ``Empirical``) on a generator of its own: ``samples /
    perf_factor`` in float64 (the values of the script's in-place ``/=``), ``draw()`` is ``np.random.choice(samples)``
    after ``np.random.seed(seed)``, and the global numpy state is left alone."""

    def __init__(self, samples, perf_factor=1, seed=0):
        if not perf_factor > 0:
            raise ValueError(f"perf_factor must be positive, not {perf_factor}")
        self.samples = np.asarray(samples, np.float64) / perf_factor
        self.rng = np.random.RandomState(seed)

    def draw(self):
        return self.rng.choice(self.samples)

    def mean(self):
        return self.samples.mean()


def load_runtime(path, perf_factor=1, seed=0):
    """a pickled runtime distribution -> ``Empirical``; ValueError for any type but 'empirical', as dist_from_dict"""
    with open(path, "rb") as f:
        dist = pickle.load(f)
    if dist["type"] != "empirical":
        raise ValueError(f'Unknown distribution type "{dist["type"]}"')
    return Empirical(dist["samples"], perf_factor, seed)


def sequences(dataset):
    """Each sequence's images (the annotation file's dicts) in the driver's order: ``[img for img in db.imgs.values() if
    img['sid'] == sid]`` (:128), where ``COCO.imgs`` maps id -> image in the order of ``dataset['images']`` (a repeated
    id keeps its first position and its last dict)."""
    imgs = {}
    for img in dataset["images"]:
        imgs[img["id"]] = img
    return [[img for img in imgs.values() if img["sid"] == sid] for sid in range(len(dataset["sequences"]))]


def wall_sequence(det, frames, n_frame, fps, det_stride, dynamic_schedule, clock=time.perf_counter):
    """One sequence through the driver's real-time loop (:138-195): ``frames[fidx]`` is frame fidx as ``det.step`` takes
    it (the device-decoded sequence), ``clock`` the host clock.  -> the sequence's pickle dict (:199-205)."""
    timestamps, results_raw, results_parsed, input_fidx, runtime = [], [], [], [], []
    last_fidx = None
    stride_cnt = 0
    t_total = n_frame / fps
    det.reset()                                       # buffer = None (:150)
    t_start = clock()
    while True:
        t1 = clock()
        t_elapsed = t1 - t_start
        if t_elapsed >= t_total:
            break
        fidx_continuous = t_elapsed * fps             # the latest frame out
        fidx = int(np.floor(fidx_continuous))
        if fidx == last_fidx:
            continue
        last_fidx = fidx
        if dynamic_schedule:
            if fidx_continuous - fidx > 0.5:
                continue
        elif stride_cnt % det_stride == 0:
            stride_cnt = 1
        else:
            stride_cnt += 1
            continue
        bboxes, scores, labels = det.step(frames[fidx])[0]      # resize, on_pipe forward, NMS; synchronises
        t2 = clock()
        t_elapsed = t2 - t_start
        if t_elapsed >= t_total:
            break
        timestamps.append(t_elapsed)
        results_raw.append(det.last_raw())
        results_parsed.append((bboxes, scores, labels, None))
        input_fidx.append(fidx)
        runtime.append(t2 - t1)
    return {"results_raw": results_raw, "results_parsed": results_parsed, "timestamps": timestamps,
            "input_fidx": input_fidx, "runtime": runtime}


def simulated_schedule(n_frame, fps, det_stride, dynamic_schedule, runtime):
    """srt_det.py:102-165.  ``runtime`` is a number, the seconds every frame takes -> (input_fidx, timestamps); or an
    ``Empirical`` that each frame's runtime is drawn from -> (input_fidx, timestamps, runtime), the last the draws of
    the frames kept.  The detector's outputs take no part in the schedule: it is a function of these arguments (and of
    the generator's state, which moves on by one draw per frame run, the one that ends the sequence included)."""
    draws = None if np.isscalar(runtime) else []
    input_fidx, timestamps = [], []
    last_fidx = None
    t_total = n_frame / fps
    t_elapsed = 0
    mean_rtf = (runtime if draws is None else runtime.mean()) * fps
    stride_cnt = 0
    while t_elapsed < t_total:
        fidx_continuous = t_elapsed * fps
        fidx = int(np.floor(fidx_continuous))
        if fidx == last_fidx:                         # the detector is idle until the next frame arrives
            fidx += 1
            if fidx == n_frame:
                break
            t_elapsed = fidx / fps
        last_fidx = fidx
        if dynamic_schedule:
            # with the runtime above one frame interval, wait for the next frame when this one's result would not be out
            # any earlier (fidx_continuous is the time the loop last read, as in srt_det.py)
            if mean_rtf > 1 and mean_rtf < np.floor(fidx_continuous - fidx + mean_rtf):
                continue
        elif stride_cnt % det_stride == 0:
            stride_cnt = 1
        else:
            stride_cnt += 1
            continue
        rt_this = runtime if draws is None else runtime.draw()
        t_elapsed += rt_this
        if t_elapsed >= t_total:
            break
        timestamps.append(t_elapsed)
        input_fidx.append(fidx)
        if draws is not None:
            draws.append(rt_this)
    return (input_fidx, timestamps) if draws is None else (input_fidx, timestamps, draws)


def infinite_order(out):
    """srt_det_inf.py:127-134: a sequence's pickle dict, its frames in detection order, reordered in place by
    ``np.argsort(timestamps)`` (the default, unstable kind: ties fall as they fall in the script)"""
    idx = np.argsort(out["timestamps"])
    for k in ("timestamps", "results_raw", "results_parsed", "input_fidx", "runtime"):
        out[k] = [out[k][i] for i in idx]
    return out


def pack_ticks(lengths, streams):
    """Sequences of ``lengths`` ticks onto ``streams`` streams, in order, each stream taking the next sequence when its
    own ends -> one list per tick of ``streams`` entries: ``(sequence, k)`` (the k-th scheduled frame of that sequence; k
    = 0 starts it) or None (the stream is idle).  Sequences of length 0 take no stream."""
    queue = deque(q for q, n in enumerate(lengths) if n > 0)
    cur, pos = [None] * streams, [0] * streams
    ticks = []
    while True:
        row = []
        for s in range(streams):
            if cur[s] is not None and pos[s] == lengths[cur[s]]:
                cur[s] = None
            if cur[s] is None and queue:
                cur[s], pos[s] = queue.popleft(), 0
            row.append(None if cur[s] is None else (cur[s], pos[s]))
            if cur[s] is not None:
                pos[s] += 1
        if all(e is None for e in row):
            return ticks
        ticks.append(row)


def run_simulated(det, files, schedules, runtime, done):
    """Run every sequence's scheduled frames on the streams of ``det`` (a StreamDetector built with ``jpeg_max_bytes``),
    packed by ``pack_ticks``.  ``files[q]`` are sequence q's file paths, ``schedules[q]`` its (input_fidx, timestamps)
    with ``runtime`` the runtime of every frame, or its (input_fidx, timestamps, runtimes) with ``runtime`` None;
    ``done(q, out)`` gets sequence q's pickle dict as soon as its last frame has run (and every empty sequence first).

    A host thread reads the files of tick k + 1 while tick k runs.  Only the files are held: S decoded sequences (6.2 GB
    each at 900 frames of 1200 x 1920) would not fit, so each tick's replay decodes its S files itself."""
    outs = [{"results_raw": [], "results_parsed": [], "timestamps": list(s[1]), "input_fidx": list(s[0]),
             "runtime": [runtime] * len(s[0]) if runtime is not None else list(s[2])} for s in schedules]
    for q, (fi, *_) in enumerate(schedules):
        if not fi:
            done(q, outs[q])
    lengths = [len(s[0]) for s in schedules]
    ticks = pack_ticks(lengths, det.streams) if any(lengths) else []

    def path(e):
        q, k = e
        return files[q][schedules[q][0][k]]

    def read(row):
        return [None if e is None else np.fromfile(path(e), np.uint8) for e in row]

    with ThreadPoolExecutor(max_workers=1) as reader:
        nxt = reader.submit(read, ticks[0]) if ticks else None
        for t, row in enumerate(ticks):
            tick_files = nxt.result()
            if t + 1 < len(ticks):
                nxt = reader.submit(read, ticks[t + 1])
            for s, e in enumerate(row):
                if e is not None and e[1] == 0:
                    det.reset(s)
            got = det.step_jpeg(tick_files)
            status, raw = det.last_status(), det.last_raw()
            for s, e in enumerate(row):
                if e is None:
                    continue
                if status[s] != 0:
                    raise RuntimeError(f"sAP: {path(e)} did not decode: {data.JPEG_STATUS.get(int(status[s]), status[s])}")
                q, k = e
                outs[q]["results_raw"].append(raw[s:s + 1].clone() if det.streams > 1 else raw)
                outs[q]["results_parsed"].append((*got[s], None))
                if k + 1 == len(schedules[q][0]):
                    done(q, outs[q])
                    outs[q] = None


def decode_sequence(paths, hw, device, batch=DECODE_BATCH):
    """The sequence's files -> uint8 [n, h, w, 3] on the device, what cv2.imread returns for each (data.decode_jpeg, in
    batches of ``batch`` files); RuntimeError naming the first file that does not decode."""
    h, w = hw
    frames = torch.empty((len(paths), h, w, 3), dtype=torch.uint8, device=device)
    if not paths:
        return frames
    max_bytes = feed.default_max_bytes(paths)
    status = torch.empty((len(paths),), dtype=torch.int32, device=device)
    ws = torch.empty(max(ops.jpeg_decode_workspace_bytes(n, max_bytes, h, w) for n in {min(batch, len(paths)),
                         len(paths) % batch or batch}), dtype=torch.uint8, device=device)
    for k in range(0, len(paths), batch):
        chunk = paths[k:k + batch]
        rows, lengths = data.pack_jpeg([np.fromfile(p, np.uint8) for p in chunk], max_bytes)
        data.decode_jpeg(torch.from_numpy(rows).to(device), torch.from_numpy(lengths).to(device), hw,
                         out=frames[k:k + len(chunk)], status=status[k:k + len(chunk)], workspace=ws)
    for i, s in enumerate(status.tolist()):
        if s != 0:
            raise RuntimeError(f"sAP: {paths[i]} did not decode: {data.JPEG_STATUS.get(s, f'status {s}')}")
    return frames


def frame_paths(opts, dataset):
    """-> (sequence names, each sequence's file paths in the driver's order); ValueError for a frame that is not 1200 x
    1920 by the annotation file"""
    seqs, seq_dirs = dataset["sequences"], dataset["seq_dirs"]
    paths = []
    for sid, imgs in enumerate(sequences(dataset)):
        for img in imgs:
            if (img["height"], img["width"]) != DRIVER_HW:
                raise ValueError(f"sAP: {img['name']} is {img['height']}x{img['width']}; the driver's input size "
                                 f"(int(1200 * in_scale), int(1920 * in_scale)) is that of 1200x1920 frames")
        paths.append([os.path.join(opts.data_root, seq_dirs[sid], img["name"]) for img in imgs])
    return seqs, paths


def dump(path, obj, overwrite):
    """the driver's ``if opts.overwrite or not isfile(out_path): pickle.dump(...)``"""
    if overwrite or not os.path.isfile(path):
        with open(path, "wb") as f:
            pickle.dump(obj, f)


def _stats(var, name, cvt):
    """the line util.print_stats prints (format %.3g; std with one degree of freedom)"""
    var = np.asarray(var)
    if len(var) == 1:
        print(f"{name}: scalar: {cvt(var[0]):.3g}")
    else:
        print(f"{name}: mean: {cvt(var.mean()):.3g}; std: {cvt(var.std(ddof=1)):.3g}; min: {cvt(var.min()):.3g}; "
              f"max: {cvt(var.max()):.3g}")


def run(opts, model, clock=time.perf_counter, detector=stream.StreamDetector):
    """The driver's main() after the model is built (:93-229): every sequence's pickle and time_info.pkl written to
    ``opts.out_dir`` (``parse_args``' namespace) and the driver's summary printed.  ``model``: YOLOX in eval mode on the
    GPU with its weights loaded.  ``clock`` is the wall clock's timer, ``detector`` the StreamDetector class (tests pass
    fakes of both).  -> the time_info dict."""
    os.makedirs(opts.out_dir, exist_ok=True)
    with open(opts.annot_path) as f:
        dataset = json.load(f)
    seqs, paths = frame_paths(opts, dataset)
    runtimes = [None] * len(paths)                # each sequence's runtimes, for time_info in the driver's order

    def done(q, out):
        dump(os.path.join(opts.out_dir, seqs[q] + ".pkl"), out, opts.overwrite)
        runtimes[q] = out["runtime"]

    if opts.clock == "wall":
        det = detector(model, frame_hw=DRIVER_HW, in_scale=opts.in_scale)
        device = next(model.parameters()).device
        for q, p in enumerate(paths):
            frames = decode_sequence(p, DRIVER_HW, device)
            done(q, wall_sequence(det, frames, len(p), opts.fps, opts.det_stride, opts.dynamic_schedule, clock))
            del frames
    else:
        # every schedule first, in the sequences' order: the draws carry the generator from one sequence to the next
        rt = None if opts.runtime is None else load_runtime(opts.runtime, opts.perf_factor, opts.seed)
        const = opts.runtime_ms / 1000.0 if rt is None else None
        if opts.clock == "simulated":
            schedules = [simulated_schedule(len(p), opts.fps, opts.det_stride, opts.dynamic_schedule,
                                            const if rt is None else rt) for p in paths]
        else:                                     # srt_det_inf.py:98-125: every frame, out at ii / fps + draw
            schedules = []
            for p in paths:
                draws = [rt.draw() for _ in range(len(p))]
                schedules.append((list(range(len(p))), [ii / opts.fps + d for ii, d in enumerate(draws)], draws))
        finish = done if opts.clock == "simulated" else lambda q, out: done(q, infinite_order(out))
        used = [p[i] for p, s in zip(paths, schedules) for i in s[0]]
        busy = sum(1 for s in schedules if s[0])
        det = None if not used else detector(model, frame_sizes=[DRIVER_HW] * min(opts.streams, busy),
                                             in_scale=opts.in_scale, jpeg_max_bytes=feed.default_max_bytes(used))
        run_simulated(det, paths, schedules, const, finish)
    runtime_all = [r for rs in runtimes for r in rs]
    n_processed, n_total = len(runtime_all), sum(len(p) for p in paths)
    runtime_all_np = np.asarray(runtime_all)
    n_small_runtime = (runtime_all_np < 1.0 / opts.fps).sum()
    info = {"runtime_all": runtime_all, "n_processed": n_processed, "n_total": n_total, "n_small_runtime": n_small_runtime}
    dump(os.path.join(opts.out_dir, "time_info.pkl"), info, opts.overwrite)
    print(f"{n_processed}/{n_total} frames processed")
    if n_processed:
        _stats(runtime_all_np, "Runtime (ms)", cvt=lambda x: 1e3 * x)
        print(f"Runtime smaller than unit time interval: {n_small_runtime}/{n_processed} "
              f"({100.0 * n_small_runtime / n_processed:.4g}%)")
    return info


def build_model(config, weights):
    """The driver's model (:100-111) on this package's YOLOX: ``get_exp(config).get_model()`` with the checkpoint's
    ``model`` weights, in eval mode on the GPU, with fp16 activation storage (the driver's ``model.half()``)."""
    from . import dropin
    dropin.install()                              # the cfg's ``from exps.model.yolox import YOLOX`` is this package's
    from yolox.exp import get_exp
    exp = get_exp(config, None)
    model = exp.get_model()
    model.cuda()
    model.eval()
    ckpt = torch.load(weights, map_location="cpu", weights_only=False)
    model.load_state_dict(ckpt["model"])
    print("loaded checkpoint done.")
    model.activation_dtype = torch.float16
    return model


def main(argv=None):
    opts = parse_args(argv)
    return run(opts, build_model(opts.config, opts.weights))


if __name__ == "__main__":
    main()
