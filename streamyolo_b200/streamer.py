"""The sAP toolkit's streamer (sAP/forecast/streamer.py) on the device: StreamYOLO detections forecast to every frame at
a fixed output rate, the per-sequence pickles and time_info.pkl out for the toolkit's streaming_eval.py to score.

    python -m streamyolo_b200.streamer --data-root ... --annot-path .../val.json --fps 30 --eta 0 \\
        --config cfgs/l_s50_onex_dfp_tal_flip.py --weights l_s50_one_x.pth --runtime rt.pkl --out-dir ... --overwrite
    python -m streamyolo_b200.streamer ... --clock simulated --runtime-ms 33 --streams 8

The streamer's loop (:176-321): the detector runs asynchronously; each non-idle iteration submits the latest frame when
no detection is in flight, waits up to one frame interval less ``--forecast-rt-ub`` for the result, and emits the tracks
of the last detection that has arrived, extrapolated to the query frame ``fidx + eta + 1``.  A detection still in flight
does not change what is emitted.  The tracks follow the streamer's rules: its Kalman filter and IoU association
(pps_forecast_kf.py's, on the device: sy_forecast_update), an empty detection leaves no track (``clear_on_empty``), a
fractional query offset is rounded to fp32 (sy_forecast_extrap_queries).  Outputs are ltrb boxes clipped to the size of
the annotation file's image 0, as the streamer's are.

It takes the streamer's arguments (``--cpu-pre`` and ``--no-mask`` are ignored) and four more:

  --clock wall       (default) the loop on ``time.perf_counter``, one sequence at a time.  A sequence's files are decoded
                     on the device before its clock starts (``sap.decode_sequence``).  The detector is a
                     ``StreamDetector(forecast=True, clear_on_empty=True)``: a detection is a ``submit`` (one graph
                     replay that ends with the track update) and ``poll`` / ``receive``; on receipt ``publish`` copies
                     the tracks to buffers of their own, and each emission is one ``query`` (one launch, one
                     synchronisation) on them, so that it neither waits for nor reads from a tick in flight.
  --clock simulated  the same loop on a virtual clock with a constant detector runtime ``--runtime-ms``: host work takes
                     no time, a detection submitted at t arrives at t + R, a wait for it returns at its arrival or
                     timeout, an idle iteration moves the clock to the next frame.  The schedule then depends on the
                     frame count, fps, R, ``--forecast-rt-ub`` and the dynamic schedule alone, so it is computed first
                     (``simulated_schedule``) and up to ``--streams`` sequences run at once, one stream each, in one
                     ``StreamDetector(jpeg_max_bytes=..., forecast=True, clear_on_empty=True, queries=Q)``: each tick
                     decodes, detects, updates the tracks and extrapolates them to every emission made between this
                     detection's arrival and the next one's, with one synchronisation.  time_info records the virtual
                     durations (``t_det`` = R, the others 0).  It is reproducible; it claims no latency.
  --max-tracks       the most detections one update takes (StreamDetector's ``max_tracks``); more raise RuntimeError

``--runtime`` (a runtime pickle, ``{'type': 'empirical', 'samples': [...]}``) feeds ``--dynamic-schedule`` only:
``mean_rtf`` is the mean of its samples divided by ``--perf-factor``, times fps (util/runtime_dist.py).  Frames must be
1200 x 1920, as for ``streamyolo_b200.sap``.
"""
import argparse
import json
import os
import pickle
import time

import numpy as np

from . import data, feed, sap, stream


def parse_args(argv=None):
    """The streamer's arguments (streamer.py:40-64) and ``--clock``, ``--runtime-ms``, ``--streams``, ``--max-tracks``."""
    p = argparse.ArgumentParser(prog="python -m streamyolo_b200.streamer")
    p.add_argument("--data-root", type=str, required=True)
    p.add_argument("--annot-path", type=str, required=True)
    p.add_argument("--fps", type=float, default=30)
    p.add_argument("--eta", type=float, default=0, help="eta >= -1")
    p.add_argument("--config", type=str, required=True)
    p.add_argument("--weights", type=str, required=True)
    p.add_argument("--in-scale", type=float, default=None)
    p.add_argument("--no-mask", action="store_true", default=False)
    p.add_argument("--cpu-pre", action="store_true", default=False)
    p.add_argument("--dynamic-schedule", action="store_true", default=False)
    p.add_argument("--runtime", type=str, required=True)
    p.add_argument("--perf-factor", type=float, default=1)
    p.add_argument("--match-iou-th", type=float, default=0.3)
    p.add_argument("--forecast-rt-ub", type=float, default=0.003)
    p.add_argument("--out-dir", type=str, required=True)
    p.add_argument("--overwrite", action="store_true", default=False)
    p.add_argument("--clock", choices=("wall", "simulated"), default="wall")
    p.add_argument("--runtime-ms", type=float, default=None, help="simulated clock: the runtime of every detection")
    p.add_argument("--streams", type=int, default=1, help="simulated clock: sequences run at once")
    p.add_argument("--max-tracks", type=int, default=1024, help="the most detections one track update takes")
    opts = p.parse_args(argv)
    if opts.clock == "wall" and (opts.runtime_ms is not None or opts.streams != 1):
        p.error("--runtime-ms and --streams take --clock simulated; the wall clock runs one sequence at a time")
    if opts.clock == "simulated" and (opts.runtime_ms is None or not opts.runtime_ms > 0):
        p.error("--clock simulated needs a positive --runtime-ms")
    if opts.streams < 1:
        p.error("--streams must be at least 1")
    if not 1 <= opts.max_tracks <= 1 << 20:
        p.error("--max-tracks must be in [1, 2^20]")
    if not opts.perf_factor > 0:
        p.error("--perf-factor must be positive")
    if opts.in_scale is None:
        opts.in_scale = 0.5
    return opts


def mean_rtf(runtime_path, perf_factor, fps):
    """streamer.py:127-130: the runtime pickle's mean (util/runtime_dist.py's Empirical, samples / perf_factor) times fps"""
    with open(runtime_path, "rb") as f:
        dist = pickle.load(f)
    if dist["type"] != "empirical":
        raise ValueError(f'Unknown distribution type "{dist["type"]}"')
    samples = np.array(dist["samples"])
    if perf_factor != 1:
        samples /= perf_factor
    return samples.mean() * fps


def next_frame_time(t, fps):
    """the virtual clock after an idle iteration at t: the first time whose floor(t * fps) is the next frame, (f + 1) /
    fps moved up while its product with fps rounds below f + 1"""
    f = int(np.floor(t * fps)) + 1
    u = f / fps
    while np.floor(u * fps) < f:
        u = float(np.nextafter(u, np.inf))
    return u


def _wait_for_next(fidx_continuous, fidx, fidx_latest, dynamic_schedule, rtf):
    """streamer.py:185-196: an idle iteration"""
    if fidx == fidx_latest:
        return True                               # the algorithm is fast and has some idle time
    if dynamic_schedule and rtf >= 1:             # with runtime < 1 every frame is processed
        return bool(rtf < np.floor(fidx_continuous - fidx + rtf))
    return False


def simulated_schedule(n_frame, fps, runtime, forecast_rt_ub=0.003, dynamic_schedule=False, rtf=None):
    """The streamer's loop on the virtual clock (see the module doc) -> dict of
      det_fidx    the input frame of each detection that arrives, in order
      timestamps  each emission's time (the loop's t3)
      emit_det    the detection each emission extrapolates (an index into det_fidx)
      emit_fidx   the latest frame at each emission's loop head (its query is emit_fidx + eta + 1)
      n_forecast  the non-idle iterations (time_info's t_forecast count; t_det has len(det_fidx))"""
    t_total, t_unit = n_frame / fps, 1 / fps
    wait_time = t_unit - forecast_rt_ub
    t = 0.0
    det_fidx, timestamps, emit_det, emit_fidx = [], [], [], []
    n_forecast = 0
    fidx_latest = done_at = None
    while t < t_total:
        fidx_continuous = t * fps
        fidx = int(np.floor(fidx_continuous))
        if _wait_for_next(fidx_continuous, fidx, fidx_latest, dynamic_schedule, rtf):
            t = next_frame_time(t, fps)
            continue
        if done_at is None:                        # submit
            done_at, fidx_latest = t + runtime, fidx
        if done_at <= t + wait_time:               # arrives within the wait
            t = max(t, done_at)
            done_at = None
            det_fidx.append(fidx_latest)
        else:
            t = t + wait_time
        n_forecast += 1
        if t >= t_total:
            break
        if det_fidx:
            timestamps.append(t)
            emit_det.append(len(det_fidx) - 1)
            emit_fidx.append(fidx)
    return {"det_fidx": det_fidx, "timestamps": timestamps, "emit_det": emit_det, "emit_fidx": emit_fidx,
            "n_forecast": n_forecast}


def empty_rows():
    """the streamer's output for a sequence without tracks (:303-306)"""
    return (np.empty((0, 4), dtype=np.float32), np.empty((0,), dtype=np.float32), np.empty((0,), dtype=np.int32), None,
            np.empty((0,), dtype=np.int32))


def output_rows(q):
    """one extrapolation (``StreamDetector.query`` / ``last_queries`` entry) -> the streamer's results_parsed entry:
    ltrb boxes (ltwh2ltrb_ in fp32), scores, labels, None, uint32 track ids; empty arrays without tracks"""
    if q is None:
        return empty_rows()
    b, s, lab, tr = q
    b = b.copy()
    if len(b):
        b[:, 2:] += b[:, :2]
    return b, s, lab, None, tr.astype(np.uint32)


def query_offset(fidx, eta, fidx_t2):
    """``query_pointer - fidx_t2`` (:287-290) as the Python float the streamer computes; numpy rounds it to fp32"""
    return fidx + eta + 1 - fidx_t2


def new_times():
    return {"t_det": [], "t_send_frame": [], "t_recv_res": [], "t_assoc": [], "t_forecast": []}


def wall_sequence(det, frames, n_frame, fps, eta=0.0, forecast_rt_ub=0.003, dynamic_schedule=False, rtf=None,
                  clock=time.perf_counter):
    """One sequence through the streamer's loop (:145-321) on ``clock``: ``det`` a one-stream StreamDetector built with
    ``forecast=True, clear_on_empty=True`` (or an object with its reset / submit / poll / receive / publish / query),
    ``frames[fidx]`` frame fidx as ``det.submit`` takes it.  -> (the sequence's pickle dict, its time_info lists)."""
    times = new_times()
    timestamps, results_parsed, input_fidx = [], [], []
    processing = False
    fidx_t2 = fidx_latest = None
    has_tracks = False
    t_total, t_unit = n_frame / fps, 1 / fps
    wait_time = t_unit - forecast_rt_ub
    det.reset()
    t_start = clock()
    while True:
        t1 = clock()
        t_elapsed = t1 - t_start
        if t_elapsed >= t_total:
            break
        fidx_continuous = t_elapsed * fps
        fidx = int(np.floor(fidx_continuous))
        if _wait_for_next(fidx_continuous, fidx, fidx_latest, dynamic_schedule, rtf):
            continue
        if not processing:
            t_start_frame = clock()
            det.submit(frames[fidx], fidx)
            t_sent = clock()
            fidx_latest = fidx
            processing = True
        if det.poll(wait_time):
            t_res = clock()
            det.receive()
            processing = False
            t_det_end = clock()
            times["t_det"].append(t_det_end - t_start_frame)
            times["t_send_frame"].append(t_sent - t_start_frame)
            times["t_recv_res"].append(t_det_end - t_res)
            t_assoc_start = clock()
            det.publish()                         # the update ran in the tick; publish its tracks to the queries
            t_assoc_end = clock()
            times["t_assoc"].append(t_assoc_end - t_assoc_start)
            fidx_t2 = fidx_latest
            has_tracks = True
        t_forecast_start = clock()
        rows = output_rows(det.query(query_offset(fidx, eta, fidx_t2))[0]) if has_tracks else empty_rows()
        t_forecast_end = clock()
        times["t_forecast"].append(t_forecast_end - t_forecast_start)
        t3 = clock()
        t_elapsed = t3 - t_start
        if t_elapsed >= t_total:
            break
        if fidx_t2 is not None:
            timestamps.append(t_elapsed)
            results_parsed.append(rows)
            input_fidx.append(fidx_t2)
    if processing:
        det.receive()                             # the streamer drops a result still in flight at the sequence's end
    return {"results_parsed": results_parsed, "timestamps": timestamps, "input_fidx": input_fidx}, times


def run_simulated(det, files, schedules, eta, runtime, done):
    """Run every sequence's scheduled detections on the streams of ``det`` (a StreamDetector built with
    ``jpeg_max_bytes``, ``forecast=True``, ``clear_on_empty=True`` and ``queries`` at least the most emissions of one
    detection), packed by ``sap.pack_ticks``.  ``files[q]`` are sequence q's file paths, ``schedules[q]`` its
    ``simulated_schedule``; ``done(q, out, times)`` gets sequence q's pickle dict and time_info lists once its last
    detection has run (and every sequence without a detection first)."""
    def times_of(sch):
        n = len(sch["det_fidx"])
        return {"t_det": [runtime] * n, "t_send_frame": [0.0] * n, "t_recv_res": [0.0] * n, "t_assoc": [0.0] * n,
                "t_forecast": [0.0] * sch["n_forecast"]}

    outs = []
    for q, sch in enumerate(schedules):
        per_det = [[] for _ in sch["det_fidx"]]
        for e, k in enumerate(sch["emit_det"]):
            per_det[k].append(e)
        outs.append({"per_det": per_det, "rows": [None] * len(sch["timestamps"])})
        if not sch["det_fidx"]:
            done(q, {"results_parsed": [], "timestamps": list(sch["timestamps"]), "input_fidx": []}, times_of(sch))
    lengths = [len(sch["det_fidx"]) for sch in schedules]
    ticks = sap.pack_ticks(lengths, det.streams) if any(lengths) else []

    def path(e):
        q, k = e
        return files[q][schedules[q]["det_fidx"][k]]

    for row in ticks:
        for s, e in enumerate(row):
            if e is not None and e[1] == 0:
                det.reset(s)
        fidx, query_dt = [0] * det.streams, [None] * det.streams
        for s, e in enumerate(row):
            if e is None:
                continue
            q, k = e
            sch = schedules[q]
            fidx[s] = sch["det_fidx"][k]
            query_dt[s] = [query_offset(sch["emit_fidx"][x], eta, fidx[s]) for x in outs[q]["per_det"][k]]
        det.step_jpeg([None if e is None else np.fromfile(path(e), np.uint8) for e in row], fidx, query_dt)
        status, got = det.last_status(), det.last_queries()
        for s, e in enumerate(row):
            if e is None:
                continue
            if status[s] != 0:
                raise RuntimeError(f"streamer: {path(e)} did not decode: "
                                   f"{data.JPEG_STATUS.get(int(status[s]), status[s])}")
            q, k = e
            for x, r in zip(outs[q]["per_det"][k], got[s]):
                outs[q]["rows"][x] = output_rows(r)
            if k + 1 == lengths[q]:
                sch = schedules[q]
                done(q, {"results_parsed": outs[q]["rows"], "timestamps": list(sch["timestamps"]),
                         "input_fidx": [sch["det_fidx"][k] for k in sch["emit_det"]]}, times_of(sch))
                outs[q] = None


def _print_stats(times):
    """streamer.py:345-351"""
    def ms(x):
        return 1e3 * x
    for key, name in (("t_det", "Runtime detection (ms)"), ("t_send_frame", "Runtime sending the frame (ms)"),
                      ("t_recv_res", "Runtime receiving the result (ms)"), ("t_assoc", "Runtime association (ms)"),
                      ("t_forecast", "Runtime forecasting (ms)")):
        sap._stats(times[key], name, cvt=ms)


def run(opts, model, clock=time.perf_counter, detector=stream.StreamDetector):
    """The streamer's main() after the model is built: every sequence's pickle and time_info.pkl written to
    ``opts.out_dir`` (``parse_args``' namespace) and its stats printed.  ``model``: YOLOX in eval mode on the GPU with its
    weights loaded.  ``clock`` is the wall clock's timer, ``detector`` the StreamDetector class (tests pass fakes of
    both).  -> the time_info dict."""
    os.makedirs(opts.out_dir, exist_ok=True)
    with open(opts.annot_path) as f:
        dataset = json.load(f)
    seqs, paths = sap.frame_paths(opts, dataset)      # every frame 1200 x 1920: db.imgs[0]'s size, which boxes clip to
    rtf = mean_rtf(opts.runtime, opts.perf_factor, opts.fps) if opts.dynamic_schedule else None
    per_seq = [None] * len(paths)

    def done(q, out, times):
        sap.dump(os.path.join(opts.out_dir, seqs[q] + ".pkl"), out, opts.overwrite)
        per_seq[q] = times

    kw = dict(in_scale=opts.in_scale, forecast=True, match_iou_th=opts.match_iou_th, max_tracks=opts.max_tracks,
              clear_on_empty=True)
    if opts.clock == "wall":
        det = detector(model, frame_hw=sap.DRIVER_HW, **kw)
        device = next(model.parameters()).device
        for q, p in enumerate(paths):
            frames = sap.decode_sequence(p, sap.DRIVER_HW, device)
            done(q, *wall_sequence(det, frames, len(p), opts.fps, opts.eta, opts.forecast_rt_ub, opts.dynamic_schedule,
                                   rtf, clock))
            del frames
    else:
        rt = opts.runtime_ms / 1000.0
        schedules = [simulated_schedule(len(p), opts.fps, rt, opts.forecast_rt_ub, opts.dynamic_schedule, rtf)
                     for p in paths]
        used = [p[i] for p, sch in zip(paths, schedules) for i in sch["det_fidx"]]
        busy = sum(1 for sch in schedules if sch["det_fidx"])
        n_q = max([1] + [int(np.bincount(sch["emit_det"]).max()) for sch in schedules if sch["emit_det"]])
        det = None if not used else detector(model, frame_sizes=[sap.DRIVER_HW] * min(opts.streams, busy),
                                             jpeg_max_bytes=feed.default_max_bytes(used), queries=n_q, **kw)
        run_simulated(det, paths, schedules, opts.eta, rt, done)
    info = {"n_total": sum(len(p) for p in paths)}
    info.update({k: [v for t in per_seq for v in t[k]] for k in new_times()})
    sap.dump(os.path.join(opts.out_dir, "time_info.pkl"), info, opts.overwrite)
    _print_stats(info)
    return info


def main(argv=None):
    opts = parse_args(argv)
    return run(opts, sap.build_model(opts.config, opts.weights))


if __name__ == "__main__":
    main()
