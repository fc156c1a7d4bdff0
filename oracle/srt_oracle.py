"""The sAP toolkit's sampled-runtime protocols, restated for tests/test_sap_runtime.py.

``srt_det``      sAP/det/srt_det.py:72-181, the simulated-time loop over every sequence, each frame's runtime drawn from
                 an empirical distribution
``srt_det_inf``  sAP/det/srt_det_inf.py:68-149, the same protocol with infinite GPUs

Each returns, per sequence, which frames the detector ran, when each result is out and what each run took, nothing else:
the detector's outputs do not take part in either schedule.
"""
import math

import numpy as np


def srt_det(lengths, fps, det_stride, dynamic_schedule, samples, perf_factor, seed):
    """srt_det.py:72-181, the whole run: ``lengths[q]`` frames in sequence q, each frame's runtime drawn from the
    empirical ``samples`` (util/runtime_dist.py) scaled by ``perf_factor``, numpy's global generator seeded once (:72)
    and carried across the sequences.  The draws come from a RandomState of their own, the same stream.

    -> one (input_fidx, timestamps, runtime) per sequence"""
    rng = np.random.RandomState(seed)                                  # :72 np.random.seed
    pool = np.array(samples)                                           # runtime_dist.py:10-13
    if perf_factor != 1:
        pool = pool / perf_factor
    out = []
    for n_frame in lengths:
        input_fidx, timestamps, runtime = [], [], []
        previous = None                      # :96 last_fidx
        length = n_frame / fps               # :102 t_total
        clock = 0                            # :103 t_elapsed
        ratio = pool.mean() * fps            # :105 mean_rtf
        count = 0                            # :107 stride_cnt
        while True:
            if clock >= length:              # :110-111
                break
            position = clock * fps           # :114-115
            frame = int(math.floor(position))
            if frame == previous:            # :116-121 idle until the next frame arrives; no next frame: done
                frame += 1
                if frame == n_frame:
                    break
                clock = frame / fps
            previous = frame
            if dynamic_schedule:             # :125-131
                if ratio > 1 and ratio < np.floor(position - frame + ratio):
                    continue
            elif count % det_stride == 0:    # :132-137
                count = 1
            else:
                count += 1
                continue
            took = rng.choice(pool)          # :155 runtime_dist.draw(), taken even when it ends the sequence
            clock += took                    # :156-158
            if clock >= length:
                break
            timestamps.append(clock)         # :160-165
            input_fidx.append(frame)
            runtime.append(took)
        out.append((input_fidx, timestamps, runtime))
    return out


def srt_det_inf(lengths, fps, samples, perf_factor, seed):
    """srt_det_inf.py:68-149, the whole run with infinite GPUs: every frame ii detected, its result out at ii / fps +
    a draw (the generator as in ``srt_det``), each sequence then ordered by np.argsort of those times (:127-134).

    -> one (input_fidx, timestamps, runtime) per sequence"""
    rng = np.random.RandomState(seed)
    pool = np.array(samples)
    if perf_factor != 1:
        pool = pool / perf_factor
    out = []
    for n_frame in lengths:
        input_fidx, timestamps, runtime = [], [], []
        for ii in range(n_frame):            # :98-125
            took = rng.choice(pool)
            timestamps.append(ii / fps + took)
            input_fidx.append(ii)
            runtime.append(took)
        order = np.argsort(timestamps)       # :128-134
        out.append(([input_fidx[i] for i in order], [timestamps[i] for i in order], [runtime[i] for i in order]))
    return out
