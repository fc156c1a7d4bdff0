"""The frame schedules of the reference's two sAP drivers, restated for tests/test_sap_driver.py.

``wall_schedule``       sAP/streamyolo/streamyolo_det.py:152-195, the real-time loop, on a modelled clock
``simulated_schedule``  sAP/det/srt_det.py:102-165, the simulated-time loop, with a runtime that is the same every frame

Both return which frames the detector ran and when it finished them, nothing else: the detector's outputs do not take part
in either schedule.
"""
import math


def wall_schedule(n_frame, fps, det_stride, dynamic_schedule, durations, poll):
    """streamyolo_det.py:152-195 with time modelled: every read of the clock (perf_counter, :148, :153, :186) returns the
    current time and then moves it on by ``poll`` seconds; the detector's work on a frame (:176-184) moves it on by the
    next entry of ``durations`` (cycled).

    -> (input_fidx, timestamps, ticks): the frames kept and the elapsed time at which each was kept (:191-194), and how
    many frames the detector ran, which is one more than kept when the last one ran past the sequence's end (:187-189)."""
    now = [0.0]

    def read():
        t = now[0]
        now[0] += poll
        return t

    input_fidx, timestamps = [], []
    ticks = 0
    previous = None                          # :143 last_fidx
    count = 0                                # :145 stride_cnt
    length = n_frame / fps                   # :147 t_total
    origin = read()                          # :148 t_start
    while True:
        begin = read()                       # :153
        elapsed = begin - origin
        if elapsed >= length:                # :155-156 the sequence is over
            break
        position = elapsed * fps             # :159-160 the newest frame out
        frame = int(math.floor(position))
        if frame == previous:                # :161-162 already seen: ask the clock again
            continue
        previous = frame
        if dynamic_schedule:                 # :165-168 skip a frame already more than half gone
            if position - frame > 0.5:
                continue
        elif count % det_stride == 0:        # :169-174 run every det_stride-th new frame
            count = 1
        else:
            count += 1
            continue
        now[0] += durations[ticks % len(durations)]        # :176-184 the detector
        ticks += 1
        end = read()                         # :186
        elapsed = end - origin
        if elapsed >= length:                # :188-189 finished after the sequence's end: dropped
            break
        timestamps.append(elapsed)           # :191-194
        input_fidx.append(frame)
    return input_fidx, timestamps, ticks


def simulated_schedule(n_frame, fps, det_stride, dynamic_schedule, runtime):
    """srt_det.py:102-165 with ``runtime_dist.draw()`` and ``runtime_dist.mean()`` both ``runtime`` seconds.

    -> (input_fidx, timestamps): the frames processed and the simulated time at which each result is out."""
    input_fidx, timestamps = [], []
    previous = None                          # :96 last_fidx
    length = n_frame / fps                   # :102 t_total
    clock = 0                                # :103 t_elapsed
    ratio = runtime * fps                    # :105 mean_rtf: frames that go by during one run
    count = 0                                # :107 stride_cnt
    while True:
        if clock >= length:                  # :110-111
            break
        position = clock * fps               # :114-115
        frame = int(math.floor(position))
        if frame == previous:                # :116-121 idle until the next frame arrives; no next frame: done
            frame += 1
            if frame == n_frame:
                break
            clock = frame / fps              # position is not recomputed (:114 is not revisited)
        previous = frame
        if dynamic_schedule:                 # :125-131 wait for the next frame when it finishes no later than this one
            if ratio > 1 and ratio < math.floor(position - frame + ratio):
                continue
        elif count % det_stride == 0:        # :132-137
            count = 1
        else:
            count += 1
            continue
        clock += runtime                     # :155-158
        if clock >= length:
            break
        timestamps.append(clock)             # :160-164
        input_fidx.append(frame)
    return input_fidx, timestamps
