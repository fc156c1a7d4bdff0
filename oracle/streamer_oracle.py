"""Restatement of the sAP toolkit's streamer (sAP/forecast/streamer.py:139-343) on a virtual clock -- TEST
INFRASTRUCTURE.

The clock: host work takes no time; a detection submitted at t completes at t + runtime; ``poll(w)`` returns at
min(t + w, completion) (at once when the detection completed during an idle wait); an idle iteration moves the clock to
the first time whose floor(t * fps) has advanced; each sequence starts at 0.  ``detect(fidx)`` gives the detection of
input frame fidx as (ltrb fp32 [n, 4], scores [n], labels [n]); the Kalman filter, the association and the
extrapolation are forecast_oracle's, with the streamer's empty-detection rule (``StreamerTracks``)."""
import numpy as np

from oracle.forecast_oracle import Tracks


class StreamerTracks(Tracks):
    """forecast_oracle.Tracks with the streamer's rule for an empty detection (sAP/forecast/streamer.py:247-280):
    iou_assoc with no detection matches nothing, and the "start from scratch" branch then leaves no track; n_matched is
    0 and the id counter stays.  pps_forecast_kf.py's ``if n:`` guard (Tracks.update) keeps the predicted tracks
    instead.  Any other detection updates the tracks as Tracks.update does."""

    def update(self, bboxes, scores, labels, dt, th=0.3, log=None):
        if len(bboxes):
            return super().update(bboxes, scores, labels, dt, th, log)
        m = len(self.x)
        if log is not None:
            log.append((0, m, 0 if m else None, [], [], []))
        if m:
            self.n_matched = 0
        self.x, self.P = self.x[:0], self.P[:0]
        self.labels, self.scores = np.asarray(labels)[:0], np.asarray(scores)[:0]
        self.tracks = np.zeros(0, np.uint32)


def next_frame_time(t, fps):
    """the first time after t whose floor(t * fps) is the next frame: (f + 1) / fps, moved up while its product with fps
    rounds below f + 1"""
    f = int(np.floor(t * fps)) + 1
    u = f / fps
    while np.floor(u * fps) < f:
        u = float(np.nextafter(u, np.inf))
    return u


def empty_rows():
    """the streamer's output without tracks (:303-306)"""
    return (np.empty((0, 4), dtype=np.float32), np.empty((0,), dtype=np.float32), np.empty((0,), dtype=np.int32), None,
            np.empty((0,), dtype=np.int32))


def sequence(detect, n_frame, w_img, h_img, fps=30.0, eta=0.0, runtime=0.075, forecast_rt_ub=0.003,
             dynamic_schedule=False, mean_rtf=None, th=0.3, log=None):
    """One sequence of the loop (:145-329) -> (the pickle dict, time_info counts {t_det, t_forecast})"""
    t_total, t_unit = n_frame / fps, 1 / fps
    t = 0.0
    timestamps, results_parsed, input_fidx = [], [], []
    processing, done_at = False, None
    fidx_t2 = fidx_latest = None
    st = StreamerTracks()
    n_det = n_forecast = 0
    while True:
        t_elapsed = t                                          # :177-180
        if t_elapsed >= t_total:
            break
        fidx_continous = t_elapsed * fps
        fidx = int(np.floor(fidx_continous))
        if fidx == fidx_latest:                                # :185-200
            wait_for_next = True
        else:
            wait_for_next = False
            if dynamic_schedule and mean_rtf >= 1:
                if mean_rtf < np.floor(fidx_continous - fidx + mean_rtf):
                    wait_for_next = True
        if wait_for_next:
            t = next_frame_time(t, fps)
            continue
        if not processing:                                     # :202-206
            done_at = t + runtime
            fidx_latest = fidx
            processing = True
        wait_time = t_unit - forecast_rt_ub                    # :209-210
        if done_at <= t + wait_time:
            t = max(t, done_at)
            processing = False
            n_det += 1
            b, s, lab = detect(fidx_latest)
            st.update(np.asarray(b, np.float32), np.asarray(s), np.asarray(lab),
                      0 if fidx_t2 is None else fidx_latest - fidx_t2, th, log)
            fidx_t2 = fidx_latest
        else:
            t = t + wait_time
        n_forecast += 1
        query_pointer = fidx + eta + 1                         # :287-306
        rows = empty_rows()
        if fidx_t2 is not None:
            q = st.query(query_pointer - fidx_t2, w_img, h_img)
            if q is not None:
                b, s, lab, tr = q
                b = b.copy()
                if len(b):
                    b[:, 2:] += b[:, :2]                       # ltwh2ltrb_
                rows = (b, s, lab, None, tr)
        if t >= t_total:                                       # :311-314
            break
        if fidx_t2 is not None:
            timestamps.append(t)
            results_parsed.append(rows)
            input_fidx.append(fidx_t2)
    return ({"results_parsed": results_parsed, "timestamps": timestamps, "input_fidx": input_fidx},
            {"t_det": n_det, "t_forecast": n_forecast})
