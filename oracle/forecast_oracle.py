"""Restatement of the sAP toolkit's offline forecast (sAP/forecast/pps_forecast_kf.py:134-287 with
--forecast-before-assoc and --assoc iou), fed from parsed results -- TEST INFRASTRUCTURE.

``dtype=torch.float32`` runs the reference's own arithmetic: torch CPU fp32 matrices for the Kalman filter, numpy fp32
for the boxes and the extrapolation, pycocotools' fp64 bbIou.  ``dtype=torch.float64`` runs the same loop with the
Kalman state, the extrapolation and the clean-up in fp64 (the boxes still enter as the fp32 ltwh rows), the yardstick the
fp32 results are measured against.

Score ties sort as a stable ascending argsort reversed (the higher index first); the reference's default argsort is not
stable above 16 elements, so fixtures keep their scores distinct.  ``stale=True`` reproduces the reference's rows for a
frame whose latest detection exists while its sequence has no track yet: the previous frame's rows again (its
``if len(kf_x)`` branch leaves ``bboxes_t3`` as it was); the default emits nothing there, as the device does."""
import numpy as np
import torch


def query_schedule(n_frames, timestamps, input_fidx, eta, fps):
    """:155-170 -> per frame (index of the latest detection or -1, new detection?, dt of its update or None, dt of the
    query)"""
    out, det_latest_p1, det_t2 = [], 0, None
    for ii in range(n_frames):
        t = (ii - eta) / fps
        while det_latest_p1 < len(timestamps) and timestamps[det_latest_p1] <= t:
            det_latest_p1 += 1
        if det_latest_p1 == 0:
            out.append((-1, False, None, None))
            continue
        d = det_latest_p1 - 1
        new = d != det_t2
        dt_up = int(input_fidx[d] - input_fidx[det_t2]) if new and det_t2 is not None else None
        if new:
            det_t2 = d
        out.append((d, new, dt_up, ii - input_fidx[d]))
    return out


def bb_iou(b1, b2):
    """pycocotools' bbIou (maskApi.c) with iscrowd = 0: [m, n] IoUs of ltwh boxes b1 [m, 4] (dt) and b2 [n, 4] (gt) in
    fp64"""
    D = np.asarray(b1, np.float64)[:, None, :]
    G = np.asarray(b2, np.float64)[None, :, :]
    da, ga = D[..., 2] * D[..., 3], G[..., 2] * G[..., 3]
    w = np.fmin(D[..., 2] + D[..., 0], G[..., 2] + G[..., 0]) - np.fmax(D[..., 0], G[..., 0])
    h = np.fmin(D[..., 3] + D[..., 1], G[..., 3] + G[..., 1]) - np.fmax(D[..., 1], G[..., 1])
    i = w * h
    with np.errstate(divide="ignore", invalid="ignore"):
        o = i / (da + ga - i)
    return np.where((w <= 0) | (h <= 0), 0.0, o)


def iou_assoc(ious, labels1, labels2, th):
    """track/__init__.py:90-133 with no_unmatched1 on the IoU matrix -> (order1, order2, n_matched, margins): margins[j]
    = (|best eligible IoU - th|, best - runner-up when the runner-up is >= th, else inf) of detection j's decision"""
    m, n = ious.shape
    match_fwd = [None] * m
    matched1, matched2, unmatched2, margins = [], [], [], []
    for j in range(n):
        best_iou, match_i, elig = th, None, []
        for i in range(m):
            if match_fwd[i] is not None or labels1[i] != labels2[j]:
                continue
            elig.append(ious[i, j])
            if ious[i, j] < best_iou:
                continue
            best_iou, match_i = ious[i, j], i
        e = sorted(elig, reverse=True)
        margins.append((abs(e[0] - th) if e else np.inf,
                        e[0] - e[1] if len(e) > 1 and e[1] >= th else np.inf))
        if match_i is None:
            unmatched2.append(j)
        else:
            matched1.append(match_i)
            matched2.append(j)
            match_fwd[match_i] = j
    return matched1, matched2 + unmatched2, len(matched2), margins


def kf_predict(x, P, dt):
    """x [N, 8, 1], P [N, 8, 8] -> F x, F P F' + Q (:64-79)"""
    F = torch.eye(8, dtype=x.dtype)
    F[[0, 1, 2, 3], [4, 5, 6, 7]] = dt
    Q = torch.eye(8, dtype=x.dtype)
    Q[range(8), range(8)] = dt * dt
    return F @ x, F @ P @ F.t() + Q


def kf_update(z, x, P):
    """batch_kf_update (:81-97) with R = 10 I; z [N, 4, 1]"""
    R = 10 * torch.eye(4, dtype=x.dtype)
    x, P = x.clone(), P.clone()
    y = z - x[:, :4]
    S = P[:, :4, :4] + R
    K = P[:, :, :4] @ S.inverse()
    x += K @ y
    P -= K @ P[:, :4]
    return x, P


def extrap(xm, n_matched, dt, w_img, h_img, min_size=75):
    """:265-270 and extrap_clean_up(..., lt=True) (forecast/__init__.py:33-56) on the means xm [N, 8] (numpy) -> (ltwh
    rows kept, keep mask)"""
    b = xm[:n_matched, :4] + dt * xm[:n_matched, 4:]
    if n_matched < len(xm):
        b = np.concatenate((b, xm[n_matched:, :4]))
    wh_nz = b[:, 2:] > 0
    keep = np.logical_and(wh_nz[:, 0], wh_nz[:, 1])
    b[:, 2:] = b[:, :2] + b[:, 2:]
    b[:, [0, 2]] = b[:, [0, 2]].clip(0, w_img)
    b[:, [1, 3]] = b[:, [1, 3]].clip(0, h_img)
    b[:, 2:] = b[:, 2:] - b[:, :2]
    keep = np.logical_and(keep, b[:, 2].astype(np.int64) * b[:, 3].astype(np.int64) >= min_size)
    return b[keep], keep


class Tracks:
    """One sequence's forecast state: Kalman mean / covariance, labels, scores, track ids, n_matched, the id counter."""

    def __init__(self, dtype=torch.float32):
        self.dtype = dtype
        self.x = torch.empty((0, 8, 1), dtype=dtype)
        self.P = torch.empty((0, 8, 8), dtype=dtype)
        self.labels = self.scores = self.tracks = None
        self.n_matched, self.tkidx = 0, 0

    def _new(self, b):
        x = torch.cat((torch.from_numpy(b).to(self.dtype), torch.zeros(b.shape, dtype=self.dtype)), dim=1).unsqueeze_(2)
        return x, 100 * torch.eye(8, dtype=self.dtype).unsqueeze(0).expand(len(b), -1, -1)

    def update(self, bboxes, scores, labels, dt, th=0.3, log=None):
        """one new detection (:175-256): ``bboxes`` ltrb fp32 [n, 4], ``scores``, ``labels`` [n]; ``dt`` the frames since
        the previous detection.  ``log`` (a list) gets (n, n_tracks before, n_matched, order1, order2, margins)."""
        if len(self.x):
            self.x, self.P = kf_predict(self.x, self.P, dt)
        n = len(bboxes)
        if not n:
            if log is not None:
                log.append((0, len(self.x), None, [], [], []))
            return
        order = np.argsort(scores, kind="stable")[::-1]
        b = np.array(bboxes[order], np.float32)
        s, lab = scores[order], labels[order]
        b[:, 2:] -= b[:, :2]                                      # ltrb2ltwh_ in fp32
        m = len(self.x)
        if m:
            bf = self.x[:, :4, 0].numpy()
            order1, order2, nm, margins = iou_assoc(bb_iou(bf, b), self.labels, lab, th)
            tracks = np.concatenate((self.tracks[order1][:nm],
                                     np.arange(self.tkidx, self.tkidx + n - nm, dtype=np.uint32)))
            self.tkidx += n - nm
            self.n_matched = nm
            if log is not None:
                log.append((n, m, nm, order1, order2, margins))
            if nm:
                x, P = self.x[order1], self.P[order1]
                z = torch.from_numpy(b[order2[:nm]]).to(self.dtype).unsqueeze_(2)
                x, P = kf_update(z, x, P)
                xn, Pn = self._new(b[order2[nm:]])
                self.x, self.P = torch.cat((x, xn)), torch.cat((P, Pn))
                self.labels, self.scores, self.tracks = lab[order2], s[order2], tracks
                return
        elif log is not None:
            log.append((n, 0, None, [], list(range(n)), []))
        self.x, self.P = self._new(b)
        self.labels, self.scores = lab, s
        self.tracks = np.arange(self.tkidx, self.tkidx + n, dtype=np.uint32)
        self.tkidx += n

    def query(self, dt, w_img, h_img):
        """(ltwh [k, 4], scores, labels, tracks) extrapolated dt frames ahead, or None without tracks"""
        if not len(self.x):
            return None
        xm = self.x[:, :, 0].numpy()
        b, keep = extrap(xm.copy(), self.n_matched, dt, w_img, h_img)
        return b, self.scores[keep], self.labels[keep], self.tracks[keep]


def run(sequences, eta=0.0, fps=30.0, th=0.3, dtype=torch.float32, stale=False, log=None):
    """The offline loop over ``sequences``: each a dict with ``images`` (the annotation dicts in COCO.imgs order) and the
    driver pickle's ``results_parsed``, ``timestamps``, ``input_fidx``.  -> one entry per annotated frame: (image_id,
    ltwh, scores, labels, tracks), empty arrays where nothing is emitted."""
    out = []
    empty = (np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros(0, np.int64), np.zeros(0, np.uint32))
    last = empty
    for seq in sequences:
        st = Tracks(dtype)
        sched = query_schedule(len(seq["images"]), seq["timestamps"], seq["input_fidx"], eta, fps)
        for img, (d, new, dt_up, dt_q) in zip(seq["images"], sched):
            rows = empty
            if d >= 0:
                if new:
                    bb, sc, lb = seq["results_parsed"][d][:3]
                    st.update(np.asarray(bb), np.asarray(sc), np.asarray(lb), dt_up if dt_up is not None else 0, th, log)
                q = st.query(dt_q, img["width"], img["height"])
                rows = q if q is not None else (last if stale else empty)
            last = rows
            out.append((img["id"],) + tuple(rows))
    return out
