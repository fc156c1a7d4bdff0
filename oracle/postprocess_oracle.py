"""CPU restatement of the detection post-processing (TEST INFRASTRUCTURE ONLY: imported by tests/ and never by the
product).  It follows

  * [yolox 0.3.0] yolox/utils/boxes.py: postprocess (not vendored in /root/reference; call sites
    /root/reference/exps/evaluators/onex_stream_evaluator.py:148, sAP/streamyolo/streamyolo_det.py:62-83; restated from
    the published source): cxcywh -> xyxy, class_conf / class_pred = max over classes, conf mask on obj * class_conf,
    detections [x1, y1, x2, y2, obj, class_conf, class_pred], batched_nms (class-aware) or nms (class-agnostic), gather;
  * torchvision 0.26's batched_nms as it runs on the reference's CUDA tensors (nms_reference): up to 100 000 box
    coordinates (25 000 candidates; the device kernel takes at most 16 384) it is _batched_nms_coordinate_trick: every
    box is shifted by class * (boxes.max() + 1) in fp32 and one class-agnostic nms runs on the shifted boxes.  The CUDA
    nms (torchvision/csrc/ops/cuda/nms_kernel.cu, devIoU; sm_90 SASS of nms_kernel_impl<float>) sorts the scores
    descending with a stable sort and suppresses a later box b by a kept earlier box a iff
        inter / (fma(w_b, h_b, w_a * h_a) - inter) > float(thr),
    the later box's area fused into the sum, w = x2 - x1 and h = y2 - y1 rounded, IEEE division, fmaxf / fminf (NaN-
    ignoring) for the intersection.  fma=False restates the CPU nms (torchvision/csrc/ops/cpu/nms_kernel.cpp): areas
    rounded, std::max / std::min, the fp32 ratio compared with the double threshold.
  * nms_greedy: per-class greedy NMS with rounded areas = batched_nms's vanilla path on the CPU (per-class
    torchvision.ops.nms), which tests/golden/nms_*.npz pin.

Pinned by tests/test_postprocess.py and tests/test_nms_reference.py against torchvision itself (installed in this
image) and against the committed fixtures."""
from fractions import Fraction

import numpy as np
import torch


def nms_greedy(boxes: np.ndarray, scores: np.ndarray, classes: np.ndarray, thr: float, class_agnostic=False) -> np.ndarray:
    """Indices kept, in decreasing score order (ties: lower index first).  fp32 arithmetic, per class."""
    order = np.lexsort((np.arange(len(scores)), -scores.astype(np.float64)))
    b = boxes.astype(np.float32)
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    areas = ((x2 - x1).astype(np.float32) * (y2 - y1).astype(np.float32)).astype(np.float32)
    removed = np.zeros(len(scores), bool)
    keep = []
    thr = np.float32(thr)
    for oi, i in enumerate(order):
        if removed[i]:
            continue
        keep.append(i)
        rest = order[oi + 1:]
        rest = rest[~removed[rest]]
        if not class_agnostic:
            rest = rest[classes[rest] == classes[i]]
        if len(rest) == 0:
            continue
        xx1, yy1 = np.maximum(x1[i], x1[rest]), np.maximum(y1[i], y1[rest])
        xx2, yy2 = np.minimum(x2[i], x2[rest]), np.minimum(y2[i], y2[rest])
        w = np.maximum(np.float32(0), (xx2 - xx1).astype(np.float32))
        h = np.maximum(np.float32(0), (yy2 - yy1).astype(np.float32))
        inter = (w * h).astype(np.float32)
        ovr = inter / ((areas[i] + areas[rest]).astype(np.float32) - inter).astype(np.float32)
        removed[rest[ovr > thr]] = True
    return np.array(keep, np.int64)


def round_f32(x: Fraction) -> np.float32:
    """x rounded to the nearest fp32, ties to even (one rounding)."""
    r = np.float32(float(x))                        # within one fp32 ulp of x
    cands = [v for v in (np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))) if np.isfinite(v)]
    return min(cands, key=lambda v: (abs(Fraction(float(v)) - x), int(np.float32(v).view(np.uint32)) & 1))


def fma_f32(a, b, c) -> np.ndarray:
    """Elementwise a * b + c for fp32 operands with one rounding to fp32, as __fmaf_rn.  The product is exact in float64,
    so the float64 sum has rounded once; rounding that to fp32 is correct unless the float64 sum lies exactly halfway
    between two fp32 values (the first rounding may have moved it there): those elements are recomputed exactly."""
    a, b, c = (np.ascontiguousarray(v, np.float32) for v in np.broadcast_arrays(a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        s = a.astype(np.float64) * b + c
        r = s.astype(np.float32)
        fin = np.isfinite(s) & np.isfinite(r)
        nb = np.nextafter(r, np.where(s > r, np.float32(np.inf), np.float32(-np.inf)))
        mid = fin & (s != r) & (np.abs(nb.astype(np.float64) - s) == np.abs(s - r.astype(np.float64)))
    for k in np.flatnonzero(mid):
        r.flat[k] = round_f32(Fraction(float(a.flat[k])) * Fraction(float(b.flat[k])) + Fraction(float(c.flat[k])))
    return r


def nms_reference(boxes: np.ndarray, scores: np.ndarray, classes: np.ndarray, thr: float, class_agnostic=False, fma=True,
                  offsets=True, propagate_nan=True, class_test=False) -> np.ndarray:
    """Indices kept by torchvision's batched_nms (class_agnostic: nms) on CUDA tensors, in decreasing score order (ties:
    lower index first).  fma=False: the same on CPU tensors (_batched_nms_coordinate_trick / nms).

    offsets=False, propagate_nan=False (boxes.max() ignoring NaN) and class_test=True (a box only suppresses boxes of its
    own class) each remove one rule of that path; tests use them to show which rule a case depends on."""
    b = np.asarray(boxes, np.float32).reshape(-1, 4)
    scores = np.asarray(scores, np.float32)
    classes = np.asarray(classes)
    n = len(b)
    if n == 0:
        return np.zeros(0, np.int64)
    if not class_agnostic and offsets:
        mx = b.max() if propagate_nan else np.fmax.reduce(b.ravel())      # torch.max propagates NaN
        off = classes.astype(np.float32) * (np.float32(mx) + np.float32(1))
        b = b + off[:, None]
    order = np.lexsort((np.arange(n), -scores.astype(np.float64)))          # stable, descending
    x1, y1, x2, y2 = (np.ascontiguousarray(b[:, k]) for k in range(4))
    bw, bh = x2 - x1, y2 - y1
    area = bw * bh
    removed = np.zeros(n, bool)
    keep = []
    zero = np.float32(0)
    for oi, i in enumerate(order):
        if removed[i]:
            continue
        keep.append(i)
        rest = order[oi + 1:]
        rest = rest[~removed[rest]]
        if class_test and not class_agnostic:
            rest = rest[classes[rest] == classes[i]]
        if len(rest) == 0:
            continue
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            if fma:     # CUDA max / min on floats: fmaxf / fminf
                w = np.fmax(np.fmin(x2[i], x2[rest]) - np.fmax(x1[i], x1[rest]), zero)
                h = np.fmax(np.fmin(y2[i], y2[rest]) - np.fmax(y1[i], y1[rest]), zero)
                inter = w * h
                ovr = inter / (fma_f32(bw[rest], bh[rest], area[i]) - inter)
                hit = ovr > np.float32(thr)
            else:       # std::max(a, b) = a < b ? b : a, std::min(a, b) = b < a ? b : a
                xx1 = np.where(x1[i] < x1[rest], x1[rest], x1[i])
                yy1 = np.where(y1[i] < y1[rest], y1[rest], y1[i])
                xx2 = np.where(x2[rest] < x2[i], x2[rest], x2[i])
                yy2 = np.where(y2[rest] < y2[i], y2[rest], y2[i])
                dw, dh = xx2 - xx1, yy2 - yy1
                w = np.where(zero < dw, dw, zero)
                h = np.where(zero < dh, dh, zero)
                inter = w * h
                ovr = inter / ((area[i] + area[rest]) - inter)
                hit = ovr.astype(np.float64) > float(thr)
        removed[rest[hit]] = True
    return np.array(keep, np.int64)


def postprocess_oracle(prediction: torch.Tensor, num_classes: int, conf_thre=0.7, nms_thre=0.45, class_agnostic=False,
                       nms=nms_reference):
    """yolox.utils.postprocess; nms(boxes, scores, classes, thr, class_agnostic) -> kept indices (default: the CUDA path)"""
    pred = prediction.detach().float().cpu()
    out = []
    for p in pred:
        half_w, half_h = p[:, 2] / 2, p[:, 3] / 2
        xyxy = torch.stack([p[:, 0] - half_w, p[:, 1] - half_h, p[:, 0] + half_w, p[:, 1] + half_h], 1)
        class_conf, class_pred = torch.max(p[:, 5:5 + num_classes], 1)
        score = p[:, 4] * class_conf
        mask = score >= conf_thre
        idx = mask.nonzero().flatten()
        if idx.numel() == 0:
            out.append(None)
            continue
        keep = nms(xyxy[idx].numpy(), score[idx].numpy(), class_pred[idx].numpy(), nms_thre, class_agnostic)
        sel = idx[torch.from_numpy(keep)]
        out.append(torch.cat([xyxy[sel], p[sel, 4:5], class_conf[sel, None], class_pred[sel, None].float()], 1))
    return out
