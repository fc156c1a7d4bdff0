"""Numpy restatement of the sAP toolkit's detection drawing -- TEST INFRASTRUCTURE.

``draw`` is the box branch of vis_obj_fancy (sAP/vis/vis_det_th.py:99-120, masks None, show_label / show_score False):
  1. every box's filled rectangle [min(x1, x2), max(x1, x2)] x [min(y1, y2), max(y1, y2)] (inclusive, clipped) in its
     label's colour, later boxes over earlier ones (cv2.rectangle thickness -1), blended as cv2.addWeighted(orig, 0.8,
     filled, 0.2, 0): rint(0.8f * v + 0.2f * p) in fp32 with each product rounded (``blend``);
  2. every box's thickness-2 outline in its colour, later over earlier (cv2.rectangle thickness 2): the pixels within
     Chebyshev distance 1 of the rectangle's border except the four diagonally outside its corners.
tests/test_vis.py pins both against cv2 itself.  ``script_rows`` and ``tick_rows`` are the host paths from a result
row list / a streaming tick's NMS rows to the rounded boxes and labels the drawing takes."""
import numpy as np


def blend(orig, paint):
    """cv2.addWeighted(orig, 0.8, paint, 0.2, 0) on uint8 arrays"""
    v = orig.astype(np.float32) * np.float32(0.8) + paint.astype(np.float32) * np.float32(0.2)
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)


def _norm(b):
    x1, y1, x2, y2 = (int(v) for v in b)
    return min(x1, x2), min(y1, y2), max(x1, x2), max(y1, y2)


def _owner_maps(h, w, boxes):
    """(fill, line): int [h, w] maps of the last box whose filled rectangle / outline covers each pixel, -1 for none"""
    fill = np.full((h, w), -1, np.int64)
    line = np.full((h, w), -1, np.int64)
    for i, b in enumerate(boxes):
        x1, y1, x2, y2 = _norm(b)
        fx0, fx1, fy0, fy1 = max(x1, 0), min(x2, w - 1), max(y1, 0), min(y2, h - 1)
        if fx0 <= fx1 and fy0 <= fy1:
            fill[fy0:fy1 + 1, fx0:fx1 + 1] = i
        ox0, ox1, oy0, oy1 = max(x1 - 1, 0), min(x2 + 1, w - 1), max(y1 - 1, 0), min(y2 + 1, h - 1)
        if ox0 > ox1 or oy0 > oy1:
            continue
        xx = np.arange(ox0, ox1 + 1)[None, :]
        yy = np.arange(oy0, oy1 + 1)[:, None]
        inner = (xx >= x1 + 2) & (xx <= x2 - 2) & (yy >= y1 + 2) & (yy <= y2 - 2)
        corner = ((xx == x1 - 1) | (xx == x2 + 1)) & ((yy == y1 - 1) | (yy == y2 + 1))
        sub = line[oy0:oy1 + 1, ox0:ox1 + 1]
        sub[~inner & ~corner] = i
    return fill, line


def draw(img, boxes, labels, palette):
    """vis_obj_fancy's drawing of int boxes [k, 4] with labels [k] on a uint8 [h, w, 3] image (a new array); ``palette``
    [P, 3] in the image's channel order"""
    img = np.asarray(img, np.uint8)
    boxes, labels = np.asarray(boxes).reshape(-1, 4), np.asarray(labels).reshape(-1)
    palette = np.asarray(palette, np.uint8).reshape(-1, 3)
    if len(boxes) == 0:
        return img.copy()
    fill, line = _owner_maps(img.shape[0], img.shape[1], boxes)
    col = palette[labels]
    out = img.copy()
    m = fill >= 0
    out[m] = blend(img[m], col[fill[m]])
    m = line >= 0
    out[m] = col[line[m]]
    return out


def script_rows(dets, score_th, gt=False):
    """vis_det_th.py:228-242 and vis_obj_fancy :75-97 on the rows of one frame (dicts with 'bbox' ltwh, 'category_id'
    and 'score' or 'iscrowd'), in the script's own numpy expressions on the rows' own dtypes -> (int32 boxes [k, 4],
    labels [k]); k = 0 where the script writes the frame unchanged"""
    bboxes = np.array([d["bbox"] for d in dets])
    if len(bboxes):
        bboxes[:, 2:] += bboxes[:, :2]
    labels = np.array([d["category_id"] for d in dets])
    scores = None if gt else np.array([d["score"] for d in dets])
    bboxes, labels = np.asarray(bboxes), np.asarray(labels)
    empty = len(bboxes) == 0
    if not empty and scores is not None and score_th > 0:
        sel = scores >= score_th
        bboxes, labels = bboxes[sel], labels[sel]
        empty = len(bboxes) == 0
    if empty:
        return np.zeros((0, 4), np.int32), np.zeros((0,), np.int64)
    return bboxes.round().astype(np.int32), labels


def tick_rows(det, count, score_th):
    """a streaming tick's NMS rows of one stream (fp32 [A, 7], first ``count`` valid) -> (int32 boxes, labels) as the
    host computes them: stream.sized_output's (bboxes, scores, labels), the ltwh rows streaming_eval.py stores, then
    vis_det_th.py's ltrb and vis_obj_fancy's threshold and rounding"""
    det = np.asarray(det, np.float32)[:count]
    bboxes, scores, labels = det[:, :4].copy(), det[:, 4] * det[:, 5], det[:, 6].astype(np.int32)
    ltwh = bboxes.copy()
    ltwh[:, 2:] -= ltwh[:, :2]
    rows = [{"bbox": ltwh[i], "score": scores[i], "category_id": labels[i]} for i in range(len(det))]
    if not rows:
        return np.zeros((0, 4), np.int32), np.zeros((0,), np.int32)
    return script_rows(rows, score_th)
