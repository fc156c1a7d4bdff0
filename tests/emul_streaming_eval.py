"""CPU emulation of the kernels behind ``python -m streamyolo_b200.streaming_eval``: ops.draw_outlines
(sy_draw_outlines) restated in numpy, ops.resize_sized (sy_resize_sized) as cv2.resize, and the command's device pass
with them (PIL's decode and encode, which the device's decode and quality-75 encode equal).  Kept apart from
emul_ops.NAMES, whose list the emulation conformance test builds its cases from."""
import io

import numpy as np
import torch


def outline_mask(h, w, boxes):
    """bool [h, w]: the pixels cv2.rectangle(img, (x1, y1), (x2, y2), color, thickness=1) sets for each int box, the
    corners in any order, clipped to the image"""
    m = np.zeros((h, w), bool)
    for x1, y1, x2, y2 in np.asarray(boxes, np.int64).reshape(-1, 4):
        xa, xb, ya, yb = min(x1, x2), max(x1, x2), min(y1, y2), max(y1, y2)
        cxa, cxb, cya, cyb = max(xa, 0), min(xb, w - 1), max(ya, 0), min(yb, h - 1)
        for y in {y1, y2}:
            if 0 <= y < h and cxa <= cxb:
                m[y, cxa:cxb + 1] = True
        for x in {x1, x2}:
            if 0 <= x < w and cya <= cyb:
                m[cya:cyb + 1, x] = True
    return m


def draw_outlines(img, sizes, boxes, counts, points, n_points, color):
    """ops.draw_outlines on the host: the same tensors (any device), the same pixels written"""
    out = img.cpu().numpy()
    sizes, boxes, counts = sizes.cpu().numpy(), boxes.cpu().numpy(), counts.cpu().numpy()
    points, n_points = points.cpu().numpy(), n_points.cpu().numpy()
    n, mh, mw, _ = out.shape
    for i in range(n):
        h, w = (int(v) for v in sizes[i])
        if h < 1 or w < 1 or h > mh or w > mw:
            continue
        m = outline_mask(h, w, boxes[i, :min(max(int(counts[i]), 0), boxes.shape[1])])
        q = points[i, :min(max(int(n_points[i]), 0), points.shape[1])].astype(np.int64)
        q = q[(q >= 0) & (q < h * w)]
        m.reshape(-1)[q] = True
        out[i, :h, :w][m] = np.asarray(color, np.uint8)
    img.copy_(torch.from_numpy(out))
    return img


def resize_sized(src, sizes, out):
    """ops.resize_sized on the host: cv2.resize(INTER_LINEAR) of each frame into the top-left of its out slot"""
    import cv2
    s, o = src.cpu().numpy(), out.cpu().numpy()
    _, sh, sw, _ = s.shape
    _, oh, ow, _ = o.shape
    for i, (h, w, dh, dw) in enumerate(sizes.cpu().numpy().tolist()):
        if min(h, w, dh, dw) < 1 or h > sh or w > sw or dh > oh or dw > ow:
            continue
        o[i, :dh, :dw] = cv2.resize(np.ascontiguousarray(s[i, :h, :w]), (dw, dh), interpolation=cv2.INTER_LINEAR)
    out.copy_(torch.from_numpy(o))
    return out


def device_pass(files, frames, scale):
    """streaming_eval.device_pass on the host: PIL's decode, cv2's resize, the drawing above, PIL's save"""
    from PIL import Image
    out = []
    for b, f in zip(files, frames):
        img = np.array(Image.open(io.BytesIO(b)))
        assert img.shape[:2] == tuple(f.hw)
        t = torch.from_numpy(img)[None].contiguous()
        if scale != 1:
            r = torch.empty((1, f.out_hw[0], f.out_hw[1], 3), dtype=torch.uint8)
            t = resize_sized(t, torch.tensor([[*f.hw, *f.out_hw]], dtype=torch.int32), r)
        boxes = torch.from_numpy(np.asarray(f.boxes, np.int32).reshape(1, -1, 4)) if len(f.boxes) else \
            torch.zeros((1, 1, 4), dtype=torch.int32)
        pts = torch.from_numpy(np.asarray(f.points, np.int32).reshape(1, -1)) if len(f.points) else \
            torch.zeros((1, 1), dtype=torch.int32)
        draw_outlines(t, torch.tensor([f.out_hw], dtype=torch.int32), boxes, torch.tensor([len(f.boxes)], dtype=torch.int32),
                      pts, torch.tensor([len(f.points)], dtype=torch.int32), (0, 255, 0))
        buf = io.BytesIO()
        Image.fromarray(t[0].numpy()).save(buf, format="JPEG")
        out.append(buf.getvalue())
    return out
