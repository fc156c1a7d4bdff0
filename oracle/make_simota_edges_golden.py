"""Generate tests/golden/simota_edges.npz -- TEST INFRASTRUCTURE.  Run in the build container:

    python oracle/make_simota_edges_golden.py

Label assignment (SimOTA) and Trend-Aware loss cases at the edges where an implementation can take the wrong branch, and
what the UNMODIFIED reference computes on each: TALHead.get_losses of /root/reference/exps/model/tal_head.py, imported on
top of the yolox stand-in in oracle/ref_shim and run on CPU fp32, with the assignment captured per image as
oracle/make_golden.py captures it.  The inputs are not stored: ``edge_cases()`` rebuilds them from fixed seeds (the
fixture keeps a checksum of each case's tensors), so the tests can run the device kernel on exactly these tensors.

Every case names the rule its answer depends on ("rule"); tests/test_simota_reference.py shows that changing that rule in
a restatement of the reference changes the recorded answer:

  grid_<h>x<w>        every multi-scale training size (train.multiscale_sizes), B = 2, 50 label rows, one image full:
                      dynamic k truncates (``.int()``) rather than rounds ("trunc")
  box_edge_on_centre  a ground-truth edge on anchor centres, and a ground-truth centre 2.5 strides from one (">": the
                      strict in-box and in-centre tests)
  box_below_stride    a 3 x 2 px ground truth whose corner is an anchor centre: no anchor strictly inside (">")
  whole_image         a ground truth covering the 688 x 1120 image: every anchor a candidate, identical predictions
                      ("ties": lowest anchor index first)
  border              ground truths hanging over the image edges and ending on the last 16 x 25 anchor row and column
                      below the 496 px image (">")
  crowd               25 identical ground truths of cycling classes and 25 overlapping ones ("ties" between equal cost
                      columns: lowest ground-truth index)
  pred_ties           duplicated predictions, and an image where every IoU is 0 and every logit equal ("ties")
  dk_sum_order        a top-10 IoU set whose fp32 sum truncates differently in torch's CPU order and in ATen's CUDA
                      order ("sum_order"); found by a seeded search (find_dk_boundary) and kept as numbers, both
                      dynamic k recorded
  dk_trunc            a top-10 IoU sum with fractional part above one half ("trunc")
  saturated           obj / cls logits at +-30 and +-100: p is 0 or 1 and the -100 clamp of the BCE decides ("clamp")
  tal_thr05, tal_thr04_g15
                      a current box inside its future box with IoU exactly ignore_thr, future labels without current
                      ones, current labels without future ones; gamma 1 and 1.5 ("ignore_thr": the strict <); the
                      TAL weights cancel out of the loss values and reach only the gradient, so the fixture also keeps
                      the reference's d total_loss / d box at the foreground anchors
  classes_c8, classes_c80
                      ground truths of class 0 and NC - 1 with one box and equal logits for both classes ("ties")
  degenerate_preds    zero-width and zero-height predicted boxes (exp underflow): every IoU 0 ("ties")
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from streamyolo_b200 import synth  # noqa: E402
from streamyolo_b200.ops import conv_out_hw  # noqa: E402
from streamyolo_b200.train import multiscale_sizes  # noqa: E402

STRIDES = (8, 16, 32)
LOSSES = ["total_loss", "iou_loss", "conf_loss", "cls_loss", "l1_loss", "num_fg"]     # get_losses' return order
F32 = np.float32


def level_hw(h, w):
    """(h, w) of the three head levels for an h x w input: Focus halves, then the stride-2 3x3 convs of dark2 ... dark5"""
    hw = [((h + 1) // 2, (w + 1) // 2)]
    for _ in range(4):
        hw.append(conv_out_hw(*hw[-1], 3, 2))
    return hw[2:]


def anchor_grid(hw):
    """gx, gy, stride per anchor (level-major, row-major), fp32"""
    xs, ys, ss = [], [], []
    for (h, w), s in zip(hw, STRIDES):
        yv, xv = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        xs.append(xv.ravel()), ys.append(yv.ravel()), ss.append(np.full(h * w, s))
    return np.concatenate(xs).astype(F32), np.concatenate(ys).astype(F32), np.concatenate(ss).astype(F32)


def anchor_index(hw, level, ix, iy):
    return sum(h * w for h, w in hw[:level]) + iy * hw[level][1] + ix


def synthetic_outputs(rng, hw, b, nc, fut):
    """decoded head outputs [b, A, 5 + nc] (boxes near their anchors, low logits) and the raw regression [b, A, 4]; the
    12 anchors nearest each ground truth predict its box well"""
    gx, gy, gs = anchor_grid(hw)
    a = gx.shape[0]
    raw = (rng.standard_normal((b, a, 4)) * 0.4).astype(F32)
    out = np.empty((b, a, 5 + nc), F32)
    out[..., 0] = (raw[..., 0] + gx) * gs
    out[..., 1] = (raw[..., 1] + gy) * gs
    out[..., 2] = np.exp(raw[..., 2] + F32(1.2)) * gs
    out[..., 3] = np.exp(raw[..., 3] + F32(1.2)) * gs
    out[..., 4:] = rng.standard_normal((b, a, 1 + nc)) * 1.5 - 3.0
    for bi in range(b):
        for gt in fut[bi]:
            if gt[3] <= 0:
                continue
            d = np.abs(out[bi, :, 0] - gt[1]) + np.abs(out[bi, :, 1] - gt[2])
            idx = np.argsort(d, kind="stable")[:12]
            out[bi, idx, 0:4] = gt[1:5] * (1 + 0.05 * rng.standard_normal((12, 4))).astype(F32)
            out[bi, idx, 4] = 1.0
            out[bi, idx, 5 + int(gt[0])] = 1.5
    return out, raw


def labels(rows, n_rows):
    """[n_rows, 5] fp32 label block from (cls, cx, cy, w, h) tuples"""
    t = np.zeros((n_rows, 5), F32)
    if rows:
        t[:len(rows)] = np.array(rows, F32)
    return t


def case(name, rule, hw, nc, fut, cur, out, raw, gamma=1.0, thr=0.5, val=1.5):
    return dict(name=name, rule=rule, hw=[tuple(map(int, x)) for x in hw], nc=nc, gamma=gamma, thr=thr, val=val,
                outputs=np.ascontiguousarray(out, F32), origin=np.ascontiguousarray(raw, F32),
                fut=np.ascontiguousarray(fut, F32), cur=np.ascontiguousarray(cur, F32))


def checksum(c):
    h = hashlib.sha256()
    for k in ("outputs", "origin", "fut", "cur"):
        h.update(c[k].tobytes())
    return h.hexdigest()[:16]


def _put(out, bi, a, box, obj, cls):
    out[bi, a, 0:4] = box
    out[bi, a, 4] = obj
    out[bi, a, 5:] = cls


def grid_cases():
    cases = []
    f0, c0 = synth.synth_labels(1, 600, 960, n_obj=50, seed=3)
    f1, c1 = synth.synth_labels(1, 600, 960, n_obj=12, seed=4)
    fut0 = np.concatenate([f0.numpy(), f1.numpy()], 0)[:, :50]
    cur0 = np.concatenate([c0.numpy(), c1.numpy()], 0)[:, :50]
    for k, (h, w) in enumerate(multiscale_sizes()):
        fut, cur = fut0.copy(), cur0.copy()
        for t in (fut, cur):                              # ops.scale_labels_: fp32 products
            t[..., 1::2] *= F32(w / 960.0)
            t[..., 2::2] *= F32(h / 600.0)
        hw = level_hw(h, w)
        out, raw = synthetic_outputs(np.random.default_rng(100 + k), hw, 2, 8, fut)
        cases.append(case(f"grid_{h}x{w}", "trunc", hw, 8, fut, cur, out, raw))
    return cases


def base(h, w, b, nc, fut, seed):
    hw = level_hw(h, w)
    out, raw = synthetic_outputs(np.random.default_rng(seed), hw, b, nc, fut)
    return hw, out, raw


def edge_cases_geometry():
    cases = []
    # --- an edge on anchor centres (stride 8 centres at 8 i + 4) and a centre 2.5 strides from one
    fut = np.stack([labels([(2, 172.0, 252.0, 16.0, 16.0), (5, 504.0, 344.0, 120.0, 120.0)], 120),
                    labels([(1, 300.0, 200.0, 64.0, 48.0)], 120)])
    cur = fut.copy()
    hw, out, raw = base(600, 960, 2, 8, fut, 201)
    good = np.full(8, -4.0, F32)
    for ix in (20, 21, 22):
        for iy in (30, 31, 32):
            if (ix, iy) != (21, 31):
                _put(out, 0, anchor_index(hw, 0, ix, iy), fut[0, 0, 1:5], 5.0, np.where(np.arange(8) == 2, 5.0, -4.0))
    _put(out, 0, anchor_index(hw, 0, 21, 31), (176.0, 256.0, 16.0, 16.0), 0.0, good)
    _put(out, 0, anchor_index(hw, 0, 60, 40), fut[0, 1, 1:5], 5.0, np.where(np.arange(8) == 5, 5.0, -4.0))
    cases.append(case("box_edge_on_centre", ">", hw, 8, fut, cur, out, raw))
    # --- a 3 x 2 px box [100, 103] x [100, 102]: its corner is the stride-8 centre (12, 12), no centre strictly inside
    fut = np.stack([labels([(4, 101.5, 101.0, 3.0, 2.0)], 120), labels([(0, 700.0, 400.0, 90.0, 60.0)], 120)])
    cur = fut.copy()
    hw, out, raw = base(600, 960, 2, 8, fut, 202)
    _put(out, 0, anchor_index(hw, 0, 12, 12), (300.0, 300.0, 4.0, 4.0), -2.0, np.full(8, -2.0, F32))
    _put(out, 0, anchor_index(hw, 0, 13, 12), (101.5, 101.0, 3.0, 2.0), 4.0, np.where(np.arange(8) == 4, 4.0, -4.0))
    cases.append(case("box_below_stride", ">", hw, 8, fut, cur, out, raw))
    # --- a box the size of the 688 x 1120 image: every anchor is a candidate; identical predictions everywhere
    fut = np.stack([labels([(3, 560.0, 344.0, 1120.0, 688.0)], 50), labels([(1, 200.0, 150.0, 80.0, 60.0)], 50)])
    cur = fut.copy()
    hw, out, raw = base(688, 1120, 2, 8, fut, 203)
    out[0, :, 0:4] = fut[0, 0, 1:5]
    out[0, :, 4:] = 0.0
    cases.append(case("whole_image", "ties", hw, 8, fut, cur, out, raw))
    # --- over the border of the 496 x 800 image; the bottom-right box ends on the last stride-32 anchor row (y 496)
    # and column (x 784)
    fut = np.stack([labels([(6, 10.0, 12.0, 60.0, 50.0), (2, 736.0, 472.0, 96.0, 48.0), (7, 790.0, 300.0, 40.0, 80.0)], 50),
                    labels([(0, 400.0, 490.0, 100.0, 30.0)], 50)])
    cur = fut.copy()
    hw, out, raw = base(496, 800, 2, 8, fut, 204)
    assert hw[2] == (16, 25)
    _put(out, 0, anchor_index(hw, 2, 24, 15), fut[0, 1, 1:5], 5.0, np.where(np.arange(8) == 2, 5.0, -4.0))
    cases.append(case("border", ">", hw, 8, fut, cur, out, raw))
    return cases


def edge_cases_ties():
    cases = []
    rng = np.random.default_rng(5)
    # --- crowd: 25 identical boxes (classes cycling 0..7) and 25 overlapping ones
    rows = [(k % 8, 480.0, 300.0, 120.0, 90.0) for k in range(25)]
    rows += [(int(rng.integers(0, 8)), float(F32(600 + rng.uniform(-3, 3))), float(F32(250 + rng.uniform(-3, 3))),
              float(F32(100 + rng.uniform(-4, 4))), float(F32(80 + rng.uniform(-4, 4)))) for _ in range(25)]
    fut = np.stack([labels(rows, 50), labels(rows[:3], 50)])
    cur = fut.copy()
    hw, out, raw = base(600, 960, 2, 8, fut, 205)
    cases.append(case("crowd", "ties", hw, 8, fut, cur, out, raw))
    # --- duplicated predictions; all-zero IoUs with equal logits
    fut = np.stack([labels([(1, 320.0, 240.0, 96.0, 64.0), (6, 640.0, 420.0, 50.0, 120.0)], 50),
                    labels([(2, 480.0, 300.0, 60.0, 60.0)], 50)])
    cur = fut.copy()
    hw, out, raw = base(600, 960, 2, 8, fut, 206)
    gx, gy, gs = anchor_grid(hw)
    d = np.abs(out[0, :, 0] - 320.0) + np.abs(out[0, :, 1] - 240.0)
    idx = np.argsort(d, kind="stable")[:12]
    for k in range(0, 12, 2):                                 # pairs of identical rows
        out[0, idx[k + 1]] = out[0, idx[k]]
    out[1, :, 0] = gx * gs + 0.5 * gs
    out[1, :, 1] = gy * gs + 0.5 * gs
    out[1, :, 2:4] = 1.0
    far = (np.abs(out[1, :, 0] - 480.0) < 40) & (np.abs(out[1, :, 1] - 300.0) < 40)
    out[1, far, 0] += 200.0                                   # no prediction touches the box
    out[1, :, 4:] = -1.0
    cases.append(case("pred_ties", "ties", hw, 8, fut, cur, out, raw))
    # --- class 0 and class NC - 1 on one box, equal logits for both classes
    for nc in (8, 80):
        fut = np.stack([labels([(0, 400.0, 300.0, 80.0, 80.0), (nc - 1, 400.0, 300.0, 80.0, 80.0),
                                (nc - 1, 700.0, 200.0, 60.0, 90.0)], 50),
                        labels([(nc - 1, 150.0, 450.0, 70.0, 40.0), (0, 800.0, 100.0, 40.0, 40.0)], 50)])
        cur = fut.copy()
        hw, out, raw = base(600, 960, 2, nc, fut, 207 + nc)
        out[0, :, 5 + nc - 1] = out[0, :, 5]
        cases.append(case(f"classes_c{nc}", "ties", hw, nc, fut, cur, out, raw))
    # --- zero-width / zero-height predicted boxes (exp underflow of the raw size)
    fut = np.stack([labels([(3, 500.0, 300.0, 90.0, 70.0)], 50), labels([(5, 100.0, 100.0, 50.0, 50.0)], 50)])
    cur = fut.copy()
    hw, out, raw = base(600, 960, 2, 8, fut, 210)
    raw[:, ::2, 2] = -200.0
    raw[:, 1::2, 3] = -200.0
    gx, gy, gs = anchor_grid(hw)
    out[..., 2] = np.exp(raw[..., 2]) * gs
    out[..., 3] = np.exp(raw[..., 3]) * gs
    out[..., 4:] = -2.0
    assert (out[..., 2] == 0).any() and (out[..., 3] == 0).any()
    cases.append(case("degenerate_preds", "ties", hw, 8, fut, cur, out, raw))
    return cases


def tree_sum(v):
    """fp32 sum in ATen's CUDA reduction order for up to 127 terms (aten_sum in head_loss.cu): 32 accumulators, term i
    into accumulator i % 32 left to right, combined by halving"""
    acc = [F32(0)] * 32
    for i, x in enumerate(v):
        acc[i % 32] = F32(acc[i % 32] + F32(x))
    while len(acc) > 1:
        h = len(acc) // 2
        acc = [F32(acc[i] + acc[i + h]) for i in range(h)]
    return acc[0]


def iou_np(gt, boxes):
    """yolox bboxes_iou(xyxy=False) of one box against many, fp32 in the reference's operation order"""
    half = F32(2)
    tlx = np.maximum(gt[0] - gt[2] / half, boxes[:, 0] - boxes[:, 2] / half)
    tly = np.maximum(gt[1] - gt[3] / half, boxes[:, 1] - boxes[:, 3] / half)
    brx = np.minimum(gt[0] + gt[2] / half, boxes[:, 0] + boxes[:, 2] / half)
    bry = np.minimum(gt[1] + gt[3] / half, boxes[:, 1] + boxes[:, 3] / half)
    en = ((tlx < brx) & (tly < bry)).astype(F32)
    ai = (brx - tlx) * (bry - tly) * en
    return (ai / ((gt[2] * gt[3]) + boxes[:, 2] * boxes[:, 3] - ai)).astype(F32)


def dk_boxes(rng, gt, target):
    """ten boxes centred on gt (its height, random widths) whose fp32 IoUs with it sum near ``target``"""
    while True:
        u = rng.uniform(0.2, 0.95, 10)
        u *= target / u.sum()
        if u.max() >= 1.0:
            continue
        boxes = np.tile(gt, (10, 1)).astype(F32)
        boxes[:, 2] = (gt[2] * u).astype(F32)
        boxes[:, 2] += rng.integers(-3, 4, 10).astype(F32) * np.spacing(boxes[:, 2])
        return boxes


def dynamic_k_sums(gt, boxes):
    """dynamic k of the ten boxes' IoUs with gt, summed by torch on the CPU and in ATen's CUDA order"""
    v = np.sort(iou_np(gt, boxes))[::-1].copy()
    return int(torch.from_numpy(v)[None].sum(1)[0]), int(tree_sum(v))


def find_dk_boundary(seed=11, gt=np.array([480.0, 296.0, 160.0, 96.0], F32)):
    """the seeded search that found DK_SUM_ORDER_WIDTHS: ten boxes whose IoU sum truncates differently in torch's CPU
    order and in ATen's CUDA order"""
    rng = np.random.default_rng(seed)
    for _ in range(200000):
        boxes = dk_boxes(rng, gt, 4.0)
        a, b = dynamic_k_sums(gt, boxes)
        if a != b:
            return boxes
    raise RuntimeError("no dynamic-k boundary found")


# widths of the ten boxes (centred on the ground truth 480, 296, 160 x 96, its height) found by find_dk_boundary(); kept
# as numbers so that the case does not depend on the summation order of the CPU that rebuilds it: the fp32 IoUs sum to
# 4 as torch 2.11 adds them on an x86-64 CPU, and to 4 - 2^-22 in ATen's CUDA order
DK_SUM_ORDER_WIDTHS = np.array([28.064960479736328, 106.55349731445312, 70.62858581542969, 37.95305633544922,
                                96.9292984008789, 44.54884719848633, 31.662460327148438, 83.35657501220703,
                                112.01058959960938, 28.2921085357666], F32)


def edge_cases_arith():
    cases = []
    rng = np.random.default_rng(11)
    # --- dynamic k on a summation-order boundary, and one with a fractional part above one half
    for name, rule in (("dk_sum_order", "sum_order"), ("dk_trunc", "trunc")):
        gt = np.array([480.0, 296.0, 160.0, 96.0], F32)
        fut = np.stack([labels([(2,) + tuple(map(float, gt))], 50), labels([(4, 200.0, 200.0, 50.0, 50.0)], 50)])
        cur = fut.copy()
        hw, out, raw = base(600, 960, 2, 8, fut, 212)
        gx, gy, gs = anchor_grid(hw)
        inside = np.nonzero((gs == 8) & (np.abs(gx * 8 + 4 - gt[0]) < 60) & (np.abs(gy * 8 + 4 - gt[1]) < 30))[0]
        near = (np.abs(out[0, :, 0] - gt[0]) < 200) & (np.abs(out[0, :, 1] - gt[1]) < 150)
        out[0, near, 0] += 400.0                              # only the ten crafted boxes overlap the ground truth
        if name == "dk_sum_order":
            boxes = np.tile(gt, (10, 1)).astype(F32)
            boxes[:, 2] = DK_SUM_ORDER_WIDTHS
        else:
            boxes = dk_boxes(rng, gt, 3.7)
        sel = inside[rng.choice(len(inside), 10, replace=False)]
        out[0, sel, 0:4] = boxes
        out[0, sel, 4] = 0.5
        c = case(name, rule, hw, 8, fut, cur, out, raw)
        c["dk_cpu"], c["dk_cuda"] = dynamic_k_sums(gt, boxes)
        cases.append(c)
    # --- saturated logits: p rounds to 0 or 1 and the -100 clamp decides the class cost
    fut = np.stack([labels([(0, 400.0, 240.0, 80.0, 64.0), (3, 700.0, 400.0, 60.0, 60.0)], 50),
                    labels([(5, 300.0, 300.0, 100.0, 100.0)], 50)])
    cur = fut.copy()
    hw, out, raw = base(600, 960, 2, 8, fut, 213)
    gx, gy, gs = anchor_grid(hw)
    for bi, (cx, cy, w, h, cls) in ((0, (400.0, 240.0, 80.0, 64.0, 0)), (0, (700.0, 400.0, 60.0, 60.0, 3)),
                                    (1, (300.0, 300.0, 100.0, 100.0, 5))):
        cand = np.nonzero((np.abs(gx * gs + gs / 2 - cx) < 2.5 * gs) & (np.abs(gy * gs + gs / 2 - cy) < 2.5 * gs))[0]
        out[bi, cand, 0:4] = (cx, cy, w * 0.8, h * 0.8)
        out[bi, cand, 4] = 30.0
        out[bi, cand, 5:] = -100.0                           # target class p = 0: clamped target term
        hit = cand[len(cand) // 2:]                          # the later half: a perfect box, target class saturated at 1,
        out[bi, hit, 0:4] = (cx, cy, w, h)                   # and one other class at +30 (p = 1: clamped non-target term)
        out[bi, hit, 5 + cls] = 100.0
        out[bi, hit, 5 + (cls + 1) % 8] = 30.0
    cases.append(case("saturated", "clamp", hw, 8, fut, cur, out, raw))
    return cases


def edge_cases_tal():
    cases = []
    for name, thr, gamma in (("tal_thr05", 0.5, 1.0), ("tal_thr04_g15", 0.4, 1.5)):
        fw, fh = 100.0, 40.0
        cw = fw * thr                                       # same height, width thr * fw, inside: IoU = thr exactly
        fut = np.stack([labels([(1, 300.0, 200.0, fw, fh), (4, 600.0, 380.0, 70.0, 90.0)], 50),
                        labels([(2, 500.0, 300.0, 80.0, 80.0)], 50),
                        labels([], 50)])
        cur = np.stack([labels([(1, 300.0 - (fw - cw) / 2, 200.0, cw, fh), (4, 604.0, 384.0, 70.0, 90.0)], 50),
                        labels([], 50),
                        labels([(3, 200.0, 200.0, 50.0, 50.0)], 50)])
        hw, out, raw = base(600, 960, 3, 8, fut, 214)
        cases.append(case(name, "ignore_thr", hw, 8, fut, cur, out, raw, gamma=gamma, thr=thr, val=1.7))
    return cases


def edge_cases():
    return grid_cases() + edge_cases_geometry() + edge_cases_ties() + edge_cases_arith() + edge_cases_tal()


# ------------------------------------------------------------------------------------------------ reference run
def reference_losses(c):
    """the unmodified reference's get_losses on CPU fp32, then total_loss.backward(): six losses, the per-image
    assignment and d total_loss / d outputs"""
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, "/root/reference")
    from exps.model.tal_head import TALHead
    head = TALHead(c["nc"], 0.125, in_channels=[256, 512, 1024], gamma=c["gamma"], ignore_thr=c["thr"],
                   ignore_value=c["val"])
    head.use_l1 = True
    rec = []
    orig = head.get_assignments

    def wrapped(batch_idx, *a, **k):
        out = orig(batch_idx, *a, **k)
        _, fg_mask, pred_ious, matched, _ = out
        rec.append((int(batch_idx), fg_mask.nonzero()[:, 0].numpy().astype(np.int32), matched.numpy().astype(np.int32),
                    pred_ious.numpy().astype(np.float32)))
        return out
    head.get_assignments = wrapped
    xs, ys, ss, org = [], [], [], []
    off = 0
    for (h, w), s in zip(c["hw"], STRIDES):
        yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        xs.append(xv.reshape(1, -1).float())
        ys.append(yv.reshape(1, -1).float())
        ss.append(torch.zeros(1, h * w).fill_(s))
        org.append(torch.from_numpy(c["origin"][:, off:off + h * w]).clone())
        off += h * w
    outputs = torch.from_numpy(c["outputs"]).clone().requires_grad_(True)
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda t, *a, **k: t                 # tal_head.py:395 moves a CPU tensor with .cuda()
    try:
        res = head.get_losses(None, xs, ys, ss, (torch.from_numpy(c["fut"]), torch.from_numpy(c["cur"])), outputs, org,
                              torch.float32)
    finally:
        torch.Tensor.cuda = cuda
    res[0].backward()                                        # the training step's loss.backward()
    return np.array([float(v) for v in res], np.float64), rec, outputs.grad.numpy()


if __name__ == "__main__":
    cases = edge_cases()
    arrays = {"names": np.array([c["name"] for c in cases]), "rule": np.array([c["rule"] for c in cases]),
              "checksum": np.array([checksum(c) for c in cases]), "torch": np.array(torch.__version__)}
    for k, c in enumerate(cases):
        loss, rec, grad = reference_losses(c)
        arrays[f"loss_{k}"] = loss
        arrays[f"fg_image_{k}"] = np.concatenate([np.full(len(r[1]), r[0], np.int32) for r in rec])
        arrays[f"fg_anchor_{k}"] = np.concatenate([r[1] for r in rec])
        arrays[f"fg_gt_{k}"] = np.concatenate([r[2] for r in rec])
        arrays[f"fg_iou_{k}"] = np.concatenate([r[3] for r in rec])
        if c["rule"] == "ignore_thr":    # the TAL weights reach only the gradient: d total / d box of the foreground
            bi, ai = arrays[f"fg_image_{k}"], arrays[f"fg_anchor_{k}"]
            arrays[f"grad_box_{k}"] = grad[bi, ai, 0:4].astype(np.float32)
        if "dk_cpu" in c:
            arrays[f"dk_cpu_{k}"], arrays[f"dk_cuda_{k}"] = np.array(c["dk_cpu"]), np.array(c["dk_cuda"])
        print(f"{c['name']:20s} {c['rule']:10s} A {sum(h * w for h, w in c['hw']):5d} fg {len(arrays[f'fg_anchor_{k}']):4d} "
              f"loss {np.round(loss, 5).tolist()}")
    path = os.path.join(ROOT, "tests", "golden", "simota_edges.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path) // 1024, "KiB")
