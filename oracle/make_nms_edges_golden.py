"""Generate tests/golden/nms_edges.npz -- TEST INFRASTRUCTURE.  Run in the build container:

    python oracle/make_nms_edges_golden.py

Crafted head outputs [A, 5 + nc] (cxcywh, obj, one-hot class scores, so a box's score is its obj) at the edges where an
NMS can take the wrong path, and the anchors that torchvision's batched_nms keeps on CUDA tensors
(oracle.postprocess_oracle.nms_reference, through postprocess_oracle), in output order.  Each case names the rule of that
path it depends on ("rule"): removing it, or for "class_test" adding back a per-class test, changes the kept list:

  fma_*, agnostic_fma_*, ties_*  a pair whose IoU lies within an ulp or two of the threshold, where the later box's area
                                 fused into the sum (fma) decides; fma_045 also holds zero-area boxes (0 / 0 IoU) and a
                                 NaN box below the confidence threshold (the max coordinate is taken after the mask);
                                 ties_065 two overlapping boxes of equal score (the lower anchor index comes first)
  trick_*                        a pair where rounding the class-shifted corners decides (offsets); trick_045 lies at
                                 negative coordinates
  cross_class                    class 0 and class 1 boxes reaching below -(max + 1): their shifted boxes overlap, and
                                 the class-1 box is suppressed across classes (class_test)
  nan, nan_c1                    a NaN box makes boxes.max() NaN, every offset NaN, and nothing is suppressed (nan)

The pairs are found by a seeded search; a rerun writes the same file."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.postprocess_oracle import nms_reference, postprocess_oracle  # noqa: E402

# the nms_reference switch that removes (or, class_test, adds) each rule
ABLATION = {"fma": {"fma": False}, "offsets": {"offsets": False}, "nan": {"propagate_nan": False},
            "class_test": {"class_test": True}}


def rows(nc, boxes):
    """boxes: (cx, cy, w, h, score, class) -> [A, 5 + nc] fp32"""
    p = np.zeros((len(boxes), 5 + nc), np.float32)
    for k, (cx, cy, w, h, s, c) in enumerate(boxes):
        p[k, :5] = (cx, cy, w, h, s)
        p[k, 5 + c] = 1.0
    return p


def keep(pred, nc, conf, thr, agnostic, **rule):
    """anchors kept by the reference path (rule: nms_reference switches), in output order"""
    p = torch.from_numpy(pred)
    half_w, half_h = p[:, 2] / 2, p[:, 3] / 2
    xyxy = torch.stack([p[:, 0] - half_w, p[:, 1] - half_h, p[:, 0] + half_w, p[:, 1] + half_h], 1)
    cconf, cls = torch.max(p[:, 5:5 + nc], 1)
    score = p[:, 4] * cconf
    idx = (score >= conf).nonzero().flatten().numpy()
    k = nms_reference(xyxy.numpy()[idx], score.numpy()[idx], cls.numpy()[idx], thr, agnostic, **rule)
    return idx[k]


def pair_near(rng, thr, cls, cls_b, rel, x_lo=100.0):
    """box A and box B of the same size, B shifted right so that the IoU (w - d) / (w + d) lies near thr, d jittered by a
    relative rel; B's size moved by a few fp32 ulps"""
    w = np.float32(rng.uniform(20, 200))
    h = np.float32(rng.uniform(20, 200))
    cx = np.float32(rng.uniform(x_lo, x_lo + 700))
    cy = np.float32(rng.uniform(100, 500))
    d = w * (1 - thr) / (1 + thr) * (1 + rel * rng.uniform(-1, 1))
    wb = np.float32(w) + np.float32(rng.integers(-4, 5)) * np.spacing(w)
    hb = np.float32(h) + np.float32(rng.integers(-4, 5)) * np.spacing(h)
    return [(cx, cy, w, h, 0.9, cls), (np.float32(cx + d), cy, wb, hb, 0.8, cls_b)]


def search(name, nc, conf, thr, agnostic, rule, make, tries=200000, seed=0):
    rng = np.random.default_rng(seed)
    for _ in range(tries):
        pred = rows(nc, make(rng))
        want = keep(pred, nc, conf, thr, agnostic)
        if not np.array_equal(want, keep(pred, nc, conf, thr, agnostic, **ABLATION[rule])):
            return pred
    raise RuntimeError(f"{name}: no case found")


def case_list():
    nanbox = (np.nan, 300.0, 50.0, 50.0, 0.95, 5)
    low_nan = (np.nan, 100.0, 40.0, 40.0, 0.001, 3)           # below every conf used here: not a candidate
    zero_area = [(400.0, 300.0, 0.0, 80.0, 0.7, 6), (400.0, 300.0, 0.0, 80.0, 0.6, 6), (420.0, 310.0, 60.0, 0.0, 0.5, 6)]
    far = (880.0, 540.0, 150.0, 100.0, 0.5, 0)                 # another class setting the max coordinate (955)
    cases = []

    def add(name, nc, conf, thr, agnostic, rule, pred):
        cases.append(dict(name=name, nc=nc, conf=conf, thr=thr, agnostic=agnostic, rule=rule, pred=pred))

    add("fma_045", 8, 0.01, 0.45, False, "fma",
        search("fma_045", 8, 0.01, 0.45, False, "fma",
               lambda r: pair_near(r, 0.45, 6, 6, 4e-7) + zero_area + [low_nan, far], seed=1))
    add("fma_065_c80", 80, 0.01, 0.65, False, "fma",
        search("fma_065_c80", 80, 0.01, 0.65, False, "fma", lambda r: pair_near(r, 0.65, 41, 41, 4e-7) + [far], seed=2))
    add("fma_065_c1", 1, 0.3, 0.65, False, "fma",
        search("fma_065_c1", 1, 0.3, 0.65, False, "fma", lambda r: pair_near(r, 0.65, 0, 0, 4e-7), seed=3))
    add("agnostic_fma_045_c80", 80, 0.001, 0.45, True, "fma",
        search("agnostic_fma_045_c80", 80, 0.001, 0.45, True, "fma",
               lambda r: pair_near(r, 0.45, 12, 57, 4e-7) + [far], seed=4))
    add("trick_045_c80", 80, 0.01, 0.45, False, "offsets",
        search("trick_045_c80", 80, 0.01, 0.45, False, "offsets",
               lambda r: [(c[0] - np.float32(800), c[1], c[2], c[3], c[4], c[5]) for c in pair_near(r, 0.45, 79, 79, 2e-4, 0.0)]
               + [far], seed=5))
    add("trick_065", 8, 0.01, 0.65, False, "offsets",
        search("trick_065", 8, 0.01, 0.65, False, "offsets", lambda r: pair_near(r, 0.65, 7, 7, 2e-4) + [far], seed=6))
    # the issue's example: [-30000, -30000, 900, 580] for classes 0 and 1, [10, 10, 960, 590] for class 2
    add("cross_class", 8, 0.01, 0.65, False, "class_test",
        rows(8, [(-14550.0, -14710.0, 30900.0, 30580.0, 0.9, 0), (-14550.0, -14710.0, 30900.0, 30580.0, 0.8, 1),
                 (485.0, 300.0, 950.0, 580.0, 0.7, 2)]))
    add("nan", 8, 0.01, 0.45, False, "nan",
        rows(8, [(200.0, 200.0, 100.0, 80.0, 0.9, 3), (205.0, 202.0, 100.0, 80.0, 0.8, 3), nanbox, far]))
    add("nan_c1", 1, 0.01, 0.65, False, "nan",
        rows(1, [(200.0, 200.0, 100.0, 80.0, 0.9, 0), (203.0, 201.0, 100.0, 80.0, 0.8, 0), nanbox[:5] + (0,)]))
    ties = [(600.0, 200.0, 90.0, 70.0, 0.75, 4), (602.0, 201.0, 90.0, 70.0, 0.75, 4), (601.0, 199.0, 90.0, 70.0, 0.75, 4)]
    add("ties_065", 8, 0.01, 0.65, False, "fma",
        search("ties_065", 8, 0.01, 0.65, False, "fma", lambda r: pair_near(r, 0.65, 2, 2, 4e-7) + ties + [far], seed=7))
    for c in cases:
        c["keep"] = keep(c["pred"], c["nc"], c["conf"], c["thr"], c["agnostic"])
        out = postprocess_oracle(torch.from_numpy(c["pred"])[None], c["nc"], c["conf"], c["thr"], c["agnostic"])[0]
        assert out.shape[0] == len(c["keep"])
    return cases


if __name__ == "__main__":
    import torchvision
    cases = case_list()
    arrays = {"names": np.array([c["name"] for c in cases]), "rule": np.array([c["rule"] for c in cases]),
              "nc": np.array([c["nc"] for c in cases], np.int32), "conf": np.array([c["conf"] for c in cases], np.float64),
              "thr": np.array([c["thr"] for c in cases], np.float64),
              "agnostic": np.array([c["agnostic"] for c in cases], bool), "torchvision": np.array(torchvision.__version__)}
    for k, c in enumerate(cases):
        arrays[f"pred_{k}"] = c["pred"]
        arrays[f"keep_{k}"] = c["keep"].astype(np.int64)
    path = os.path.join(ROOT, "tests", "golden", "nms_edges.npz")
    np.savez_compressed(path, **arrays)
    for c in cases:
        print(f"{c['name']:22s} nc {c['nc']:2d} thr {c['thr']} {c['rule']:10s} {len(c['pred'])} anchors -> keep {c['keep'].tolist()}")
    print(path)
