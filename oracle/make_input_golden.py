"""Generate tests/golden/input_pairs.npz FROM THE UNMODIFIED REFERENCE (test infrastructure).

Runs only in the build container, where /root/reference is mounted and cv2 is installed:

    python oracle/make_input_golden.py

It imports /root/reference/exps/data/data_augment_flip.py untouched (``yolox.utils.xyxy2cxcywh``, restated below, is added
to the stand-in package of oracle/ref_shim before that import), runs DoubleTrainTransform(max_labels, hsv=False, flip=True) and DoubleValTransform with cv2 on seeded
small frames, with ``random.randrange(2)`` replaced by the case's mirror bit, and records images and labels.  The dataset's
load_resized_img (exps/dataset/tal_flip_one_future_argoversedataset.py:179-187) and the streaming driver's preproc
(sAP/streamyolo/streamyolo_det.py:57-60) live in modules that import pycocotools / mmcv, so their few lines are restated
here.  Every case asserts that the situation it is named for actually occurs.

Keys per case ``c``: c_frames uint8 [2, h, w, 3], c_ann float64 [2, M, 5] (zero-padded), c_counts int32 [2],
c_meta int32 [H, W, max_labels, mirror, raw, train], c_x uint8 [6, H, W] (the fp32 image; every value is an integer),
c_labels float32 [2, max_labels, 5] (train cases).  Streaming cases ``s<i>``: s<i>_frame uint8, s<i>_out uint8 [3, H, W].
"""
import os
import sys
import types

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "ref_shim"))
sys.path.insert(0, "/root/reference")

import yolox.utils  # noqa: E402  (the stand-in of oracle/ref_shim)


def xyxy2cxcywh(bboxes):
    """yolox==0.3.0 yolox.utils.xyxy2cxcywh restated from memory of the published sources (call site
    /root/reference/exps/data/data_augment_flip.py:14,190,201): in place on an [n, >=4] array, x1, y1, x2, y2 -> cx, cy, w, h"""
    bboxes[:, 2] = bboxes[:, 2] - bboxes[:, 0]
    bboxes[:, 3] = bboxes[:, 3] - bboxes[:, 1]
    bboxes[:, 0] = bboxes[:, 0] + bboxes[:, 2] * 0.5
    bboxes[:, 1] = bboxes[:, 1] + bboxes[:, 3] * 0.5
    return bboxes


yolox.utils.xyxy2cxcywh = xyxy2cxcywh          # the one yolox symbol data_augment_flip.py imports

from exps.data import data_augment_flip as daf  # noqa: E402
from oracle import input_oracle  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "input_pairs.npz")


def load_resized_img(img, img_size):
    r = min(img_size[0] / img.shape[0], img_size[1] / img.shape[1])
    return cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR).astype(np.uint8)


def stream_preproc(img, input_size, swap=(2, 0, 1)):
    resized_img = cv2.resize(img, (input_size[1], input_size[0]), interpolation=cv2.INTER_LINEAR,)
    resized_img = resized_img.transpose(swap)
    return resized_img


def frames(g, h, w):
    """two correlated BGR frames: smooth content plus noise, the second one shifted"""
    lo = g.uniform(0, 255, (h // 4 + 2, w // 4 + 2, 3))
    a = cv2.resize(lo, (w, h), interpolation=cv2.INTER_CUBIC) * 0.8 + g.uniform(0, 50, (h, w, 3))
    b = np.roll(a, (1, 2), axis=(0, 1)) * 0.9 + g.uniform(0, 25, (h, w, 3))
    return np.stack([np.clip(a, 0, 255), np.clip(b, 0, 255)]).astype(np.uint8)


def boxes(g, n, h, w, tiny=False):
    """n rows x1, y1, x2, y2, cls inside an h x w image (``tiny``: every box under one pixel wide)"""
    x1 = g.uniform(0, w - 2, n)
    y1 = g.uniform(0, h - 2, n)
    bw = g.uniform(0.05, 0.5, n) if tiny else g.uniform(2, w / 3, n)
    bh = g.uniform(2, h / 3, n)
    return np.stack([x1, y1, np.minimum(x1 + bw, w - 1), np.minimum(y1 + bh, h - 1), g.integers(0, 8, n)], 1)


def run_train(imgs, targets, size, max_labels, mirror):
    daf.random = types.SimpleNamespace(randrange=lambda n: mirror)
    t = daf.DoubleTrainTransform(max_labels=max_labels, hsv=False, flip=True)
    img1, img2, l1, l2 = t((imgs[0], imgs[1]), (targets[0].copy(), targets[1].copy()), size)
    return np.concatenate([img1, img2], 0), np.stack([l1, l2])


def as_u8(x):
    assert np.array_equal(x, np.round(x)) and x.min() >= 0 and x.max() <= 255
    return x.astype(np.uint8)


def main():
    g = np.random.default_rng(20261015)
    out = {}
    size = (60, 96)
    f45 = frames(g, 45, 80)                        # r = 1.2: upscaled to 54 x 96, 6 pad rows

    def add(name, imgs, targets, mirror, max_labels=6, raw=False, train=True, check=None):
        src = [load_resized_img(i, size) for i in imgs] if raw else list(imgs)
        m = max(1, max(len(t) for t in targets))
        ann = np.zeros((2, m, 5))
        for i, t in enumerate(targets):
            ann[i, :len(t)] = t
        if train:
            x, lab = run_train(src, targets, size, max_labels, mirror)
            out[name + "_labels"] = lab
            want = input_oracle.pair_transform(imgs, targets, size, max_labels, mirror, raw=raw)
            assert np.array_equal(want[0], x) and np.array_equal(want[1], lab[0]) and np.array_equal(want[2], lab[1]), name
            if check is not None:
                assert check(src, targets, want[3]), name
        else:
            t = daf.DoubleValTransform()
            img1, img2, _, _ = t((src[0], src[1]), (None, None), size)
            x = np.concatenate([img1, img2], 0)
            assert np.array_equal(input_oracle.val_pair(imgs, size, raw=raw), x), name
        out[name + "_frames"] = np.ascontiguousarray(imgs)
        out[name + "_ann"] = ann
        out[name + "_counts"] = np.array([len(t) for t in targets], np.int32)
        out[name + "_meta"] = np.array([size[0], size[1], max_labels, mirror, int(raw), int(train)], np.int32)
        out[name + "_x"] = as_u8(x)

    t0, t1 = boxes(g, 5, 45, 80), boxes(g, 4, 45, 80)
    add("mirror0", f45, [t0, t1], 0, check=lambda s, t, a: a == (0, 0))
    add("mirror1", f45, [t0, t1], 1, check=lambda s, t, a: a == (1, 1))
    add("no_annotations", f45, [np.zeros((0, 5)), t1], 1, check=lambda s, t, a: a == (0, 1))
    add("all_filtered", f45, [boxes(g, 3, 45, 80, tiny=True), t1], 1, check=lambda s, t, a: a == (0, 1))
    mixed = np.concatenate([boxes(g, 7, 45, 80), boxes(g, 3, 45, 80, tiny=True)])[g.permutation(10)]

    def overflow(s, t, a):                         # more surviving rows than max_labels (6), and some filtered
        r = min(size[0] / 45, size[1] / 80)
        kept = int((np.minimum(t[0][:, 2] - t[0][:, 0], t[0][:, 3] - t[0][:, 1]) * r > 1).sum())
        return a == (1, 1) and 6 < kept < len(t[0])
    add("too_many_rows", f45, [mixed, t1], 1, check=overflow)

    f20 = frames(g, 20, 94)

    def two_resizes(s, t, a):
        mid = s[0].shape[:2]
        r = min(size[0] / mid[0], size[1] / mid[1])
        return mid != (20, 94) and (int(mid[0] * r), int(mid[1] * r)) != mid and a == (1, 1)
    add("two_resizes", f20, [boxes(g, 3, 20, 95), boxes(g, 2, 20, 95)], 1, raw=True, check=two_resizes)
    f75 = frames(g, 75, 133)
    add("raw", f75, [boxes(g, 4, 54, 96), boxes(g, 4, 54, 96)], 1, raw=True,          # 75 x 133 -> 54 x 96, then only the pad
        check=lambda s, t, a: s[0].shape[:2] == (54, 96) and a == (1, 1))
    add("val", f45, [np.zeros((0, 5)), np.zeros((0, 5))], 0, train=False)
    add("val_raw", f75, [np.zeros((0, 5)), np.zeros((0, 5))], 0, raw=True, train=False)

    for i, (h, w, H, W) in enumerate([(30, 48, 15, 24), (37, 53, 50, 70), (45, 80, 30, 77), (12, 20, 12, 20)]):
        fr = frames(g, h, w)[0]
        o = stream_preproc(fr, (H, W))
        assert np.array_equal(input_oracle.stream_frame(fr, (H, W))[0], o.astype(np.float32))
        out[f"s{i}_frame"], out[f"s{i}_out"] = fr, np.ascontiguousarray(o)

    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
