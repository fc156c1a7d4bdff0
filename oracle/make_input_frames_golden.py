"""Generate tests/golden/input_frames.npz FROM THE UNMODIFIED REFERENCE (test infrastructure).

Runs only in the build container, where /root/reference is mounted and cv2 is installed:

    python oracle/make_input_frames_golden.py

The single-frame counterpart of oracle/make_input_golden.py (same imports, same frame / box generators): it runs the
still-image baseline's dataset transforms, TrainTransform(max_labels, hsv=False, flip=True) with the case's mirror bit and
ValTransform (/root/reference/exps/data/data_augment_flip.py:170-263, cfgs/l_s50_still_dfp_flip.py:72, 122), with cv2 on
seeded small frames, and records images and labels.  Every case asserts that the situation it is named for occurs and that
``oracle.input_oracle.train_frame`` reproduces the reference.

Keys per case ``c``: c_frame uint8 [h, w, 3], c_ann float64 [M, 5] (zero-padded), c_count int32 [1],
c_meta int32 [H, W, max_labels, mirror, raw, train], c_x uint8 [3, H, W] (the fp32 image; every value is an integer),
c_labels float32 [max_labels, 5] (train cases).
"""
import os

import numpy as np

from make_input_golden import ROOT, as_u8, boxes, daf, frames, load_resized_img  # noqa: E402  (sets up the reference import)
from oracle import input_oracle  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "input_frames.npz")


def main():
    g = np.random.default_rng(20261016)
    out = {}
    size = (60, 96)
    f45 = frames(g, 45, 80)[0]                     # r = 1.2: upscaled to 54 x 96, 6 pad rows

    def add(name, img, tg, mirror, max_labels=6, raw=False, train=True, check=None):
        src = load_resized_img(img, size) if raw else img
        ann = np.zeros((max(1, len(tg)), 5))
        ann[:len(tg)] = tg
        if train:
            x, lab = daf.TrainTransform(max_labels=max_labels, hsv=False, flip=True)(src, tg.copy(), size, mirror=mirror)
            out[name + "_labels"] = lab
            want = input_oracle.train_frame(src, tg, size, max_labels, mirror)
            assert np.array_equal(want[0], x) and np.array_equal(want[1], lab), name
            if check is not None:
                assert check(src, tg, want[2]), name
        else:
            x, _ = daf.ValTransform()(src, None, size)
            assert np.array_equal(input_oracle.letterbox(src, size)[0], x), name
        out[name + "_frame"] = np.ascontiguousarray(img)
        out[name + "_ann"] = ann
        out[name + "_count"] = np.array([len(tg)], np.int32)
        out[name + "_meta"] = np.array([size[0], size[1], max_labels, mirror, int(raw), int(train)], np.int32)
        out[name + "_x"] = as_u8(x)

    t0 = boxes(g, 5, 45, 80)
    add("mirror0", f45, t0, 0, check=lambda s, t, a: a == 0)
    add("mirror1", f45, t0, 1, check=lambda s, t, a: a == 1)
    add("no_annotations", f45, np.zeros((0, 5)), 1, check=lambda s, t, a: a == 0)
    add("all_filtered", f45, boxes(g, 3, 45, 80, tiny=True), 1, check=lambda s, t, a: a == 0)
    mixed = np.concatenate([boxes(g, 7, 45, 80), boxes(g, 3, 45, 80, tiny=True)])[g.permutation(10)]

    def overflow(s, t, a):                         # more surviving rows than max_labels (6), and some filtered
        r = min(size[0] / 45, size[1] / 80)
        kept = int((np.minimum(t[:, 2] - t[:, 0], t[:, 3] - t[:, 1]) * r > 1).sum())
        return a == 1 and 6 < kept < len(t)
    add("too_many_rows", f45, mixed, 1, check=overflow)

    f20 = frames(g, 20, 94)[0]

    def two_resizes(s, t, a):
        mid = s.shape[:2]
        r = min(size[0] / mid[0], size[1] / mid[1])
        return mid != (20, 94) and (int(mid[0] * r), int(mid[1] * r)) != mid and a == 1
    add("two_resizes", f20, boxes(g, 3, 20, 95), 1, raw=True, check=two_resizes)
    f75 = frames(g, 75, 133)[0]
    add("raw", f75, boxes(g, 4, 54, 96), 1, raw=True,                                   # 75 x 133 -> 54 x 96, then only the pad
        check=lambda s, t, a: s.shape[:2] == (54, 96) and a == 1)
    add("val", f45, np.zeros((0, 5)), 0, train=False)
    add("val_raw", f75, np.zeros((0, 5)), 0, raw=True, train=False)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
