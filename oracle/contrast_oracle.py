"""Numpy restatement of the sAP toolkit's split-screen composition (sAP/vis/vis_contrast.py) -- TEST INFRASTRUCTURE.

``split_at`` is one frame's split position (:130-135): --split-pos in pixels above 1, otherwise a fraction of the frame's
extent ``l`` along the split axis, moved by the swing animation (:45-92) at time ``ii / fps``, rounded half to even.
``compose`` is the frame (:137-165): B alone for a split at or before 0, otherwise A with B's pixels from the split on,
then the 14-pixel band [split - 7, split + 7) in the line colour where it overlaps [0, l).  ``swing`` takes an array of
times and evaluates the animation's keyframe table with the script's float64 operations, so it is an independent
restatement of streamyolo_b200.contrast.split_anime_swing.  tests/test_contrast.py pins both against the files the
unmodified script wrote (tests/golden/contrast_script.npz)."""
import numpy as np

LINE_WIDTH = 15
LINE_RGB = (241, 159, 93)


def swing(t, split_pos, l, line_width=LINE_WIDTH):
    """the swing animation's position at times ``t`` (array) -> float64 array"""
    t = np.asarray(t, np.float64)
    far, near = l + line_width // 2, (-line_width) // 2 - 1    # l + 7 and -9: the band wholly outside the frame
    keys = np.array([0, 4, 5, 8, 10, 13, 14])               # the phases' start times; durations 4, 1, 3, 2, 3, 1
    frm = np.array([split_pos, split_pos, far, far, near, near, split_pos], np.float64)
    to = np.array([split_pos, far, far, near, near, split_pos, split_pos], np.float64)
    k = np.clip(np.searchsorted(keys, t, side="right") - 1, 0, len(keys) - 1)
    dur = np.append(np.diff(keys), 1)[k]
    p = -np.cos(np.pi * ((t - keys[k]) / dur)) / 2 + 0.5
    moving = frm[k] != to[k]
    return np.where(moving, frm[k] + p * (to[k] - frm[k]), frm[k])


def split_at(ii, l, split_pos=0.5, animation=None, fps=30.0):
    """the int split of frame ``ii`` (its index in the sequence) for frames ``l`` pixels along the split axis"""
    pos = split_pos if split_pos > 1 else l * split_pos
    if animation is not None:
        assert animation == "swing", animation
        pos = float(swing([ii / fps], pos, l)[0])
    return int(np.round(np.float64(pos)))


def compose(img_a, img_b, split, horizontal=False, color=LINE_RGB):
    """the frame the script saves for images A and B ([h, w, 3] uint8, ``color`` in their channel order)"""
    a, b = np.asarray(img_a, np.uint8), np.asarray(img_b, np.uint8)
    assert a.shape == b.shape, (a.shape, b.shape)
    if horizontal:                                          # rows are the split axis: work on the transpose
        return compose(a.transpose(1, 0, 2), b.transpose(1, 0, 2), split, False, color).transpose(1, 0, 2).copy()
    l = a.shape[1]
    cols = np.arange(l)
    take_b = cols >= split                                  # every column for split <= 0
    band = (cols >= split - 7) & (cols < split + 7)
    out = np.where(take_b[None, :, None], b, a)
    out[:, band] = np.asarray(color, np.uint8)
    return out
