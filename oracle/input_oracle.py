"""CPU ORACLE OF THE INPUT TRANSFORMS -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A numpy restatement of what the reference does to a frame pair before the model sees it:

    /root/reference/exps/data/data_augment_flip.py:141-234     _mirror, preproc, TrainTransform, DoubleTrainTransform,
                                                               ValTransform, DoubleValTransform
    /root/reference/exps/dataset/tal_flip_one_future_argoversedataset.py:179-187   load_resized_img
    /root/reference/sAP/streamyolo/streamyolo_det.py:57-60,176-181                  the streaming driver's preproc

with cv2.resize(..., interpolation=cv2.INTER_LINEAR) on uint8 BGR restated as OpenCV's 8-bit fixed-point bilinear
resize (``resize_linear_u8``).  ``tests/test_input_pipeline.py`` pins the resize against cv2 itself and the transforms
against ``tests/golden/input_pairs.npz``, which ``oracle/make_input_golden.py`` writes from the unmodified reference.
"""
import numpy as np

PAD_VALUE = 114


def _axis(src, dst, clamp):
    """Source taps and 11-bit weights of one axis: (s0, s1, w0, w1) int64 arrays of length dst."""
    scale = 1.0 / (dst / src)                                        # double, as cv2 computes it
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:                                                        # columns: taps and weight clamped at both borders
        lo, hi = s < 0, s >= src - 1
        s[lo], f[lo] = 0, 0
        s[hi], f[hi] = src - 1, 0
    w0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    w1 = np.rint(f * np.float32(2048)).astype(np.int64)
    # rows keep their weights; only the two rows fetched are clamped
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), w0, w1


def resize_linear_u8(img, dsize):
    """cv2.resize(img, dsize=(W, H), interpolation=cv2.INTER_LINEAR) for a uint8 [h, w, C] image."""
    dw, dh = dsize
    h, w = img.shape[:2]
    xs0, xs1, xa0, xa1 = _axis(w, dw, True)
    ys0, ys1, yb0, yb1 = _axis(h, dh, False)
    p = img.astype(np.int64)
    S = p[:, xs0] * xa0[None, :, None] + p[:, xs1] * xa1[None, :, None]           # horizontal pass, [h, dw, C]
    v = (((yb0[:, None, None] * (S[ys0] >> 4)) >> 16) + ((yb1[:, None, None] * (S[ys1] >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def load_resized(img, input_size):
    """load_resized_img: the raw frame scaled to fit input_size (int() truncation of both sides)."""
    r = min(input_size[0] / img.shape[0], input_size[1] / img.shape[1])
    return resize_linear_u8(img, (int(img.shape[1] * r), int(img.shape[0] * r)))


def letterbox(img, input_size):
    """preproc: resize to fit, top-left on a 114 canvas, HWC -> CHW float32.  -> (image, r)"""
    out = np.full((input_size[0], input_size[1], 3), PAD_VALUE, np.uint8)
    r = min(input_size[0] / img.shape[0], input_size[1] / img.shape[1])
    nh, nw = int(img.shape[0] * r), int(img.shape[1] * r)
    out[:nh, :nw] = resize_linear_u8(img, (nw, nh))
    return np.ascontiguousarray(out.transpose(2, 0, 1), dtype=np.float32), r


def _cxcywh(b):
    b = b.copy()
    b[:, 2] = b[:, 2] - b[:, 0]
    b[:, 3] = b[:, 3] - b[:, 1]
    b[:, 0] = b[:, 0] + b[:, 2] * 0.5
    b[:, 1] = b[:, 1] + b[:, 3] * 0.5
    return b


def train_frame(img, targets, input_size, max_labels, mirror, flip=True):
    """TrainTransform(max_labels, hsv=False, flip) on one frame.  -> (image [3, H, W] f32, labels [max_labels, 5] f32,
    effective mirror bit)"""
    labels = np.zeros((max_labels, 5), np.float64)
    if len(targets) == 0:
        return letterbox(img, input_size)[0], labels.astype(np.float32), 0
    boxes, cls = targets[:, :4].copy(), targets[:, 4].copy()
    a = bool(flip and mirror)
    src = img
    if a:
        width = img.shape[1]
        src = img[:, ::-1]
        boxes[:, 0::2] = width - boxes[:, 2::-2]
    image, r = letterbox(src, input_size)
    boxes = _cxcywh(boxes) * r
    keep = np.minimum(boxes[:, 2], boxes[:, 3]) > 1
    boxes, cls = boxes[keep], cls[keep]
    if len(boxes) == 0:                                              # every row filtered: the unmirrored frame
        a = False
        image, r = letterbox(img, input_size)
        boxes, cls = _cxcywh(targets[:, :4]) * r, targets[:, 4]
    rows = np.hstack((cls[:, None], boxes))[:max_labels]
    labels[:len(rows)] = rows
    return image, labels.astype(np.float32), int(a)


def pair_transform(images, targets, input_size, max_labels, mirror, flip=True, raw=False):
    """DoubleTrainTransform(max_labels, hsv=False, flip)((img, support_img), (target, support_target), input_size) with
    random.randrange(2) -> ``mirror``; ``raw``: the frames are what cv2.imread returned and load_resized_img runs first.
    -> (x [6, H, W] f32 (current frame first), labels_fut, labels_cur, effective mirror bits (2,))"""
    out = []
    for img, tg in zip(images, targets):
        if raw:
            img = load_resized(img, input_size)
        out.append(train_frame(img, tg, input_size, max_labels, mirror, flip))
    return (np.concatenate([out[0][0], out[1][0]], 0), out[0][1], out[1][1], (out[0][2], out[1][2]))


def val_pair(images, input_size, raw=False):
    """DoubleValTransform: both frames letterboxed, no mirror, no labels.  -> x [6, H, W] f32"""
    if raw:
        images = [load_resized(i, input_size) for i in images]
    return np.concatenate([letterbox(i, input_size)[0] for i in images], 0)


def stream_frame(frame, size=(600, 960)):
    """streamyolo_det.preproc(frame, size) + torch.from_numpy(.).float()[None]: a plain (possibly non-uniform) resize, no
    pad, no mirror.  -> [1, 3, H, W] f32"""
    r = resize_linear_u8(frame, (size[1], size[0]))
    return np.ascontiguousarray(r.transpose(2, 0, 1), dtype=np.float32)[None]
