"""Deterministic synthetic weights / frame pairs / labels for StreamYOLO.

There is no dataset and no checkpoint in this environment, so every test,
``bench.py`` and ``__graft_entry__.smoke()`` run on synthetic data of the
reference's shapes (SURVEY.md section 8d).  Everything here is a pure function of
(name, shape, seed) so that three independent implementations -- the
unmodified reference (imported only by ``oracle/make_golden.py``), the CPU
oracle and the CUDA product -- can be fed bit-identical inputs without
shipping tensors around.

Shapes follow the reference:
  * images ``[B, 6, H, W]`` float32 in 0..255, channels 0:3 = frame t,
    3:6 = frame t-1 (/root/reference/exps/dataset/tal_flip_one_future_argoversedataset.py:260)
  * labels: tuple ``(future[B,120,5], current[B,120,5])`` rows ``(cls, cx, cy, w, h)``
    in input pixels, zero padded (/root/reference/exps/data/data_augment_flip.py:224-234,
    max_labels=120 at /root/reference/cfgs/s_s50_onex_dfp_tal_flip.py:80)
"""
import zlib

import numpy as np
import torch

MAX_LABELS = 120


def _rng(name: str, seed: int) -> np.random.Generator:
    return np.random.default_rng([zlib.crc32(name.encode()), seed])


def synth_tensor(name: str, shape, seed: int = 0) -> torch.Tensor:
    """Value for one state_dict entry, chosen by the role its key name implies."""
    shape = tuple(int(s) for s in shape)
    g = _rng(name, seed)
    leaf = name.rsplit(".", 1)[-1]
    if leaf == "num_batches_tracked":
        return torch.zeros((), dtype=torch.long)
    is_bn = ".bn." in name
    if is_bn and leaf == "weight":
        a = g.uniform(0.6, 1.4, shape)
    elif is_bn and leaf == "bias":
        a = g.uniform(-0.3, 0.3, shape)
    elif leaf == "running_mean":
        a = g.uniform(-0.2, 0.2, shape)
    elif leaf == "running_var":
        a = g.uniform(0.5, 1.5, shape)
    elif leaf == "weight":  # conv OIHW: uniform(+-sqrt(3/fan_in)) keeps unit gain
        fan_in = int(np.prod(shape[1:]))
        b = (3.0 / fan_in) ** 0.5
        a = g.uniform(-b, b, shape)
    elif leaf == "bias":  # the three prediction convs (tal_head.py:105-131,141-150)
        if "cls_preds" in name or "obj_preds" in name:
            a = -4.59512 + g.uniform(-0.5, 0.5, shape)
        else:
            a = g.uniform(-0.2, 0.2, shape)
    else:
        raise KeyError(f"no synthetic rule for {name}")
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))


def synth_state_dict(shapes: dict, seed: int = 0) -> dict:
    """``shapes`` maps state_dict key -> shape (e.g. from ``model.state_dict()``)."""
    return {k: synth_tensor(k, s, seed) for k, s in shapes.items()}


def synth_frames(batch: int, height: int = 600, width: int = 960, seed: int = 1234) -> torch.Tensor:
    """``[B,6,H,W]`` float32 in [0,255).  Smooth-ish content (low-res noise upsampled
    plus pixel noise) so that BatchNorm statistics are not degenerate; the support
    frame is the current frame shifted by (3, 5) pixels plus fresh noise."""
    g = _rng("frames", seed)
    lo = g.uniform(0, 255, (batch, 3, height // 8 + 2, width // 8 + 2)).astype(np.float32)
    cur = np.repeat(np.repeat(lo, 8, axis=2), 8, axis=3)[:, :, 4:4 + height, 4:4 + width]
    cur = 0.7 * cur + 0.3 * g.uniform(0, 255, cur.shape).astype(np.float32)
    sup = np.roll(cur, (3, 5), axis=(2, 3))
    sup = 0.9 * sup + 0.1 * g.uniform(0, 255, cur.shape).astype(np.float32)
    x = np.concatenate([cur, sup], axis=1).astype(np.float32)
    return torch.from_numpy(np.ascontiguousarray(x))


def synth_labels(batch: int, height: int = 600, width: int = 960, n_obj: int = 12,
                 seed: int = 1, empty_image: int = -1, num_classes: int = 8):
    """(future, current) label tensors.  Current-frame boxes are the future boxes
    shifted by (+4,+4) px; two per image are replaced by far-away boxes so both TAL
    branches (iou>=thr and iou<thr -> ignore_value, tal_head.py:401-403) fire.
    ``empty_image`` >= 0 zeroes that image's labels (tal_head.py:309-315)."""
    g = _rng("labels", seed)
    fut = np.zeros((batch, MAX_LABELS, 5), np.float32)
    cur = np.zeros((batch, MAX_LABELS, 5), np.float32)
    sx, sy = width / 960.0, height / 600.0
    for b in range(batch):
        n = n_obj
        cls = g.integers(0, num_classes, n).astype(np.float32)
        cx = g.uniform(30 * sx, 930 * sx, n)
        cy = g.uniform(30 * sy, 570 * sy, n)
        w = g.uniform(10, 160, n) * max(sx, 0.35)
        h = g.uniform(10, 130, n) * max(sy, 0.35)
        fut[b, :n] = np.stack([cls, cx, cy, w, h], 1)
        c = fut[b, :n].copy()
        c[:, 1] += 4.0
        c[:, 2] += 4.0
        for j in (1, n - 2):  # far-away replacements
            c[j, 1] = (c[j, 1] + 0.5 * width) % (width - 40) + 20
            c[j, 2] = (c[j, 2] + 0.5 * height) % (height - 40) + 20
        cur[b, :n] = c
        if b == empty_image:
            fut[b] = 0
            cur[b] = 0
    return torch.from_numpy(fut), torch.from_numpy(cur)


def synth_uint8_pairs(batch: int, height: int = 600, width: int = 960, rows: int = 60, seed: int = 1):
    """What the data loader hands ``data.pair_transform`` for ``batch`` pairs already at ``(height, width)``: uint8 BGR
    frames ``[B, 2, h, w, 3]``, float64 annotations ``[B, 2, rows, 5]`` (x1, y1, x2, y2, cls; zero padded), int32 counts
    ``[B, 2]`` and int32 mirror bits ``[B]``, as CPU tensors."""
    g = _rng("uint8_pairs", seed)
    lo = g.integers(0, 256, (batch, 2, height // 16 + 1, width // 16 + 1, 3)).astype(np.uint8)
    frames = np.repeat(np.repeat(lo, 16, 2), 16, 3)[:, :, :height, :width] ^ g.integers(0, 64, (batch, 2, height, width, 3),
                                                                                         dtype=np.uint8)
    ann = np.zeros((batch, 2, rows, 5))
    counts = g.integers(4, 20, (batch, 2)).astype(np.int32)
    for i in range(batch):
        for f in range(2):
            n = counts[i, f]
            x1, y1 = g.uniform(0, 0.9 * width, n), g.uniform(0, 0.9 * height, n)
            bw, bh = g.uniform(8, 0.2 * width, n), g.uniform(8, 0.2 * height, n)
            ann[i, f, :n] = np.stack([x1, y1, np.minimum(x1 + bw, width - 1), np.minimum(y1 + bh, height - 1),
                                      g.integers(0, 8, n)], 1)
    mirror = g.integers(0, 2, batch).astype(np.int32)
    return (torch.from_numpy(np.ascontiguousarray(frames)), torch.from_numpy(ann), torch.from_numpy(counts),
            torch.from_numpy(mirror))
