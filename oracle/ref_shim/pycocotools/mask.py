import numpy as np


def iou(dt, gt, iscrowd):
    """maskApi.c bbIou for [m, 4] / [n, 4] ltwh boxes in fp64 -> [m, n]; crowd gts divide by the dt area"""
    D = np.asarray(dt, np.float64).reshape(-1, 4)[:, None, :]
    G = np.asarray(gt, np.float64).reshape(-1, 4)[None, :, :]
    crowd = np.asarray(iscrowd, bool).reshape(1, -1)
    da, ga = D[..., 2] * D[..., 3], G[..., 2] * G[..., 3]
    w = np.fmin(D[..., 2] + D[..., 0], G[..., 2] + G[..., 0]) - np.fmax(D[..., 0], G[..., 0])
    h = np.fmin(D[..., 3] + D[..., 1], G[..., 3] + G[..., 1]) - np.fmax(D[..., 1], G[..., 1])
    i = w * h
    u = np.where(crowd, da, da + ga - i)
    with np.errstate(divide="ignore", invalid="ignore"):
        o = i / u
    return np.where((w <= 0) | (h <= 0), 0.0, o)


def _absent(*args, **kwargs):
    raise NotImplementedError("pycocotools stand-in: only mask.iou is provided")


encode = decode = area = toBbox = frPyObjects = merge = _absent
