"""numpy restatement of cv2.cvtColor(frame, COLOR_YUV2BGR_{NV12, NV21, I420, YV12, YUY2, UYVY}): OpenCV's BT.601
limited-range fixed-point formula (modules/imgproc/src/color_yuv.simd.hpp, ITUR_BT_601_*), chroma replicated over its
2x2 (4:2:0) or 2x1 (4:2:2) pixel group.

    bgr = yuv_to_bgr("nv12", frame)      # frame: uint8 [h * 3 // 2, w] (4:2:0) or [h, w, 2] (4:2:2), as cv2 takes it
"""
import numpy as np

FORMATS = ("nv12", "nv21", "i420", "yv12", "yuyv", "uyvy")
CV2_CODES = {"nv12": "COLOR_YUV2BGR_NV12", "nv21": "COLOR_YUV2BGR_NV21", "i420": "COLOR_YUV2BGR_I420",
             "yv12": "COLOR_YUV2BGR_YV12", "yuyv": "COLOR_YUV2BGR_YUY2", "uyvy": "COLOR_YUV2BGR_UYVY"}
CY, CUB, CUG, CVG, CVR, SHIFT = 1220542, 2116026, -409993, -852492, 1673527, 20


def is420(fmt):
    return fmt in ("nv12", "nv21", "i420", "yv12")


def frame_shape(fmt, h, w):
    """the uint8 array cv2 takes for an h x w frame of ``fmt``"""
    return (h * 3 // 2, w) if is420(fmt) else (h, w, 2)


def planes(fmt, frame):
    """-> Y [h, w], U and V [h, w] (each chroma sample replicated over its group), all int64"""
    f = np.asarray(frame, np.uint8)
    if is420(fmt):
        h, w = f.shape[0] * 2 // 3, f.shape[1]
        y, rest = f[:h], f[h:].reshape(-1)
        if fmt in ("nv12", "nv21"):
            c = rest.reshape(h // 2, w // 2, 2)
            u, v = (c[..., 0], c[..., 1]) if fmt == "nv12" else (c[..., 1], c[..., 0])
        else:
            q = (h // 2) * (w // 2)
            a, b = rest[:q].reshape(h // 2, w // 2), rest[q:].reshape(h // 2, w // 2)
            u, v = (a, b) if fmt == "i420" else (b, a)
        u, v = (np.repeat(np.repeat(c, 2, 0), 2, 1) for c in (u, v))
    else:
        g = f.reshape(f.shape[0], f.shape[1] // 2, 4)
        oy, ou = (0, 1) if fmt == "yuyv" else (1, 0)
        y = np.stack([g[..., oy], g[..., oy + 2]], -1).reshape(f.shape[0], f.shape[1])
        u, v = (np.repeat(g[..., k], 2, 1) for k in (ou, ou + 2))
    return y.astype(np.int64), u.astype(np.int64), v.astype(np.int64)


def yuv_to_bgr(fmt, frame):
    """uint8 [h, w, 3] BGR, what cv2.cvtColor(frame, CV2_CODES[fmt]) returns"""
    y, u, v = planes(fmt, frame)
    y = np.maximum(y - 16, 0) * CY
    u, v = u - 128, v - 128
    rnd = 1 << (SHIFT - 1)
    b = (y + CUB * u + rnd) >> SHIFT
    g = (y + CVG * v + CUG * u + rnd) >> SHIFT
    r = (y + CVR * v + rnd) >> SHIFT
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)
