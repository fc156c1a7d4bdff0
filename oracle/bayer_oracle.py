"""numpy restatement of cv2.cvtColor(raw, COLOR_Bayer{RGGB, BGGR, GBRG, GRBG}2BGR[_EA]): the bilinear and the edge-aware
demosaicing of 8-bit Bayer mosaics, as OpenCV computes them (modules/imgproc/src/demosaicing.cpp).

    bgr = bayer_to_bgr("rggb", "bilinear", raw)      # raw: uint8 [h, w], top-left 2x2 = R G / G B

Both algorithms compute the pixels off the frame's border, rows 1..h-2 and columns 1..w-2, from the 3x3 neighbourhood:
  * a pixel's own colour is its raw value;
  * at a green pixel, the colour of its left and right neighbours is their mean (a + b + 1) >> 1, and the colour of its
    upper and lower neighbours theirs;
  * at a red or blue pixel, the other of the two is the mean of the four diagonal neighbours (a + b + c + d + 2) >> 2,
    and green is
      bilinear:   the mean of the four edge neighbours, (l + r + u + d + 2) >> 2;
      edge-aware: the mean of the vertical pair, (u + d + 1) >> 1, where |l - r| > |u - d|, else of the horizontal pair.
The border is a copy: column 0 of column 1 and column w-1 of column w-2, then row 0 of row 1 and row h-1 of row h-2.
A frame of fewer than three rows or columns is all zeros.

This is cv2 on a C-contiguous frame, whatever the bytes around it; that is the layout the detector stages.  (cv2's _EA
on a strided view -- a crop of a wider image -- reads its second and later rows at the wrong pitch.)
"""
import numpy as np

PATTERNS = ("rggb", "bggr", "gbrg", "grbg")
ALGOS = ("bilinear", "ea")
# the colour order of the top-left 2x2 -> cv2's code: COLOR_BayerRGGB2BGR is COLOR_BayerBG2BGR, and so on
CV2_CODES = {("rggb", "bilinear"): "COLOR_BayerRGGB2BGR", ("bggr", "bilinear"): "COLOR_BayerBGGR2BGR",
             ("gbrg", "bilinear"): "COLOR_BayerGBRG2BGR", ("grbg", "bilinear"): "COLOR_BayerGRBG2BGR",
             ("rggb", "ea"): "COLOR_BayerRGGB2BGR_EA", ("bggr", "ea"): "COLOR_BayerBGGR2BGR_EA",
             ("gbrg", "ea"): "COLOR_BayerGBRG2BGR_EA", ("grbg", "ea"): "COLOR_BayerGRBG2BGR_EA"}
B, G, R = 0, 1, 2


def colours(pattern, h, w):
    """int [h, w]: the BGR channel index (B, G or R) each mosaic site samples"""
    c = np.array([{"r": R, "g": G, "b": B}[ch] for ch in pattern]).reshape(2, 2)
    return np.tile(c, ((h + 1) // 2, (w + 1) // 2))[:h, :w]


def bayer_to_bgr(pattern, algo, raw):
    """uint8 [h, w, 3] BGR, what cv2.cvtColor(raw, getattr(cv2, CV2_CODES[pattern, algo])) returns"""
    f = np.asarray(raw, np.uint8)
    h, w = f.shape
    out = np.zeros((h, w, 3), np.uint8)
    if h < 3 or w < 3:
        return out
    v = f.astype(np.int32)
    col = colours(pattern, h, w)
    c, right = col[1:-1, 1:-1], col[1:-1, 2:]                 # each site's colour and its right neighbour's
    ctr = v[1:-1, 1:-1]
    up, dn, lf, rt = v[:-2, 1:-1], v[2:, 1:-1], v[1:-1, :-2], v[1:-1, 2:]
    diag = (v[:-2, :-2] + v[:-2, 2:] + v[2:, :-2] + v[2:, 2:] + 2) >> 2
    hor, ver = (lf + rt + 1) >> 1, (up + dn + 1) >> 1
    if algo == "bilinear":
        cross = (up + dn + lf + rt + 2) >> 2
    elif algo == "ea":
        cross = np.where(np.abs(lf - rt) > np.abs(up - dn), ver, hor)
    else:
        raise ValueError(f"unknown demosaicing {algo!r} (one of {', '.join(ALGOS)})")
    green = c == G
    inner = np.empty((h - 2, w - 2, 3), np.int32)
    for ch in (B, R):
        inner[..., ch] = np.where(green, np.where(right == ch, hor, ver), np.where(c == ch, ctr, diag))
    inner[..., G] = np.where(green, ctr, cross)
    out[1:-1, 1:-1] = inner
    out[1:-1, 0], out[1:-1, -1] = out[1:-1, 1], out[1:-1, -2]
    out[0], out[-1] = out[1], out[-2]
    return out
