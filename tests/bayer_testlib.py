"""numpy restatement of the Bayer formats' demosaic (include/adcensus_b200.h, "Bayer mosaics"): what
cv::cvtColor(raw, COLOR_Bayer*2BGR) gives for 8-bit mosaics, bilinear, with or without IPP.

A pattern names the colours of the view's own top-left 2x2 block (GenICam's BayerRG8 = "rggb"), so the colour of pixel
(x, y) is PATTERNS[p][y & 1][x & 1].  Frames narrower or lower than 3 pixels are all zero.  Otherwise pixel (x, y)
takes the interior rule at (clamp(x, 1, W - 2), clamp(y, 1, H - 2)):
  - its own colour is the raw value;
  - at an R or B site, G = (N + S + W + E + 2) >> 2 and the other of R / B = (NW + NE + SW + SE + 2) >> 2;
  - at a G site, the colour of the horizontal neighbours = (W + E + 1) >> 1, that of the vertical ones = (N + S + 1) >> 1.
"""
from __future__ import annotations

import numpy as np

# pattern name -> colours of rows 0 and 1 of its 2x2 block
PATTERNS = {"bayer_rggb": ("RG", "GB"), "bayer_grbg": ("GR", "BG"), "bayer_bggr": ("BG", "GR"),
            "bayer_gbrg": ("GB", "RG")}
NAMES = list(PATTERNS)
CODE = {"bayer_rggb": 16, "bayer_grbg": 17, "bayer_bggr": 18, "bayer_gbrg": 19}
# OpenCV's conversion code for each pattern.  OpenCV's legacy names count from the second row's second and third
# pixels: COLOR_BayerBG2BGR is the RGGB sensor (= COLOR_BayerRGGB2BGR in OpenCV >= 4.x aliases).
CV_NAME = {"bayer_rggb": "COLOR_BayerBG2BGR", "bayer_grbg": "COLOR_BayerGB2BGR", "bayer_bggr": "COLOR_BayerRG2BGR",
           "bayer_gbrg": "COLOR_BayerGR2BGR"}
_BGR = {"B": 0, "G": 1, "R": 2}


def colour_at(pattern, y, x) -> str:
    return PATTERNS[pattern][y & 1][x & 1]


def demosaic(raw, pattern) -> np.ndarray:
    """BGR u8 [H][W][3] of the u8 mosaic raw [H][W] (any strides)."""
    raw = np.asarray(raw, np.uint8)
    H, W = raw.shape
    out = np.zeros((H, W, 3), np.uint8)
    if H < 3 or W < 3:
        return out
    r = raw.astype(np.int32)
    c = r[1:-1, 1:-1]
    n, s, w, e = r[:-2, 1:-1], r[2:, 1:-1], r[1:-1, :-2], r[1:-1, 2:]
    cross = (n + s + w + e + 2) >> 2
    diag = (r[:-2, :-2] + r[:-2, 2:] + r[2:, :-2] + r[2:, 2:] + 2) >> 2
    hor, ver = (w + e + 1) >> 1, (n + s + 1) >> 1
    inner = np.zeros((H - 2, W - 2, 3), np.int32)
    for py in (0, 1):           # parity of the frame row y = 1 + i
        for px in (0, 1):
            sl = (slice((py - 1) & 1, None, 2), slice((px - 1) & 1, None, 2))
            own = colour_at(pattern, py, px)
            inner[sl + (_BGR[own],)] = c[sl]
            if own == "G":
                inner[sl + (_BGR[colour_at(pattern, py, px + 1)],)] = hor[sl]
                inner[sl + (_BGR[colour_at(pattern, py + 1, px)],)] = ver[sl]
            else:
                inner[sl + (1,)] = cross[sl]
                inner[sl + (_BGR["B" if own == "R" else "R"],)] = diag[sl]
    out[:] = np.pad(inner, ((1, 1), (1, 1), (0, 0)), mode="edge")
    return out


def mosaic(bgr, pattern) -> np.ndarray:
    """The u8 [H][W] mosaic that samples BGR image bgr [H][W][3] through the pattern."""
    bgr = np.asarray(bgr, np.uint8)
    H, W = bgr.shape[:2]
    out = np.empty((H, W), np.uint8)
    for py in (0, 1):
        for px in (0, 1):
            out[py::2, px::2] = bgr[py::2, px::2, _BGR[colour_at(pattern, py, px)]]
    return out


def cv_demosaic(cv2, raw, pattern) -> np.ndarray:
    """cv2.cvtColor(raw, <the pattern's code>): the live OpenCV call the restatement stands for."""
    return cv2.cvtColor(np.asarray(raw, np.uint8), getattr(cv2, CV_NAME[pattern]))
