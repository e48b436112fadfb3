"""Test infrastructure of the per-pixel side maps (adc_match_outputs*): what the confidence maps must hold, the outlier
map in the form of the reference's mismatch / occlusion lists, and the demo's 8-bit rendering of a map
(adc_render_disparity)."""
from __future__ import annotations

import numpy as np


def confidence(vol_hwd: np.ndarray):
    """(MIN_COST, PEAK_RATIO), float32 [H][W], of an f32 [H][W][D] volume, by the header's definitions: d1 = the first
    index of the minimum, c1 = C(d1), c2 = min C(d) over |d - d1| >= 2, ratio = c1 / c2 rounded to nearest in f32, and 1
    where no such d exists or c2 == 0."""
    v = np.asarray(vol_hwd, np.float32)
    H, W, D = v.shape
    c1 = np.empty((H, W), np.float32)
    ratio = np.empty((H, W), np.float32)
    idx = np.arange(D, dtype=np.int32)
    for y0 in range(0, H, 32):                          # blocks of rows keep the temporaries small on large volumes
        b = np.ascontiguousarray(v[y0:y0 + 32])
        d1 = np.argmin(b, axis=-1).astype(np.int32)     # numpy's argmin takes the first minimum
        m = np.take_along_axis(b, d1[..., None], -1)[..., 0]
        far = np.abs(idx - d1[..., None]) >= 2
        c2 = np.where(far, b, np.float32(np.inf)).min(axis=-1)
        has = far.any(axis=-1) & (c2 != 0)
        c1[y0:y0 + 32] = m
        ratio[y0:y0 + 32] = np.where(has, m / np.where(has, c2, np.float32(1)), np.float32(1))
    return c1, ratio


def confidence_loop(vol_hwd: np.ndarray):
    """The same definitions as a plain per-pixel Python loop (the check on confidence())."""
    v = np.asarray(vol_hwd, np.float32)
    H, W, D = v.shape
    c1s = np.empty((H, W), np.float32)
    rs = np.empty((H, W), np.float32)
    for y in range(H):
        for x in range(W):
            col = [np.float32(c) for c in v[y, x]]
            d1 = 0
            for d in range(1, D):
                if col[d] < col[d1]:
                    d1 = d
            c1 = col[d1]
            far = [col[d] for d in range(D) if abs(d - d1) >= 2]
            c2 = min(far) if far else None
            c1s[y, x] = c1
            rs[y, x] = np.float32(1.0) if c2 is None or c2 == 0 else np.float32(c1) / np.float32(c2)
    return c1s, rs


def outlier_lists(label: np.ndarray):
    """The mismatch and occlusion lists of an outlier map: int32 [n][2] (x, y) in raster order, as the reference builds
    mismatches_ / occlusions_ and the MISMATCHES / OCCLUSIONS debug taps return them."""
    out = []
    for want in (1, 2):
        ys, xs = np.nonzero(np.asarray(label) == want)
        out.append(np.ascontiguousarray(np.stack([xs, ys], 1).astype(np.int32).reshape(-1, 2)))
    return out


def gray8(disp: np.ndarray, width: int):
    """ShowDisparityMap / SaveDisparityMap (main.cpp:147-170, 180-201) in float32."""
    d = np.abs(disp.astype(np.float32))
    valid = ~np.isinf(d)                                   # disp != Invalid_Float
    mn = np.float32(min(np.float32(width), d[valid].min())) if valid.any() else np.float32(width)
    mx = np.float32(max(np.float32(-width), d[valid].max())) if valid.any() else np.float32(-width)
    out = np.zeros(d.shape, np.uint8)
    with np.errstate(invalid="ignore", divide="ignore"):
        v = (d - mn) / np.float32(mx - mn) * np.float32(255)
    ok = valid & np.isfinite(v)
    out[ok] = v[ok].astype(np.uint8)                       # static_cast<uchar>: truncation
    return out, float(mn), float(mx)
