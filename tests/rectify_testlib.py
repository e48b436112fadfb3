"""numpy restatement of the rectified entries' resampling (include/adcensus_b200.h, "rectification on the way in"):
cv::remap(src, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) for float (CV_32FC1 x / y) and fixed (CV_16SC2 +
CV_16UC1) maps, plus map builders for tests that need no OpenCV.

Every map reduces to one fixed form per output pixel: the integer corner (x0, y0) and the 5-bit fractions (ax, ay).
Float maps: X = round_half_even(x * 32) saturated to int32, INT_MIN for NaN and anything outside int32 (x86's
conversion), x0 = sat_int16(X >> 5), ax = X & 31.  Fixed maps: (x0, y0) = map1, a = map2 & 1023, ax = a & 31,
ay = a >> 5.  out = (sum of w * s + 512) >> 10 over the four neighbours, w = (dx ? ax : 32 - ax) * (dy ? ay : 32 - ay),
s = 0 outside the frame.
"""
from __future__ import annotations

import numpy as np

INT_MIN = -(1 << 31)


def coord_x32(v) -> np.ndarray:
    """cvRound(v * 32) on x86 for float32 map values, as int64."""
    v = np.asarray(v, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        t = np.rint(v * np.float32(32)).astype(np.float64)
    ok = np.isfinite(t) & (t >= INT_MIN) & (t <= (1 << 31) - 1)
    return np.where(ok, np.nan_to_num(t), INT_MIN).astype(np.int64)


def sat16(v) -> np.ndarray:
    return np.clip(v, -32768, 32767)


def fixed_from_f32(mx, my):
    """(x0, y0, a) of float maps, a = ax | ay << 5."""
    X, Y = coord_x32(mx), coord_x32(my)
    return sat16(X >> 5), sat16(Y >> 5), (X & 31) | (Y & 31) << 5


def fixed_from_cv(m1, m2):
    """(x0, y0, a) of CV_16SC2 + CV_16UC1 maps (the high bits of m2 are ignored)."""
    m1 = np.asarray(m1, np.int16).astype(np.int64)
    return m1[..., 0], m1[..., 1], np.asarray(m2).astype(np.int64) & 1023


def convert_maps(mx, my):
    """cv2.convertMaps(mx, my, CV_16SC2) restated: (int16 [H][W][2], uint16 [H][W])."""
    x0, y0, a = fixed_from_f32(mx, my)
    return np.stack([x0, y0], axis=-1).astype(np.int16), a.astype(np.uint16)


def blend(src, x0, y0, a) -> np.ndarray:
    """The resampled image: src [h][w] or [h][w][c] u8, the fixed form over the output [H][W]."""
    src = np.asarray(src, np.uint8)
    flat = src.ndim == 2
    s3 = src[:, :, None] if flat else src
    h, w = s3.shape[:2]
    ax, ay = a & 31, a >> 5
    acc = np.full(np.shape(a) + (s3.shape[2],), 512, np.int64)
    for dy in (0, 1):
        for dx in (0, 1):
            wt = (ax if dx else 32 - ax) * (ay if dy else 32 - ay)
            xx, yy = x0 + dx, y0 + dy
            ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            v = s3[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.int64)
            acc += np.where(ok[..., None], v, 0) * wt[..., None]
    out = (acc >> 10).astype(np.uint8)
    return out[:, :, 0] if flat else out


def remap(src, map1, map2) -> np.ndarray:
    """cv2.remap(src, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) for float32 x / y maps or int16 [H][W][2] +
    uint16 maps."""
    if np.asarray(map1).dtype == np.float32:
        return blend(src, *fixed_from_f32(map1, map2))
    return blend(src, *fixed_from_cv(map1, map2))


def identity_maps(W, H, fixed=False):
    """Maps that send output pixel (x, y) to source pixel (x, y)."""
    mx, my = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32))
    return convert_maps(mx, my) if fixed else (mx, my)


def warp_maps(W, H, src_w, src_h, seed, fixed=False, specials=True):
    """A smooth made-up rectification (scale to the source, a small rotation and radial term) from a W x H output into
    a src_w x src_h frame: part of the border falls outside the frame.  specials: a few NaN / inf / huge coordinates,
    exact ties at odd multiples of 1/64 and (fixed) junk in the high bits of map2."""
    rng = np.random.default_rng(seed)
    u, v = np.meshgrid((np.arange(W) + 0.5) / W - 0.5, (np.arange(H) + 0.5) / H - 0.5)
    th = rng.uniform(-0.04, 0.04)
    k = rng.uniform(-0.12, 0.12)
    r2 = u * u + v * v
    uu = (np.cos(th) * u - np.sin(th) * v) * (1 + k * r2) * 1.06
    vv = (np.sin(th) * u + np.cos(th) * v) * (1 + k * r2) * 1.06
    mx = ((uu + 0.5) * src_w - 0.5 + rng.uniform(-0.3, 0.3)).astype(np.float32)
    my = ((vv + 0.5) * src_h - 0.5 + rng.uniform(-0.3, 0.3)).astype(np.float32)
    if specials:
        t = rng.random((H, W)) < 0.05
        mx[t] = np.round(mx[t] * 32) / np.float32(32) + np.float32(1 / 64)
        sp = rng.random((H, W)) < 0.01
        mx[sp] = rng.choice(np.array([np.nan, np.inf, -np.inf, 1e9, -1e9, 70000.0, -0.0], np.float32), sp.sum())
        sp = rng.random((H, W)) < 0.005
        my[sp] = rng.choice(np.array([np.nan, -np.inf, 3e9, -1.5], np.float32), sp.sum())
    if not fixed:
        return mx, my
    m1, m2 = convert_maps(mx, my)
    if specials:
        m2 = m2 | (rng.integers(0, 64, (H, W)).astype(np.uint16) << 10)
    return m1, m2


def cone_rig(cv2, sw, sh, W, H, t, baseline):
    """initUndistortRectifyMap maps (map type t) of one view of a made-up rig: a camera of sw x sh with some
    distortion, rotated a little (baseline +1 / -1 picks the view), rectified into W x H."""
    K = np.array([[0.9 * sw, 0, sw / 2 - 3.3], [0, 0.9 * sw, sh / 2 + 2.1], [0, 0, 1]], np.float64)
    dist = np.array([-0.12, 0.05, 0.0008, -0.0006, -0.004])
    R1, _ = cv2.Rodrigues(np.array([0.004, -0.011 * baseline, 0.002]))
    P = np.array([[0.95 * W, 0, W / 2, 0], [0, 0.95 * W, H / 2, 0], [0, 0, 1, 0]], np.float64)
    return cv2.initUndistortRectifyMap(K, dist, R1, P, (W, H), t)
