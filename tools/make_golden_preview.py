#!/usr/bin/env python
"""Writes tests/golden/golden_preview_cases.npz: what OpenCV itself gives for the previews, for machines without OpenCV.

Per case <name>: the map ("m"), the parameters ("p": colormap, MINMAX 0 / NORM_INF 1, alpha, width, height, format
index into preview_testlib.FORMATS, invalid B, G, R) and OpenCV's frame ("out"):
  cv2.normalize(m, zeros, 0, 255, NORM_MINMAX, CV_8U, mask = isfinite(m))    (MINMAX)
  cv2.normalize(m, zeros, alpha, 0, NORM_INF, CV_8U, mask)                    (a fixed scale alpha / max|m|, shift 0)
  -> cv2.applyColorMap (or gray) -> invalid colour -> cv2.resize(INTER_NEAREST) -> cv2.cvtColor.
Also "luts": cv2.applyColorMap(arange(256), k) for k = 0..21, and "nearest/<n_src>_<n_dst>" index rows.

  python tools/make_golden_preview.py [output path]
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import preview_testlib as PV  # noqa: E402

OUT = ROOT / "tests" / "golden" / "golden_preview_cases.npz"
CONVERT = {"bgr": None, "bgra": "COLOR_BGR2BGRA", "rgba": "COLOR_BGR2RGBA", "gray": "COLOR_BGR2GRAY",
           "i420": "COLOR_BGR2YUV_I420", "yv12": "COLOR_BGR2YUV_YV12"}


def cv_g(m, mode=0, alpha=0.0):
    """OpenCV's 8-bit map: NORM_MINMAX (mode 0) or NORM_INF with alpha (mode 1), over the finite pixels."""
    import cv2
    mask = np.isfinite(m).astype(np.uint8)
    g = np.zeros(m.shape, np.uint8)
    if mode == 0:
        cv2.normalize(m, g, 0, 255, cv2.NORM_MINMAX, cv2.CV_8U, mask)
    else:
        cv2.normalize(m, g, alpha, 0, cv2.NORM_INF, cv2.CV_8U, mask)
    return g


def inf_scale(m, alpha):
    """NORM_INF's (scale, shift): alpha / max|m| over the finite pixels (0 when that is at most DBL_EPSILON), 0."""
    v = m[np.isfinite(m)]
    norm = float(np.abs(v).max()) if v.size else 0.0
    return (alpha / norm if norm > PV.DBL_EPSILON else 0.0), 0.0


def cv_preview(m, colormap, mode, alpha, size, fmt, invalid):
    """The whole preview through OpenCV's own calls."""
    import cv2
    g = cv_g(m, mode, alpha)
    bgr = cv2.cvtColor(g, cv2.COLOR_GRAY2BGR) if colormap < 0 else cv2.applyColorMap(g, colormap)
    bgr[~np.isfinite(m)] = invalid
    w, h = size
    if (w, h) != (m.shape[1], m.shape[0]):
        bgr = cv2.resize(bgr, (w, h), interpolation=cv2.INTER_NEAREST)
    if fmt in ("nv12", "nv21"):
        i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
        flat, q = i420.reshape(-1), h * w // 4
        u, v = flat[h * w:h * w + q], flat[h * w + q:]
        pair = np.stack([u, v] if fmt == "nv12" else [v, u], -1).reshape(h // 2, w)
        return np.concatenate([i420[:h], pair])
    return bgr if CONVERT[fmt] is None else cv2.cvtColor(bgr, getattr(cv2, CONVERT[fmt]))


def designed_maps(rng):
    """name -> float32 map: random with invalid pixels, constant, one valid, none valid, +-1e30, subnormals and
    negatives, a range at DBL_EPSILON, NaN depth."""
    H, W = 24, 34
    r = (rng.random((H, W)) * 200 - 40).astype(np.float32)
    r[rng.random((H, W)) < 0.2] = np.inf
    maps = {"random": r, "constant": np.full((H, W), 7.25, np.float32)}
    one = np.full((H, W), np.inf, np.float32)
    one[5, 9] = -3.5
    maps["one_valid"] = one
    maps["none_valid"] = np.full((H, W), np.inf, np.float32)
    big = r.copy()
    big[0, 0], big[1, 1] = np.float32(1e30), np.float32(-1e30)
    maps["huge"] = big
    sub = (rng.integers(1, 1 << 23, (H, W)).astype(np.uint32) | (rng.integers(0, 2, (H, W)).astype(np.uint32) << 31))
    maps["subnormal"] = sub.view(np.float32)
    neg = -np.abs(r)
    neg[3, 3] = -np.inf
    maps["negative"] = neg
    eps = np.full((H, W), 1.0, np.float32)
    eps[0, :5] = np.float32(1.0) + np.float32(2.0 ** -23)
    maps["eps_range"] = eps
    nan = r.copy()
    nan[rng.random((H, W)) < 0.3] = np.nan
    maps["nan_depth"] = nan
    return maps


def cases():
    rng = np.random.default_rng(23)
    out = {}
    maps = designed_maps(rng)
    for i, (name, m) in enumerate(sorted(maps.items())):
        H, W = m.shape
        for j, fmt in enumerate(PV.FORMATS):
            cm = [-1, 2, 20, 21, 13, 9, 0, 18][(i + j) % 8]
            size = [(W, H), (64, 40), (16, 10), (33, 17) if fmt not in PV.YUV420 else (34, 18)][(i + 2 * j) % 4]
            mode, alpha = (1, [-255.0, 1000.0, 255.0][j % 3]) if (i + j) % 5 == 4 else (0, 0.0)
            invalid = (int(rng.integers(0, 256)), int(rng.integers(0, 256)), int(rng.integers(0, 256)))
            out[f"{name}_{fmt}/m"] = m
            out[f"{name}_{fmt}/p"] = np.array([cm, mode, alpha, size[0], size[1], j, *invalid], np.float64)
            out[f"{name}_{fmt}/out"] = cv_preview(m, cm, mode, alpha, size, fmt, invalid)
    import cv2
    ramp = np.arange(256, dtype=np.uint8).reshape(256, 1)
    out["luts"] = np.stack([cv2.applyColorMap(ramp, k).reshape(256, 3) for k in range(22)])
    for n_src, n_dst in ((450, 1920), (375, 1080), (375, 17), (7, 512), (512, 7), (49, 256), (300, 299)):
        row = np.arange(n_src, dtype=np.int32).reshape(1, n_src)
        out[f"nearest/{n_src}_{n_dst}"] = cv2.resize(row, (n_dst, 1), interpolation=cv2.INTER_NEAREST)[0]
    return out


def main(path=OUT):
    np.savez_compressed(path, **cases())


if __name__ == "__main__":
    p = Path(sys.argv[1]) if len(sys.argv) > 1 else OUT
    main(p)
    print("wrote", p)
