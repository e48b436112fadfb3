"""Numpy restatement of the previews (adc_preview*, include/adcensus_b200_preview.h): cv::normalize's scale and shift
over the finite pixels, convertTo(CV_8U) as one fused multiply-add rounded half to even, the colormap tables of
adcensus_b200/csrc/colormap_lut.h, cv::resize INTER_NEAREST's index rule and cv::cvtColor's BGR -> gray / BGRA / RGBA /
I420 / YV12 / NV12 / NV21 integer rules.  Needs no OpenCV; tests/test_preview.py pins every step to live cv2 (and to
tests/golden/golden_preview_cases.npz where cv2 is absent).
"""
from __future__ import annotations

import functools
import re
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
LUT_HEADER = ROOT / "adcensus_b200" / "csrc" / "colormap_lut.h"
DBL_EPSILON = float(np.finfo(np.float64).eps)
FORMATS = ("bgr", "bgra", "rgba", "gray", "nv12", "nv21", "i420", "yv12")
YUV420 = ("nv12", "nv21", "i420", "yv12")


@functools.cache
def header_luts() -> np.ndarray:
    """uint8 [22][256][3] (B, G, R): the tables of colormap_lut.h, as the kernel sees them."""
    body = LUT_HEADER.read_text().split("= {", 1)[1]
    vals = [int(v) for v in re.findall(r"\b\d+\b", re.sub(r"//[^\n]*", "", body))]
    a = np.array(vals, np.uint8)
    assert a.size == 22 * 256 * 3, a.size
    return a.reshape(22, 256, 3)


def colour_table(colormap: int) -> np.ndarray:
    """uint8 [256][3] (B, G, R) of g for a colormap value (-1 = gray)."""
    if colormap < 0:
        return np.repeat(np.arange(256, dtype=np.uint8)[:, None], 3, 1)
    return header_luts()[colormap]


def minmax_scale_shift(m: np.ndarray):
    """cv::normalize(NORM_MINMAX, 0, 255, mask = isfinite(m))'s (scale, shift) in double; (0, 0) without a valid pixel
    (minMaxIdx over an empty mask gives 0 and 0)."""
    v = m[np.isfinite(m)]
    smin, smax = (float(v.min()), float(v.max())) if v.size else (0.0, 0.0)
    scale = 255.0 * (1.0 / (smax - smin) if smax - smin > DBL_EPSILON else 0.0)
    return scale, 0.0 - smin * scale


def fmaf(v: np.ndarray, a, b) -> np.ndarray:
    """float32 fma(v, a, b) rounded once: the exact product in double, the sum rounded to odd (TwoSum), then to float."""
    p = v.astype(np.float64) * np.float64(np.float32(a))
    c = np.float64(np.float32(b))
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        odd = (e != 0) & np.isfinite(s) & ((s.view(np.int64) & 1) == 0)
        s = np.where(odd, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(np.float32)


def mul_add(v: np.ndarray, a, b) -> np.ndarray:
    """The unfused form, m * scale rounded, then + shift rounded (an SSE-baseline build of OpenCV)."""
    with np.errstate(invalid="ignore", over="ignore"):
        return (v.astype(np.float32) * np.float32(a)).astype(np.float32) + np.float32(b)


def sat_u8(t: np.ndarray) -> np.ndarray:
    """round_half_even(t) saturated to 0..255; 0 where t is outside int32 or NaN (x86's cvtps2dq gives INT_MIN)."""
    with np.errstate(invalid="ignore"):
        inside = t < np.float32(2.0 ** 31)
        r = np.clip(np.rint(np.where(inside, t, 0)), 0, 255)
    return np.where(inside, r, 0).astype(np.uint8)


def convert_u8(m: np.ndarray, scale, shift, fused=True) -> np.ndarray:
    """convertTo(CV_8U, scale, shift) of a float32 map: sat_u8(fmaf(m, (float)scale, (float)shift))."""
    with np.errstate(over="ignore"):
        a, b = np.float32(scale), np.float32(shift)
    return sat_u8((fmaf if fused else mul_add)(np.asarray(m, np.float32), a, b))


def nearest(n_src: int, n_dst: int) -> np.ndarray:
    """cv::resize INTER_NEAREST's source index of every destination index: min(floor(d * (1.0 / (n_dst / n_src))),
    n_src - 1), in double."""
    inv = 1.0 / (n_dst / n_src)
    return np.minimum(np.floor(np.arange(n_dst) * inv).astype(np.int64), n_src - 1)


def gray(bgr: np.ndarray) -> np.ndarray:
    b, g, r = (bgr[..., i].astype(np.int64) for i in range(3))
    return ((9798 * r + 19235 * g + 3735 * b + (1 << 14)) >> 15).astype(np.uint8)


def yuv(bgr: np.ndarray):
    """(Y, U, V) of every pixel by COLOR_BGR2YUV_I420's integer rule (BT.601, limited range)."""
    b, g, r = (bgr[..., i].astype(np.int64) for i in range(3))
    h = 1 << 19
    y = (269484 * r + 528482 * g + 102760 * b + h + (16 << 20)) >> 20
    u = (-155188 * r - 305135 * g + 460324 * b + h + (128 << 20)) >> 20
    v = (460324 * r - 385875 * g - 74448 * b + h + (128 << 20)) >> 20
    return tuple(np.clip(c, 0, 255).astype(np.uint8) for c in (y, u, v))


def convert(bgr: np.ndarray, fmt: str) -> np.ndarray:
    """cv2.cvtColor(bgr, COLOR_BGR2<fmt>) as a tight frame; NV12 / NV21 are I420 with U and V interleaved."""
    H, W, _ = bgr.shape
    if fmt == "bgr":
        return bgr.copy()
    if fmt in ("bgra", "rgba"):
        px = bgr if fmt == "bgra" else bgr[..., ::-1]
        return np.concatenate([px, np.full((H, W, 1), 255, np.uint8)], -1)
    if fmt == "gray":
        return gray(bgr)
    assert fmt in YUV420 and H % 2 == 0 and W % 2 == 0, (fmt, H, W)
    y, u, v = yuv(bgr)
    u, v = u[0::2, 0::2], v[0::2, 0::2]
    if fmt in ("i420", "yv12"):
        first, second = (u, v) if fmt == "i420" else (v, u)
        chroma = np.concatenate([first.reshape(-1), second.reshape(-1)]).reshape(H // 2, W)
    else:
        pair = np.stack([u, v] if fmt == "nv12" else [v, u], -1)
        chroma = pair.reshape(H // 2, W)
    return np.concatenate([y, chroma])


def g_map(m: np.ndarray, value_range=None) -> np.ndarray:
    """Step 3 over the whole map (invalid pixels included, they are replaced later)."""
    scale, shift = minmax_scale_shift(m) if value_range is None else value_range
    with np.errstate(invalid="ignore"):
        return convert_u8(np.where(np.isfinite(m), m, 0).astype(np.float32), scale, shift)


def preview(m: np.ndarray, colormap: int = 20, value_range=None, size=None, fmt: str = "bgr",
            invalid=(0, 0, 0)) -> np.ndarray:
    """The preview frame of one map (tight): steps 1 to 6 of the header."""
    m = np.asarray(m, np.float32)
    H, W = m.shape
    bgr = colour_table(colormap)[g_map(m, value_range)]
    bgr[~np.isfinite(m)] = np.array(invalid, np.uint8)
    w, h = (W, H) if size is None else size
    bgr = bgr[nearest(H, h)][:, nearest(W, w)]
    return convert(bgr, fmt)
