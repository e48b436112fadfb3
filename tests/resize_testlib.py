"""Resizing on the way in, restated in numpy: cv::resize's INTER_AREA at integer factors and INTER_LINEAR_EXACT on 8-bit
images of any channel count (the rules in include/adcensus_b200.h), and one view of every ADC_IMG_* format (a random
raw frame in the shape the host entries take, its format conversion to packed BGR, its bytes laid into a pitched
buffer) through the format restatements of images_testlib, bayer_testlib, yuv_video_testlib and rawdepth_testlib.
"""
import numpy as np

import bayer_testlib as B
import images_testlib as IT
import rawdepth_testlib as RD
import yuv_video_testlib as V

AREA, LINEAR_EXACT = 16, 17
CODE = {**IT.CODE, **B.CODE, **V.ALL, **RD.CODE}   # every format name -> its ADC_IMG_* code (without flags)
ENC = V.ENC


def area(src, kx, ky) -> np.ndarray:
    """cv2.resize(src, (W, H), interpolation=INTER_AREA) for src of shape [ky*H][kx*W][...] with both factors exact
    (area_exact): per channel the block sum s, (s + 2) >> 2 for 2 x 2, otherwise round_half_even(float32(s) *
    float32(1 / n)) saturated to 255."""
    src = np.asarray(src)
    H, W = src.shape[0] // ky, src.shape[1] // kx
    assert src.shape[:2] == (H * ky, W * kx)
    rest = src.shape[2:]
    s = src.astype(np.int64).reshape((H, ky, W, kx) + rest).sum((1, 3))
    if (kx, ky) == (2, 2):
        return ((s + 2) >> 2).astype(np.uint8)
    v = np.rint(s.astype(np.float32) * np.float32(1.0 / np.float32(kx * ky))).astype(np.int64)
    return np.minimum(v, 255).astype(np.uint8)


def area_exact(k, n_dst=1) -> bool:
    """Whether cv::resize takes its integer-block INTER_AREA path on an axis of n_dst outputs downscaled by k: its scale
    1 / (n_dst / (k * n_dst)), in double, is k exactly.  (n_dst / (k * n_dst) rounds the same real number as 1 / k, so
    the answer does not depend on n_dst.)  The engine rejects the other factors."""
    return 1.0 / (n_dst / (k * n_dst)) == k


def taps(n_src, n_dst):
    """(i0, i1, c1) per destination index of one axis of INTER_LINEAR_EXACT: f = (d + 0.5) * scale - 0.5 in float64
    (two roundings, no fused multiply-add) with scale = 1 / (n_dst / n_src) (two divisions, as OpenCV inverts its
    inv_scale; n_src / n_dst differs in the last bit for some sizes, e.g. 49 -> 256), i = floor(f),
    c1 = round_half_even((f - i) * 256), clamped into the source with c1 = 0 at both borders."""
    f = (np.arange(n_dst, dtype=np.float64) + 0.5) * (1.0 / (n_dst / n_src)) - 0.5
    i = np.floor(f)
    c1 = np.rint((f - i) * 256).astype(np.int64)
    i = i.astype(np.int64)
    c1[i < 0] = 0
    i[i < 0] = 0
    hi = i >= n_src - 1
    i[hi], c1[hi] = n_src - 1, 0
    return i, np.minimum(i + 1, n_src - 1), c1


def linear_exact(src, W, H) -> np.ndarray:
    """cv2.resize(src, (W, H), interpolation=INTER_LINEAR_EXACT) of an 8-bit [h][w][...] image."""
    src = np.asarray(src).astype(np.int64)
    extra = (None,) * (src.ndim - 2)
    x0, x1, cx = taps(src.shape[1], W)
    y0, y1, cy = taps(src.shape[0], H)
    cx, cy = cx[(None, slice(None)) + extra], cy[(slice(None), None) + extra]
    rows0, rows1 = src[y0], src[y1]
    h0 = rows0[:, x0] * (256 - cx) + rows0[:, x1] * cx
    h1 = rows1[:, x0] * (256 - cx) + rows1[:, x1] * cx
    return ((h0 * (256 - cy) + h1 * cy + (1 << 15)) >> 16).astype(np.uint8)


def resize(bgr, W, H, interp) -> np.ndarray:
    """The resize of one converted frame to W x H under AREA or LINEAR_EXACT."""
    if interp == AREA:
        return area(bgr, bgr.shape[1] // W, bgr.shape[0] // H)
    return linear_exact(bgr, W, H)


# ---- one raw view of any format ---------------------------------------------------------------------------------------
def random_frame(rng, fmt, W, H) -> np.ndarray:
    """A random raw view of `fmt` (a name of CODE) in the shape the host entries take."""
    if fmt in V.ALL:
        return V.random_frame(rng, fmt, W, H)
    if fmt in RD.CODE:
        return RD.random_frame(rng, fmt, W, H)
    if fmt in B.CODE or fmt == "gray":
        return rng.integers(0, 256, (H, W), dtype=np.uint8)
    if fmt == "rgb_planar":
        return rng.integers(0, 256, (3, H, W), dtype=np.uint8)
    return rng.integers(0, 256, (H, W, IT.BPP[fmt]), dtype=np.uint8)


def decode(frame, fmt, W, H, enc=0) -> np.ndarray:
    """The packed BGR u8 [H][W][3] of one raw view: its format's conversion (encoding flags `enc` for YUV)."""
    if fmt in V.ALL:
        return V.decode(frame, fmt, W, H, enc)
    if fmt in RD.CODE:
        return RD.decode(frame, fmt, W, H)
    if fmt in B.CODE:
        return B.demosaic(frame, fmt)
    if fmt == "gray":
        return IT.gray_to_bgr(frame)
    if fmt == "rgb_planar":
        return np.stack([frame[2], frame[1], frame[0]], -1)
    return np.ascontiguousarray(frame[..., 2::-1] if fmt in ("rgb", "rgba") else frame[..., :3])


def tight_row(fmt, W) -> int:
    """The tight (and least) row pitch in bytes of a W pixel wide view."""
    if fmt in V.ALL:
        return V.tight_row(fmt, W)
    if fmt in RD.CODE:
        return RD.tight_row(fmt, W)
    return W * (IT.BPP[fmt] if fmt in IT.BPP else 1)


def planes(fmt) -> bool:
    """Whether a view of `fmt` has a plane pitch."""
    return fmt == "rgb_planar" or (fmt in V.ALL and V.is420(fmt))


def footprint(fmt, H, row_pitch, plane_pitch=0) -> int:
    if fmt in V.ALL:
        return V.footprint(fmt, H, row_pitch, plane_pitch)
    return IT.footprint(fmt, H, row_pitch, plane_pitch) if fmt in IT.CODE else H * row_pitch


def write_view(buf, frame, fmt, W, H, row_pitch, plane_pitch=0, off=0):
    """Lays the view `frame` into the flat u8 buffer `buf` at byte `off` with the given pitches, writing only the
    view's own bytes."""
    if fmt in V.ALL:
        return V.write_view(buf, frame, fmt, W, H, row_pitch, plane_pitch, off)
    if fmt in RD.CODE:
        return RD.write_view(buf, frame, fmt, W, H, row_pitch, off)
    if fmt in IT.CODE:
        return IT.write_view(buf, frame, fmt, row_pitch, plane_pitch, off)
    rows = np.ascontiguousarray(frame).reshape(H, -1)
    for y in range(H):
        buf[off + y * row_pitch:off + y * row_pitch + W] = rows[y]
    return buf
