"""numpy restatement of the YUV formats (include/adcensus_b200.h, "YUV video and camera frames"): what
cv::cvtColor(frame, COLOR_YUV2BGR_<F>) gives for NV12 / NV21 and packed 4:2:2 frames, and the geometry of a view.

Conversion (OpenCV's BT.601 limited-range fixed-point rule), per pixel from its own Y and its chroma sample's U, V:
  y' = max(0, Y - 16) * 1220542, u = U - 128, v = V - 128, h = 1 << 19
  R = sat_u8((y' + h + 1673527 v) >> 20), G = sat_u8((y' + h - 852492 v - 409993 u) >> 20), B = sat_u8((y' + h + 2116026 u) >> 20)
Pixel (x, y) takes the chroma sample (x >> 1, y >> 1) (NV12 / NV21) or (x >> 1, y) (4:2:2), relative to the view's own
(0, 0).  An odd-sized view is the crop of cvtColor on any even frame that holds it at its top-left.

Frames are numpy arrays in the shapes the Python host entries take:
  NV12 / NV21: [H + ceil(H/2)][2*ceil(W/2)] u8, the luma rows, then the interleaved chroma rows;
  4:2:2:       [H][2*ceil(W/2)][2] u8 (OpenCV's CV_8UC2), the macropixels' bytes in order.
"""
from __future__ import annotations

import numpy as np

CODE = {"nv12": 32, "nv21": 33, "yuyv": 34, "uyvy": 35, "yvyu": 36}
NAMES = list(CODE)
CV_NAME = {"nv12": "COLOR_YUV2BGR_NV12", "nv21": "COLOR_YUV2BGR_NV21", "yuyv": "COLOR_YUV2BGR_YUYV",
           "uyvy": "COLOR_YUV2BGR_UYVY", "yvyu": "COLOR_YUV2BGR_YVYU"}
# 4:2:2: byte offsets of Y0, U, Y1, V in the 4-byte macropixel
PACKED = {"yuyv": (0, 1, 2, 3), "uyvy": (1, 0, 3, 2), "yvyu": (0, 3, 2, 1)}
# sample values at the rule's corners: the clamp of Y at 16, the chroma zero at 128, the limited range's ends
CORNERS = np.array([0, 1, 15, 16, 17, 127, 128, 129, 235, 240, 254, 255], np.uint8)


def is420(fmt) -> bool:
    return fmt in ("nv12", "nv21")


def half(n) -> int:
    return (n + 1) // 2


def tight_row(fmt, W) -> int:
    """The tight (and least) row pitch of a W-pixel-wide view."""
    return 2 * half(W) if is420(fmt) else 4 * half(W)


def footprint(fmt, H, row_pitch, plane_pitch=0) -> int:
    """The bytes a view occupies from its base: plane_pitch + ceil(H/2) * row_pitch (4:2:0), H * row_pitch (4:2:2)."""
    return (plane_pitch or H * row_pitch) + half(H) * row_pitch if is420(fmt) else H * row_pitch


def frame_shape(fmt, W, H) -> tuple:
    return (H + half(H), 2 * half(W)) if is420(fmt) else (H, 2 * half(W), 2)


def convert(Y, U, V) -> np.ndarray:
    """BGR u8 [...][3] of equal-shaped Y, U, V sample arrays."""
    y = np.maximum(0, Y.astype(np.int64) - 16) * 1220542 + (1 << 19)
    u, v = U.astype(np.int64) - 128, V.astype(np.int64) - 128
    r = (y + 1673527 * v) >> 20
    g = (y - 852492 * v - 409993 * u) >> 20
    b = (y + 2116026 * u) >> 20
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)


def samples(frame, fmt, W, H):
    """(Y, U, V) [H][W] of each pixel of a W x H view held by `frame` (the shapes above, any strides)."""
    frame = np.asarray(frame, np.uint8)
    assert frame.shape == frame_shape(fmt, W, H), (frame.shape, fmt, W, H)
    ys, xs = np.arange(H)[:, None], np.arange(W)[None, :]
    if is420(fmt):
        Y = frame[:H, :W]
        c = frame[H:]
        c0, c1 = c[ys >> 1, 2 * (xs >> 1)], c[ys >> 1, 2 * (xs >> 1) + 1]
        return (Y, c0, c1) if fmt == "nv12" else (Y, c1, c0)
    m = frame.reshape(H, -1)   # the row's bytes
    oy, ou, _, ov = PACKED[fmt]
    Y = m[ys, 4 * (xs >> 1) + oy + 2 * (xs & 1)]
    return Y, m[ys, 4 * (xs >> 1) + ou], m[ys, 4 * (xs >> 1) + ov]


def decode(frame, fmt, W, H) -> np.ndarray:
    """BGR u8 [H][W][3] of the W x H view held by `frame`."""
    return convert(*samples(frame, fmt, W, H))


def cv_decode(cv2, frame, fmt, W, H) -> np.ndarray:
    """The live OpenCV path the restatement stands for: cv2.cvtColor on the even frame that holds the view (the luma
    plane of an odd-height 4:2:0 view grown by one row), cropped to W x H."""
    frame = np.ascontiguousarray(frame, np.uint8)
    if is420(fmt) and H % 2:
        frame = np.concatenate([frame[:H], np.zeros((1, frame.shape[1]), np.uint8), frame[H:]])
    return cv2.cvtColor(frame, getattr(cv2, CV_NAME[fmt]))[:H, :W]


def random_frame(rng, fmt, W, H, corners=False) -> np.ndarray:
    """A random frame (uniform bytes, or drawn from CORNERS) of the tight shape."""
    shape = frame_shape(fmt, W, H)
    if corners:
        return rng.choice(CORNERS, shape).astype(np.uint8)
    return rng.integers(0, 256, shape, dtype=np.uint8)


def encode(bgr, fmt) -> np.ndarray:
    """A YUV frame of BGR u8 [H][W][3] (BT.601 limited range, rounded; chroma averaged over its 2 x 2 or 2 x 1 block,
    the last column / row repeated for odd sizes): a plausible camera frame, not an exact inverse."""
    bgr = np.asarray(bgr, np.float64)
    H, W = bgr.shape[:2]
    b, g, r = bgr[..., 0], bgr[..., 1], bgr[..., 2]
    Y = 16 + (65.481 * r + 128.553 * g + 24.966 * b) / 255
    U = 128 + (-37.797 * r - 74.203 * g + 112.0 * b) / 255
    V = 128 + (112.0 * r - 93.786 * g - 18.214 * b) / 255
    ev = np.pad(np.stack([U, V], -1), ((0, H % 2), (0, W % 2), (0, 0)), mode="edge")
    q = lambda a: np.clip(np.rint(a), 0, 255).astype(np.uint8)   # noqa: E731
    Yq = q(np.pad(Y, ((0, 0), (0, W % 2)), mode="edge"))
    if is420(fmt):
        c = q((ev[0::2, 0::2] + ev[1::2, 0::2] + ev[0::2, 1::2] + ev[1::2, 1::2]) / 4)   # [H/2][W/2][U V]
        if fmt == "nv21":
            c = c[..., ::-1]
        return np.concatenate([Yq, c.reshape(half(H), -1)])
    c = q((ev[:H, 0::2] + ev[:H, 1::2]) / 2)   # [H][W/2][U V]
    out = np.empty((H, half(W), 4), np.uint8)
    oy, ou, oy1, ov = PACKED[fmt]
    out[..., oy], out[..., oy1] = Yq[:, 0::2], Yq[:, 1::2]
    out[..., ou], out[..., ov] = c[..., 0], c[..., 1]
    return out.reshape(H, 2 * half(W), 2)


def write_view(buf, frame, fmt, W, H, row_pitch, plane_pitch=0, off=0):
    """Lays the view held by `frame` into the flat u8 buffer `buf` at byte `off` with the given pitches, writing only
    the view's own samples: W luma bytes a row and 2*ceil(W/2) chroma bytes a chroma row (4:2:0), 4*ceil(W/2) bytes a
    row (4:2:2).  Every other byte of buf keeps its value."""
    frame = np.asarray(frame, np.uint8)
    rows = frame.reshape(frame.shape[0], -1)
    if is420(fmt):
        pp = plane_pitch or H * row_pitch
        for y in range(H):
            buf[off + y * row_pitch:off + y * row_pitch + W] = rows[y, :W]
        for y in range(half(H)):
            o = off + pp + y * row_pitch
            buf[o:o + 2 * half(W)] = rows[H + y]
    else:
        for y in range(H):
            buf[off + y * row_pitch:off + y * row_pitch + 4 * half(W)] = rows[y]
    return buf
