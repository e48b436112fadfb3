"""numpy restatement of the video-decoder YUV containers and the colour encodings (include/adcensus_b200.h, "YUV video
and camera frames"): I420 / YV12 (a Y plane, then two chroma planes of half the row pitch), P016 (NV12's layout in
16-bit words, reduced to 8 bits first), and BT.601 / BT.709 in limited and full range for all eight YUV containers.

Conversion, u = U - 128, v = V - 128, int arithmetic with floor shifts, sat = clip to 0..255:
  limited range: y' = max(0, Y - 16) * 1220542, R = sat((y' + 2^19 + Rv v) >> 20), G = sat((y' + 2^19 + Gu u + Gv v) >> 20),
                 B = sat((y' + 2^19 + Bu u) >> 20)
  full range:    R = sat(Y + ((Rv v + 8192) >> 14)), G = sat(Y + ((Gu u + Gv v + 8192) >> 14)), B = sat(Y + ((Bu u + 8192) >> 14))
with the constant row of the encoding (COEF).  No flag (BT.601 limited) is yuv_testlib's rule.

Frames are numpy arrays in the shapes the Python host entries take:
  I420 / YV12: [H + ceil(H/2)][2*ceil(W/2)] u8: the luma rows, then the first and the second chroma plane, each
               ceil(H/2) rows of ceil(W/2) bytes, back to back (OpenCV's (H*3/2, W) Mat, FFmpeg's yuv420p buffer);
  P016:        [H + ceil(H/2)][2*ceil(W/2)] uint16: the luma rows, then the interleaved U V rows;
  the others:  as in yuv_testlib.
"""
from __future__ import annotations

import numpy as np

import rawdepth_testlib as X
import yuv_testlib as Y

CODE = {"i420": 38, "yv12": 39, "p016": 40}
NAMES = list(CODE)
ALL = {**Y.CODE, **CODE}                 # every YUV container
BT709, FULL = 0x100, 0x200
ENC = {"bt601": 0, "bt709": BT709, "bt601_full": FULL, "bt709_full": BT709 | FULL}
# (Rv, Gu, Gv, Bu) by encoding
COEF = {0: (1673527, -409993, -852492, 2116026), BT709: (1879825, -223607, -558796, 2215014),
        FULL: (22987, -5636, -11698, 29049), BT709 | FULL: (25802, -3069, -7670, 30402)}
KR_KB = {0: (0.299, 0.114), BT709: (0.2126, 0.0722)}
# P016 words at the to8 rule's corners: 0, the half-way points of 0 -> 1 and 254 -> 255 with both parities, the
# saturation, MSB-aligned 10-bit extremes
P016_CORNERS = np.array([0, 127, 128, 383, 384, 0x8000, 0x807F, 0x8080, 0x8180, 0xFE7F, 0xFE80, 0xFF7F, 0xFF80, 0xFFC0,
                         0xFFFF, 64 << 6, 940 << 6, 512 << 6], np.uint16)


def half(n) -> int:
    return (n + 1) // 2


def is_planar(fmt) -> bool:
    return fmt in ("i420", "yv12")


def tight_row(fmt, W) -> int:
    """The tight (and least) row pitch in bytes."""
    if fmt in CODE:
        return (4 if fmt == "p016" else 2) * half(W)
    return Y.tight_row(fmt, W)


def is420(fmt) -> bool:
    return fmt in CODE or Y.is420(fmt)


def footprint(fmt, H, row_pitch, plane_pitch=0) -> int:
    """plane_pitch + ceil(H/2) * row_pitch for every 4:2:0 container, H * row_pitch for 4:2:2."""
    return (plane_pitch or H * row_pitch) + half(H) * row_pitch if is420(fmt) else H * row_pitch


def read_bytes(fmt, W, H) -> int:
    """The bytes of a view the ingestion kernels read."""
    if is420(fmt):
        return (2 if fmt == "p016" else 1) * (W * H + 2 * half(W) * half(H))
    return 4 * half(W) * H


def frame_shape(fmt, W, H) -> tuple:
    return (H + half(H), 2 * half(W)) if fmt in CODE else Y.frame_shape(fmt, W, H)


def convert(Yv, U, V, enc=0) -> np.ndarray:
    """BGR u8 [...][3] of equal-shaped Y, U, V 8-bit sample arrays under encoding `enc` (flag bits)."""
    rv, gu, gv, bu = COEF[enc]
    Yi = Yv.astype(np.int64)
    u, v = U.astype(np.int64) - 128, V.astype(np.int64) - 128
    if enc & FULL:
        r = Yi + ((rv * v + 8192) >> 14)
        g = Yi + ((gu * u + gv * v + 8192) >> 14)
        b = Yi + ((bu * u + 8192) >> 14)
    else:
        y = np.maximum(0, Yi - 16) * 1220542 + (1 << 19)
        r = (y + rv * v) >> 20
        g = (y + gu * u + gv * v) >> 20
        b = (y + bu * u) >> 20
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)


def float_convert(Yv, U, V, enc) -> np.ndarray:
    """The floating-point matrix of the encoding, rounded half away from zero and saturated: what the BT.709 rules are
    bounded against."""
    kr, kb = KR_KB[enc & BT709]
    kg = 1 - kr - kb
    Yf, u, v = Yv.astype(np.float64), U.astype(np.float64) - 128, V.astype(np.float64) - 128
    if not enc & FULL:
        Yf, u, v = (Yf - 16) * 255 / 219, u * 255 / 224, v * 255 / 224
    r = Yf + 2 * (1 - kr) * v
    g = Yf - 2 * (1 - kb) * kb / kg * u - 2 * (1 - kr) * kr / kg * v
    b = Yf + 2 * (1 - kb) * u
    out = np.stack([b, g, r], -1)
    return np.clip(np.sign(out) * np.floor(np.abs(out) + 0.5), 0, 255).astype(np.uint8)


def samples(frame, fmt, W, H):
    """(Y, U, V) 8-bit [H][W] of each pixel of a W x H view held by `frame` (the shapes above), P016 reduced."""
    if fmt not in CODE:
        return Y.samples(frame, fmt, W, H)
    frame = np.asarray(frame)
    assert frame.shape == frame_shape(fmt, W, H), (frame.shape, fmt, W, H)
    ys, xs = np.arange(H)[:, None], np.arange(W)[None, :]
    if fmt == "p016":
        assert frame.dtype == np.uint16
        return Y.samples(X.to8(frame, 8), "nv12", W, H)
    assert frame.dtype == np.uint8
    c = np.ascontiguousarray(frame[H:]).reshape(-1)
    cw = half(W)
    first = c[(ys >> 1) * cw + (xs >> 1)]
    second = c[half(H) * cw + (ys >> 1) * cw + (xs >> 1)]
    return (frame[:H, :W], first, second) if fmt == "i420" else (frame[:H, :W], second, first)


def decode(frame, fmt, W, H, enc=0) -> np.ndarray:
    """BGR u8 [H][W][3] of the W x H view held by `frame` under encoding `enc`."""
    return convert(*samples(frame, fmt, W, H), enc)


def cv_decode(cv2, frame, fmt, W, H, enc=0) -> np.ndarray:
    """The live OpenCV path the restatement stands for, where OpenCV has one (BT.601, limited or full range):
      I420 / YV12: cvtColor(COLOR_YUV2BGR_I420 / _YV12) on the even frame holding the view, cropped;
      P016: convertScaleAbs(alpha=1/256) (= convertTo(CV_8U, 1/256)), then COLOR_YUV2BGR_NV12;
      full range: nearest chroma upsampling, then cvtColor(COLOR_YCrCb2BGR) on the pixels (Y, V, U);
      the others: yuv_testlib.cv_decode."""
    assert not enc & BT709, "OpenCV has no BT.709 YUV conversion"
    if enc & FULL:
        if fmt == "p016":
            frame = cv2.convertScaleAbs(np.ascontiguousarray(frame), alpha=1.0 / 256).reshape(frame.shape)
            fmt = "nv12"
        Yv, U, V = samples(frame, fmt, W, H)
        return cv2.cvtColor(np.ascontiguousarray(np.stack([Yv, V, U], -1)), cv2.COLOR_YCrCb2BGR)
    if fmt == "p016":
        return Y.cv_decode(cv2, cv2.convertScaleAbs(np.ascontiguousarray(frame), alpha=1.0 / 256).reshape(frame.shape),
                           "nv12", W, H)
    if fmt not in CODE:
        return Y.cv_decode(cv2, frame, fmt, W, H)
    frame = np.ascontiguousarray(frame, np.uint8)
    wp = frame.shape[1]
    luma = np.concatenate([frame[:H], np.zeros((H % 2, wp), np.uint8)])
    even = np.concatenate([luma.reshape(-1), frame[H:].reshape(-1)]).reshape(-1, wp)
    name = "COLOR_YUV2BGR_I420" if fmt == "i420" else "COLOR_YUV2BGR_YV12"
    return cv2.cvtColor(even, getattr(cv2, name))[:H, :W]


def random_frame(rng, fmt, W, H, corners=False) -> np.ndarray:
    """A random frame (uniform samples, or drawn from the rule's corner values) of the tight shape."""
    if fmt not in CODE:
        return Y.random_frame(rng, fmt, W, H, corners)
    shape = frame_shape(fmt, W, H)
    if fmt == "p016":
        if corners:
            return rng.choice(P016_CORNERS, shape).astype(np.uint16)
        return rng.integers(0, 1 << 16, shape, dtype=np.uint16)
    if corners:
        return rng.choice(Y.CORNERS, shape).astype(np.uint8)
    return rng.integers(0, 256, shape, dtype=np.uint8)


def encode(bgr, fmt) -> np.ndarray:
    """A plausible camera frame of BGR u8 [H][W][3] (BT.601 limited range, yuv_testlib.encode): I420 / YV12 from the
    NV12 encoding with its chroma de-interleaved, P016 as those samples MSB-aligned."""
    if fmt not in CODE:
        return Y.encode(bgr, fmt)
    nv = Y.encode(bgr, "nv12")
    H, W = bgr.shape[:2]
    if fmt == "p016":
        return nv.astype(np.uint16) << 8
    c = nv[H:].reshape(half(H), half(W), 2)
    first, second = (c[..., 0], c[..., 1]) if fmt == "i420" else (c[..., 1], c[..., 0])
    return np.concatenate([nv[:H].reshape(-1), first.reshape(-1), second.reshape(-1)]).reshape(nv.shape)


def write_view(buf, frame, fmt, W, H, row_pitch, plane_pitch=0, off=0):
    """Lays the view held by `frame` into the flat u8 buffer `buf` at byte `off` with the given pitches, writing only
    the view's own samples: W luma samples a row; ceil(W/2) bytes a chroma row of each I420 / YV12 plane (row pitch
    row_pitch / 2, the second plane ceil(H/2) * row_pitch / 2 after the first); 2*ceil(W/2) words a P016 chroma row.
    Every other byte of buf keeps its value."""
    if fmt not in CODE:
        return Y.write_view(buf, frame, fmt, W, H, row_pitch, plane_pitch, off)
    frame = np.asarray(frame)
    pp = plane_pitch or H * row_pitch
    if fmt == "p016":
        rows = frame.astype("<u2").view(np.uint8).reshape(frame.shape[0], -1)
        for y in range(H):
            buf[off + y * row_pitch:off + y * row_pitch + 2 * W] = rows[y, :2 * W]
        for y in range(half(H)):
            o = off + pp + y * row_pitch
            buf[o:o + 4 * half(W)] = rows[H + y]
        return buf
    assert row_pitch % 2 == 0
    for y in range(H):
        buf[off + y * row_pitch:off + y * row_pitch + W] = frame[y, :W]
    c = np.ascontiguousarray(frame[H:]).reshape(2, half(H), half(W))
    cp = row_pitch // 2
    for k in range(2):
        for y in range(half(H)):
            o = off + pp + k * half(H) * cp + y * cp
            buf[o:o + half(W)] = c[k, y]
    return buf
