"""numpy restatement of the image formats of adc_match_images* (include/adcensus_b200.h): what packed BGR image a view
in a given format and geometry stands for, and how to lay pixels out in a format, for building test inputs.

Byte addressing of one view inside a flat u8 buffer, as the header defines it (pitches already resolved, no zero
defaults): packed / gray pixel (x, y) at offset + y*row_pitch + x*bytes_per_pixel; planar channel c (0 = R, 1 = G,
2 = B) at offset + c*plane_pitch + y*row_pitch + x.
"""
from __future__ import annotations

import numpy as np

FORMATS = ["bgr", "rgb", "bgra", "rgba", "gray", "rgb_planar"]
CODE = {f: i for i, f in enumerate(FORMATS)}
BPP = {"bgr": 3, "rgb": 3, "bgra": 4, "rgba": 4, "gray": 1, "rgb_planar": 1}
# source channel of output B, G, R for the packed colour formats
_ORDER = {"bgr": (0, 1, 2), "rgb": (2, 1, 0), "bgra": (0, 1, 2), "rgba": (2, 1, 0)}


def footprint(fmt, H, row_pitch, plane_pitch=0) -> int:
    """Bytes one view spans (the tight image stride): H*row_pitch, or 3*plane_pitch for planar images."""
    return 3 * plane_pitch if fmt == "rgb_planar" else H * row_pitch


def to_bgr(buf, fmt, H, W, row_pitch, plane_pitch=0, offset=0) -> np.ndarray:
    """The packed BGR u8 [H][W][3] image the view of format `fmt` at byte `offset` of `buf` stands for."""
    buf = np.asarray(buf).view(np.uint8).reshape(-1)
    ys = np.arange(H)[:, None] * row_pitch + offset
    xs = np.arange(W)[None, :]
    out = np.empty((H, W, 3), np.uint8)
    if fmt == "gray":
        out[:] = buf[ys + xs][:, :, None]
    elif fmt == "rgb_planar":
        for c, src in enumerate((2, 1, 0)):            # B, G, R from planes 2, 1, 0
            out[:, :, c] = buf[ys + xs + src * plane_pitch]
    else:
        for c, src in enumerate(_ORDER[fmt]):
            out[:, :, c] = buf[ys + xs * BPP[fmt] + src]
    return out


def from_bgr(bgr, fmt, alpha=None) -> np.ndarray:
    """Tight array of a packed BGR image in `fmt`: [H][W][3 or 4], [3][H][W] for rgb_planar.  Gray images take the
    first channel (callers pass images whose channels are equal).  alpha: the fourth byte of bgra / rgba (default: a
    pattern that differs from pixel to pixel, so that a kernel that read it would be caught)."""
    bgr = np.asarray(bgr, np.uint8)
    H, W, _ = bgr.shape
    if fmt == "bgr":
        return bgr.copy()
    if fmt == "rgb":
        return np.ascontiguousarray(bgr[:, :, ::-1])
    if fmt == "gray":
        return bgr[:, :, 0].copy()
    if fmt == "rgb_planar":
        return np.ascontiguousarray(bgr[:, :, ::-1].transpose(2, 0, 1))
    if alpha is None:
        alpha = ((np.arange(H)[:, None] * 7 + np.arange(W)[None, :] * 13) % 251).astype(np.uint8)
    base = bgr if fmt == "bgra" else bgr[:, :, ::-1]
    return np.ascontiguousarray(np.concatenate([base, np.broadcast_to(alpha, (H, W))[:, :, None]], axis=2))


def write_view(buf, img, fmt, row_pitch, plane_pitch=0, offset=0):
    """Writes a tight image `img` (as from_bgr returns it) into the flat u8 buffer `buf` at byte `offset` with the given
    pitches; bytes between rows and planes are left as they are."""
    buf = buf.reshape(-1)
    if fmt == "rgb_planar":
        _, H, W = img.shape
        for c in range(3):
            for y in range(H):
                o = offset + c * plane_pitch + y * row_pitch
                buf[o:o + W] = img[c, y]
        return
    H, W = img.shape[:2]
    rb = W * BPP[fmt]
    flat = img.reshape(H, rb)
    for y in range(H):
        o = offset + y * row_pitch
        buf[o:o + rb] = flat[y]


def gray_to_bgr(gray) -> np.ndarray:
    """A gray image replicated to BGR: pixel v -> (v, v, v)."""
    g = np.asarray(gray, np.uint8)
    return np.ascontiguousarray(np.repeat(g[:, :, None], 3, axis=2))
