"""numpy restatement of the high-bit-depth formats (include/adcensus_b200.h, "High-bit-depth mono and Bayer frames"):
the 10p / 12p bit streams, the depth reduction and the full-depth demosaic, i.e. what unpacking to CV_16UC1,
cv::cvtColor(raw16, COLOR_Bayer*2BGR) and cv::Mat::convertTo(CV_8U, 2^-s) give.

A format name is <colour><depth>[p]: colour mono, bayer_rg, bayer_gr, bayer_bg or bayer_gb (the view's own top-left 2x2
block, as GenICam names it); depth 10, 12 or 16 bits in one little-endian uint16 per sample, or 10p / 12p, a
little-endian bit stream per row (sample x in bits [x*b, x*b + b) of the row's bytes).
  to8(v) = min(255, (v + 2^(s-1) - 1 + ((v >> s) & 1)) >> s), s = depth - 8: round half to even, saturated.
  mono: to8 of each sample, three times.  Bayer: the 8-bit mosaics' rule on the full-depth samples, then to8.

Frames are numpy arrays in the shapes the Python host entries take: uint16 [H][W] for the 16-bit containers, uint8
[H][ceil(b*W/8)] for the packed ones.
"""
from __future__ import annotations

import numpy as np

COLOURS = ("mono", "bayer_rg", "bayer_gr", "bayer_bg", "bayer_gb")
CONTAINERS = (("10", 10, False), ("12", 12, False), ("16", 16, False), ("10p", 10, True), ("12p", 12, True))
CODE = {f"{c}{suffix}": 64 + 5 * k + i for k, (suffix, _, _) in enumerate(CONTAINERS) for i, c in enumerate(COLOURS)}
NAMES = list(CODE)
# colours of rows 0 and 1 of each pattern's 2x2 block, and OpenCV's (legacy-named) conversion code for it
PATTERNS = {"bayer_rg": ("RG", "GB"), "bayer_gr": ("GR", "BG"), "bayer_bg": ("BG", "GR"), "bayer_gb": ("GB", "RG")}
CV_NAME = {"bayer_rg": "COLOR_BayerBG2BGR", "bayer_gr": "COLOR_BayerGB2BGR", "bayer_bg": "COLOR_BayerRG2BGR",
           "bayer_gb": "COLOR_BayerGR2BGR"}
_BGR = {"B": 0, "G": 1, "R": 2}


def info(name) -> tuple:
    """(colour, bits, packed) of a format name."""
    k, i = divmod(CODE[name] - 64, 5)
    return COLOURS[i], CONTAINERS[k][1], CONTAINERS[k][2]


def tight_row(name, W) -> int:
    """The tight (and least) row pitch in bytes of a W-sample row."""
    _, bits, packed = info(name)
    return (bits * W + 7) // 8 if packed else 2 * W


def frame_shape(name, W, H) -> tuple:
    return (H, tight_row(name, W)) if info(name)[2] else (H, W)


def pack(v, bits) -> np.ndarray:
    """uint8 [H][ceil(bits*W/8)]: the rows of samples v [H][W] (< 2^bits) as little-endian bit streams, each row starting
    on a byte; the unused high bits of a row's last byte are 0."""
    v = np.asarray(v, np.uint32)
    H, W = v.shape
    stream = ((v[..., None] >> np.arange(bits, dtype=np.uint32)) & 1).astype(np.uint8).reshape(H, W * bits)
    stream = np.pad(stream, ((0, 0), (0, -(W * bits) % 8)))
    return np.packbits(stream, axis=1, bitorder="little")


def unpack(rows, bits, W) -> np.ndarray:
    """uint16 [H][W] of packed rows [H][>= ceil(bits*W/8)], by the header's two-byte rule."""
    rows = np.asarray(rows, np.uint8).astype(np.uint32)
    o = np.arange(W) * bits
    k = o >> 3
    v = ((rows[:, k] | rows[:, k + 1] << 8) >> (o & 7)) & ((1 << bits) - 1)
    return np.ascontiguousarray(v, np.uint16)


def samples(frame, name, W, H) -> np.ndarray:
    """uint16 [H][W]: the samples of the view held by `frame` (a 16-bit container's whole words, bits above the depth
    included)."""
    _, bits, packed = info(name)
    frame = np.asarray(frame)
    assert frame.shape == frame_shape(name, W, H) and frame.dtype == (np.uint8 if packed else np.uint16), \
        (frame.shape, frame.dtype, name)
    return unpack(frame, bits, W) if packed else frame


def to8(v, s) -> np.ndarray:
    """round_half_even(v / 2^s) saturated to uint8."""
    v = np.asarray(v).astype(np.int64)
    return np.minimum(255, (v + (1 << (s - 1)) - 1 + ((v >> s) & 1)) >> s).astype(np.uint8)


def demosaic16(raw, colour) -> np.ndarray:
    """int64 [H][W][3] BGR at full depth of the mosaic raw [H][W]: zero below 3 x 3, else the interior rule at the
    position clamped to [1, W - 2] x [1, H - 2]."""
    r = np.asarray(raw).astype(np.int64)
    H, W = r.shape
    if H < 3 or W < 3:
        return np.zeros((H, W, 3), np.int64)
    pat = PATTERNS[colour]
    c = r[1:-1, 1:-1]
    n, s, w, e = r[:-2, 1:-1], r[2:, 1:-1], r[1:-1, :-2], r[1:-1, 2:]
    cross = (n + s + w + e + 2) >> 2
    diag = (r[:-2, :-2] + r[:-2, 2:] + r[2:, :-2] + r[2:, 2:] + 2) >> 2
    hor, ver = (w + e + 1) >> 1, (n + s + 1) >> 1
    inner = np.zeros((H - 2, W - 2, 3), np.int64)
    for py in (0, 1):           # parity of the frame row y = 1 + i
        for px in (0, 1):
            sl = (slice((py - 1) & 1, None, 2), slice((px - 1) & 1, None, 2))
            own = pat[py][px]
            inner[sl + (_BGR[own],)] = c[sl]
            if own == "G":
                inner[sl + (_BGR[pat[py][px ^ 1]],)] = hor[sl]
                inner[sl + (_BGR[pat[py ^ 1][px]],)] = ver[sl]
            else:
                inner[sl + (1,)] = cross[sl]
                inner[sl + (_BGR["B" if own == "R" else "R"],)] = diag[sl]
    return np.pad(inner, ((1, 1), (1, 1), (0, 0)), mode="edge")


def decode(frame, name, W, H) -> np.ndarray:
    """BGR u8 [H][W][3] of the W x H view held by `frame`."""
    colour, bits, _ = info(name)
    v = samples(frame, name, W, H)
    if colour == "mono":
        return np.repeat(to8(v, bits - 8)[..., None], 3, -1)
    return to8(demosaic16(v, colour), bits - 8)


def cv_decode(cv2, frame, name, W, H) -> np.ndarray:
    """The live OpenCV path the restatement stands for: cvtColor on the unpacked uint16 mosaic, then convertScaleAbs
    (= convertTo(CV_8U, 2^-s) for non-negative input)."""
    colour, bits, _ = info(name)
    v = np.ascontiguousarray(samples(frame, name, W, H))
    if colour != "mono":
        v = cv2.cvtColor(v, getattr(cv2, CV_NAME[colour]))
    out = cv2.convertScaleAbs(v, alpha=2.0 ** -(bits - 8)).reshape(v.shape)
    return out if colour != "mono" else np.repeat(out[..., None], 3, -1)


def from_samples(v, name) -> np.ndarray:
    """The frame (host-entry shape) that holds samples v [H][W]; packed formats keep the low `bits` bits."""
    _, bits, packed = info(name)
    v = np.asarray(v, np.uint16)
    return pack(v & ((1 << bits) - 1), bits) if packed else v.copy()


def random_frame(rng, name, W, H, corners=False) -> np.ndarray:
    """A random frame: samples uniform over the depth, or (corners) drawn from the half-way values of the reduction,
    the depth's ends and, for the 16-bit containers, words above the nominal depth."""
    _, bits, packed = info(name)
    top = (1 << bits) - 1
    if corners:
        s = bits - 8
        pool = [0, 1, top - 1, top, 1 << (s - 1), 3 << (s - 1), 5 << (s - 1), (509 << (s - 1)) & top, 254 << s]
        if not packed and bits < 16:
            pool += [top + 1, 2 * top, 0xFFFF]
        v = rng.choice(np.array(pool, np.uint16), (H, W))
    else:
        v = rng.integers(0, top + 1, (H, W)).astype(np.uint16)
    return from_samples(v, name)


def encode(bgr, name, rng) -> np.ndarray:
    """A frame of BGR u8 [H][W][3]: each pixel's own colour (mono: its green) scaled to the depth, plus random low bits
    so that the reduction has something to round."""
    colour, bits, _ = info(name)
    bgr = np.asarray(bgr, np.uint8)
    H, W = bgr.shape[:2]
    if colour == "mono":
        v8 = bgr[..., 1]
    else:
        v8 = np.empty((H, W), np.uint8)
        for py in (0, 1):
            for px in (0, 1):
                v8[py::2, px::2] = bgr[py::2, px::2, _BGR[PATTERNS[colour][py][px]]]
    s = bits - 8
    return from_samples((v8.astype(np.uint16) << s) | rng.integers(0, 1 << s, (H, W)).astype(np.uint16), name)


def write_view(buf, frame, name, W, H, row_pitch, off=0):
    """Lays the view held by `frame` into the flat u8 buffer `buf` at byte `off` with the given row pitch, writing only
    the tight bytes of each row."""
    rows = np.ascontiguousarray(frame).view(np.uint8).reshape(H, -1)
    t = tight_row(name, W)
    assert rows.shape[1] == t
    for y in range(H):
        buf[off + y * row_pitch:off + y * row_pitch + t] = rows[y]
    return buf
