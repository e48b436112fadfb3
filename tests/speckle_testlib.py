"""numpy / scipy restatement of speckle removal (adc_filter_speckles*, include/adcensus_b200.h): cv2.filterSpeckles on
int16 maps (OpenCV's plain C++ path, or its IPP path with ipp=True), and the engine's f32 rules, as connected components
of the 4-neighbour graph."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

INT_MIN = -(2 ** 31)


def cv_round(v) -> int:
    """cvRound on x86 (cvtsd2si): round half to even, INT_MIN for NaN and for anything outside int32."""
    v = float(v)
    if np.isnan(v):
        return INT_MIN
    r = float(np.rint(v))
    return int(r) if -(2.0 ** 31) <= r <= 2.0 ** 31 - 1 else INT_MIN


def wrap16(v: int) -> int:
    """(int16)v: the low 16 bits, signed."""
    return (int(v) + 32768) % 65536 - 32768


def removed(missing: np.ndarray, right: np.ndarray, down: np.ndarray, max_size: int) -> np.ndarray:
    """bool [H][W]: the pixels of components of at most max_size pixels; the graph's vertices are the pixels that are not
    missing, its edges the pairs (x, x + 1) where right [H][W-1] is set and (y, y + 1) where down [H-1][W] is set."""
    H, W = missing.shape
    idx = np.arange(H * W).reshape(H, W)
    rows = np.concatenate([idx[:, :-1][right], idx[:-1, :][down]])
    cols = np.concatenate([idx[:, 1:][right], idx[1:, :][down]])
    g = coo_matrix((np.ones(rows.size, np.int8), (rows, cols)), shape=(H * W, H * W))
    _, lab = connected_components(g, directed=False)
    sizes = np.bincount(lab, minlength=lab.max() + 1)
    return (~missing) & (sizes[lab].reshape(H, W) <= max_size)


def filter_s16(img: np.ndarray, new_val, max_size: int, max_diff, ipp: bool = False) -> np.ndarray:
    """cv2.filterSpeckles(img, new_val, max_size, max_diff) on an int16 map, returned as a copy.  new_val and max_diff go
    through cvRound; the missing test and the differences are in int; the value written is (int16)new_val.  ipp=True:
    OpenCV's IPP path, which wraps cvRound(max_diff) and cvRound(new_val) to int16 first (the second matters only for
    a new_val outside int16, where the plain path marks nothing as missing and IPP the pixels equal to the wrapped
    value)."""
    nv, md = cv_round(new_val), cv_round(max_diff)
    miss_val = nv
    if ipp:
        md, miss_val = wrap16(md), wrap16(nv)
    a = img.astype(np.int64)
    miss = a == miss_val
    right = ~miss[:, :-1] & ~miss[:, 1:] & (np.abs(a[:, :-1] - a[:, 1:]) <= md)
    down = ~miss[:-1, :] & ~miss[1:, :] & (np.abs(a[:-1, :] - a[1:, :]) <= md)
    out = img.copy()
    out[removed(miss, right, down, int(max_size))] = np.int16(wrap16(nv))
    return out


def filter_f32(img: np.ndarray, new_val, max_size: int, max_diff) -> np.ndarray:
    """The F32 rules on a float32 map, returned as a copy: nv = (float)new_val; missing = v == nv; connected = neither
    missing and (double)fabsf(a - b) <= max_diff, a - b in float."""
    img = np.asarray(img, np.float32)
    with np.errstate(all="ignore"):
        nv = np.float32(new_val)
        miss = img == nv
        dx = np.abs(img[:, :-1] - img[:, 1:]).astype(np.float64) <= float(max_diff)
        dy = np.abs(img[:-1, :] - img[1:, :]).astype(np.float64) <= float(max_diff)
    right = ~miss[:, :-1] & ~miss[:, 1:] & dx
    down = ~miss[:-1, :] & ~miss[1:, :] & dy
    out = img.copy()
    out[removed(miss, right, down, int(max_size))] = nv
    return out


def filter_any(img: np.ndarray, new_val, max_size: int, max_diff) -> np.ndarray:
    """filter_s16 or filter_f32 by the map's dtype."""
    return filter_s16(img, new_val, max_size, max_diff) if img.dtype == np.int16 else \
        filter_f32(img, new_val, max_size, max_diff)


def same_bits(a: np.ndarray, b: np.ndarray) -> bool:
    """Equal shape, dtype and bits (NaN payloads included: the filter copies or writes values, it computes none)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    return a.tobytes() == b.tobytes()
