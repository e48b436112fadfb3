"""numpy restatement of the reprojection entries (adc_reproject*, include/adcensus_b200.h): what
cv2.reprojectImageTo3D(disp, Q) gives, its Z plane, and the StereoSGBM "disparity * 16" encoding, bit for bit apart from
NaN payloads."""
import numpy as np

INT16_MIN, INT16_MAX = -32768, 32767


def points(disp: np.ndarray, Q) -> np.ndarray:
    """float32 [H][W][3]: h_i = (((+0.0 + Q[i][0]*x) + Q[i][1]*y) + Q[i][2]*d) + Q[i][3]*1.0 in double, one rounding per
    operation; P_c = (float)((double)(float)h_c * (1.0 / h_3)); P_z = 10000 where d is exactly FLT_MAX."""
    Q = np.asarray(Q).astype(np.float64)
    H, W = disp.shape
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    d = disp.astype(np.float64)
    with np.errstate(all="ignore"):
        h = [(((np.zeros_like(d) + Q[i, 0] * xs) + Q[i, 1] * ys) + Q[i, 2] * d) + Q[i, 3] * 1.0 for i in range(4)]
        ia = 1.0 / h[3]
        P = np.stack([(h[c].astype(np.float32).astype(np.float64) * ia).astype(np.float32) for c in range(3)], -1)
    # OpenCV's bigZ: Z = 10000 where |d - minDisparity| <= FLT_EPSILON, minDisparity = FLT_MAX without handleMissingValues
    P[disp == np.finfo(np.float32).max, 2] = 10000.0
    return P


def depth(disp: np.ndarray, Q) -> np.ndarray:
    """float32 [H][W]: the Z plane of points()."""
    return np.ascontiguousarray(points(disp, Q)[:, :, 2])


def saturate_s16(disp: np.ndarray) -> np.ndarray:
    """int16: cv::saturate_cast<short>(d * 16) as x86 computes it: t = d * 16 rounded half to even, saturated when it
    fits in int32, -32768 otherwise (NaN, +-inf, |t| >= 2^31: the integer indefinite value)."""
    with np.errstate(all="ignore"):
        t = disp.astype(np.float32) * np.float32(16)
        out = np.full(disp.shape, INT16_MIN, np.int16)
        ok = (t < np.float32(2.0 ** 31)) & (t >= np.float32(-(2.0 ** 31)))
        out[ok] = np.clip(np.rint(t[ok].astype(np.float64)), INT16_MIN, INT16_MAX).astype(np.int16)
    return out


def disp_s16(disp: np.ndarray, min_disparity: int) -> np.ndarray:
    """int16 [H][W]: saturate_s16, with +inf (the engine's invalid value) as (min_disparity - 1) * 16 saturated."""
    out = saturate_s16(disp)
    out[np.isposinf(disp)] = np.clip((int(min_disparity) - 1) * 16, INT16_MIN, INT16_MAX)
    return out


def same_nan(got: np.ndarray, want: np.ndarray) -> bool:
    """Bit-equal, except that any NaN equals any NaN (payloads differ between x86 and the GPU)."""
    if got.shape != want.shape or got.dtype != want.dtype:
        return False
    if got.dtype.kind != "f":
        return np.array_equal(got, want)
    gn, wn = np.isnan(got), np.isnan(want)
    return bool(np.array_equal(gn, wn) and np.array_equal(got[~gn].view(np.uint32), want[~wn].view(np.uint32)))

