"""Writes tests/golden/golden_reproject_cases.npz: small disparity maps, Q matrices and what OpenCV gives for them, so
that the numpy restatement of the reprojection entries (tests/reproject_testlib.py) is checked against OpenCV where
OpenCV is not installed, and the GPU tests compare the kernel with OpenCV's own output.

Cases (keys "<name>/disp" f32 [H][W], "<name>/Q" f64 [4][4], "<name>/min_disparity", "<name>/points" =
cv2.reprojectImageTo3D(disp, Q), "<name>/s16" = cv2.multiply(disp, 16.0, dtype=CV_16S) with +inf pixels replaced by
(min_disparity - 1) * 16 saturated):
  rand_*   random Q with entries from 1e-30 to 1e30 and +-0 entries, maps with +-inf, NaN, +-0, f32 subnormals, +-3e38;
  rig_*    the Q of cv2.stereoRectify for a made-up rig, with CALIB_ZERO_DISPARITY on ("zero") and off ("free"), on
           engine-like maps (quarter-pixel disparities, +inf = invalid);
  line_*   1 x 1, 1 x N and N x 1 maps;
  s16_*    S16 ties (odd multiples of 1/32), saturation, int32 overflow, for several min_disparity values.

    python tools/make_golden_reproject.py [out.npz]
"""
import sys
from pathlib import Path

import cv2
import numpy as np

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "golden_reproject_cases.npz"
SPECIALS = np.array([np.inf, -np.inf, np.nan, 0.0, -0.0, 1e-40, -1e-42, 1.4e-45, 3e38, -3e38], np.float32)
S16_VALUES = np.array([2047.96875, 2048.0, 2047.9375, -2048.03125, -2048.0625, 0.03125, 0.09375, -0.03125, -0.09375,
                       0.15625, 1.03125, -1.03125, 2 ** 27, -2 ** 27, 2 ** 27 - 8, 134217720.0, 3e38, -3e38, 1e30,
                       np.inf, -np.inf, np.nan, 0.0, -0.0, 1.4e-45, 63.75, -4.25, 12.5, 2047.0, -2049.0], np.float32)


def random_Q(rng):
    """4x4 with entries of random sign from 1e-30 to 1e30, about a quarter of them +0 or -0."""
    Q = rng.choice([-1.0, 1.0], (4, 4)) * 10.0 ** rng.uniform(-30, 30, (4, 4))
    z = rng.random((4, 4))
    Q[z < 0.25] = 0.0
    Q[z < 0.1] = -0.0
    return Q


def random_disp(rng, H, W):
    """Uniform values in [-300, 300) with about a fifth replaced by SPECIALS."""
    d = rng.uniform(-300, 300, (H, W)).astype(np.float32)
    m = rng.random((H, W)) < 0.2
    d[m] = rng.choice(SPECIALS, int(m.sum()))
    return d


def engine_disp(rng, H, W, dmin=0, D=64):
    """An engine-like final map: quarter-pixel values in [dmin, dmin + D), about a fifth +inf."""
    d = (dmin + rng.integers(0, 4 * D, (H, W)) / 4.0).astype(np.float32)
    d[rng.random((H, W)) < 0.2] = np.inf
    return d


def rig_Q(W, H, zero_disparity=True, baseline=0.12):
    """Q of cv2.stereoRectify for a made-up rig of two slightly different cameras imaging W x H."""
    K1 = np.array([[0.92 * W, 0, W / 2 - 2.5], [0, 0.92 * W, H / 2 + 1.5], [0, 0, 1]], np.float64)
    K2 = np.array([[0.91 * W, 0, W / 2 + 3.1], [0, 0.91 * W, H / 2 - 0.7], [0, 0, 1]], np.float64)
    d1 = np.array([-0.11, 0.04, 0.0007, -0.0005, -0.003])
    d2 = np.array([-0.09, 0.03, -0.0004, 0.0006, -0.002])
    R, _ = cv2.Rodrigues(np.array([0.003, -0.009, 0.002]))
    T = np.array([-baseline, 0.002, 0.001])
    flags = cv2.CALIB_ZERO_DISPARITY if zero_disparity else 0
    return cv2.stereoRectify(K1, d1, K2, d2, (W, H), R, T, flags=flags, alpha=0)[4]


def cv_points(disp, Q):
    return cv2.reprojectImageTo3D(disp, Q)


def cv_s16(disp, min_disparity):
    out = cv2.multiply(disp, 16.0, dtype=cv2.CV_16S).reshape(disp.shape)
    out[np.isposinf(disp)] = np.clip((min_disparity - 1) * 16, -32768, 32767)
    return out


def cases():
    rng = np.random.default_rng(20261015)
    out = {}
    for i in range(16):
        H, W = (int(v) for v in rng.integers(1, 28, 2))
        out[f"rand_{i}"] = (random_disp(rng, H, W), random_Q(rng), int(rng.integers(-20, 21)))
    for i, (W, H, dmin) in enumerate([(48, 32, 0), (33, 21, -4), (40, 24, 2)]):
        for name, zero in (("zero", True), ("free", False)):
            out[f"rig_{name}_{i}"] = (engine_disp(rng, H, W, dmin), rig_Q(W, H, zero), dmin)
    for name, (H, W) in (("1x1", (1, 1)), ("1xN", (1, 600)), ("Nx1", (37, 1))):
        out[f"line_{name}"] = (random_disp(rng, H, W), random_Q(rng), 0)
    for i, dmin in enumerate([0, -3000, 3000, 7]):
        d = rng.permutation(np.tile(S16_VALUES, 4)).reshape(8, 15)
        out[f"s16_{i}"] = (d, rig_Q(15, 8, i % 2 == 0), dmin)
    return out


def main(path=OUT):
    arrays = {}
    for name, (disp, Q, dmin) in cases().items():
        arrays.update({f"{name}/disp": disp, f"{name}/Q": Q, f"{name}/min_disparity": np.int32(dmin),
                       f"{name}/points": cv_points(disp, Q), f"{name}/s16": cv_s16(disp, dmin)})
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len(arrays) // 5} cases, opencv {cv2.__version__}")


if __name__ == "__main__":
    main(Path(sys.argv[1]) if len(sys.argv) > 1 else OUT)
