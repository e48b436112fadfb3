"""Writes tests/golden/golden_resize_cases.npz: small 8-bit images and what cv2.resize gives for them with INTER_AREA at
integer factors and with INTER_LINEAR_EXACT, so that the numpy restatement (tests/resize_testlib.py) is checked against
OpenCV where OpenCV is not installed.

Cases (keys "<name>/src" (uint8 [h][w] or [h][w][c]), "<name>/interp" (16 = AREA, 17 = LINEAR_EXACT), "<name>/size"
(W, H of the output), "<name>/out"):
  area_*     factors 1 x 1, 2 x 2, 3 x 3, 2 x 3, 3 x 2, 4 x 4, 5 x 7, 8 x 1, 1 x 8, 16 x 16, 64 x 64 and 4096 x 1 on
             1, 3 and 4 channels, uniform samples and samples of 127 and 128 only;
  linear_*   random sizes 1..64 up and down, 1 x 1, 1 x N and N x 1 sources and outputs, on 1, 3 and 4 channels.

    python tools/make_golden_resize.py [out.npz]
"""
import sys
from pathlib import Path

import cv2
import numpy as np

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "golden_resize_cases.npz"
AREA, LINEAR_EXACT = 16, 17


def cases():
    rng = np.random.default_rng(2026)
    out = {}
    factors = [(1, 1), (2, 2), (3, 3), (2, 3), (3, 2), (4, 4), (5, 7), (8, 1), (1, 8), (16, 16), (64, 64), (4096, 1)]
    for kx, ky in factors:
        for c in (1, 3, 4):
            W, H = (1, 1) if kx * ky >= 4096 else (2, 1) if kx * ky >= 256 else (5, 4)
            shape = (H * ky, W * kx) + ((c,) if c > 1 else ())
            src = rng.integers(0, 256, shape, dtype=np.uint8)
            if c == 4:   # samples of 127 and 128 only: sums near the rounding points
                src[:] = 127 + rng.integers(0, 2, shape, dtype=np.uint8)
            out[f"area_{kx}x{ky}_c{c}"] = (src, AREA, W, H)
    sizes = [(1, 1, 5, 3), (7, 1, 1, 4), (1, 9, 6, 1), (13, 2, 1, 1), (2, 2, 64, 3)]
    sizes += [tuple(int(v) for v in rng.integers(1, 65, 4)) for _ in range(24)]
    for k, (sw, sh, W, H) in enumerate(sizes):
        c = (1, 3, 4)[k % 3]
        shape = (sh, sw) + ((c,) if c > 1 else ())
        out[f"linear_{k}_{sw}x{sh}_to_{W}x{H}_c{c}"] = (rng.integers(0, 256, shape, dtype=np.uint8), LINEAR_EXACT, W, H)
    return out


def main(path=OUT):
    arrays = {}
    interp = {AREA: cv2.INTER_AREA, LINEAR_EXACT: cv2.INTER_LINEAR_EXACT}
    for name, (src, t, W, H) in cases().items():
        got = cv2.resize(src, (W, H), interpolation=interp[t]).reshape((H, W) + src.shape[2:])
        arrays.update({f"{name}/src": src, f"{name}/interp": np.int32(t), f"{name}/size": np.int32([W, H]),
                       f"{name}/out": got})
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len({k.split('/')[0] for k in arrays})} cases, opencv {cv2.__version__}")


if __name__ == "__main__":
    main(Path(sys.argv[1]) if len(sys.argv) > 1 else OUT)
