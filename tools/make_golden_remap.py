"""Writes tests/golden/golden_remap_cases.npz: small sources, remap tables and what cv2.remap(src, map1, map2,
INTER_LINEAR, BORDER_CONSTANT, 0) gives for them, so that the numpy restatement of the rectified entries' resampling
(tests/rectify_testlib.py) is checked against OpenCV where OpenCV is not installed.

Cases (keys "<name>/src", "<name>/map1", "<name>/map2", "<name>/out"):
  f32_*    random float maps, 1 / 3 / 4 channels, with exact ties at odd multiples of 1/64, NaN, +-inf, +-1e9, 70000,
           -0.0 and neighbours partly outside the frame;
  fixed_*  random CV_16SC2 + CV_16UC1 maps with saturated int16 corners and junk in the high bits of map2;
  rig_*    initUndistortRectifyMap maps of a made-up camera (both map types);
  line_*   1 x 1, 1 x N and N x 1 sources.

    python tools/make_golden_remap.py [out.npz]
"""
import sys
from pathlib import Path

import cv2
import numpy as np

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "golden_remap_cases.npz"
SPECIALS = np.array([np.nan, np.inf, -np.inf, 1e9, -1e9, 70000.0, -0.0], np.float32)


def cv_remap(src, m1, m2):
    out = cv2.remap(src, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    return out.reshape(m2.shape + src.shape[2:])


def random_f32(rng, h, w, H, W, c):
    src = rng.integers(0, 256, (h, w, c) if c > 1 else (h, w), dtype=np.uint8)
    mx = rng.uniform(-3, w + 2, (H, W)).astype(np.float32)
    my = rng.uniform(-3, h + 2, (H, W)).astype(np.float32)
    t = rng.random((H, W)) < 0.2
    mx[t] = (rng.integers(-200, 64 * w, t.sum()) * 2 + 1) / np.float32(64)
    t = rng.random((H, W)) < 0.1
    my[t] = (rng.integers(-200, 64 * h, t.sum()) * 2 + 1) / np.float32(64)
    sp = rng.random((H, W)) < 0.03
    mx[sp] = rng.choice(SPECIALS, sp.sum())
    sp = rng.random((H, W)) < 0.02
    my[sp] = rng.choice(SPECIALS, sp.sum())
    return src, mx, my


def random_fixed(rng, h, w, H, W, c):
    src = rng.integers(0, 256, (h, w, c) if c > 1 else (h, w), dtype=np.uint8)
    m1 = rng.integers(-4, max(w, h) + 3, (H, W, 2)).astype(np.int16)
    m1[rng.random((H, W)) < 0.02] = [-32768, 32767]
    m1[rng.random((H, W)) < 0.02] = [32767, -32768]
    m2 = rng.integers(0, 65536, (H, W)).astype(np.uint16)
    return src, m1, m2


def rig_maps(src_w, src_h, W, H, m1type):
    """initUndistortRectifyMap of a made-up camera: focal length ~0.9 * width, radial and tangential distortion, a
    small rectifying rotation, output W x H."""
    K = np.array([[0.9 * src_w, 0, src_w / 2 - 3.3], [0, 0.9 * src_w, src_h / 2 + 2.1], [0, 0, 1]], np.float64)
    dist = np.array([-0.21, 0.08, 0.0012, -0.0009, -0.011])
    R, _ = cv2.Rodrigues(np.array([0.011, -0.024, 0.006]))
    P = np.array([[0.8 * W, 0, W / 2, 0], [0, 0.8 * W, H / 2, 0], [0, 0, 1, 0]], np.float64)
    return cv2.initUndistortRectifyMap(K, dist, R, P, (W, H), m1type)


def cases():
    rng = np.random.default_rng(20261015)
    out = {}
    for i in range(6):
        h, w = (int(v) for v in rng.integers(5, 40, 2))
        H, W = (int(v) for v in rng.integers(5, 40, 2))
        out[f"f32_{i}"] = random_f32(rng, h, w, H, W, [1, 3, 4][i % 3])
        out[f"fixed_{i}"] = random_fixed(rng, h, w, H, W, [1, 3, 4][i % 3])
    for i, (sw, sh) in enumerate([(40, 30), (24, 18)]):
        src = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        for name, t in (("f32", cv2.CV_32FC1), ("fixed", cv2.CV_16SC2)):
            m1, m2 = rig_maps(sw, sh, 32, 24, t)
            out[f"rig_{name}_{i}"] = (src, m1, m2)
    for name, (h, w) in (("1x1", (1, 1)), ("1xN", (1, 23)), ("Nx1", (19, 1))):
        src, mx, my = random_f32(rng, h, w, 9, 11, 3)
        out[f"line_{name}"] = (src, mx, my)
        out[f"line_{name}_fixed"] = (src, *cv2.convertMaps(mx, my, cv2.CV_16SC2))
    return out


def main(path=OUT):
    arrays = {}
    for name, (src, m1, m2) in cases().items():
        arrays.update({f"{name}/src": src, f"{name}/map1": m1, f"{name}/map2": m2, f"{name}/out": cv_remap(src, m1, m2)})
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len(arrays) // 4} cases, opencv {cv2.__version__}")


if __name__ == "__main__":
    main(Path(sys.argv[1]) if len(sys.argv) > 1 else OUT)
