"""Writes tests/golden/golden_speckle_cases.npz: small int16 maps, filterSpeckles arguments and what OpenCV gives for
them, so that the restatement of the speckle entries (tests/speckle_testlib.py) is checked against OpenCV where OpenCV is
not installed, and the GPU tests compare the kernels with OpenCV's own output.

Cases (keys "<name>/map" int16 [H][W], "<name>/args" f64 [new_val, max_size, max_diff], "<name>/want" =
cv2.filterSpeckles with IPP off, the plain C++ path the engine follows; "<name>/want_ipp" = the same with IPP on, for the
cases where the two paths may differ, max_diff or new_val outside int16):
  tie_*      cvRound ties of new_val (2.5 -> 2, 3.5 -> 4) and of max_diff;
  nv_*       new_val outside int16 (40000 wraps to -25536 when written; nothing is missing on the plain path);
  md_*       max_diff negative, and outside int16 (40000, 65536, 70000, 1e10, NaN);
  size_*     max_size 0, negative, and >= H*W;
  extreme_*  values +-32767 and -32768;
  line_*     1 x 1, 1 x N and N x 1 maps;
  engine_*   S16 maps of engine-like content: (min_disparity - 1) * 16 invalid, smooth surfaces, speckles.

    python tools/make_golden_speckles.py [out.npz]
"""
import sys
from pathlib import Path

import cv2
import numpy as np

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "golden_speckle_cases.npz"


def small_map(rng, H, W, lo=-6, hi=7, scale=1):
    """Random values in [lo, hi) * scale: plenty of small components and of equal neighbours."""
    return (rng.integers(lo, hi, (H, W)) * scale).astype(np.int16)


def engine_s16(rng, H, W, dmin=0, D=64, speckle_frac=0.03):
    """An engine-like S16 map: a few planes of disparity * 16 at quarter-pixel steps, about a tenth invalid
    ((dmin - 1) * 16) in blobs, and small speckles of unrelated values."""
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    d = np.zeros((H, W))
    for _ in range(3):
        cx, cy = rng.uniform(0, W), rng.uniform(0, H)
        plane = dmin + D * (0.3 + 0.4 * rng.random()) + rng.uniform(-0.1, 0.1) * (xs - cx) + rng.uniform(-0.1, 0.1) * (ys - cy)
        mask = (xs - cx) ** 2 + (ys - cy) ** 2 < (rng.uniform(0.2, 0.6) * max(H, W)) ** 2
        d[mask] = plane[mask]
    s16 = (np.round(np.clip(d, dmin, dmin + D - 1) * 4) * 4).astype(np.int16)
    inv = rng.random((H, W)) < 0.03
    inv = inv | np.roll(inv, 1, 0) | np.roll(inv, 1, 1)
    s16[inv] = (dmin - 1) * 16
    sp = rng.random((H, W)) < speckle_frac
    s16[sp] = rng.integers(dmin * 16, (dmin + D) * 16, int(sp.sum()))
    return s16


def run(img, new_val, max_size, max_diff, ipp):
    cv2.ipp.setUseIPP(ipp)
    out = img.copy()
    cv2.filterSpeckles(out, new_val, max_size, max_diff)
    return out


def cases(rng):
    c = {}
    c["tie_nv_2_5"] = (small_map(rng, 23, 31, 0, 6), 2.5, 4, 1.0)
    c["tie_nv_3_5"] = (small_map(rng, 23, 31, 0, 6), 3.5, 4, 1.0)
    c["tie_md_0_5"] = (small_map(rng, 19, 27), 0.0, 5, 0.5)
    c["tie_md_1_5"] = (small_map(rng, 19, 27), 0.0, 5, 1.5)
    m = small_map(rng, 21, 33, -3, 4, 3000)
    m[rng.random(m.shape) < 0.2] = -25536
    c["nv_40000"] = (m, 40000.0, 6, 20000.0)
    c["nv_m40000"] = (small_map(rng, 21, 33, -3, 4), -40000.0, 3, 1.0)
    c["md_neg"] = (small_map(rng, 17, 25), 0.0, 1, -1.0)
    for md in (40000.0, 65536.0, 70000.0, 1e10, float("nan")):
        c[f"md_{md:g}"] = (small_map(rng, 24, 29, -3, 4, 2500), 0.0, 2, md)
    c["size_0"] = (small_map(rng, 16, 16), 0.0, 0, 2.0)
    c["size_neg"] = (small_map(rng, 16, 16), 0.0, -3, 2.0)
    c["size_all"] = (small_map(rng, 16, 20, -2, 3), 0.0, 320, 1.0)
    e = rng.choice(np.array([32767, -32767, -32768, 0, 32766, -32766], np.int16), (20, 24))
    c["extreme_md_1"] = (e, 0.0, 3, 1.0)
    c["extreme_md_32767"] = (e, -32768.0, 5, 32767.0)
    c["line_1x1"] = (np.array([[5]], np.int16), 0.0, 1, 1.0)
    c["line_1x1_missing"] = (np.array([[5]], np.int16), 5.0, 1, 1.0)
    c["line_1xN"] = (small_map(rng, 1, 97, -2, 3), 0.0, 3, 1.0)
    c["line_Nx1"] = (small_map(rng, 89, 1, -2, 3), 0.0, 3, 1.0)
    for i, (H, W, dmin) in enumerate([(60, 80, 0), (75, 90, -8), (48, 130, 5)]):
        c[f"engine_{i}"] = (engine_s16(rng, H, W, dmin), float((dmin - 1) * 16), 30, 32.0)
    c["engine_opencv_default"] = (engine_s16(rng, 96, 128, 0), -16.0, 200, 32.0)
    return c


def main():
    out = Path(sys.argv[1]) if len(sys.argv) > 1 else OUT
    rng = np.random.default_rng(16)
    z = {}
    for name, (img, nv, ms, md) in cases(rng).items():
        z[f"{name}/map"] = img
        z[f"{name}/args"] = np.array([nv, ms, md], np.float64)
        z[f"{name}/want"] = run(img, nv, ms, md, False)
        if not (-32768 <= np.nan_to_num(md, nan=1e30) <= 32767 and -32768 <= nv <= 32767):
            z[f"{name}/want_ipp"] = run(img, nv, ms, md, True)
    cv2.ipp.setUseIPP(True)
    np.savez_compressed(out, **z)
    print(f"wrote {out}: {len({k.split('/')[0] for k in z})} cases, OpenCV {cv2.__version__}")


if __name__ == "__main__":
    main()
