"""Writes tests/golden/golden_bayer_cases.npz: small raw Bayer mosaics and what cv2.cvtColor(raw, COLOR_Bayer*2BGR)
gives for them, plus cvtColor followed by cv2.remap(INTER_LINEAR, BORDER_CONSTANT, 0), so that the numpy restatement of
the Bayer formats (tests/bayer_testlib.py, composed with tests/rectify_testlib.py for the rectified entries) is checked
against OpenCV where OpenCV is not installed.

Cases (keys "<name>/raw", "<name>/pattern" (the ADC_IMG_BAYER_* code), "<name>/out", and for rect_* also
"<name>/map1", "<name>/map2"):
  tiny_*   every pattern at 1 x 1, 2 x 2, 1 x 7, 6 x 2, 3 x 3, 3 x 8, 9 x 3 (sizes below 3 give zeros);
  odd_*    every pattern at random odd and even sizes up to 40, taken as crops of a larger frame at odd offsets;
  rect_*   cvtColor -> remap with random float maps (specials included) and CV_16SC2 maps, frames larger and smaller
           than the output, maps reaching past the last row and column; a 2 x N and a 1 x 1 frame (all-zero views).

    python tools/make_golden_bayer.py [out.npz]
"""
import sys
from pathlib import Path

import cv2
import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import bayer_testlib as B  # noqa: E402
import make_golden_remap as MG  # noqa: E402

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "golden_bayer_cases.npz"


def cases():
    """{name: (raw, pattern name, map1 or None, map2 or None)}"""
    rng = np.random.default_rng(20261016)
    out = {}
    for p in B.NAMES:
        for h, w in ((1, 1), (2, 2), (1, 7), (6, 2), (3, 3), (3, 8), (9, 3)):
            out[f"tiny_{p}_{h}x{w}"] = (rng.integers(0, 256, (h, w), dtype=np.uint8), p, None, None)
        for i in range(3):
            h, w = (int(v) for v in rng.integers(3, 41, 2))
            big = rng.integers(0, 256, (h + 3, w + 5), dtype=np.uint8)
            out[f"odd_{p}_{i}"] = (np.ascontiguousarray(big[1:1 + h, 3:3 + w]), p, None, None)
    sizes = [(31, 23), (12, 17), (40, 29), (9, 13), (2, 25), (1, 1)]   # (h, w) of the raw frame; output 19 x 21
    for i, (h, w) in enumerate(sizes):
        p = B.NAMES[i % 4]
        raw = rng.integers(0, 256, (h, w), dtype=np.uint8)
        _, mx, my = MG.random_f32(rng, h, w, 19, 21, 1)
        if i % 2:
            mx, my = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        out[f"rect_{i}"] = (raw, p, mx, my)
    return out


def expected(raw, p, m1, m2):
    bgr = B.cv_demosaic(cv2, raw, p)
    if m1 is None:
        return bgr
    return cv2.remap(bgr, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def main(path=OUT):
    arrays = {}
    for name, (raw, p, m1, m2) in cases().items():
        arrays.update({f"{name}/raw": raw, f"{name}/pattern": np.int32(B.CODE[p]), f"{name}/out": expected(raw, p, m1, m2)})
        if m1 is not None:
            arrays.update({f"{name}/map1": m1, f"{name}/map2": m2})
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len({k.split('/')[0] for k in arrays})} cases, opencv {cv2.__version__}")


if __name__ == "__main__":
    main(Path(sys.argv[1]) if len(sys.argv) > 1 else OUT)
