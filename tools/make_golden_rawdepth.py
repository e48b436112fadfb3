"""Writes tests/golden/golden_rawdepth_cases.npz: small high-bit-depth frames (10 / 12 / 16 bits per uint16, 10p / 12p,
mono and the four Bayer patterns) and what OpenCV gives for them -- cv2.cvtColor(raw16, COLOR_Bayer*2BGR) on the
unpacked uint16 mosaic, then cv2.convertScaleAbs(v, alpha=2**-(bits - 8)) -- plus the same followed by
cv2.remap(INTER_LINEAR, BORDER_CONSTANT, 0), so that the numpy restatement (tests/rawdepth_testlib.py, composed with
tests/rectify_testlib.py for the rectified entries) is checked against OpenCV where OpenCV is not installed.  The
unpacking itself has no OpenCV counterpart; tests/test_rawdepth.py checks it against byte vectors written out by hand.

Cases (keys "<name>/frame" (the host entries' array), "<name>/format" (the ADC_IMG_* code), "<name>/size" (W, H),
"<name>/out", and for rect_* also "<name>/map1", "<name>/map2"):
  tiny_*    every format at 1 x 1, 2 x 5, 3 x 3 and 5 x 7 (H x W);
  odd_*     every format at two random sizes up to 40, uniform samples and the reduction's corner values (half-way
            values of both parities, the depth's ends, words above the nominal depth);
  rect_*    decode -> remap with random float maps (specials included) and CV_16SC2 maps, frames larger and smaller
            than the output, maps reaching past the last row and column, a 1 x N, a 2 x 2 and a 1 x 1 frame.

    python tools/make_golden_rawdepth.py [out.npz]
"""
import sys
from pathlib import Path

import cv2
import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import make_golden_remap as MG  # noqa: E402
import rawdepth_testlib as X  # noqa: E402

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "golden_rawdepth_cases.npz"


def cases():
    """{name: (frame, format name, W, H, map1 or None, map2 or None)}"""
    rng = np.random.default_rng(20261017)
    out = {}
    for f in X.NAMES:
        for h, w in ((1, 1), (2, 5), (3, 3), (5, 7)):
            out[f"tiny_{f}_{h}x{w}"] = (X.random_frame(rng, f, w, h), f, w, h, None, None)
        for i in range(2):
            h, w = (int(v) for v in rng.integers(3, 41, 2))
            out[f"odd_{f}_{i}"] = (X.random_frame(rng, f, w, h, corners=i == 1), f, w, h, None, None)
    sizes = [(31, 23), (12, 17), (40, 29), (9, 13), (1, 25), (1, 1), (24, 30), (2, 2), (7, 8), (33, 3)]   # (h, w); output 19 x 21
    picks = ["bayer_rg12p", "mono12p", "bayer_gb10p", "bayer_gr12", "mono10p", "bayer_bg12p", "bayer_bg16", "bayer_rg10p",
             "mono16", "bayer_gr10"]
    for i, ((h, w), f) in enumerate(zip(sizes, picks)):
        frame = X.random_frame(rng, f, w, h, corners=i == 6)
        _, mx, my = MG.random_f32(rng, h, w, 19, 21, 1)
        if i % 2:
            mx, my = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        out[f"rect_{i}"] = (frame, f, w, h, mx, my)
    return out


def expected(frame, f, w, h, m1, m2):
    bgr = X.cv_decode(cv2, frame, f, w, h)
    if m1 is None:
        return bgr
    return cv2.remap(bgr, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0).reshape(m2.shape[:2] + (3,))


def main(path=OUT):
    arrays = {}
    for name, (frame, f, w, h, m1, m2) in cases().items():
        arrays.update({f"{name}/frame": frame, f"{name}/format": np.int32(X.CODE[f]), f"{name}/size": np.int32([w, h]),
                       f"{name}/out": expected(frame, f, w, h, m1, m2)})
        if m1 is not None:
            arrays.update({f"{name}/map1": m1, f"{name}/map2": m2})
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len({k.split('/')[0] for k in arrays})} cases, opencv {cv2.__version__}")


if __name__ == "__main__":
    main(Path(sys.argv[1]) if len(sys.argv) > 1 else OUT)
