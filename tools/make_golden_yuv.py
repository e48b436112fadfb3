"""Writes tests/golden/golden_yuv_cases.npz: small YUV frames (NV12, NV21, YUYV, UYVY, YVYU) and what
cv2.cvtColor(frame, COLOR_YUV2BGR_*) gives for them, plus cvtColor followed by cv2.remap(INTER_LINEAR, BORDER_CONSTANT,
0), so that the numpy restatement of the YUV formats (tests/yuv_testlib.py, composed with tests/rectify_testlib.py for
the rectified entries) is checked against OpenCV where OpenCV is not installed.

Cases (keys "<name>/frame" (the host entries' array shape), "<name>/format" (the ADC_IMG_* code), "<name>/size" (W, H),
"<name>/out", and for rect_* also "<name>/map1", "<name>/map2"):
  tiny_*    every format at 1 x 1, 1 x 7, 2 x 2, 6 x 1, 3 x 5 and 4 x 6 (H x W);
  odd_*     every format at random odd and even sizes up to 40, uniform bytes and the rule's corner values; odd views
            are the crop of cvtColor on the even frame that holds them;
  rect_*    cvtColor -> remap with random float maps (specials included) and CV_16SC2 maps, frames larger and smaller
            than the output, maps reaching past the last row and column (the border is BGR 0, not the conversion of
            YUV 0), odd source sizes, a 1 x N and a 1 x 1 frame.

    python tools/make_golden_yuv.py [out.npz]
"""
import sys
from pathlib import Path

import cv2
import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import make_golden_remap as MG  # noqa: E402
import yuv_testlib as Y  # noqa: E402

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "golden_yuv_cases.npz"


def cases():
    """{name: (frame, format name, W, H, map1 or None, map2 or None)}"""
    rng = np.random.default_rng(20261016)
    out = {}
    for f in Y.NAMES:
        for h, w in ((1, 1), (1, 7), (2, 2), (6, 1), (3, 5), (4, 6)):
            out[f"tiny_{f}_{h}x{w}"] = (Y.random_frame(rng, f, w, h), f, w, h, None, None)
        for i in range(4):
            h, w = (int(v) for v in rng.integers(1, 41, 2))
            out[f"odd_{f}_{i}"] = (Y.random_frame(rng, f, w, h, corners=i % 2 == 1), f, w, h, None, None)
    sizes = [(31, 23), (12, 17), (40, 29), (9, 13), (1, 25), (1, 1), (24, 30), (7, 8)]   # (h, w) of the raw frame; output 19 x 21
    for i, (h, w) in enumerate(sizes):
        f = Y.NAMES[i % 5]
        frame = Y.random_frame(rng, f, w, h, corners=i == 6)
        _, mx, my = MG.random_f32(rng, h, w, 19, 21, 1)
        if i % 2:
            mx, my = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        out[f"rect_{i}"] = (frame, f, w, h, mx, my)
    return out


def expected(frame, f, w, h, m1, m2):
    bgr = Y.cv_decode(cv2, frame, f, w, h)
    if m1 is None:
        return bgr
    return cv2.remap(bgr, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def main(path=OUT):
    arrays = {}
    for name, (frame, f, w, h, m1, m2) in cases().items():
        arrays.update({f"{name}/frame": frame, f"{name}/format": np.int32(Y.CODE[f]), f"{name}/size": np.int32([w, h]),
                       f"{name}/out": expected(frame, f, w, h, m1, m2)})
        if m1 is not None:
            arrays.update({f"{name}/map1": m1, f"{name}/map2": m2})
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len({k.split('/')[0] for k in arrays})} cases, opencv {cv2.__version__}")


if __name__ == "__main__":
    main(Path(sys.argv[1]) if len(sys.argv) > 1 else OUT)
