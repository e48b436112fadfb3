"""Writes tests/golden/golden_yuv_video_cases.npz: small I420, YV12 and P016 frames and what OpenCV gives for them, and
frames of every YUV container under full-range BT.601 and what OpenCV gives for those, plus each followed by
cv2.remap(INTER_LINEAR, BORDER_CONSTANT, 0), so that the numpy restatement (tests/yuv_video_testlib.py, composed with
tests/rectify_testlib.py for the rectified entries) is checked against OpenCV where OpenCV is not installed.

OpenCV paths: I420 / YV12 cvtColor(COLOR_YUV2BGR_I420 / _YV12); P016 convertScaleAbs(alpha=1/256) (= convertTo(CV_8U,
1/256)), then cvtColor(COLOR_YUV2BGR_NV12); full range nearest chroma upsampling, then cvtColor(COLOR_YCrCb2BGR) on
(Y, V, U).  Odd views are the crop of the conversion of the even frame that holds them.  OpenCV has no BT.709 YUV
conversion, so the BT.709 rules have no fixture.

Cases (keys "<name>/frame" (the host entries' array shape), "<name>/format" (the ADC_IMG_* container code),
"<name>/encoding" (the flag bits), "<name>/size" (W, H), "<name>/out", and for rect_* also "<name>/map1", "<name>/map2"):
  tiny_*    I420, YV12, P016 (BT.601 limited) and every container at full range, at 1 x 1, 1 x 7, 2 x 2, 6 x 1, 3 x 5
            and 4 x 6 (H x W);
  odd_*     the same at random odd and even sizes up to 40, uniform samples and the rules' corner values;
  rect_*    conversion -> remap with random float maps (specials included) and CV_16SC2 maps, frames larger and smaller
            than the output, maps reaching past the last row and column, odd source sizes, a 1 x N and a 1 x 1 frame.

    python tools/make_golden_yuv_video.py [out.npz]
"""
import sys
from pathlib import Path

import cv2
import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import make_golden_remap as MG  # noqa: E402
import yuv_video_testlib as V  # noqa: E402

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "golden_yuv_video_cases.npz"
# (container, encoding) pairs OpenCV can state
COMBOS = [(f, 0) for f in V.NAMES] + [(f, V.FULL) for f in V.ALL]


def cases():
    """{name: (frame, container, encoding, W, H, map1 or None, map2 or None)}"""
    rng = np.random.default_rng(20261017)
    out = {}
    for f, enc in COMBOS:
        tag = f"{f}_{enc:x}"
        for h, w in ((1, 1), (1, 7), (2, 2), (6, 1), (3, 5), (4, 6)):
            out[f"tiny_{tag}_{h}x{w}"] = (V.random_frame(rng, f, w, h), f, enc, w, h, None, None)
        for i in range(3):
            h, w = (int(v) for v in rng.integers(1, 41, 2))
            out[f"odd_{tag}_{i}"] = (V.random_frame(rng, f, w, h, corners=i % 2 == 1), f, enc, w, h, None, None)
    sizes = [(31, 23), (12, 17), (40, 29), (9, 13), (1, 25), (1, 1), (24, 30), (7, 8), (15, 20), (2, 3), (33, 9)]
    for i, (f, enc) in enumerate(COMBOS):
        h, w = sizes[i % len(sizes)]
        frame = V.random_frame(rng, f, w, h, corners=i % 4 == 3)
        _, mx, my = MG.random_f32(rng, h, w, 19, 21, 1)
        if i % 2:
            mx, my = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        out[f"rect_{i}"] = (frame, f, enc, w, h, mx, my)
    return out


def expected(frame, f, enc, w, h, m1, m2):
    bgr = V.cv_decode(cv2, frame, f, w, h, enc)
    if m1 is None:
        return bgr
    return cv2.remap(bgr, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def main(path=OUT):
    arrays = {}
    for name, (frame, f, enc, w, h, m1, m2) in cases().items():
        arrays.update({f"{name}/frame": frame, f"{name}/format": np.int32(V.ALL[f]), f"{name}/encoding": np.int32(enc),
                       f"{name}/size": np.int32([w, h]), f"{name}/out": expected(frame, f, enc, w, h, m1, m2)})
        if m1 is not None:
            arrays.update({f"{name}/map1": m1, f"{name}/map2": m2})
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len({k.split('/')[0] for k in arrays})} cases, opencv {cv2.__version__}")


if __name__ == "__main__":
    main(Path(sys.argv[1]) if len(sys.argv) > 1 else OUT)
