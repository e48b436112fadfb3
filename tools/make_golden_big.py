#!/usr/bin/env python
"""Generates the large-configuration goldens from the UNMODIFIED reference (oracle/_ref):

  tests/golden/real_pairs.npz      the reference's bundled Middlebury pairs besides Cone -- Cloth3 view1/view5
                                   (D = 128, the reference's own usage example, main.cpp:30), Wood2 view1/view5
                                   (D = 128), Piano im0/im1 (D = 64) -- as packed BGR u8, their ground-truth
                                   disparity PNGs where the reference ships them, and the author's published 8-bit
                                   result images doc/exp/res/{cone,cloth,piano}-d.png (the weak known-answer pin of
                                   SURVEY.md 4.2)
  tests/golden/golden_big.json     sha256 of every tap after every stage (and of the stock Match output) for
                                   those pairs and for the BASELINE.json configs 3 / 4 inputs: synthetic 1242x375x128
                                   seeds 1-2, synthetic 1920x1080x192 seed 1

Needs a checkout of the reference (ADC_REFERENCE_DIR) and oracle/_ref built from it; the fixtures are committed so that
the tests, which have neither, can compare the CUDA path with the real reference's outputs.
"""
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import adc_testlib as T  # noqa: E402

REAL = {  # name: (dir, left, right, dmax, gt_left or None)
    "cloth3": ("Cloth3", "view1.png", "view5.png", 128, "disp1.png"),
    "wood2": ("Wood2", "view1.png", "view5.png", 128, "disp1.png"),
    "piano": ("Piano", "im0.png", "im1.png", 64, None),
}
SYNTH = {  # name: (W, H, D, seed)
    "kitti_s1": (1242, 375, 128, 1),
    "kitti_s2": (1242, 375, 128, 2),
    "p1080_s1": (1920, 1080, 192, 1),
}


def run_case(name, left, right, dmax, out):
    h, w, _ = left.shape
    opt = T.default_option(max_disparity=dmax)
    t0 = time.time()
    ref = T.Reference(w, h, opt)
    ref.begin(left, right)
    hashes = {}
    for st in T.STAGES:
        ref.step()
        for tap in T.STAGE_TAPS[st]:
            hashes[f"{st}/{tap}"] = T.sha(ref.tap(tap))
    final = ref.tap("DISP_L").copy()
    ref.close()
    out[name] = {"width": w, "height": h, "max_disparity": dmax, "hashes": hashes,
                 "input_sha": [T.sha(left), T.sha(right)]}
    print(name, w, h, dmax, "final", hashes["MEDIAN/DISP_L"][:16], f"{time.time() - t0:.1f}s", flush=True)
    return final


def main():
    import cv2
    T.build_oracle()
    assert T.have_ref(), "oracle/_ref is required: set ADC_REFERENCE_DIR to a checkout of the reference"
    only = set(sys.argv[1:])
    jpath = T.GOLDEN_DIR / "golden_big.json"
    out = json.loads(jpath.read_text()) if jpath.exists() else {}
    arrays = {}
    data = T.REFERENCE_ROOT / "Data"
    for name, (d, l, r, dmax, gt) in REAL.items():
        left = cv2.imread(str(data / d / l), cv2.IMREAD_COLOR)
        right = cv2.imread(str(data / d / r), cv2.IMREAD_COLOR)
        arrays[f"{name}_left"], arrays[f"{name}_right"] = left, right
        if gt:
            arrays[f"{name}_gt"] = cv2.imread(str(data / d / gt), cv2.IMREAD_GRAYSCALE)
        if not only or name in only:
            final = run_case(name, left, right, dmax, out)
            arrays[f"{name}_final"] = final   # the reference's float map (for the accuracy / render checks)
    res = T.REFERENCE_ROOT / "doc" / "exp" / "res"
    for nm in ("cone", "cloth", "piano"):
        arrays[f"doc_{nm}_d"] = cv2.imread(str(res / f"{nm}-d.png"), cv2.IMREAD_GRAYSCALE)
    if not only:
        np.savez_compressed(T.GOLDEN_DIR / "real_pairs.npz", **arrays)
    jpath.write_text(json.dumps(out, indent=1, sort_keys=True))
    for name, (w, h, D, seed) in SYNTH.items():
        if only and name not in only:
            continue
        left, right = T.synthetic_pair(w, h, D, seed)
        run_case(name, left, right, D, out)
        jpath.write_text(json.dumps(out, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
