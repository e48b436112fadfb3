#!/usr/bin/env python
"""Generates tests/golden/golden_gray_cases.json from the UNMODIFIED reference (oracle/_ref) on gray images.

A gray image goes into the reference the only way the reference takes images: replicated to packed BGR, pixel v ->
(v, v, v), which is what adc_match_images defines a gray view to be.  Two cases:
  * cone_gray: the reference's own GRAY_L / GRAY_R taps of the Cone pair (its fp64 luma, truncated), replicated;
  * synth_gray_odd: an odd-width synthetic gray pair (the green channel of a synthetic pair, with a band of 128s).
For every case: the sha256 of both gray input planes and of every tap after every stage.
"""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import adc_testlib as T  # noqa: E402
import images_testlib as IT  # noqa: E402
import make_golden as G  # noqa: E402

GRAY_CASES = {"cone_gray": {}, "synth_gray_odd": {"max_disparity": 24}}


def synth_gray_pair(w=97, h=61, D=24, seed=5):
    """Green channel of a synthetic pair, with rows 10..13 set to 128 in both views (gray(128, 128, 128) = 127)."""
    left, right = T.synthetic_pair(w, h, D, seed)
    gl, gr = left[:, :, 1].copy(), right[:, :, 1].copy()
    gl[10:14] = 128
    gr[10:14] = 128
    return gl, gr


def cone_gray_pair(checker):
    """The Cone pair's GRAY_L / GRAY_R taps of `checker` (the reference, or the restatement that reproduces it)."""
    left, right = T.load_cone()
    h, w, _ = left.shape
    c = checker(w, h, T.default_option())
    c.begin(left, right)
    c.run_to("COST")
    gl, gr = c.tap("GRAY_L").copy(), c.tap("GRAY_R").copy()
    c.close()
    return gl, gr


def gray_case_inputs(name, checker=None):
    """(gray left, gray right, option) of a case; cone_gray needs a checker (T.Oracle in the tests)."""
    opt = T.default_option(**GRAY_CASES[name])
    if name == "cone_gray":
        gl, gr = cone_gray_pair(checker or T.Oracle)
    else:
        gl, gr = synth_gray_pair()
    return gl, gr, opt


def main():
    assert T.have_ref() or (T.build_oracle() or T.have_ref()), "oracle/_ref is required: set ADC_REFERENCE_DIR to a checkout of the reference"
    out = {}
    for name in GRAY_CASES:
        gl, gr, opt = gray_case_inputs(name, T.Reference)
        h, w = gl.shape
        ref = T.Reference(w, h, opt)
        ref.begin(IT.gray_to_bgr(gl), IT.gray_to_bgr(gr))
        hashes = {}
        for st in T.STAGES:
            ref.step()
            for tap in T.STAGE_TAPS[st]:
                hashes[f"{st}/{tap}"] = T.sha(G.ref_case_tap(opt, tap, ref.tap(tap)))
        ref.close()
        out[name] = {"width": w, "height": h, "max_disparity": opt.max_disparity, "input_sha": [T.sha(gl), T.sha(gr)],
                     "hashes": hashes}
        print(name, w, h, "final sha", hashes["MEDIAN/DISP_L"][:16], flush=True)
    (T.GOLDEN_DIR / "golden_gray_cases.json").write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
