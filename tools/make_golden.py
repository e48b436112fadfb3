#!/usr/bin/env python
"""Generates tests/golden/golden_*.npz from the UNMODIFIED reference (oracle/_ref, built by oracle/Makefile from the
checkout ADC_REFERENCE_DIR names).  The fixtures are committed, so the tests check against the real reference's outputs
without the reference itself.

For every case: sha256 of every tap after every stage (bit-exact pin for all intermediates,
including the cost volumes) plus the full arrays of the small per-pixel maps and the final map.
"""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import adc_testlib as T  # noqa: E402

CASES = {
    # name: (source, W, H, option overrides, seed or crop)
    "cone_full": ("cone", None, None, {}, None),
    "cone_crop": ("cone", 140, 100, {"max_disparity": 32}, (150, 120)),
    "synth_a": ("synth", 97, 61, {"max_disparity": 24}, 2),
    "synth_b": ("synth", 130, 70, {"max_disparity": 37}, 3),
    "synth_opts": ("synth", 120, 90, {"max_disparity": 48, "lambda_ad": 7, "lambda_census": 20, "so_p1": 0.7,
                                       "so_p2": 2.5, "irv_ts": 10, "irv_th": 0.3, "lrcheck_thres": 0.5,
                                       "cross_L1": 20, "cross_L2": 9}, 11),
    "synth_disc": ("synth", 80, 60, {"max_disparity": 32, "do_discontinuity_adjustment": 1}, 10),
}
FULL_TAPS = {"ARMS", "SUPCNT_H", "SUPCNT_V", "DISP_L", "DISP_R", "MISMATCHES", "OCCLUSIONS", "CENSUS_L"}
# synthetic cases (W, H, D, option overrides, seed) whose every tap after every stage is pinned by sha256 in
# tests/golden/golden_ref_cases.json: small sizes, option switches, dmin > 0 and dmin < 0
REF_CASES = [(70, 50, 20, {}, 21), (64, 40, 16, {"min_disparity": 0, "do_lr_check": 0}, 22),
             (90, 64, 40, {"do_filling": 0}, 23), (33, 30, 48, {}, 24), (9, 9, 8, {}, 25),
             (80, 60, 32, {"min_disparity": 2, "max_disparity": 34}, 31),
             (80, 60, 32, {"min_disparity": -4, "max_disparity": 28}, 32)]


def ref_case_id(case):
    return f"{case[0]}x{case[1]}x{case[2]}-s{case[4]}"


def ref_case_tap(opt, tap, a):
    """The part of a tap the reference defines.  Right pixels x >= W - dmin (and x < 1 - dmax) have no candidate column
    at all: the reference then runs its parabola on an uninitialised cost_local[], or reads past it (ADCensusStereo.cpp:
    271-300, SURVEY 8a A10) -- whatever the heap held; the restatement writes the integer 0 there.  Undefined in the
    reference, so not pinned."""
    if tap == "DISP_R" and (opt.min_disparity > 0 or opt.max_disparity <= 0):
        lo = max(0, 1 - opt.max_disparity)
        a = a[:, lo:max(lo, a.shape[1] - max(opt.min_disparity, 0))]
    return a


def ref_case_inputs(case):
    w, h, D, over, seed = case
    opt = T.default_option(**{"max_disparity": D, **over})
    left, right = T.synthetic_pair(w, h, D, seed)
    return left, right, opt


def case_inputs(name):
    src, w, h, over, extra = CASES[name]
    opt = T.default_option(**over)
    if src == "cone":
        left, right = T.load_cone()
        if w is not None:
            left, right = T.crop_pair(left, right, extra[0], extra[1], w, h)
    else:
        left, right = T.synthetic_pair(w, h, opt.max_disparity - opt.min_disparity, extra)
    return left, right, opt


def main():
    assert T.have_ref() or (T.build_oracle() or T.have_ref()), "oracle/_ref is required: set ADC_REFERENCE_DIR to a checkout of the reference"
    out_dir = T.GOLDEN_DIR
    for name in CASES:
        left, right, opt = case_inputs(name)
        h, w, _ = left.shape
        ref = T.Reference(w, h, opt)
        ref.begin(left, right)
        arrays, hashes = {}, {}
        for st in T.STAGES:
            ref.step()
            for tap in T.STAGE_TAPS[st]:
                a = ref.tap(tap)
                hashes[f"{st}/{tap}"] = T.sha(a)
                if tap in FULL_TAPS and (name != "cone_full" or (st in ("WTA", "MEDIAN") and tap in ("DISP_L", "DISP_R"))):
                    arrays[f"{st}__{tap}"] = a.copy()
        stock = ref.stock_match(left, right)
        assert T.sha(stock) == hashes["MEDIAN/DISP_L"], "staged runner and stock Match disagree"
        np.savez_compressed(out_dir / f"golden_{name}.npz", hashes=json.dumps(hashes), **arrays)
        print(name, w, h, "final sha", hashes["MEDIAN/DISP_L"][:16], "arrays", len(arrays))
    ref_cases = {}
    for case in REF_CASES:
        left, right, opt = ref_case_inputs(case)
        h, w, _ = left.shape
        ref = T.Reference(w, h, opt)
        ref.begin(left, right)
        hashes = {}
        for st in T.STAGES:
            ref.step()
            for tap in T.STAGE_TAPS[st]:
                hashes[f"{st}/{tap}"] = T.sha(ref_case_tap(opt, tap, ref.tap(tap)))
        ref_cases[ref_case_id(case)] = hashes
        print(ref_case_id(case), "final sha", hashes["MEDIAN/DISP_L"][:16])
    (out_dir / "golden_ref_cases.json").write_text(json.dumps(ref_cases, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
