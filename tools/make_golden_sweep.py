#!/usr/bin/env python
"""Generates tests/golden/golden_sweep_ref.json from the UNMODIFIED reference (oracle/_ref, built by oracle/Makefile from
the checkout ADC_REFERENCE_DIR names): sha256 of every tap after every stage for the first (textured) pair of the
disparity-sweep cases of tests/test_kernel_sweep.py whose range the other fixtures do not reach.

The sweep's cases are defined here, so that the tests and this generator build the same inputs.
"""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import adc_testlib as T  # noqa: E402
import make_golden as G  # noqa: E402

# disparity ranges whose sweep case is narrower than the range (W < D: no pixel has every candidate in the image)
NARROW = (40, 96, 150, 224, 256)
# the sweep cases pinned to the reference: ranges none of the other fixtures reach (D 80: dmin > 0, D 31: dmin < 0)
GOLDEN_DS = (1, 2, 7, 19, 29, 31, 40, 44, 56, 61, 65, 80, 96, 113, 127, 160, 161, 224, 253)
FLAT, NOISE = 1, 3          # positions of the two poison pairs among the five pairs of a case


def sweep_case(D):
    """(W, H, option, seed) of the sweep case of disparity range D: W and H not multiples of 4, H odd and not a multiple
    of 3 (so not a multiple of any scanline slot length T), W > D except for NARROW, min_disparity != 0 on every seventh
    range (alternately positive and negative)."""
    H = (13, 17, 19, 23, 25, 29)[D % 6]
    W = max(D - 9, 10) if D in NARROW else D + 11 + D % 5
    if W % 4 == 0:
        W += 1
    over = {"max_disparity": D}
    if D % 7 == 3:
        dmin = 3 if (D // 7) % 2 else -(D // 2)
        over = {"min_disparity": dmin, "max_disparity": dmin + D}
    return W, H, T.default_option(**over), 1000 + D


def sweep_pairs(W, H, D, seed):
    """Five distinct pairs: three textured synthetic pairs, and between them a flat pair (every in-image cost 0, arms as
    long as the options allow) at FLAT and a white-noise pair (short arms, no match) at NOISE.  In a batch, a pair's
    neighbours are then always different inputs, so a sum that reaches into a neighbouring pair's rows changes the result."""
    tex = [T.synthetic_pair(W, H, D, seed + 7919 * i) for i in range(3)]
    flat = np.full((H, W, 3), 128, np.uint8)
    rng = np.random.default_rng(seed)
    noise = (rng.integers(0, 256, (H, W, 3), dtype=np.uint8), rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
    pairs = [tex[0], tex[1], tex[2]]
    pairs.insert(FLAT, (flat, flat.copy()))
    pairs.insert(NOISE, noise)
    return pairs


def staged_hashes(checker, opt, left, right):
    """sha256 of every tap after every stage of one pair (DISP_R cut to the part the reference defines)."""
    checker.begin(left, right)
    hashes = {}
    for st in T.STAGES:
        checker.step()
        for tap in T.STAGE_TAPS[st]:
            hashes[f"{st}/{tap}"] = T.sha(G.ref_case_tap(opt, tap, checker.tap(tap)))
    return hashes


def main():
    assert T.have_ref() or (T.build_oracle() or T.have_ref()), "oracle/_ref is required: set ADC_REFERENCE_DIR to a checkout of the reference"
    out = {}
    for D in GOLDEN_DS:
        W, H, opt, seed = sweep_case(D)
        left, right = sweep_pairs(W, H, D, seed)[0]
        ref = T.Reference(W, H, opt)
        out[str(D)] = staged_hashes(ref, opt, left, right)
        ref.close()
        print(f"D={D} {W}x{H} dmin={opt.min_disparity} final sha {out[str(D)]['MEDIAN/DISP_L'][:16]}")
    (T.GOLDEN_DIR / "golden_sweep_ref.json").write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
