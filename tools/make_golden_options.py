#!/usr/bin/env python
"""Generates tests/golden/golden_options_ref.json from the UNMODIFIED reference (oracle/_ref, built by oracle/Makefile from
the checkout ADC_REFERENCE_DIR names): sha256 of every tap after every stage for the first (textured) pair of every
option-space case of tests/test_option_space.py that is pinned (PINNED).

The option-space cases are defined here, so that the tests and this generator build the same inputs.  Every case runs
the sweep's five pairs (make_golden_sweep.sweep_pairs: textured, flat, textured, noise, textured).
"""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import adc_testlib as T  # noqa: E402
import make_golden_sweep as GS  # noqa: E402

INT32_MAX = 2**31 - 1
NAN, INF = float("nan"), float("inf")

# ---- arm-length sweep: cross_L1 over 0..256 and beyond, on rows about two arms wide ---------------------------------
ARM_L1S = list(range(0, 257)) + [-1, 300, 1000]
ARM_T = dict(cross_t1=64, cross_t2=48)      # high enough that the flat pair's arms (and most textured ones) run to L1
ARM_PINNED_L1S = (-1, 0, 1, 2, 3, 6, 127, 128, 254, 255, 256, 300)


def arm_case(L1, tall=False):
    """(W, H, overrides, seed) of the arm-length case: W = 2 min(L1, 255) + 5, 7 or 9 (odd), H = 5 or 7, D = 5..7;
    tall = the same case transposed, so that the vertical arms reach L1."""
    Lc = min(max(L1, 0), 255)
    W, H = 2 * Lc + 5 + 2 * (L1 % 3), 5 + 2 * (L1 % 2)
    D = 5 + L1 % 3
    over = dict(ARM_T, cross_L1=L1, max_disparity=D)
    if L1 % 5 == 2:
        over.update(min_disparity=-2, max_disparity=D - 2)
    return (H, W, over, 3000 + L1) if tall else (W, H, over, 3000 + L1)


# ---- field edges: one option field at an edge value per case, on a textured shape ----------------------------------
EDGE_W, EDGE_H = 71, 29


def _edge(i, **over):
    """D = 21 (not a multiple of 4); every third case with dmin != 0, alternately negative and positive."""
    D = 21
    r = {0: dict(max_disparity=D), 1: dict(min_disparity=-5, max_disparity=D - 5), 2: dict(min_disparity=3, max_disparity=D + 3)}[i % 3]
    return dict(r, **over)


_EDGE_ROWS = (
    [("cross_L2", v) for v in (-1, 0, 1, 34, 35, 1000)]
    + [("cross_t1", v) for v in (-1, 0, 1, 2, 255, 256)]
    + [("cross_t2", v) for v in (-1, 0, 21)]
    + [(f, v) for f in ("lambda_ad", "lambda_census") for v in (1, 2, 255, 256, 10000, INT32_MAX)]
    + [(("so_p1", "so_p2"), v) for v in ((0.0, 0.0), (2.0, 2.0), (3.0, 1.0), (0.1, 0.3), (1e30, 1e30))]
    + [("so_tso", v) for v in (-1, 0, 1, 255, 256)]
    + [(("irv_ts", "cross_L1"), (v, L1)) for L1 in (34, 160) for v in (-1, 0, 1, 65535, 65536, INT32_MAX)]
    + [("irv_th", v) for v in (-1.0, 0.0, 0.25, 0.5, 1.0, NAN)]
    + [("lrcheck_thres", v) for v in (-1.0, 0.0, 1e-7, 0.5, INF, NAN)]
)


def _edge_name(field, v):
    fields, vals = (field, v) if isinstance(field, tuple) else ((field,), (v,))
    return "edge_" + "_".join(f"{f}={x!r}" for f, x in zip(fields, vals))


def _edge_over(field, v):
    fields, vals = (field, v) if isinstance(field, tuple) else ((field,), (v,))
    return dict(zip(fields, vals))


# ---- flags and range placement ------------------------------------------------------------------------------------
def _flag_cases():
    out = {}
    for bits in range(8):
        lr, fill, disc = bits & 1, (bits >> 1) & 1, (bits >> 2) & 1
        for dmin in (0, -7):
            over = dict(do_lr_check=lr, do_filling=fill, do_discontinuity_adjustment=disc, min_disparity=dmin, max_disparity=dmin + 23)
            out[f"flags_lr{lr}_fill{fill}_disc{disc}_dmin{dmin}"] = (EDGE_W, EDGE_H, over, 4100 + 2 * bits + (dmin != 0))
    return out


# max_search = max(|dmax|, |dmin|) decides whether interpolation walks its rays through the integer offset table (< 4096)
RAY_TABLE_LIMIT = 4096
RANGE_CASES = {
    "range_dmax0": (EDGE_W, EDGE_H, dict(min_disparity=-20, max_disparity=0), 4200),
    "range_all_negative": (EDGE_W, EDGE_H, dict(min_disparity=-30, max_disparity=-9), 4201),
    "range_dmin_eq_W": (EDGE_W, EDGE_H, dict(min_disparity=EDGE_W, max_disparity=EDGE_W + 19), 4202),
    "range_dmin_past_W": (EDGE_W, EDGE_H, dict(min_disparity=100, max_disparity=117), 4203),
    # rows wide enough for matches at |d| about 4090, on either side of the ray-table rule
    "range_search_4095": (4151, 5, dict(min_disparity=4079, max_disparity=4095), 4204),
    "range_search_4096": (4151, 5, dict(min_disparity=4080, max_disparity=4096), 4205),
    "range_search_neg_4095": (4151, 5, dict(min_disparity=-4095, max_disparity=-4078), 4206),
    "range_search_5000": (5101, 3, dict(min_disparity=4990, max_disparity=5000), 4207),
    # D > 254 with L1 <= 127: the wide voting instantiation without forced enumeration
    "range_D256": (301, 13, dict(min_disparity=-3, max_disparity=253), 4208),
}


def cases():
    """name -> (W, H, option overrides, seed), every case of tests/test_option_space.py."""
    out = {}
    for L1 in ARM_L1S:
        out[f"arm_L1={L1}"] = arm_case(L1)
        if L1 % 8 == 0 or L1 in (-1, 300):
            out[f"arm_L1={L1}_tall"] = arm_case(L1, tall=True)
    for i, (f, v) in enumerate(_EDGE_ROWS):
        out[_edge_name(f, v)] = (EDGE_W, EDGE_H, _edge(i, **_edge_over(f, v)), 4000 + i)
    out.update(_flag_cases())
    out.update(RANGE_CASES)
    return out


def option(over):
    return T.default_option(**over)


PINNED = sorted([n for n in cases() if not n.startswith("arm_")] + [f"arm_L1={L1}" for L1 in ARM_PINNED_L1S])


def first_pair(name):
    W, H, over, seed = cases()[name]
    opt = option(over)
    return W, H, opt, GS.sweep_pairs(W, H, opt.max_disparity - opt.min_disparity, seed)[0]


def main():
    assert T.have_ref() or (T.build_oracle() or T.have_ref()), "oracle/_ref is required: set ADC_REFERENCE_DIR to a checkout of the reference"
    out = {}
    for name in PINNED:
        W, H, opt, (left, right) = first_pair(name)
        ref = T.Reference(W, H, opt)
        out[name] = GS.staged_hashes(ref, opt, left, right)
        ref.close()
        print(f"{name} {W}x{H} [{opt.min_disparity},{opt.max_disparity}) final sha {out[name]['MEDIAN/DISP_L'][:16]}")
    (T.GOLDEN_DIR / "golden_options_ref.json").write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
