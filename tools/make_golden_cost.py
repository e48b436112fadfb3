#!/usr/bin/env python
"""Generates tests/golden/golden_cost_cases.json from the UNMODIFIED reference with an injected cost volume.

tests/c/ref_cost_harness.cpp (oracle/ref_harness.cpp plus a COST step that writes the given volume into the
reference's cost_init_) is compiled here with the reference's sources from the checkout ADC_REFERENCE_DIR names, with
oracle/Makefile's flags, into a temporary directory.  For every case: sha256 of every tap after every stage (GRAY and
CENSUS excluded: cost-input mode does not compute them) for the volume tests/cost_testlib.synthetic_cost generates.
"""
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import adc_testlib as T  # noqa: E402
import cost_testlib as CT  # noqa: E402
import make_golden as G  # noqa: E402

# (W, H, D, option overrides, seed): D % 4 != 0, dmin < 0 and dmin > 0, 8 / 16 / 32 lanes per scanline (D <= 64,
# <= 128, <= 256), D = 256 (region voting with int state), no LR check, discontinuity adjustment
COST_CASES = [(70, 50, 22, {}, 41),
              (80, 40, 32, {"min_disparity": -4, "max_disparity": 28}, 42),
              (80, 40, 32, {"min_disparity": 3, "max_disparity": 35}, 43),
              (70, 30, 64, {"do_lr_check": 0}, 44),
              (150, 30, 130, {"do_discontinuity_adjustment": 1}, 45),
              (300, 20, 256, {}, 46)]
COST_STAGE_TAPS = {st: [t for t in taps if not t.startswith(("GRAY", "CENSUS"))] for st, taps in T.STAGE_TAPS.items()}
REF_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-w",
             "-include", "math.h", "-include", "stdlib.h", "-include", "string.h", "-include", "stdio.h"]
REF_SRCS = ["ADCensusStereo.cpp", "adcensus_util.cpp", "cost_computor.cpp", "cross_aggregator.cpp",
            "scanline_optimizer.cpp", "multistep_refiner.cpp"]


def cost_case_id(case):
    return f"{case[0]}x{case[1]}x{case[2]}-s{case[4]}"


def cost_case_inputs(case):
    """(left, right, option, cost volume f32 [H][W][D]) of a case."""
    w, h, D, over, seed = case
    opt = T.default_option(**{"max_disparity": D, **over})
    D = opt.max_disparity - opt.min_disparity
    left, right = T.synthetic_pair(w, h, D, seed)
    return left, right, opt, CT.synthetic_cost(w, h, D, seed, opt.min_disparity)


def build_ref_cost_harness(out_dir: Path) -> Path:
    ref = Path(os.environ["ADC_REFERENCE_DIR"]) / "AD-Census"
    lib = out_dir / "libadcensus_ref_cost.so"
    subprocess.run(["g++", *REF_FLAGS, f"-I{ref}", f"-I{T.ORACLE_DIR}", "-o", str(lib),
                    str(ROOT / "tests" / "c" / "ref_cost_harness.cpp"), *[str(ref / s) for s in REF_SRCS]], check=True)
    return lib


def main():
    assert os.environ.get("ADC_REFERENCE_DIR"), "set ADC_REFERENCE_DIR to a checkout of the reference"
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_ref_cost_harness(Path(tmp))
        for case in COST_CASES:
            left, right, opt, cost = cost_case_inputs(case)
            h, w, _ = left.shape
            ref = CT.CostReference(lib, w, h, opt)
            ref.begin_cost(left, right, cost)
            hashes = {}
            for st in T.STAGES:
                ref.step()
                for tap in COST_STAGE_TAPS[st]:
                    hashes[f"{st}/{tap}"] = T.sha(G.ref_case_tap(opt, tap, ref.tap(tap)))
            assert hashes["COST/VOL_INIT"] == T.sha(cost)
            ref.close()
            out[cost_case_id(case)] = hashes
            print(cost_case_id(case), "final sha", hashes["MEDIAN/DISP_L"][:16], flush=True)
    (T.GOLDEN_DIR / "golden_cost_cases.json").write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
