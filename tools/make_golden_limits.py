#!/usr/bin/env python
"""Generates tests/golden/golden_limits.json: sha256 of the inputs and of every tap after every stage for the large
per-pair volumes of tests/test_size_limits.py, which no test can afford to recompute.

  L1   2100 x 1024 x 256, seeds 1 and 2: 550 M elements, 2.2 GB per volume -- past 2^31 bytes.  The hashes are the
       UNMODIFIED reference's (oracle/_ref), which is defined at this size.
  L2   8400 x 1024 x 256, seed 1: 2.2 G elements per volume -- past 2^31 elements.  The reference indexes its volumes
       with int32 (cost_computor.cpp: y * width_ * disp_range + ...; cross_aggregator.cpp: width_ * height_ *
       disp_range * sizeof(...)), so it is undefined here; the hashes are the oracle's (oracle/adc_oracle.c), which
       indexes with size_t and agrees with the reference wherever the reference is defined.  About 18 GB of host memory.

Usage: make_golden_limits.py [case ...]   (all cases by default; each case runs in its own process, in parallel)
Rerunning it reproduces the file byte for byte.
"""
import json
import sys
import time
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import adc_testlib as T  # noqa: E402

# name: (W, H, D, seed, checker)
CASES = {
    "L1_s1": (2100, 1024, 256, 1, "reference"),
    "L1_s2": (2100, 1024, 256, 2, "reference"),
    "L2_s1": (8400, 1024, 256, 1, "oracle"),
}


def run_case(name):
    w, h, D, seed, checker = CASES[name]
    t0 = time.time()
    left, right = T.synthetic_pair(w, h, D, seed)
    opt = T.default_option(max_disparity=D)
    c = T.Reference(w, h, opt) if checker == "reference" else T.Oracle(w, h, opt)
    assert c.ok, name
    c.begin(left, right)
    hashes = {}
    for st in T.STAGES:
        c.step()
        for tap in T.STAGE_TAPS[st]:
            hashes[f"{st}/{tap}"] = T.sha(c.tap(tap))
    c.close()
    print(name, w, h, D, checker, hashes["MEDIAN/DISP_L"][:16], f"{time.time() - t0:.0f}s", flush=True)
    return name, {"width": w, "height": h, "max_disparity": D, "seed": seed, "checker": checker, "hashes": hashes,
                  "input_sha": [T.sha(left), T.sha(right)]}


def main():
    T.build_oracle()
    names = sys.argv[1:] or list(CASES)
    if any(CASES[n][4] == "reference" for n in names):
        assert T.have_ref(), "oracle/_ref is required: set ADC_REFERENCE_DIR to a checkout of the reference"
    jpath = T.GOLDEN_DIR / "golden_limits.json"
    out = json.loads(jpath.read_text()) if jpath.exists() else {}
    with ProcessPoolExecutor(len(names)) as ex:
        for name, entry in ex.map(run_case, names):
            out[name] = entry
    jpath.write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
