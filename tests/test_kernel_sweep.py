"""Parity sweep over the kernel instantiations and launch-plan branches that the disparity range and the shape select.

The scanline, fused-cost and fused-aggregation kernels are templates whose instantiation follows from the disparity
range (the voting kernels' also from the arm length), and their launch plans (adcensus_b200/csrc/so_plan.h, ca_plan.h)
cut rows and columns differently per shape.

CPU: the instantiations compiled into the library (cuobjdump -symbols), the instantiations every GPU case of this file
reaches by the launch rules, and the assertion that together they reach every one; the plan branch each plan-branch case
is meant to take; the oracle against the reference's hashes of the sweep cases (tests/golden/golden_sweep_ref.json).
GPU: for every disparity range 1..256 and every plan-branch case, one batched call over five distinct pairs (three waves
of two, the last partial; a flat and a white-noise pair between textured ones) that exports every volume and side map,
each pair compared bit for bit with its own oracle run.
"""
import os
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E  # puts tools/ on sys.path
import make_golden_sweep as GS  # case definitions shared with the fixture generator
from sweep_testlib import Case, check_case, plans, reached, so_lanes_per_line  # noqa: F401  (plans: the fixture)


# ---- cases ----------------------------------------------------------------------------------------------------------
def _sweep_case(D):
    W, H, opt, seed = GS.sweep_case(D)
    return Case(f"D{D}", W, H, opt, seed)


def _opt(D, **kw):
    return T.default_option(max_disparity=D, **kw)


LONG_ARMS = dict(cross_L1=255, cross_L2=120, cross_t1=50, cross_t2=25)
# name -> (case, what its plans must be).  Shapes found with the plan executables; test_plan_branch_cases checks them.
PLAN_CASES = {
    # fused cost + first horizontal pass (ca_plan): rows in 2 and 3 segments at L1 = 34, qc = 8, exact and not
    "cost_rows_2seg": (Case("cost_rows_2seg", 501, 23, _opt(45), 61), dict(ca_nseg=2, ca_qc=8)),
    "cost_rows_3seg": (Case("cost_rows_3seg", 861, 19, _opt(64), 62), dict(ca_nseg=3, ca_qc=8)),
    # L1 = 130: 3 segments of 164 outputs, shorter than 2 L1, so a segment's halos span a whole neighbouring segment
    "cost_rows_l1_130": (Case("cost_rows_l1_130", 486, 17, _opt(61, cross_L1=130, cross_L2=40, cross_t1=60, cross_t2=30), 63),
                         dict(ca_nseg=3, ca_qc=8, ca_short=True)),
    # D < 32: four quads per CTA, D not a multiple of 4, rows in 2 segments
    "cost_rows_qc4": (Case("cost_rows_qc4", 825, 13, _opt(23), 64), dict(ca_nseg=2, ca_qc=4)),
    # arms too long for the fused cost plan: the separate cost kernel, exact and padded D; at W = 701 the row does not
    # fit k_arm_sum2t's plan either, so both axes take the LDG double pass with eight quads
    "cost_volume_exact": (Case("cost_volume_exact", 509, 13, _opt(32, **LONG_ARMS), 65), dict(ca_ok=False)),
    "cost_volume_padded_ldg": (Case("cost_volume_padded_ldg", 701, 13, _opt(37, **LONG_ARMS), 66),
                               dict(ca_ok=False, tmaps=False)),
    # k_arm_sum2t down columns cut into segments, one line per CTA, eight and four quads
    "cols_seg_qc8": (Case("cols_seg_qc8", 21, 709, _opt(64), 67), dict(t1_nseg=3, t1_qc=8, t1_lpc=1)),
    "cols_seg_qc4": (Case("cols_seg_qc4", 13, 809, _opt(23), 68), dict(t1_nseg=2, t1_qc=4, t1_lpc=1)),
    # the LDG double pass on rows in segments: Q = 4 (generic QC) and Q = 3 (no TMA plan at all, Q < 4)
    "ldg_rows_q4": (Case("ldg_rows_q4", 1001, 13, _opt(14), 69), dict(ldg0_nseg=2, ldg0_qc=0, t0_nseg=2)),
    "ldg_rows_q3": (Case("ldg_rows_q3", 1001, 13, _opt(11), 70), dict(ldg0_nseg=2, ldg0_qc=0, tmaps=False)),
    # scanline slots of T = 2 steps on the row passes, for 8, 16 and 32 lanes per line, K not FULL, an odd step count
    "so_t2_lps8": (Case("so_t2_lps8", 33, 1057, _opt(61), 71, wave_pairs=8, lanes=1), dict(so_T0=2, lps=8)),
    "so_t2_lps16": (Case("so_t2_lps16", 33, 659, _opt(93), 72, wave_pairs=8, lanes=1), dict(so_T0=2, lps=16)),
    "so_t2_lps32": (Case("so_t2_lps32", 33, 329, _opt(200), 73, wave_pairs=8, lanes=1), dict(so_T0=2, lps=32)),
}

SWEEP_DS = list(range(1, 257))


def _all_cases():
    return [_sweep_case(D) for D in SWEEP_DS] + [c for c, _ in PLAN_CASES.values()]


# ---- CPU ------------------------------------------------------------------------------------------------------------
_SYMBOLS = {
    "k_scanline": re.compile(r"_Z10k_scanlineILi(\d+)ELi(\d+)ELb([01])EE"),
    "k_cost_volume": re.compile(r"_Z13k_cost_volumeILb([01])EE"),
    "k_cost_arm_sum_h": re.compile(r"_Z16k_cost_arm_sum_hILb([01])ELi(\d+)EE"),
    "k_arm_sum2t": re.compile(r"_Z11k_arm_sum2tILb([01])ELi(\d+)EE"),
    "k_arm_sum2": re.compile(r"_Z10k_arm_sum2ILb([01])ELi(\d+)EE"),
    "k_vote_scan": re.compile(r"_Z11k_vote_scanILb([01])EE"),
    "k_vote_push": re.compile(r"_Z11k_vote_pushILb([01])EE"),
}


def library_instantiations():
    """{(template, args...)} of the seven templates, read from the built library's device symbols."""
    from adcensus_b200.build import build_library
    cuobjdump = Path(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")).parent / "cuobjdump"
    if not cuobjdump.exists():
        pytest.skip(f"cuobjdump not found at {cuobjdump}")
    r = subprocess.run([str(cuobjdump), "-symbols", str(build_library())], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    found = set()
    for name, rx in _SYMBOLS.items():
        for m in rx.finditer(r.stdout):
            args = tuple(int(g) for g in m.groups())
            if name == "k_scanline":
                found.add((name, args[0], args[1], bool(args[2])))
            else:
                found.add((name, bool(args[0]), *args[1:]))
    return found


def test_every_instantiation_is_reached(plans):
    """Every instantiation of k_scanline, k_cost_volume, k_cost_arm_sum_h, k_arm_sum2t, k_arm_sum2, k_vote_scan and
    k_vote_push in the library is launched by at least one GPU case of this file; one that no case reaches fails here."""
    lib = library_instantiations()
    assert sum(1 for i in lib if i[0] == "k_scanline") == 32, sorted(lib)
    assert {i[0] for i in lib} == set(_SYMBOLS), sorted(lib)
    by_case = {c.name: reached(c, plans) for c in _all_cases()}
    union = set().union(*by_case.values())
    assert union <= lib, sorted(union - lib)           # the launch rules name only instantiations that exist
    missing = sorted(lib - union)
    assert not missing, f"instantiations no GPU case reaches: {missing}"
    for inst in sorted(lib, key=str):
        print(inst, "reached by", sorted((n for n, r in by_case.items() if inst in r), key=len)[:4])


def test_plan_branch_cases(plans):
    """Each plan-branch case takes the branch it is there for (so that a plan change cannot drop the coverage quietly)."""
    for name, (c, want) in PLAN_CASES.items():
        ca, arm = plans.ca(c), plans.arm(c)
        tmaps = bool(arm[0]["t_ok"] and arm[1]["t_ok"])
        got = dict(ca_ok=bool(ca["ok"]), ca_nseg=ca["nseg"], ca_qc=ca["qc"], ca_short=ca["Ls"] < 2 * min(max(c.L1, 0), 255),
                   tmaps=tmaps, t0_nseg=arm[0]["t_nseg"], t1_nseg=arm[1]["t_nseg"], t1_qc=arm[1]["t_qc"],
                   t1_lpc=arm[1]["t_lpc"], ldg0_nseg=arm[0]["ldg_nseg"], ldg0_qc=8 if arm[0]["ldg_qc_log2"] == 3 else 0,
                   so_T0=plans.so(c, 0)["T"], lps=so_lanes_per_line(c.Dp))
        for k, v in want.items():
            assert got[k] == v, f"{name}: {k} = {got[k]}, expected {v} (plans: ca {ca}, arm {arm})"
        if "t1_lpc" in want:           # k_arm_sum2t takes the columns, one segment's worth per CTA
            assert tmaps and arm[1]["t_nseg"] > 1, (name, arm)
        if "ldg0_nseg" in want:        # the rows take the LDG double pass
            assert not tmaps or arm[0]["t_nseg"] > 1, (name, arm)
        if "so_T0" in want:            # ... with K not FULL and an odd number of steps along the row pass
            K = -(-c.Dp // want["lps"])
            assert c.D != K * want["lps"] and c.W % 2 == 1 and c.H % 2 == 1, name


def test_sweep_case_shapes(plans):
    """The sweep's shapes: W and H not multiples of 4, H not a multiple of either pass's T, W < D on a few ranges,
    min_disparity != 0 on every seventh, both signs; whole-line plans whose line counts are not multiples of lpc."""
    narrow, dmins = 0, set()
    for D in SWEEP_DS:
        c = _sweep_case(D)
        assert c.D == D and c.W % 4 and c.H % 4, (D, c.W, c.H)
        for axis in (0, 1):
            assert c.H % plans.so(c, axis)["T"], (D, c.H)
        narrow += c.W < D
        if c.opt.min_disparity:
            dmins.add(np.sign(c.opt.min_disparity))
        if D == 64:
            arm = plans.arm(c)
            assert arm[0]["t_lpc"] == arm[1]["t_lpc"] == 4 and c.H % 4 and c.W % 4, arm
    assert narrow >= 4 and dmins == {-1, 1}
    assert sum(1 for D in SWEEP_DS if _sweep_case(D).opt.min_disparity) >= len(SWEEP_DS) // 8


@pytest.mark.parametrize("D", GS.GOLDEN_DS)
def test_sweep_oracle_vs_reference(D):
    """The oracle on the sweep cases the other fixtures do not reach (D = 1, 2, 96, 161, 253, ...): every tap after every
    stage of the first pair against the unmodified reference's sha256 (tools/make_golden_sweep.py)."""
    want = E.golden("golden_sweep_ref.json")[str(D)]
    W, H, opt, seed = GS.sweep_case(D)
    left, right = GS.sweep_pairs(W, H, D, seed)[0]
    orc = T.Oracle(W, H, opt)
    got = GS.staged_hashes(orc, opt, left, right)
    orc.close()
    bad = [k for k in want if got[k] != want[k]]
    assert not bad and set(got) == set(want), f"D={D}: taps differing from the reference: {bad}"


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", SWEEP_DS)
def test_disparity_sweep(D):
    """Disparity range D through one batched call (five distinct pairs, waves of two, the last partial) against the
    oracle, every exported volume and side map bit for bit; the ranges pinned to the reference also by the final map's
    sha256."""
    got = check_case(_sweep_case(D))
    if D in GS.GOLDEN_DS:
        want = E.golden("golden_sweep_ref.json")[str(D)]
        assert T.sha(got["disp"][0]) == want["MEDIAN/DISP_L"], f"D={D}: final map differs from the reference's hash"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PLAN_CASES))
def test_plan_branch(name):
    """A shape that sends a kernel down a plan branch the sweep's small shapes do not take, checked as the sweep is."""
    check_case(PLAN_CASES[name][0])
