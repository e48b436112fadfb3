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
import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E  # puts tools/ on sys.path
import make_golden_sweep as GS  # case definitions shared with the fixture generator
from sweep_testlib import (PLAN_CASES, SWEEP_DS, SYMBOLS, all_cases, check_case, library_instantiations, plans,  # noqa: F401
                           reached, so_lanes_per_line, sweep_case)  # (plans: the fixture)


def test_every_instantiation_is_reached(plans):
    """Every instantiation of k_scanline, k_cost_volume, k_cost_arm_sum_h, k_arm_sum2t, k_arm_sum2, k_vote_scan and
    k_vote_push in the library is launched by at least one GPU case of this file; one that no case reaches fails here."""
    lib = library_instantiations()
    assert sum(1 for i in lib if i[0] == "k_scanline") == 32, sorted(lib)
    assert {i[0] for i in lib} == set(SYMBOLS), sorted(lib)
    by_case = {c.name: reached(c, plans) for c in all_cases()}
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
        c = sweep_case(D)
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
    assert sum(1 for D in SWEEP_DS if sweep_case(D).opt.min_disparity) >= len(SWEEP_DS) // 8


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
    got = check_case(sweep_case(D))
    if D in GS.GOLDEN_DS:
        want = E.golden("golden_sweep_ref.json")[str(D)]
        assert T.sha(got["disp"][0]) == want["MEDIAN/DISP_L"], f"D={D}: final map differs from the reference's hash"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PLAN_CASES))
def test_plan_branch(name):
    """A shape that sends a kernel down a plan branch the sweep's small shapes do not take, checked as the sweep is."""
    check_case(PLAN_CASES[name][0])
