"""Tie parity: the first-minimum, strict-comparison and threshold rules of the matching pipeline, on inputs built to tie.

The kernels are bit-exact with the reference only because each reproduces how the reference breaks ties: the WTA's
strict scans, the confidence maps' first minimum, the parabola's flat case, the LR check's `>` and occlusion test,
region voting's lowest-disparity peak and its two thresholds, the interpolation's earliest ray and its no-candidate 0.0,
the edge test and the discontinuity adjustment's `<`, the arm rules' byte compares.  Each differs from its neighbouring
comparison only when two values are exactly equal, which the suite's textured, flat and noise inputs almost never make.
The cases (tools/make_golden_ties.py) are input families built to tie -- periodic columns and tiles, a complementary dot
lattice, colour steps of exactly cross_t1 / cross_t2, shifts at the range ends, identical views, occlusion bars,
piecewise-constant regions, and cost volumes periodic in d, with plateaus, with minima at the range ends, in blocks
whose map steps by exactly 1.25, and in teeth whose halves vote 2k and 2k + 1 in equal counts -- each under every
option set, two of which run the defaults with region voting's enumeration or the interpolation's generic ray walk.

CPU: the oracle's tie counters (orc_tie_counts) show which rules each family decides, and that every rule is decided
somewhere in this file, against the counts on the suite's other content; the oracle reproduces the unmodified
reference's hashes on the first pair of every pinned case (tests/golden/golden_ties_ref.json).
GPU: every case through one batched call, plain and pipelined, every volume and side map (with the confidence maps)
bit for bit against each pair's oracle run; the first pair of every family through the staged debug run and the one-pair
match with its right map.
"""
import functools
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import adc_testlib as T
import cost_testlib as CT
import engine_testlib as E  # puts tools/ on sys.path
import maps_testlib as MT
import make_golden_cost as GC
import make_golden_sweep as GS
import make_golden_ties as GT  # case definitions shared with the fixture generator
from sweep_testlib import Case, check_case

CASES = GT.cases()
FAMILIES = [*GT.IMAGE_FAMILIES, *GT.COST_FAMILIES]


def _oracle(opt, w, h, cost):
    return T.Oracle(w, h, opt) if cost is None else CT.CostOracle(w, h, opt)


def _run(opt, left, right, cost, w=GT.W, h=GT.H, stop="MEDIAN"):
    """One oracle run up to `stop`: (tie counts, the checker, still open)."""
    orc = _oracle(opt, w, h, cost)
    orc.begin(left, right) if cost is None else orc.begin_cost(left, right, cost)
    orc.run_to(stop)
    return orc.tie_counts(), orc


def _counts(opt, left, right, cost=None, w=GT.W, h=GT.H):
    t, orc = _run(opt, left, right, cost, w, h)
    orc.close()
    return t


@functools.cache
def case_counts(name):
    """Tie counts of every pair of a case, summed."""
    opt = GT.option(name)
    with ThreadPoolExecutor(GT.N_PAIRS) as ex:
        per = list(ex.map(lambda p: _counts(opt, *p), GT.pairs(name)))
    return {k: sum(t[k] for t in per) for k in T.TIES}


# ---- CPU: the oracle against the reference ------------------------------------------------------------------------
@pytest.mark.parametrize("name", GT.PINNED)
def test_tie_oracle_vs_reference(name):
    """The oracle on the first pair of every case: every tap after every stage against the unmodified reference's
    sha256 (tools/make_golden_ties.py)."""
    want = E.golden("golden_ties_ref.json")[name]
    opt = GT.option(name)
    left, right, cost = GT.pairs(name)[0]
    orc = _oracle(opt, GT.W, GT.H, cost)
    got = GT.staged_hashes(orc, opt, left, right, cost)
    orc.close()
    bad = [k for k in want if got[k] != want[k]]
    assert not bad and set(got) == set(want), f"{name}: taps differing from the reference: {bad}"


def test_golden_covers_the_pinned_cases():
    assert sorted(E.golden("golden_ties_ref.json")) == GT.PINNED


# ---- CPU: the rules each family decides -----------------------------------------------------------------------------
# family -> the counters it is there for, each > 0 summed over its option sets
FAMILY_REACH = {
    "periodic_cols": ["WTA_L", "WTA_R", "SUBPIX_FLAT", "OCCL_EQ", "LR_EQ", "INTERP_DIST", "INTERP_NONE"],
    "periodic_tiles": ["WTA_L", "WTA_R", "SUBPIX_FLAT", "OCCL_EQ", "LR_EQ", "INTERP_DIST"],
    "dot_lattice": ["WTA_L", "WTA_R", "VOTE_PEAK", "VOTE_TS", "INTERP_DIST"],
    "saturated_steps": ["ARM_T1", "ARM_T2", "ARM_L2", "LR_EQ"],
    "range_ends": ["WTA_L", "SUBPIX_FLAT", "INTERP_NONE"],
    "identical": ["INTERP_NONE", "SUBPIX_FLAT"],
    "occlusion_bars": ["OCCL_EQ", "VOTE_PEAK", "VOTE_TS", "INTERP_DIST"],
    "piecewise_regions": ["WTA_L", "VOTE_TS", "INTERP_DIST"],
    "cost_periodic_d": ["WTA_L", "WTA_R", "VOTE_TS", "INTERP_DIST", "LR_EQ", "DISC_EQ"],
    "cost_plateau": ["WTA_L", "VOTE_PEAK", "VOTE_TS", "INTERP_DIST"],
    "cost_range_ends": ["INTERP_NONE", "INTERP_DIST", "OCCL_EQ"],
    "cost_blocks": ["WTA_L", "WTA_R", "EDGE_EQ", "SUBPIX_FLAT"],
    "cost_vote_pairs": ["VOTE_PAIR", "VOTE_PEAK", "VOTE_TS", "OCCL_EQ", "INTERP_DIST"],
}


def test_vote_pairs_reach_the_narrow_histogram():
    """VOTE_PAIR (bins 2k and 2k + 1 tied at a filled peak) is decided on cases that vote with the narrow histogram
    (D <= 254 and L1 <= 127: two bins per word, so the lane's own scan breaks the tie, not the cross-lane minimum)."""
    narrow = [n for n, (f, _) in CASES.items() if f == "cost_vote_pairs"
              and GT.option(n).max_disparity - GT.option(n).min_disparity <= 254 and GT.option(n).cross_L1 <= 127]
    assert sum(case_counts(n)["VOTE_PAIR"] > 0 for n in narrow) >= 5, {n: case_counts(n)["VOTE_PAIR"] for n in narrow}


@pytest.mark.parametrize("family", FAMILIES)
def test_family_reaches_its_rules(family):
    """Each family decides the rules it is there for, by the oracle's tie counters over its option sets."""
    tot = dict.fromkeys(T.TIES, 0)
    for name, (fam, _) in CASES.items():
        if fam == family:
            for k, v in case_counts(name).items():
                tot[k] += v
    missed = [k for k in FAMILY_REACH[family] if tot[k] == 0]
    assert not missed, f"{family}: no tie decided for {missed}; counts {tot}"


def test_every_tie_counter_is_reached():
    """Across the file every tie counter is > 0: every rule is decided by an exact equality on some input here."""
    tot = dict.fromkeys(T.TIES, 0)
    for name in CASES:
        for k, v in case_counts(name).items():
            tot[k] += v
    print("tie counts over the file:", tot)
    assert all(v > 0 for v in tot.values()), tot


# The counts on the suite's other content, each summed over its pairs: the sweep's five pairs at 96 x 64, D = 32
# (seed 11), the stage-parity cases (engine_testlib.PARITY_CASES) and Cone.  They are recorded so that the gap this file
# closes stays written down: there LR_EQ, EDGE_EQ and DISC_EQ are never decided, OCCL_EQ only on the parity cases,
# VOTE_TH twice and VOTE_PAIR six times.  (WTA_L counts every later d equal to the best so far, including ties the scan
# later leaves.)
EXISTING_COUNTS = {
    "sweep_pairs": {"WTA_L": 3885, "WTA_R": 1, "SUBPIX_FLAT": 29, "VOTE_PEAK": 7, "VOTE_TS": 32, "INTERP_DIST": 52,
                    "INTERP_NONE": 6423, "ARM_T1": 16188, "ARM_T2": 112, "ARM_L2": 3249},
    "parity_cases": {"WTA_L": 494553, "WTA_R": 5, "SUBPIX_FLAT": 1376, "OCCL_EQ": 78, "VOTE_PEAK": 39, "VOTE_TS": 228,
                     "ARM_T1": 89408, "ARM_T2": 2196, "ARM_L2": 25686, "VOTE_PAIR": 5},
    "cone": {"WTA_L": 55022, "WTA_R": 9, "SUBPIX_FLAT": 926, "VOTE_PEAK": 9, "VOTE_TS": 370, "VOTE_TH": 2,
             "INTERP_DIST": 859, "INTERP_NONE": 5, "ARM_T1": 68165, "ARM_T2": 4967, "ARM_L2": 35736, "VOTE_PAIR": 1},
}


@functools.cache
def existing_counts():
    out = {}
    opt = T.default_option(max_disparity=32)
    per = [_counts(opt, l, r, w=96, h=64) for l, r in GS.sweep_pairs(96, 64, 32, 11)]
    out["sweep_pairs"] = {k: sum(t[k] for t in per) for k in T.TIES}
    per = []
    for w, h, D, over, seed in E.PARITY_CASES:
        o = T.default_option(**{"max_disparity": D, **over})
        per.append(_counts(o, *T.synthetic_pair(w, h, o.max_disparity - o.min_disparity, seed), w=w, h=h))
    out["parity_cases"] = {k: sum(t[k] for t in per) for k in T.TIES}
    left, right = T.load_cone()
    out["cone"] = _counts(T.default_option(), left, right, w=left.shape[1], h=left.shape[0])
    return out


def test_tie_counts_on_the_existing_content():
    """The tie counts on the suite's other inputs are the recorded ones (EXISTING_COUNTS)."""
    got = existing_counts()
    for k, v in got.items():
        print(k, {t: n for t, n in v.items() if n})
    assert got == {k: {t: v.get(t, 0) for t in T.TIES} for k, v in EXISTING_COUNTS.items()}


def _far_tie_fraction(vol):
    """Fraction of pixels whose curve repeats its minimum at least 2 from its first minimum."""
    D = vol.shape[2]
    d1 = vol.argmin(axis=2)
    mn = np.take_along_axis(vol, d1[..., None], 2)
    far = (vol == mn) & (np.abs(np.arange(D)[None, None] - d1[..., None]) >= 2)
    return float(far.any(axis=2).mean())


# cost family -> the fraction of pixels (of the first pair under the defaults) whose SO4 curve keeps a far tie.  The
# range-end and block families are built for other rules; under the scanline penalties their far ties do not survive.
FAR_TIE_FRACTION = {"cost_periodic_d": 0.9, "cost_plateau": 0.01}


@pytest.mark.parametrize("family", list(FAR_TIE_FRACTION))
def test_cost_far_ties_survive_to_the_optimised_volume(family):
    """The cost families' exact far ties survive aggregation and all four scanline passes into the oracle's SO4
    volume (the one the WTA and the confidence maps read), on at least the stated fraction of pixels."""
    name = f"{family}/default"
    left, right, cost = GT.pairs(name)[0]
    _, orc = _run(GT.option(name), left, right, cost, stop="SO4")
    frac = _far_tie_fraction(orc.tap("VOL_AGGR"))
    orc.close()
    print(family, "far-tie fraction", frac)
    assert frac >= FAR_TIE_FRACTION[family], frac


# The families that make no PEAK_RATIO tie, and why; every other case must.  Their rows are aperiodic, or each curve has
# one designed minimum, so no d at least 2 from d1 matches it exactly after aggregation and the scanline passes.
NO_PEAK_TIE = {
    "dot_lattice": "isolated dots: a dot meets its inverse at one d only",
    "saturated_steps": "the textured strip and the 0 / 255 blocks are aperiodic",
    "range_ends": "white-noise rows: one d matches",
    "identical": "d = 0 is the only exact match",
    "piecewise_regions": "rectangles of random widths: one d matches",
    "cost_range_ends": "one designed minimum per curve",
    "cost_blocks": "one designed minimum (or plateau adjacent to it) per curve",
    "cost_vote_pairs": "one designed minimum per curve",
}


@pytest.mark.parametrize("name", [n for n, (f, _) in CASES.items() if f not in NO_PEAK_TIE])
def test_peak_ratio_meets_a_tie(name):
    """PEAK_RATIO's c2 equals c1 (a ratio of exactly 1 from a far tie) on pixels of one of the case's pairs (their SO4
    volumes), so the first-minimum rule of the confidence maps decides something there."""
    for left, right, cost in GT.pairs(name):
        _, orc = _run(GT.option(name), left, right, cost, stop="SO4")
        vol = orc.tap("VOL_AGGR").copy()
        orc.close()
        c1, ratio = MT.confidence(vol)
        if _far_tie_fraction(vol) > 0 and ((ratio == 1) & (c1 > 0)).any():
            return
    raise AssertionError(f"{name}: no pair has a far tie at its minimum")


def test_dot_lattice_reaches_the_cost_extremes():
    """The dot lattice reaches the AD sum 765 (the last entry of the table) and the largest census Hamming distance,
    62, at a valid (x, d): from the images and the oracle's CENSUS_L / CENSUS_R taps."""
    name = "dot_lattice/default"
    opt = GT.option(name)
    left, right, _ = GT.pairs(name)[0]
    _, orc = _run(opt, left, right, None, stop="COST")
    cl, cr = orc.tap("CENSUS_L").copy(), orc.tap("CENSUS_R").copy()
    orc.close()
    W = GT.W
    ad_max = ham_max = 0
    for d in range(opt.min_disparity, opt.max_disparity):
        x0, x1 = max(0, d), min(W, W + d)
        if x0 >= x1:
            continue
        ad = np.abs(left[:, x0:x1].astype(int) - right[:, x0 - d:x1 - d].astype(int)).sum(axis=2)
        ad_max = max(ad_max, int(ad.max()))
        x = np.bitwise_xor(cl[:, x0:x1], cr[:, x0 - d:x1 - d])
        ham = np.unpackbits(x.view(np.uint8), axis=-1).reshape(*x.shape, 64).sum(axis=-1)
        ham_max = max(ham_max, int(ham.max()))
    assert ad_max == 765 and ham_max == 62, (ad_max, ham_max)


# ---- GPU ------------------------------------------------------------------------------------------------------------
COST_INPUTS = [(layout, dtype) for layout in ("hwd", "dhw") for dtype in ("f32", "f16", "bf16")]


def cost_input_of(name):
    """(layout, element type) a cost case is handed to the engine in: the option sets cycle through every pair."""
    return COST_INPUTS[list(GT.OPTION_SETS).index(CASES[name][1]) % len(COST_INPUTS)]


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True], ids=["plain", "pipelined"])
@pytest.mark.parametrize("name", list(CASES))
def test_tie_case(name, pipelined):
    """Every case's five pairs through one batched call (waves of two, the last partial), every exported volume, both
    WTA maps, the outlier lists, MIN_COST / PEAK_RATIO and the final map bit for bit against each pair's oracle run;
    the first pair's final map also against the reference's hash."""
    c = Case(name, GT.W, GT.H, GT.option(name), GT.seed_of(name))
    layout, dtype = cost_input_of(name) if GT.is_cost(name) else ("hwd", "f32")
    got = check_case(c, debug_flags=GT.debug_flags(name), pairs=GT.pairs(name), confidence=True, pipelined=pipelined,
                     cost_layout=layout, cost_dtype=dtype)
    if name not in GT.REF_DIVERGES:
        fam, os_ = CASES[name]
        pinned = f"{fam}/default" if os_ in GT.DEFAULT_RUNS else name
        assert T.sha(got["disp"][0]) == E.golden("golden_ties_ref.json")[pinned]["MEDIAN/DISP_L"]


def test_cost_cases_cover_every_input_type():
    for fam in GT.COST_FAMILIES:
        assert {cost_input_of(f"{fam}/{o}") for o in GT.OPTION_SETS} == set(COST_INPUTS), fam


@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
def test_tie_family_staged(family):
    """The first pair of every family under the defaults and under the flat-penalty discontinuity set: the staged debug
    run tap by tap against the oracle, then the one-pair match and its right map."""
    for os_ in ("default", "flat_so_disc"):
        name = f"{family}/{os_}"
        opt = GT.option(name)
        left, right, cost = GT.pairs(name)[0]
        taps = T.STAGE_TAPS if cost is None else GC.COST_STAGE_TAPS
        eng = E.engine(GT.W, GT.H, opt)
        orc = _oracle(opt, GT.W, GT.H, cost)
        orc.begin(left, right) if cost is None else orc.begin_cost(left, right, cost)
        for st in T.STAGES:
            orc.step()
            eng.debug_run(left, right, st) if cost is None else eng.debug_run_cost(left, right, cost, "hwd", st)
            for tap in taps[st]:
                E.same(f"{name} {st}/{tap}", eng.tap(tap), orc.tap(tap))
        want_r = orc.tap("DISP_R").copy()
        orc.close()
        orc = _oracle(opt, GT.W, GT.H, cost)
        want = orc.match(left, right) if cost is None else orc.match_cost(left, right, cost)
        orc.close()
        got = eng.match(left, right) if cost is None else eng.match_cost(left, right, cost, "hwd")
        E.same(f"{name} match", got, want)
        E.same(f"{name} right map", eng.right_disparity(), want_r)
        eng.close()
