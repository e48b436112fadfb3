"""Option-space parity: every adc_option field at its edges, against the oracle and the reference, and the values
adc_create rejects.

The test_kernel_sweep cases run the default non-range options; the kernels also branch on option values (arm lengths,
thresholds, penalty classes, voting and refinement thresholds, the interpolation's ray table).  The cases are defined in
tools/make_golden_options.py:
  - arm-length sweep: cross_L1 over 0..256, -1, 300 and 1000 on rows about two arms wide (every 8th also transposed);
  - field edges: one field at an edge value per case (cross_L2, cross_t1, cross_t2, lambda_*, so_p1/so_p2, so_tso,
    irv_ts with L1 on both sides of 127, irv_th, lrcheck_thres), including NaN and infinities where accepted;
  - the eight flag combinations, with dmin = 0 and dmin < 0;
  - range placement: every candidate outside the image (dmax <= 0, dmin >= W), and max_search on either side of the
    interpolation's ray-table rule.

CPU: the cases reach the branches they are there for; the oracle reproduces the reference's hashes of the pinned cases
(tests/golden/golden_options_ref.json); adc_create rejects exactly the values outside the option domain.
GPU: every case through one batched call over five pairs (waves of two, the last partial), every exported volume and
side map bit for bit against each pair's oracle run, the pinned cases also by the final map's sha256; a few cases
through the staged debug run, tap by tap.
"""
import ctypes
import math

import pytest

import adc_testlib as T
import engine_testlib as E  # puts tools/ on sys.path
import make_golden_options as GO  # case definitions shared with the fixture generator
import make_golden_sweep as GS
from sweep_testlib import Case, check_case, plans, reached  # noqa: F401  (plans: the fixture)

CASES = GO.cases()
ADC_DBG_VOTE_ENUM = 2


def _case(name):
    W, H, over, seed = CASES[name]
    return Case(name, W, H, GO.option(over), seed)


def _golden():
    return E.golden("golden_options_ref.json")


def arm_rec_words(L1):
    """Words of one window record, by arm_L1c / arm_rec_words (adcensus_b200/csrc/ca_plan.h)."""
    L1c = min(max(L1, 0), 255)
    return (1 + (2 * L1c + 4 + 7) // 8 + 3) // 4 * 4


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_option_case_coverage(plans):
    """The cases reach the option branches they are there for, so that a change to the cases cannot drop one quietly:
    t1 <= 0, L2 < 0, L2 >= L1; every record size arm_rec_words takes for L1 in 0..255; both voting instantiations,
    each with and without enumeration; both sides of the ray-table rule (max_search < 4096 and >= 4096)."""
    opts = {n: GO.option(c[2]) for n, c in CASES.items()}
    assert any(o.cross_t1 <= 0 for o in opts.values())
    assert any(o.cross_L2 < 0 for o in opts.values())
    assert any(o.cross_L2 >= o.cross_L1 > 0 for o in opts.values())
    assert {arm_rec_words(o.cross_L1) for o in opts.values()} >= {arm_rec_words(L1) for L1 in range(256)}
    assert set(range(-1, 257)) | {300, 1000} <= {o.cross_L1 for o in opts.values()}
    # voting: WIDE iff D > 254 or L1 > 127 (k_vote.cu); enumeration forced for L1 > 127 or by ADC_DBG_VOTE_ENUM, which
    # the staged cases set on the narrow instantiation
    vote = set()
    for n, o in opts.items():
        L1c = min(max(o.cross_L1, 0), 255)
        wide = (o.max_disparity - o.min_disparity) > 254 or L1c > 127
        vote.add((wide, L1c > 127 or STAGED.get(n, 0) == ADC_DBG_VOTE_ENUM))
    assert vote == {(False, False), (False, True), (True, False), (True, True)}, vote
    for n in ("range_D256", "arm_L1=128", "arm_L1=127"):         # the sweep's launch rules agree on the instantiation
        wide = n != "arm_L1=127"
        assert ("k_vote_push", wide) in reached(_case(n), plans), n
    search = {max(abs(o.max_disparity), abs(o.min_disparity)) for o in opts.values()}
    assert min(search) > 1 and max(s for s in search if s < GO.RAY_TABLE_LIMIT) == GO.RAY_TABLE_LIMIT - 1
    assert GO.RAY_TABLE_LIMIT in search and max(search) > GO.RAY_TABLE_LIMIT
    # every candidate outside the image, on both sides
    assert any(o.max_disparity <= 0 for o in opts.values())
    assert any(o.min_disparity >= CASES[n][0] for n, o in opts.items())
    # all eight flag combinations, each with dmin = 0 and dmin < 0
    flags = {(o.do_lr_check, o.do_filling, o.do_discontinuity_adjustment, o.min_disparity < 0) for n, o in opts.items()
             if n.startswith("flags_")}
    assert len(flags) == 16
    # the arm-sweep shapes: rows about two arms wide, odd, small heights
    for L1 in GO.ARM_L1S:
        W, H, _, _ = CASES[f"arm_L1={L1}"]
        assert W % 2 and H % 2 and H <= 7 and 0 < W - 2 * min(max(L1, 0), 255) < 10, (L1, W, H)


@pytest.mark.parametrize("name", GO.PINNED)
def test_option_oracle_vs_reference(name):
    """The oracle on the pinned cases: every tap after every stage of the first pair against the unmodified
    reference's sha256 (tools/make_golden_options.py)."""
    want = _golden()[name]
    W, H, opt, (left, right) = GO.first_pair(name)
    orc = T.Oracle(W, H, opt)
    got = GS.staged_hashes(orc, opt, left, right)
    orc.close()
    bad = [k for k in want if got[k] != want[k]]
    assert not bad and set(got) == set(want), f"{name}: taps differing from the reference: {bad}"


def test_golden_covers_the_pinned_cases():
    assert sorted(_golden()) == GO.PINNED


INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
REJECTED = [
    # (field(s), value(s), what the message names)
    ("lambda_ad", 0, "lambda_ad"), ("lambda_ad", -1, "lambda_ad"), ("lambda_ad", INT32_MIN, "lambda_ad"),
    ("lambda_census", 0, "lambda_census"), ("lambda_census", -30, "lambda_census"),
    ("so_p1", -1.0, "so_p1"), ("so_p1", -1e-30, "so_p1"), ("so_p1", math.inf, "so_p1"), ("so_p1", -math.inf, "so_p1"),
    ("so_p1", math.nan, "so_p1"), ("so_p2", -3.0, "so_p2"), ("so_p2", math.inf, "so_p2"), ("so_p2", math.nan, "so_p2"),
    (("min_disparity", "max_disparity"), (INT32_MIN, INT32_MIN + 64), "min_disparity"),
    (("min_disparity", "max_disparity"), (-2**30 - 8, 2**30 + 8), "max - min"),
    (("min_disparity", "max_disparity"), (INT32_MIN + 1, INT32_MAX), "max - min"),
    (("min_disparity", "max_disparity"), (-INT32_MAX, -INT32_MAX + 64), "x - d"),
    (("min_disparity", "max_disparity"), (INT32_MAX - 64, INT32_MAX), "x + d"),
]


def _set(o, fields, vals):
    if not isinstance(fields, tuple):
        fields, vals = (fields,), (vals,)
    for f, v in zip(fields, vals):
        setattr(o, f, v)
    return o


@pytest.mark.parametrize("fields,vals,names", REJECTED, ids=[f"{f}={v}" for f, v, _ in REJECTED])
def test_adc_create_rejects_values_outside_the_domain(fields, vals, names):
    """Values for which the reference is undefined or its cost volume non-finite fail with ADC_ERR_ARG and a message
    naming the field, before any device work (so also on a machine without a GPU); the drop-in class's Initialize
    returns false."""
    import adcensus_b200 as A
    L = A.load_library()
    o = _set(A.ADCensusOption(), fields, vals)
    h = ctypes.c_void_p()
    assert L.adc_create(80, 40, ctypes.byref(o), None, ctypes.byref(h)) == 1 and not h.value
    msg = L.adc_last_error().decode()
    assert "adc_create" in msg and names in msg, msg
    assert A.ADCensusStereo().Initialize(80, 40, o) is False


ACCEPTED = [
    ("lambda_ad", 1), ("lambda_census", 1), ("lambda_ad", INT32_MAX), ("so_p1", 0.0), ("so_p2", 0.0), ("so_p1", -0.0),
    ("so_p2", 3.4e38), ("irv_th", math.nan), ("lrcheck_thres", math.nan), ("irv_th", -math.inf), ("lrcheck_thres", math.inf),
    ("cross_L1", INT32_MIN), ("cross_L2", INT32_MIN), ("cross_t1", INT32_MIN), ("so_tso", INT32_MIN), ("irv_ts", INT32_MIN),
    (("min_disparity", "max_disparity"), (-(INT32_MAX - 79), -(INT32_MAX - 79) + 64)),
    (("min_disparity", "max_disparity"), (INT32_MAX - 80 - 64 + 1, INT32_MAX - 80 + 1)),
]


@pytest.mark.parametrize("fields,vals", ACCEPTED, ids=[f"{f}={v}" for f, v in ACCEPTED])
def test_adc_create_accepts_the_domain_edges(fields, vals):
    """The edges of the domain pass the option checks: without a GPU adc_create then fails only at the device probe
    (ADC_ERR_CUDA); with one it creates the engine."""
    import torch
    import adcensus_b200 as A
    L = A.load_library()
    o = _set(A.ADCensusOption(), fields, vals)
    h = ctypes.c_void_p()
    rc = L.adc_create(80, 40, ctypes.byref(o), None, ctypes.byref(h))
    if torch.cuda.is_available():
        assert rc == 0, L.adc_last_error()
        L.adc_destroy(h)
    else:
        assert rc == 2 and b"no CUDA device" in L.adc_last_error(), L.adc_last_error()


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_option_case(name):
    """One option-space case through one batched call (five distinct pairs, waves of two, the last partial) against the
    oracle, every exported volume and side map bit for bit; the pinned cases also by the final map's sha256."""
    got = check_case(_case(name))
    if name in GO.PINNED:
        assert T.sha(got["disp"][0]) == _golden()[name]["MEDIAN/DISP_L"], f"{name}: final map differs from the reference's hash"


# name -> debug_flags of the staged run (ADC_DBG_VOTE_ENUM: region voting enumerates on the narrow instantiation)
STAGED = {
    "arm_L1=0": 0, "arm_L1=255": 0, "arm_L1=256_tall": 0,
    "edge_cross_t1=-1": 0, "edge_irv_th=nan": ADC_DBG_VOTE_ENUM, "edge_lrcheck_thres=nan": 0,
    "edge_so_p1=0.1_so_p2=0.3": ADC_DBG_VOTE_ENUM, "range_dmin_eq_W": 0, "range_dmax0": ADC_DBG_VOTE_ENUM,
    "range_search_4096": 0,
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STAGED))
def test_option_case_staged(name):
    """Every pair of a few cases through the staged debug run, every tap after every stage against the oracle."""
    W, H, over, seed = CASES[name]
    opt = GO.option(over)
    eng = E.engine(W, H, opt, debug_flags=STAGED[name])
    for i, (left, right) in enumerate(GS.sweep_pairs(W, H, opt.max_disparity - opt.min_disparity, seed)):
        orc = T.Oracle(W, H, opt)
        orc.begin(left, right)
        for st in T.STAGES:
            orc.step()
            eng.debug_run(left, right, st)
            for tap in T.STAGE_TAPS[st]:
                E.same(f"{name} pair {i} {st}/{tap}", eng.tap(tap), orc.tap(tap))
        orc.close()
    eng.close()
