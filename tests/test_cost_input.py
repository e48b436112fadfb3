"""Cost-input mode (adc_match_cost*): the pipeline after stage 1 run on a caller's matching-cost volume.

CPU: the C restatement with an injected volume against the unmodified reference's hashes (tests/golden/
golden_cost_cases.json, tools/make_golden_cost.py), argument errors, the volume generator.
GPU: round trips of the engine's own AD-census volume, stage parity of every layout x element type, the value domain,
the batched device entry point.
"""
import numpy as np
import pytest

import adc_testlib as T
import cost_testlib as CT
import engine_testlib as E  # puts tools/ on sys.path
import make_golden as G
import make_golden_cost as GC

LAYOUTS = ["hwd", "dhw"]
DTYPES = ["f32", "f16", "bf16"]


def _as_input(vol_hwd, layout, dtype):
    """(array, dtype argument) of a [H][W][D] f32 volume in the given layout and element type."""
    v = vol_hwd if layout == "hwd" else np.ascontiguousarray(vol_hwd.transpose(2, 0, 1))
    if dtype == "f32":
        return np.ascontiguousarray(v, np.float32), "f32"
    if dtype == "f16":
        h = v.astype(np.float16)
        assert np.array_equal(h.astype(np.float32).view(np.uint32), np.ascontiguousarray(v).view(np.uint32))
        return h, "f16"
    return CT.to_bf16_bits(v), "bf16"


# ---- CPU ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", GC.COST_CASES, ids=[GC.cost_case_id(c) for c in GC.COST_CASES])
def test_cost_oracle_vs_reference_golden(case):
    """Every tap after every stage of the restatement with an injected volume: sha256 equal to the reference's."""
    want = E.golden("golden_cost_cases.json")[GC.cost_case_id(case)]
    left, right, opt, cost = GC.cost_case_inputs(case)
    h, w, _ = left.shape
    orc = CT.CostOracle(w, h, opt)
    orc.begin_cost(left, right, cost)
    for st in T.STAGES:
        orc.step()
        for tap in GC.COST_STAGE_TAPS[st]:
            assert T.sha(G.ref_case_tap(opt, tap, orc.tap(tap))) == want[f"{st}/{tap}"], f"{st}/{tap}"
    orc.close()


def test_cost_cases_exercise_refinement():
    """The generated volumes leave outliers for region voting and interpolation to fix (not a trivial map)."""
    left, right, opt, cost = GC.cost_case_inputs(GC.COST_CASES[0])
    h, w, _ = left.shape
    orc = CT.CostOracle(w, h, opt)
    orc.begin_cost(left, right, cost)
    orc.run_to("OUTLIER")
    assert len(orc.tap("MISMATCHES")) > 100 and len(orc.tap("OCCLUSIONS")) > 0
    orc.run_to("MEDIAN")
    d = orc.tap("DISP_L")
    assert np.isfinite(d).mean() > 0.8


def test_synthetic_cost_properties():
    a = CT.synthetic_cost(60, 40, 22, 5, dmin=-3)
    assert a.shape == (40, 60, 22) and a.dtype == np.float32
    assert np.array_equal(a, CT.synthetic_cost(60, 40, 22, 5, dmin=-3))          # deterministic
    assert a.min() >= 0 and a.max() < 4 and np.array_equal(a * 32, np.floor(a * 32))
    assert np.array_equal(a.astype(np.float16).astype(np.float32), a)            # exact in f16 ...
    CT.to_bf16_bits(a)                                                           # ... and in bf16
    assert ((a < 0.5).sum(axis=2) == 1).all()                                    # one planted minimum per pixel


def test_cost_domain_restatement():
    x = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, -1.5, 2.5, 65535.99, 65536.0, 1e30, -np.nan], np.float32)
    got = CT.cost_domain(x)
    want = np.array([65536, 65536, 0, 0, 0, 0, 2.5, 65535.99, 65536, 65536, 65536], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_cost_argument_errors_need_no_gpu():
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    buf = np.zeros(16, np.float32)
    p = buf.ctypes.data
    assert L.adc_match_cost(None, p, p, p, A.COST_HWD, A.COST_F32, p) == 1
    assert b"engine is NULL" in L.adc_last_error()
    assert L.adc_match_cost(None, p, p, p, 2, A.COST_F32, p) == 1
    assert b"layout" in L.adc_last_error()
    assert L.adc_match_cost(None, p, p, p, A.COST_DHW, 3, p) == 1
    assert b"element type" in L.adc_last_error()
    assert L.adc_match_cost_batch_device(None, 1, p, p, p, -1, A.COST_F32, p, None) == 1
    assert b"layout" in L.adc_last_error()
    assert L.adc_match_cost_batch_device(None, 1, p, p, None, A.COST_HWD, A.COST_BF16, p, None) == 1
    assert L.adc_debug_run_cost(None, p, p, p, A.COST_HWD, A.COST_F16, 0) == 1
    assert L.adc_debug_run_cost(None, p, p, p, A.COST_HWD, 7, 0) == 1
    assert b"element type" in L.adc_last_error()


# ---- GPU ------------------------------------------------------------------------------------------
ROUND_TRIP = [(97, 61, 24, {}, 2), (130, 70, 37, {}, 3), (80, 60, 32, {"min_disparity": -4, "max_disparity": 28}, 32)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cone"] + [f"{c[0]}x{c[1]}x{c[2]}-s{c[4]}" for c in ROUND_TRIP])
def test_own_volume_round_trip(case, cone):
    """The engine's own AD-census volume fed back as HWD f32 and as DHW f32 reproduces match() and the right map."""
    if case == "cone":
        left, right = cone
        opt = T.default_option()
    else:
        w, h, D, over, seed = ROUND_TRIP[[f"{c[0]}x{c[1]}x{c[2]}-s{c[4]}" for c in ROUND_TRIP].index(case)]
        opt = T.default_option(**{"max_disparity": D, **over})
        left, right = T.synthetic_pair(w, h, opt.max_disparity - opt.min_disparity, seed)
    h, w, _ = left.shape
    eng = E.engine(w, h, opt)
    eng.debug_run(left, right, "COST")
    vol = eng.tap("VOL_INIT").copy()
    want = eng.match(left, right)
    want_r = eng.right_disparity()
    if case == "cone":
        assert T.sha(want).startswith("77d70a58d1aa5c71")
    for layout in LAYOUTS:
        v = vol if layout == "hwd" else np.ascontiguousarray(vol.transpose(2, 0, 1))
        got = eng.match_cost(left, right, v, layout)
        E.same(f"{layout} map", got, want)
        E.same(f"{layout} right map", eng.right_disparity(), want_r)
        if case == "cone":
            assert T.sha(got).startswith("77d70a58d1aa5c71")
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", GC.COST_CASES, ids=[GC.cost_case_id(c) for c in GC.COST_CASES])
def test_cost_stage_parity_vs_reference(case):
    """Every golden cost case, every layout x element type, every stage: the reference's hashes; VOL_INIT = the volume."""
    want = E.golden("golden_cost_cases.json")[GC.cost_case_id(case)]
    left, right, opt, cost = GC.cost_case_inputs(case)
    h, w, _ = left.shape
    eng = E.engine(w, h, opt)
    for layout in LAYOUTS:
        for dtype in DTYPES:
            v, dt = _as_input(cost, layout, dtype)
            for st in T.STAGES:
                eng.debug_run_cost(left, right, v, layout, st, dtype=dt)
                if st == "COST":
                    E.same(f"{layout}/{dtype} VOL_INIT", eng.tap("VOL_INIT"), cost)
                for tap in GC.COST_STAGE_TAPS[st]:
                    assert T.sha(G.ref_case_tap(opt, tap, eng.tap(tap))) == want[f"{st}/{tap}"], f"{layout}/{dtype} {st}/{tap}"
            got = eng.match_cost(left, right, v, layout, dtype=dt)
            assert T.sha(got) == want["MEDIAN/DISP_L"], f"{layout}/{dtype} match_cost"
    eng.close()


@pytest.mark.gpu
def test_cost_value_domain():
    """NaN, +-inf, -0.0, negatives and values >= 65536 are clamped as documented; the map equals the restatement's on
    the clamped volume."""
    w, h, D = 64, 40, 20
    opt = T.default_option(max_disparity=D)
    left, right = T.synthetic_pair(w, h, D, 51)
    cost = CT.synthetic_cost(w, h, D, 51) * np.float32(2000.0)
    rng = np.random.default_rng(5)
    specials = np.array([np.nan, np.inf, -np.inf, -0.0, -3.0, -1e-30, 65536.0, 70000.0, 1e38, 65535.5], np.float32)
    mask = rng.random(cost.shape) < 0.08
    cost[mask] = specials[rng.integers(0, len(specials), int(mask.sum()))]
    clamped = CT.cost_domain(cost)
    want = CT.CostOracle(w, h, opt).match_cost(left, right, clamped)
    eng = E.engine(w, h, opt)
    for layout in LAYOUTS:
        v = cost if layout == "hwd" else np.ascontiguousarray(cost.transpose(2, 0, 1))
        eng.debug_run_cost(left, right, v, layout, "COST")
        E.same(f"{layout} VOL_INIT", eng.tap("VOL_INIT"), clamped)
        E.same(f"{layout} map", eng.match_cost(left, right, v, layout), want)
    eng.close()


def _device_batch_check(eng, pairs, n, layout, dtype):
    """n pairs (pair i = pairs[i % len(pairs)]) through match_cost_batch_device; every map equals the single-pair
    match_cost of its own pair."""
    torch, dev = E.cuda()
    singles = [eng.match_cost(l, r, v, layout, dtype=dt) for (l, r, v, dt) in pairs]
    k = len(pairs)
    d_l = torch.from_numpy(np.stack([pairs[i % k][0] for i in range(n)])).to(dev)
    d_r = torch.from_numpy(np.stack([pairs[i % k][1] for i in range(n)])).to(dev)
    d_c = torch.from_numpy(np.stack([pairs[i % k][2] for i in range(n)])).to(dev)
    d_out = torch.full((n, eng.height, eng.width), -1.0, dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream()
    # two calls that flow into each other, joined once
    E.split_calls(eng, n, True, lambda first, count: eng.match_cost_batch_device(
        count, d_l[first:].data_ptr(), d_r[first:].data_ptr(), d_c[first:].data_ptr(), d_out[first:].data_ptr(), layout,
        dtype, st.cuda_stream))
    out = d_out.cpu().numpy()
    for i in range(n):
        E.same(f"pair {i}", out[i], singles[i % k])


@pytest.mark.gpu
def test_cost_batch_device_order_and_stride():
    """n = 3 * wave_pairs + 2 distinct pairs with wave_pairs = 4, lanes = 3, pipelined."""
    w, h, D = 72, 48, 24
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt, wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    pairs = []
    for s in range(n):
        l, r = T.synthetic_pair(w, h, D, 100 + s)
        pairs.append((l, r, CT.synthetic_cost(w, h, D, 100 + s), "f32"))
    _device_batch_check(eng, pairs, n, "hwd", "f32")
    eng.close()


@pytest.mark.gpu
def test_cost_batch_device_loaded_waves_bf16():
    """Default configuration with several waves per lane in flight, DHW bf16: every map equals its single-pair result."""
    w, h, D = 160, 120, 64
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt)
    n = 2 * eng.wave_pairs * eng.lanes + 5
    pairs = []
    for s in range(7):    # 7 distinct pairs cycled: coprime with the wave size, so every wave slot sees different pairs
        l, r = T.synthetic_pair(w, h, D, 200 + s)
        v, _ = _as_input(CT.synthetic_cost(w, h, D, 200 + s), "dhw", "bf16")
        pairs.append((l, r, v, "bf16"))
    _device_batch_check(eng, pairs, n, "dhw", "bf16")
    eng.close()
