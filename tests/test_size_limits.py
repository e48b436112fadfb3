"""Size-limit parity: the shapes at the edges of what adc_create accepts (height <= 4096, width and width + range <=
10000, range <= 256) against the oracle, and per-pair volumes past 2^31 bytes and 2^31 elements against committed hashes
(DESIGN.md 3).  adc_create promises that whatever it accepts, adc_match runs; these are the sizes that promise covers and
the rest of the suite does not reach.

CPU: region voting's list admission rule (adcensus_b200/csrc/vote_plan.h) swept over the whole accepted domain by
tests/c/vote_plan_main.cpp, and the launch-plan branches the edge shapes reach."""
from __future__ import annotations

import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E
import cloud_testlib as CL
import maps_testlib as MT
import reproject_testlib as RP
import speckle_testlib as SP


# ---- CPU: the voting admission rule ----------------------------------------------------------------------------------
def test_vote_admission_rule_over_the_accepted_domain():
    """Every D from 1 to 256 in both histogram forms, N up to the largest the shape limits allow, pending counts 0..N,
    true forward-list sizes up to N * 65535 and every counter value the saturating accumulation can leave: wherever the
    rule admits the forward lists, the entry count and every int cursor stay below 2^31, the entries k_vote_push streams
    are the entries k_vote_scan wrote, and the lists fit the idle cost volume."""
    r = subprocess.run([str(E.c_tool("vote_plan_main"))], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("ok "), r.stdout[-4000:] + r.stderr[-2000:]
    assert int(r.stdout.split()[1]) > 1_000_000, r.stdout


# ---- the edge shapes -------------------------------------------------------------------------------------------------
# name -> (W, H, option overrides, seed)
SHAPES = {
    "widest_row": (9992, 16, dict(max_disparity=8), 1),                           # W + range = 10000: 14 row segments in
    #                                                                               the fused cost pass
    "widest_row_d1": (9999, 16, dict(max_disparity=1), 12),                       # the widest row adc_create accepts
    "widest_range_256": (9744, 4, dict(max_disparity=256), 2),                    # W + range = 10000, WIDE voting
    "widest_dmin_neg": (9760, 4, dict(min_disparity=-16, max_disparity=224), 3),  # W + range = 10000, dmin < 0
    "tallest_d16": (24, 4096, dict(max_disparity=16), 4),                         # median: 4 rows per thread, full
    "tallest_d16_h4095": (24, 4095, dict(max_disparity=16), 5),
    "tallest_d256": (24, 4096, dict(max_disparity=256), 6),                       # D > W
    "tallest_d256_h4095": (24, 4095, dict(max_disparity=256), 7),
    "median_h1024": (13, 1024, dict(max_disparity=16), 8),                        # median: 1 row per thread, full
    "median_h1025": (13, 1025, dict(max_disparity=16), 9),                        # 2 rows per thread, one used
    "median_h2048": (13, 2048, dict(max_disparity=16), 10),
    "median_h2049": (13, 2049, dict(max_disparity=16), 11),                       # 4 rows per thread
}
for _w in (1, 2, 3):               # degenerate shapes: no row or column has a neighbour on both sides
    for _h in (1, 2):
        for _d in (1, 2):
            SHAPES[f"tiny_{_w}x{_h}_d{_d}"] = (_w, _h, dict(max_disparity=_d), 100 + 10 * _w + 2 * _h + _d)

N_PAIRS, WAVE = 3, 2               # a partial second wave


def _plan(exe, *args):
    r = subprocess.run([str(E.c_tool(exe)), *map(str, args)], capture_output=True, text=True)
    assert r.returncode == 0, (exe, args, r.stdout, r.stderr)
    return [list(map(int, line.split())) for line in r.stdout.strip().split("\n")]


def test_edge_shapes_reach_their_plan_branches():
    """The launch plans (ca_plan.h, so_plan.h) the widest and tallest shapes take, read from the plan executables."""
    # W = 9992 at D = 8 and W = 9999 at D = 1: the fused cost + first horizontal pass cuts the row into 14 segments of 4
    # quads; no TMA plan fits the row, so both double passes take the LDG form, the rows in 6 and 3 segments
    for W, Dp, ldg_nseg in ((9992, 8, 6), (9999, 4, 3)):
        qc, _, nseg, _, _, _, _, _, ok, _ = _plan("ca_plan_main", W, Dp, 34)[0]
        assert (ok, qc, nseg) == (1, 4, 14), W
        rows, cols = _plan("ca_plan_main", "arm", W, 16, Dp, 34)
        assert (rows[1], rows[11], rows[13], cols[13]) == (0, ldg_nseg, 0, 0), (W, rows, cols)
    # W + range = 10000 at D = 256 and D = 240: 23 segments of 8 quads
    for W, Dp in ((9744, 256), (9760, 240)):
        qc, _, nseg, _, _, _, _, _, ok, _ = _plan("ca_plan_main", W, Dp, 34)[0]
        assert (ok, qc, nseg) == (1, 8, 23), (W, Dp)
    # H = 4096: k_arm_sum2t cuts the columns into 7 segments (D = 16) and 17 (D = 256)
    for Dp, qc, nseg in ((16, 4, 7), (256, 8, 17)):
        rows, cols = _plan("ca_plan_main", "arm", 24, 4096, Dp, 34)
        assert (cols[1], cols[2], cols[4], cols[13]) == (1, qc, nseg, 1), (Dp, cols)
        assert rows[13] == 1, (Dp, rows)
    # the scanline passes of the widest row and the tallest column: slots of T = 4 steps, rings of 3
    for args in ((9992, 16, 8, WAVE, 0), (9992, 16, 8, WAVE, 1), (24, 4096, 16, WAVE, 1), (24, 4096, 256, WAVE, 1)):
        assert _plan("so_plan_main", *args)[0][:2] == [4, 3], args


def _pairs(W, H, D, seed):
    return [T.synthetic_pair(W, H, D, seed + 7919 * i) for i in range(N_PAIRS)]


def _compare(tag, got, want):
    E.same(f"{tag} COST/VOL_INIT", got["cost"], want["cost"])
    E.same(f"{tag} AGG4/VOL_AGGR", got["aggr"], want["aggr"])
    E.same(f"{tag} SO4/VOL_AGGR", got["opt"], want["opt"])
    E.same(f"{tag} WTA/DISP_L", got["wta_left"], want["wta_left"])
    E.same(f"{tag} WTA/DISP_R", got["wta_right"], want["wta_right"])
    assert set(np.unique(got["outliers"])) <= {0, 1, 2}, f"{tag} OUTLIER: labels other than 0, 1, 2"
    mis, occ = MT.outlier_lists(got["outliers"])
    E.same(f"{tag} OUTLIER/MISMATCHES", mis, want["mismatches"].reshape(-1, 2))
    E.same(f"{tag} OUTLIER/OCCLUSIONS", occ, want["occlusions"].reshape(-1, 2))
    E.same(f"{tag} MEDIAN/DISP_L", got["disp"], want["final"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_edge_shape_vs_oracle(name):
    """One batched call over 3 distinct pairs in waves of 2, plain and pipelined, exporting the three volumes, both WTA
    maps, the outlier map and the final map: each pair bit for bit against its own oracle run.  Then the one-pair match
    of the first pair and its right map."""
    W, H, over, seed = SHAPES[name]
    opt = T.default_option(**over)
    D = opt.max_disparity - opt.min_disparity
    torch, dev = E.cuda()
    pairs = _pairs(W, H, D, seed)
    with ThreadPoolExecutor(len(pairs)) as ex:     # the oracle runs overlap the GPU work (ctypes releases the GIL)
        futs = [ex.submit(E.oracle_outputs, W, H, opt, l, r) for l, r in pairs]
        d_l = torch.from_numpy(np.stack([p[0] for p in pairs])).to(dev)
        d_r = torch.from_numpy(np.stack([p[1] for p in pairs])).to(dev)
        eng = E.engine(W, H, opt, wave_pairs=WAVE, lanes=2)
        assert eng.wave_pairs == WAVE
        runs = {}
        for pipelined in (False, True):
            runs[pipelined] = E.batch_outputs(eng, eng.match_outputs_batch_device, N_PAIRS, d_l.data_ptr(), d_r.data_ptr(),
                                              3 * W * H, volumes=[(s, "hwd", "f32") for s in ("cost", "aggr", "opt")],
                                              maps=["wta_left", "wta_right", "outliers"], pipelined=pipelined)
        one = eng.match(*pairs[0])
        one_right = eng.right_disparity()
        want = [f.result() for f in futs]
        try:
            if name in POST_SHAPES:
                _check_post_processing(name, eng, pairs[0][0], want[0]["final"])
        finally:
            eng.close()
    for pipelined, got in runs.items():
        for i, w in enumerate(want):
            _compare(f"{name} ({W}x{H}x{D}, {'pipelined' if pipelined else 'plain'}) pair {i}",
                     {k: v[i] for k, v in got.items()}, w)
    E.same(f"{name} match", one, want[0]["final"])
    E.same(f"{name} right map", one_right, want[0]["wta_right"])


POST_SHAPES = ("widest_row", "widest_row_d1", "widest_range_256", "tallest_d16", "tallest_d256")
SPECKLE = (30, 0.25)


def _check_post_processing(name, eng, left, disp):
    """The map post-processing entries on the oracle's final map against their restatements: reprojection (points,
    depth, 16-bit disparity), the speckle filter, the point cloud with colours and pixel indices, and the demo's render
    and cloud."""
    import cv2
    Q = np.load(T.GOLDEN_DIR / "golden_reproject_cases.npz")["rig_zero_0/Q"]
    got = eng.reproject(disp, Q, ("points", "depth", "disp_s16"))
    assert RP.same_nan(got["points"], RP.points(disp, Q)), f"{name} points"
    assert RP.same_nan(got["depth"], RP.depth(disp, Q)), f"{name} depth"
    assert np.array_equal(got["disp_s16"], RP.disp_s16(disp, eng.option.min_disparity)), f"{name} disp_s16"
    assert SP.same_bits(eng.filter_speckles(disp, *SPECKLE), SP.filter_f32(disp, np.inf, *SPECKLE)), f"{name} speckles"
    pts, cols, pix = eng.point_cloud(disp, Q, bgr=left, pixels=True)
    wp, wc, wx = CL.cloud(disp, Q, left)
    assert RP.same_nan(pts, wp) and np.array_equal(cols, wc) and np.array_equal(pix, wx), f"{name} point cloud"
    gray, jet, (mn, mx) = eng.render_disparity(disp)
    want_gray, wmn, wmx = MT.gray8(disp, disp.shape[1])
    assert (mn, mx) == (wmn, wmx) and np.array_equal(gray, want_gray), f"{name} render"
    assert np.array_equal(jet, cv2.applyColorMap(want_gray, cv2.COLORMAP_JET)), f"{name} render jet"
    ys, xs = np.nonzero(~np.isinf(disp))
    want = np.stack([xs, ys, np.abs(disp[ys, xs]), left[ys, xs, 2], left[ys, xs, 1], left[ys, xs, 0]], 1).astype(np.float32)
    assert np.array_equal(eng.disparity_cloud(left, disp), want), f"{name} disparity cloud"


# ---- volumes past 2^31 bytes and 2^31 elements -----------------------------------------------------------------------
def _large_case(name):
    g = E.golden("golden_limits.json")[name]
    W, H, D = g["width"], g["height"], g["max_disparity"]
    left, right = T.synthetic_pair(W, H, D, g["seed"])
    assert [T.sha(left), T.sha(right)] == g["input_sha"]
    return g, left, right


def test_large_cases_cross_the_thresholds():
    """L1's volume is past 2^31 bytes, L2's past 2^31 elements, and a batch of two L1 pairs past 2^32 bytes."""
    g = E.golden("golden_limits.json")
    n1 = g["L1_s1"]["width"] * g["L1_s1"]["height"] * g["L1_s1"]["max_disparity"]
    n2 = g["L2_s1"]["width"] * g["L2_s1"]["height"] * g["L2_s1"]["max_disparity"]
    assert 4 * n1 > 2 ** 31 and n1 < 2 ** 31 and 2 * 4 * n1 > 2 ** 32
    assert n2 > 2 ** 31
    assert g["L1_s1"]["checker"] == g["L1_s2"]["checker"] == "reference" and g["L2_s1"]["checker"] == "oracle"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["L1_s1", "L2_s1"])
def test_large_volume_stage_by_stage(name):
    """Every tap after every stage against the reference's (L1) or the oracle's (L2) hashes."""
    g, left, right = _large_case(name)
    eng = E.engine(g["width"], g["height"], T.default_option(max_disparity=g["max_disparity"]))
    try:
        for st in T.STAGES:
            eng.debug_run(left, right, st)
            for tap in T.STAGE_TAPS[st]:
                assert T.sha(eng.tap(tap)) == g["hashes"][f"{st}/{tap}"], f"{name}: {st}/{tap}"
    finally:
        eng.close()


@pytest.mark.gpu
def test_large_volume_batch_entries():
    """Two distinct L1 pairs in one wave: pair offsets past 2^32 bytes, in-pair offsets past 2^31.  Against each pair's
    reference hashes: the maps of adc_match_batch_device; the maps and the optimised volumes (DHW f32) of
    adc_match_volumes_batch_device; its matching-cost volumes (DHW f32), which then go into adc_match_cost_batch_device,
    and that call's maps."""
    torch, dev = E.cuda()
    cases = [_large_case(n) for n in ("L1_s1", "L1_s2")]
    W, H, D = cases[0][0]["width"], cases[0][0]["height"], cases[0][0]["max_disparity"]
    n = len(cases)
    d_l = torch.from_numpy(np.stack([c[1] for c in cases])).to(dev)
    d_r = torch.from_numpy(np.stack([c[2] for c in cases])).to(dev)
    d_vol = torch.empty((n, D, H, W), dtype=torch.float32, device=dev)    # before the engine: its sizing sees it
    d_disp = torch.full((n, H, W), -7.0, dtype=torch.float32, device=dev)
    eng = E.engine(W, H, T.default_option(max_disparity=D), wave_pairs=2, lanes=1)
    try:
        assert eng.wave_pairs == 2
        st = torch.cuda.current_stream().cuda_stream

        def check_maps(what):
            torch.cuda.synchronize()
            for i, (g, _, _) in enumerate(cases):
                assert T.sha(d_disp[i].cpu().numpy()) == g["hashes"]["MEDIAN/DISP_L"], f"{what}: pair {i}"
            d_disp.fill_(-7.0)

        eng.match_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), d_disp.data_ptr(), stream=st)
        check_maps("adc_match_batch_device")
        eng.match_volumes_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), [(d_vol.data_ptr(), "opt", "dhw", "f32")],
                                       d_disp=d_disp.data_ptr(), stream=st)
        check_maps("adc_match_volumes_batch_device")
        for i, (g, _, _) in enumerate(cases):
            hwd = d_vol[i].permute(1, 2, 0).contiguous().cpu().numpy()
            assert T.sha(hwd) == g["hashes"]["SO4/VOL_AGGR"], f"optimised volume, pair {i}"
            del hwd
        # the matching cost as DHW f32, from the engine's own export, into the cost-input entry
        eng.match_volumes_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), [(d_vol.data_ptr(), "cost", "dhw", "f32")],
                                       stream=st)
        torch.cuda.synchronize()
        for i, (g, _, _) in enumerate(cases):
            hwd = d_vol[i].permute(1, 2, 0).contiguous().cpu().numpy()
            assert T.sha(hwd) == g["hashes"]["COST/VOL_INIT"], f"matching cost volume, pair {i}"
            del hwd
        eng.match_cost_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), d_vol.data_ptr(), d_disp.data_ptr(), "dhw", "f32",
                                    stream=st)
        check_maps("adc_match_cost_batch_device")
    finally:
        eng.close()


# ---- L3: region voting past 2^30 forward-list entries ----------------------------------------------------------------
def test_refine_runner_equals_the_staged_run():
    """orc_begin_refine (the oracle's staged runner from OUTLIER on, from given WTA maps, volumes untouched) against the
    full staged run on every stage-parity case: the outlier lists and every refinement stage's map.  A case with the
    discontinuity adjustment, which reads the aggregated volume, is refused."""
    for W, H, D, over, seed in E.PARITY_CASES:
        opt = T.default_option(**{"max_disparity": D, **over})
        left, right = T.synthetic_pair(W, H, D, seed)
        full = T.Oracle(W, H, opt)
        full.begin(left, right)
        full.run_to("WTA")
        wl, wr = full.tap("DISP_L").copy(), full.tap("DISP_R").copy()
        ref = T.Oracle(W, H, opt)
        if opt.do_discontinuity_adjustment:
            f = ref._f("begin_refine")
            assert f(ref.ctx, left.ctypes.data, right.ctypes.data, wl.ctypes.data, wr.ctypes.data) == 0
            continue
        ref.begin_refine(left, right, wl, wr)
        for st in T.STAGES[T.STAGE["OUTLIER"]:]:
            assert full.step() == ref.step() == T.STAGE[st]
            for tap in T.STAGE_TAPS[st]:
                E.same(f"{W}x{H}x{D} {over} {st}/{tap}", ref.tap(tap), full.tap(tap))
        full.close()
        ref.close()


# 9872 x 3600 at D = 128: N * Dp = 4.55 G words, so the idle cost volume would hold a saturated counter's 2^32 words of
# forward lists; a 1000 x 1000 patch of low-amplitude noise gives regions of up to 69 x 69 pixels that fail the LR check
L3 = dict(W=9872, H=3600, D=128, shift=32, y0=1300, x0=4400, P=1000, seed=1)


def _noise_patch_pair(W, H, shift, y0, x0, P, seed, **_):
    """White noise seen at a disparity of `shift`, with a P x P patch where each view carries its own noise of amplitude
    3 around 126: colour steps below cross_t2, so the arms reach cross_L1, and nothing to match."""
    rng = np.random.default_rng(seed)
    tex = rng.integers(0, 256, (H, W + 2 * shift, 3), dtype=np.uint8)
    left = np.ascontiguousarray(tex[:, shift:shift + W])
    right = np.ascontiguousarray(tex[:, 2 * shift:2 * shift + W])
    left[y0:y0 + P, x0:x0 + P] = 126 + rng.integers(0, 4, (P, P, 3), dtype=np.uint8)
    right[y0:y0 + P, x0 - shift:x0 - shift + P] = 126 + rng.integers(0, 4, (P, P, 3), dtype=np.uint8)
    return left, right


@pytest.mark.gpu
def test_voting_past_2_30_forward_entries():
    """A pair whose pending pixels' regions hold more than 2^30 entries in a volume large enough to admit a saturated
    counter: voting must enumerate and end in the oracle's outlier lists, post-voting map and final map, refined from
    the GPU's own WTA maps (no oracle run of the volumes is possible at this size)."""
    import adcensus_b200 as A
    torch, _ = E.cuda()
    torch.cuda.empty_cache()
    W, H, D = L3["W"], L3["H"], L3["D"]
    opt = T.default_option(max_disparity=D)
    left, right = _noise_patch_pair(**L3)
    try:
        eng = E.engine(W, H, opt, wave_pairs=1, lanes=1)
    except A.AdcError as e:
        if "error 4:" in str(e):           # ADC_ERR_NOMEM
            pytest.skip(f"the L3 pair does not fit this device: {e}")
        raise
    try:
        eng.debug_run(left, right, "WTA")
        wl, wr = eng.tap("DISP_L").copy(), eng.tap("DISP_R").copy()
        eng.debug_run(left, right, "OUTLIER")
        mis, occ = eng.tap("MISMATCHES").copy(), eng.tap("OCCLUSIONS").copy()
        eng.debug_run(left, right, "VOTE")
        cnt = eng.counters()
        voted = eng.tap("DISP_L").copy()
        final = eng.match(left, right)
    finally:
        eng.close()
    # preconditions: inside the regime where a saturated counter used to admit the forward lists
    ns, room, N, HW = cnt[10] + cnt[11], cnt[15] & 0xffffffff, W * H, D // 2
    fwd_off = (ns * HW + 1) & ~1
    assert 0 < ns <= len(mis) + len(occ), (ns, len(mis), len(occ))
    assert room > 2 ** 30, f"forward-list room {room} is not saturated (pending {ns})"
    assert N * ((D + 3) // 4 * 4) >= fwd_off + 2 ** 32, (N, fwd_off)
    assert cnt[13] == 0, "the adjacency lists were used"
    print(f"L3: {ns} pending pixels, room counter {room:#x}, k_vote_push {cnt[5] / 1000:.1f} ms "
          f"(derive {cnt[6] / 1000:.1f}, push {cnt[7] / 1000:.1f}), {cnt[2]} rounds, {cnt[12]} changes")
    orc = T.Oracle(W, H, opt)
    orc.begin_refine(left, right, wl, wr)
    orc.run_to("OUTLIER")
    E.same("L3 OUTLIER/MISMATCHES", mis, orc.tap("MISMATCHES"))
    E.same("L3 OUTLIER/OCCLUSIONS", occ, orc.tap("OCCLUSIONS"))
    orc.run_to("VOTE")
    E.same("L3 VOTE/DISP_L", voted, orc.tap("DISP_L"))
    orc.run_to("MEDIAN")
    E.same("L3 MEDIAN/DISP_L", final, orc.tap("DISP_L"))
    orc.close()
