"""Per-pixel side maps (adc_match_outputs*): the raw WTA maps of both views, the LR check's classification and the
cost-curve confidence, for every pair of a batch, in the same pipeline pass as the final map and the exported volumes.

CPU: the argument rules (on a NULL engine, before any device work), the constants, the confidence helper against a plain
per-pixel loop, k_confidence's register / local-memory figures.
GPU: all five maps against the C restatement (itself pinned to the reference) on every test_gpu_parity.CASES entry, Cone
and a D = 3 case; the WTA maps and outlier lists of the large shapes against the reference's hashes and their confidence
against the same call's optimised volume; the cost-input cases; batched device calls (offsets, guard bytes, pipelining);
map-only mode; the unchanged paths.
"""
import ctypes

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E  # puts tools/ on sys.path
import maps_testlib as MT
import make_golden as G
import make_golden_cost as GC

MAPS = ["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"]


# ---- CPU ------------------------------------------------------------------------------------------
def _vols(*specs):
    import adcensus_b200 as A
    arr = (A.engine.VolumeOut * max(1, len(specs)))()
    for i, (dst, stage, layout, dtype, reserved) in enumerate(specs):
        arr[i] = A.engine.VolumeOut(dst, stage, layout, dtype, reserved)
    return arr


def _maps(*specs):
    import adcensus_b200 as A
    arr = (A.engine.MapOut * max(1, len(specs)))()
    for i, (dst, kind, reserved) in enumerate(specs):
        arr[i] = A.engine.MapOut(dst, kind, reserved)
    return arr


def test_output_argument_errors_need_no_gpu():
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    F32, HWD, DHW = A.COST_F32, A.COST_HWD, A.COST_DHW
    gv = (p, A.VOL_OPT, DHW, F32, 0)
    gm = (p, A.MAP_PEAK_RATIO, 0)

    def host(maps, n_maps, vols=None, n_vols=0, disp=p, cost=None, cl=HWD, cd=F32):
        return L.adc_match_outputs(None, p, p, cost, cl, cd, disp, vols, n_vols, maps, n_maps)

    def dev(maps, n_maps, vols=None, n_vols=0, disp=p, cost=None, cl=HWD, cd=F32):
        return L.adc_match_outputs_batch_device(None, 1, p, p, cost, cl, cd, disp, vols, n_vols, maps, n_maps, None)

    for call in (host, dev):
        cases = [
            (dict(maps=_maps(gm), n_maps=6), b"n_maps"),
            (dict(maps=_maps(gm), n_maps=-1), b"n_maps"),
            (dict(maps=None, n_maps=1), b"maps is NULL"),
            (dict(maps=_maps((p, 5, 0)), n_maps=1), b"maps[0].kind"),
            (dict(maps=_maps((p, -1, 0)), n_maps=1), b"maps[0].kind"),
            (dict(maps=_maps(gm, (p, A.MAP_PEAK_RATIO, 0)), n_maps=2), b"requested twice"),
            (dict(maps=_maps(gm, (None, A.MAP_WTA_LEFT, 0)), n_maps=2), b"maps[1].dst"),
            (dict(maps=_maps((p, A.MAP_OUTLIERS, 1)), n_maps=1), b"maps[0].reserved"),
            (dict(maps=None, n_maps=0, disp=None), b"no volume or map"),
            # the volume entries' rules, under this entry's field names
            (dict(maps=_maps(gm), n_maps=1, vols=_vols(gv), n_vols=4), b"n_vols"),
            (dict(maps=_maps(gm), n_maps=1, vols=None, n_vols=1), b"vols is NULL"),
            (dict(maps=_maps(gm), n_maps=1, vols=_vols((p, 3, HWD, F32, 0)), n_vols=1), b"vols[0].stage"),
            (dict(maps=_maps(gm), n_maps=1, vols=_vols(gv, gv), n_vols=2), b"requested twice"),
            (dict(maps=_maps(gm), n_maps=1, vols=_vols((p, A.VOL_OPT, HWD, F32, 1)), n_vols=1), b"vols[0].reserved"),
            (dict(maps=_maps(gm), n_maps=1, cost=p, cl=2), b"cost_layout"),
            (dict(maps=_maps(gm), n_maps=1, cost=p, cd=5), b"cost_dtype"),
        ]
        for kw, msg in cases:
            assert call(**kw) == 1, (call.__name__, kw)
            assert msg in L.adc_last_error(), (call.__name__, kw, L.adc_last_error())
        # valid requests get as far as the engine check: maps only, volumes only, the final map only, all five maps
        every = _maps(*[(p, k, 0) for k in range(5)])
        for kw in (dict(maps=_maps(gm), n_maps=1, disp=None), dict(maps=None, n_maps=0, vols=_vols(gv), n_vols=1, disp=None),
                   dict(maps=None, n_maps=0), dict(maps=every, n_maps=5, vols=_vols(gv), n_vols=1, disp=None),
                   dict(maps=_maps(gm), n_maps=1, cost=None, cl=9)):
            assert call(**kw) == 1 and b"engine is NULL" in L.adc_last_error(), (call.__name__, kw)
    # device destinations of f32 maps must be 4-byte aligned; the u8 outlier map may start at any byte; host destinations
    # are copied into, so need not be aligned
    for k in (A.MAP_WTA_LEFT, A.MAP_WTA_RIGHT, A.MAP_MIN_COST, A.MAP_PEAK_RATIO):
        assert dev(_maps((p + 2, k, 0)), 1) == 1 and b"4-byte aligned" in L.adc_last_error(), k
        assert host(_maps((p + 2, k, 0)), 1) == 1 and b"engine is NULL" in L.adc_last_error(), k
    assert dev(_maps((p + 1, A.MAP_OUTLIERS, 0)), 1) == 1 and b"engine is NULL" in L.adc_last_error()


def test_map_constants():
    import adcensus_b200 as A
    assert (A.MAP_WTA_LEFT, A.MAP_WTA_RIGHT, A.MAP_OUTLIERS, A.MAP_MIN_COST, A.MAP_PEAK_RATIO) == (0, 1, 2, 3, 4)
    assert A.engine.MAP_KINDS == {n: i for i, n in enumerate(MAPS)}
    assert ctypes.sizeof(A.engine.MapOut) == 16
    assert A.Engine.PROFILE_KERNELS["confidence"] == 12


def _hand_volume(rng, H, W, D):
    """A volume that reaches every rule: values from a small set (ties everywhere), all-zero pixels (c2 == 0), a unique
    zero minimum, the minimum at d = 0 and d = D - 1, continuous values."""
    v = rng.choice(np.float32([0.0, 0.5, 1.0, 2.0, 3.0, 7.25]), size=(H, W, D)).astype(np.float32)
    v[0, 0] = 0.0
    v[0, 1] = 5.0
    v[0, 1, 0] = 0.0                                              # unique zero minimum at the low end
    v[0, 2] = 5.0
    v[0, 2, D - 1] = 1.5                                          # minimum at the high end
    v[1] = rng.random((W, D), dtype=np.float32) * np.float32(100)  # no ties
    v[2, :, :] = 4.0                                              # every d ties: d1 = 0
    return v


def test_confidence_helper_matches_loop():
    rng = np.random.default_rng(17)
    for D in (1, 2, 3, 4, 5, 8, 13):
        for rep in range(3):
            v = _hand_volume(rng, 6, 7, D)
            got = MT.confidence(v)
            want = MT.confidence_loop(v)
            for name, g, w in zip(("min_cost", "peak_ratio"), got, want):
                assert g.dtype == np.float32 and g.shape == (6, 7)
                E.same(f"D={D} {name}", g, w)
            r = got[1]
            assert ((r >= 0) & (r <= 1)).all()
            if D <= 2:
                assert (r == 1).all()
    # hand-computed values
    c1, r = MT.confidence(np.float32([[[3, 1, 2, 5]], [[0, 5, 5, 9]], [[2, 1, 2, 9]], [[4, 4, 4, 4]], [[0, 0, 0, 0]]]))
    assert c1.ravel().tolist() == [1, 0, 1, 4, 0]
    assert r.ravel().tolist() == [np.float32(1) / np.float32(5), 0.0, np.float32(1) / np.float32(9), 1.0, 1.0]
    _, r3 = MT.confidence(np.float32([[[2, 1, 2], [1, 2, 3], [3, 2, 0]]]))       # D = 3: d1 = 1 has no far d
    assert r3.ravel().tolist() == [1.0, np.float32(1) / np.float32(3), 0.0]


def test_outlier_lists_helper():
    lab = np.zeros((3, 4), np.uint8)
    lab[0, 3] = 1
    lab[2, 0] = 1
    lab[1, 1] = 2
    mis, occ = MT.outlier_lists(lab)
    assert mis.tolist() == [[3, 0], [0, 2]] and occ.tolist() == [[1, 1]]
    assert mis.dtype == np.int32 and MT.outlier_lists(np.zeros((2, 2), np.uint8))[0].shape == (0, 2)


def test_confidence_kernel_uses_no_local_memory():
    """ptxas -v on k_confidence.cu: no stack frame, no spills."""
    report = E.ptxas_report(T.REPO / "adcensus_b200" / "csrc" / "k_confidence.cu")
    assert report and all((f["stack"], f["spill_stores"], f["spill_loads"], f["lmem"]) == (0, 0, 0, 0)
                          for f in report.values()), report


# ---- GPU ------------------------------------------------------------------------------------------
def _check_maps(name, got, want):
    E.same(f"{name} wta_left", got["wta_left"], want["wta_left"])
    E.same(f"{name} wta_right", got["wta_right"], want["wta_right"])
    gm, go = MT.outlier_lists(got["outliers"])
    assert np.array_equal(gm, want["mismatches"].reshape(-1, 2)), f"{name}: mismatch list"
    assert np.array_equal(go, want["occlusions"].reshape(-1, 2)), f"{name}: occlusion list"
    c1, ratio = MT.confidence(want["opt"])
    E.same(f"{name} min_cost", got["min_cost"], c1)
    E.same(f"{name} peak_ratio", got["peak_ratio"], ratio)


CASES = E.PARITY_CASES + [(40, 30, 3, {}, 20)]      # D = 3: pixels with d1 = 1 have no d with |d - d1| >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("case", [f"{c[0]}x{c[1]}x{c[2]}-{i}" for i, c in enumerate(CASES)] + ["cone"])
def test_maps_parity(case, cone):
    """All five maps from one match_outputs call against the restatement: WTA maps bit for bit against WTA/DISP_L and
    WTA/DISP_R, the outlier map as raster-order lists equal to OUTLIER/MISMATCHES and OUTLIER/OCCLUSIONS, the confidence
    bit for bit against the numpy helper on SO4/VOL_AGGR, and the final map of the same call the restatement's."""
    if case == "cone":
        left, right = cone
        opt = T.default_option()
    else:
        w, h, D, over, seed = CASES[int(case.rsplit("-", 1)[1])]
        opt = T.default_option(**{"max_disparity": D, **over})
        left, right = T.synthetic_pair(w, h, D, seed)
    h, w, _ = left.shape
    want = E.oracle_outputs(w, h, opt, left, right)
    eng = E.engine(w, h, opt)
    disp, got = eng.match_outputs(left, right, maps=MAPS)
    E.same("final map", disp, want["final"])
    _check_maps(case, got, want)
    if not opt.do_lr_check:
        assert not got["outliers"].any()
    if case == "cone":
        assert T.sha(disp).startswith("77d70a58d1aa5c71")
    eng.close()


def _check_hashes(name, got, g, opt):
    """WTA maps and outlier lists against the reference's hashes (the right map only where the reference defines it)."""
    assert T.sha(got["wta_left"]) == g["WTA/DISP_L"], f"{name}: wta_left"
    assert T.sha(G.ref_case_tap(opt, "DISP_R", got["wta_right"])) == g["WTA/DISP_R"], f"{name}: wta_right"
    mis, occ = MT.outlier_lists(got["outliers"])
    assert T.sha(mis) == g["OUTLIER/MISMATCHES"], f"{name}: mismatch list"
    assert T.sha(occ) == g["OUTLIER/OCCLUSIONS"], f"{name}: occlusion list"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cloth3", "wood2", "piano", "kitti_s1", "p1080_s1"])
def test_maps_large_shapes_vs_reference_goldens(name):
    """WTA maps and outlier lists of Cloth3, Wood2, Piano, 1242x375x128 and 1920x1080x192 against the reference's
    hashes.  Cloth3 and 1242x375x128 also export the optimised volume (f32) in the same call: it must hash to the
    reference's SO4/VOL_AGGR and the confidence must equal the helper on it.  1080p goes through the batched device
    call with two pairs, so that the second pair's volume reads run past 2^31 bytes inside the arena."""
    g = E.golden("golden_big.json")[name]
    if name in ("cloth3", "wood2", "piano"):
        z = np.load(T.GOLDEN_DIR / "real_pairs.npz")
        left, right = z[f"{name}_left"], z[f"{name}_right"]
        D = g["max_disparity"]
    else:
        w, h, D = g["width"], g["height"], g["max_disparity"]
        left, right = T.synthetic_pair(w, h, D, int(name.rsplit("_s", 1)[1]))
    assert [T.sha(left), T.sha(right)] == g["input_sha"]
    h, w, _ = left.shape
    opt = T.default_option(max_disparity=D)
    hs = g["hashes"]
    if name != "p1080_s1":
        eng = E.engine(w, h, opt)
        vols = ["opt"] if name in ("cloth3", "kitti_s1") else []
        disp, got = eng.match_outputs(left, right, maps=MAPS, volumes=vols)
        assert T.sha(disp) == hs["MEDIAN/DISP_L"]
        _check_hashes(name, got, hs, opt)
        if vols:
            assert T.sha(got["opt"]) == hs["SO4/VOL_AGGR"]
            c1, ratio = MT.confidence(got["opt"])
            E.same(f"{name} min_cost", got["min_cost"], c1)
            E.same(f"{name} peak_ratio", got["peak_ratio"], ratio)
        eng.close()
        return
    import torch
    dev = torch.device("cuda", 0)
    n = 2
    eng = E.engine(w, h, opt)
    assert eng.wave_pairs >= n
    assert n * h * w * ((D + 3) // 4 * 4) * 4 > 2 ** 31
    d_l = torch.from_numpy(np.stack([left] * n)).to(dev)
    d_r = torch.from_numpy(np.stack([right] * n)).to(dev)
    d_disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    bufs = {m: torch.empty((n, h, w), dtype=torch.uint8 if m == "outliers" else torch.float32, device=dev) for m in MAPS}
    st = torch.cuda.current_stream()
    eng.match_outputs_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), maps=[(b.data_ptr(), m) for m, b in bufs.items()],
                                   d_disp=d_disp.data_ptr(), stream=st.cuda_stream)
    torch.cuda.synchronize()
    got = [{m: b[i].cpu().numpy() for m, b in bufs.items()} for i in range(n)]
    for i in range(n):
        assert T.sha(d_disp[i].cpu().numpy()) == hs["MEDIAN/DISP_L"], f"pair {i} map"
        _check_hashes(f"pair {i}", got[i], hs, opt)
    for m in ("min_cost", "peak_ratio"):
        E.same(f"pair 1 {m}", got[1][m], got[0][m])
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", GC.COST_CASES, ids=[GC.cost_case_id(c) for c in GC.COST_CASES])
def test_maps_cost_input(case):
    """A caller's cost through d_cost (two pairs, [D][H][W] bf16 and [H][W][D] f32): WTA maps and outlier lists hash to
    the reference's for that cost; the confidence equals the helper on the optimised volume of the same call, which
    hashes to the reference's SO4/VOL_AGGR."""
    import torch
    from cost_testlib import to_bf16_bits
    want = E.golden("golden_cost_cases.json")[GC.cost_case_id(case)]
    left, right, opt, cost = GC.cost_case_inputs(case)
    h, w, _ = left.shape
    D = cost.shape[2]
    dev = torch.device("cuda", 0)
    eng = E.engine(w, h, opt)
    n = 2
    d_l = torch.from_numpy(np.stack([left] * n)).to(dev)
    d_r = torch.from_numpy(np.stack([right] * n)).to(dev)
    st = torch.cuda.current_stream()
    for layout, dtype, c in (("dhw", "bf16", to_bf16_bits(np.ascontiguousarray(cost.transpose(2, 0, 1)))),
                             ("hwd", "f32", cost)):
        d_c = torch.from_numpy(np.stack([c] * n)).to(dev)
        d_disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
        d_opt = torch.empty((n, h, w, D), dtype=torch.float32, device=dev)
        bufs = {m: torch.empty((n, h, w), dtype=torch.uint8 if m == "outliers" else torch.float32, device=dev)
                for m in MAPS}
        eng.match_outputs_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), maps=[(b.data_ptr(), m) for m, b in bufs.items()],
                                       volumes=[(d_opt.data_ptr(), "opt", "hwd", "f32")], d_disp=d_disp.data_ptr(),
                                       d_cost=d_c.data_ptr(), cost_layout=layout, cost_dtype=dtype, stream=st.cuda_stream)
        torch.cuda.synchronize()
        for i in range(n):
            name = f"{layout}/{dtype} pair {i}"
            got = {m: b[i].cpu().numpy() for m, b in bufs.items()}
            vol = d_opt[i].cpu().numpy()
            assert T.sha(vol) == want["SO4/VOL_AGGR"], name
            assert T.sha(d_disp[i].cpu().numpy()) == want["MEDIAN/DISP_L"], name
            _check_hashes(name, got, want, opt)
            c1, ratio = MT.confidence(vol)
            E.same(f"{name} min_cost", got["min_cost"], c1)
            E.same(f"{name} peak_ratio", got["peak_ratio"], ratio)
    eng.close()


def _maps_batch_check(eng, pairs, n, specs, with_disp, pipelined, vol=None):
    """n pairs (pair i = pairs[i % len(pairs)]) through match_outputs_batch_device with the map requests `specs`
    [(kind, skew)], each destination `skew` elements (u8: bytes) into a buffer with 4096 elements of 0xA5 bytes on either
    side (and optionally one volume request (stage, layout, dtype)); every map equals the single-pair match_outputs
    result at its offset, the final maps the single-pair maps, and no element outside the n maps changes."""
    torch, dev = E.cuda()
    H, W, D = eng.height, eng.width, eng.D
    N = H * W
    k = len(pairs)
    kinds = [m for m, _ in specs]
    singles = []
    for (l, r) in pairs:
        disp, got = eng.match_outputs(l, r, maps=kinds, volumes=[vol[0]] if vol else [],
                                      layout=vol[1] if vol else "hwd", dtype=vol[2] if vol else "f32")
        singles.append((disp, got))
    d_l = torch.from_numpy(np.stack([pairs[i % k][0] for i in range(n)])).to(dev)
    d_r = torch.from_numpy(np.stack([pairs[i % k][1] for i in range(n)])).to(dev)
    d_out = torch.full((n, H, W), -1.0, dtype=torch.float32, device=dev) if with_disp else None
    es = {m: 1 if m == "outliers" else 4 for m in kinds}
    bufs = [E.guarded(n * N * es[m], torch.uint8, (4096 + skew) * es[m], (4096 - skew) * es[m], 0xA5) for m, skew in specs]
    if vol:
        tdt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[vol[2]]
        d_vol = torch.empty((n, H * W * D), dtype=tdt, device=dev)
    st = torch.cuda.current_stream()

    def issue(first, count):
        maps = [(data.data_ptr() + first * N * es[m], m) for (data, _), m in zip(bufs, kinds)]
        vols = [(d_vol[first:].data_ptr(), *vol)] if vol else []
        eng.match_outputs_batch_device(count, d_l[first:].data_ptr(), d_r[first:].data_ptr(), maps=maps, volumes=vols,
                                       d_disp=d_out[first:].data_ptr() if with_disp else 0, stream=st.cuda_stream)

    E.split_calls(eng, n, pipelined, issue)
    if with_disp:
        out = d_out.cpu().numpy()
        for i in range(n):
            E.same(f"pair {i} map", out[i], singles[i % k][0])
    for (data, intact), m in zip(bufs, kinds):
        assert intact(), f"{m}: bytes outside the maps written"
        got = data.cpu().numpy().view(np.uint8 if m == "outliers" else np.float32)
        for i in range(n):
            E.same(f"pair {i} {m}", got[i * N:(i + 1) * N].reshape(H, W), singles[i % k][1][m])
    if vol:
        raw = d_vol.view(torch.int32 if vol[2] == "f32" else torch.int16).cpu().numpy()
        for i in range(n):
            want = singles[i % k][1][vol[0]]
            assert np.array_equal(raw[i], want.reshape(-1).view(raw.dtype)), f"pair {i} volume"


# N = 71*47 is odd: pair i of a u8 map with an odd skew starts at every byte offset mod 4
BATCH_SPECS = [("wta_left", 0), ("wta_right", 3), ("outliers", 1), ("min_cost", 1), ("peak_ratio", 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_maps_batch_device_order_and_stride(pipelined):
    """n = 3 * wave_pairs + 2 distinct pairs, wave_pairs = 4, lanes = 3 (several waves per lane, n not a multiple of the
    wave size); all five maps at odd offsets, with the final map, then with an exported volume in the same call."""
    w, h, D = 71, 47, 23
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt, wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    pairs = [T.synthetic_pair(w, h, D, 500 + s) for s in range(n)]
    _maps_batch_check(eng, pairs, n, BATCH_SPECS, True, pipelined)
    _maps_batch_check(eng, pairs, n, [("peak_ratio", 0), ("outliers", 0)], True, pipelined, vol=("opt", "dhw", "bf16"))
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_maps_batch_device_loaded_waves(pipelined):
    """Default configuration with several waves per lane in flight: confidence and outliers plus the final map."""
    w, h, D = 160, 120, 64
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt)
    n = 2 * eng.wave_pairs * eng.lanes + 5
    pairs = [T.synthetic_pair(w, h, D, 600 + s) for s in range(7)]
    _maps_batch_check(eng, pairs, n, [("min_cost", 0), ("peak_ratio", 0), ("outliers", 0)], True, pipelined)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_maps_batch_device_map_only(pipelined):
    """No final map (d_disp NULL): the same side maps as a call with one."""
    w, h, D = 71, 47, 23
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt, wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    pairs = [T.synthetic_pair(w, h, D, 700 + s) for s in range(n)]
    _maps_batch_check(eng, pairs, n, BATCH_SPECS, False, pipelined)
    _maps_batch_check(eng, pairs, n, [("wta_left", 1), ("peak_ratio", 0)], False, pipelined)
    eng.close()


@pytest.mark.gpu
def test_map_only_mode_skips_refinement():
    """disparity=False: the maps equal those of a call with the final map, and the launch count shows where the pipeline
    stopped: at the WTA (plus k_confidence) for WTA / confidence maps, after the LR check for the outlier map."""
    w, h, D = 97, 61, 23
    opt = T.default_option(max_disparity=D)
    left, right = T.synthetic_pair(w, h, D, 2)
    eng = E.engine(w, h, opt)
    want_disp, want = eng.match_outputs(left, right, maps=MAPS)
    want_r = eng.right_disparity()
    counts = {}
    for st in ("WTA", "OUTLIER", "MEDIAN"):
        c0 = eng.launch_count
        eng.debug_run(left, right, st)
        counts[st] = eng.launch_count - c0
    assert counts["WTA"] < counts["OUTLIER"] < counts["MEDIAN"]
    for maps, extra, stop in ((["wta_left"], 0, "WTA"), (["wta_right", "wta_left"], 0, "WTA"), (["min_cost"], 1, "WTA"),
                              (["peak_ratio", "wta_right"], 1, "WTA"), (["outliers"], 0, "OUTLIER"),
                              (["outliers", "min_cost"], 1, "OUTLIER"), (MAPS, 1, "OUTLIER")):
        c0 = eng.launch_count
        none, got = eng.match_outputs(left, right, maps=maps, disparity=False)
        assert none is None
        assert eng.launch_count - c0 == counts[stop] + extra, maps
        for m in maps:
            E.same(f"{maps} {m}", got[m], want[m])
    # with the final map: the full pipeline plus k_confidence, and the same final and right-view maps as match()
    c0 = eng.launch_count
    disp, _ = eng.match_outputs(left, right, maps=["peak_ratio"])
    assert eng.launch_count - c0 == counts["MEDIAN"] + 1
    E.same("final map", disp, want_disp)
    E.same("match()", eng.match(left, right), want_disp)
    E.same("right map", eng.right_disparity(), want_r)
    E.same("right map = wta_right", want["wta_right"], want_r)
    eng.close()


@pytest.mark.gpu
def test_no_map_path_unchanged(cone):
    """A batched outputs call without map requests issues the launches of match_batch_device; the final maps of calls
    with and without side maps are bit-identical and equal the reference's."""
    import torch
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option(), wave_pairs=4, lanes=3)
    n = 9
    dev = torch.device("cuda", 0)
    d_l = torch.from_numpy(np.repeat(left[None], n, 0)).to(dev)
    d_r = torch.from_numpy(np.repeat(right[None], n, 0)).to(dev)
    st = torch.cuda.current_stream()

    def run(fn):
        d = torch.zeros((n, h, w), dtype=torch.float32, device=dev)
        c0 = eng.launch_count
        fn(d)
        torch.cuda.synchronize()
        return d.cpu().numpy(), eng.launch_count - c0

    maps0, launches0 = run(lambda d: eng.match_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), d.data_ptr(), st.cuda_stream))
    maps1, launches1 = run(lambda d: eng.match_outputs_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), d_disp=d.data_ptr(),
                                                                    stream=st.cuda_stream))
    assert launches1 == launches0
    E.same("no requests", maps1, maps0)
    side = {m: torch.empty((n, h, w), dtype=torch.uint8 if m == "outliers" else torch.float32, device=dev) for m in MAPS}
    maps2, launches2 = run(lambda d: eng.match_outputs_batch_device(
        n, d_l.data_ptr(), d_r.data_ptr(), maps=[(b.data_ptr(), m) for m, b in side.items()], d_disp=d.data_ptr(),
        stream=st.cuda_stream))
    assert launches2 == launches0 + -(-n // eng.wave_pairs)     # one k_confidence per wave
    E.same("with side maps", maps2, maps0)
    maps3, launches3 = run(lambda d: eng.match_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), d.data_ptr(), st.cuda_stream))
    assert launches3 == launches0
    E.same("after side maps", maps3, maps0)
    hashes = E.golden_hashes("cone_full")
    assert all(T.sha(maps2[i]) == hashes["MEDIAN/DISP_L"] for i in range(n))
    eng.close()
