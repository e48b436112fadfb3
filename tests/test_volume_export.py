"""Volume export (adc_match_volumes*): the matching, aggregated and optimised cost volumes handed to the caller.

CPU: the argument rules (on a NULL engine, before any device work), the bf16 rounding helper against an exact
restatement.
GPU: every stage x layout x element type against the C restatement (itself pinned to the reference) on a subset of
test_gpu_parity.CASES and Cone; the aggregated / optimised volumes of the large shapes against the reference's hashes;
the cost-input round trip; volumes-only mode; the batched device entry point (offsets, guard bytes, pipelining); the
unchanged no-export path.
"""
import ctypes
from fractions import Fraction

import numpy as np
import pytest

import adc_testlib as T
import cost_testlib as CT
import engine_testlib as E  # puts tools/ on sys.path
import export_testlib as XT
import make_golden_cost as GC

STAGES = ["cost", "aggr", "opt"]
LAYOUTS = ["hwd", "dhw"]
DTYPES = ["f32", "f16", "bf16"]


# ---- CPU ------------------------------------------------------------------------------------------
def _outs(*specs):
    import adcensus_b200 as A
    arr = (A.engine.VolumeOut * max(1, len(specs)))()
    for i, (dst, stage, layout, dtype, reserved) in enumerate(specs):
        arr[i] = A.engine.VolumeOut(dst, stage, layout, dtype, reserved)
    return arr


def test_volume_argument_errors_need_no_gpu():
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    F32, HWD, DHW = A.COST_F32, A.COST_HWD, A.COST_DHW
    good = (p, A.VOL_OPT, DHW, F32, 0)

    def host(outs, n, disp=p, cost=None, cl=HWD, cd=F32):
        return L.adc_match_volumes(None, p, p, cost, cl, cd, disp, outs, n)

    def dev(outs, n, disp=p, cost=None, cl=HWD, cd=F32):
        return L.adc_match_volumes_batch_device(None, 1, p, p, cost, cl, cd, disp, outs, n, None)

    for call in (host, dev):
        cases = [
            (dict(outs=_outs(good), n=4), b"n_outs"),
            (dict(outs=_outs(good), n=-1), b"n_outs"),
            (dict(outs=None, n=1), b"outs is NULL"),
            (dict(outs=_outs(good, (p, A.VOL_OPT, HWD, F32, 0)), n=2), b"requested twice"),
            (dict(outs=_outs((p, 3, HWD, F32, 0)), n=1), b"outs[0].stage"),
            (dict(outs=_outs((p, -1, HWD, F32, 0)), n=1), b"outs[0].stage"),
            (dict(outs=_outs(good, (p, A.VOL_COST, 2, F32, 0)), n=2), b"outs[1].layout"),
            (dict(outs=_outs((p, A.VOL_AGGR, HWD, 3, 0)), n=1), b"outs[0].dtype"),
            (dict(outs=_outs((None, A.VOL_AGGR, HWD, F32, 0)), n=1), b"outs[0].dst"),
            (dict(outs=_outs((p, A.VOL_AGGR, HWD, F32, 1)), n=1), b"outs[0].reserved"),
            (dict(outs=None, n=0, disp=None), b"disp"),
            (dict(outs=_outs(good), n=1, cost=p, cl=2), b"cost_layout"),
            (dict(outs=_outs(good), n=1, cost=p, cd=5), b"cost_dtype"),
        ]
        for kw, msg in cases:
            assert call(**kw) == 1, (call.__name__, kw)
            assert msg in L.adc_last_error(), (call.__name__, kw, L.adc_last_error())
        # valid requests get as far as the engine check: a bad cost layout is ignored without a cost, and a
        # volumes-only request (disp NULL) is valid
        assert call(_outs(good), 1, cost=None, cl=9) == 1 and b"engine is NULL" in L.adc_last_error()
        assert call(_outs(good), 1, disp=None) == 1 and b"engine is NULL" in L.adc_last_error()
        assert call(None, 0) == 1 and b"engine is NULL" in L.adc_last_error()
    # device destinations must be aligned to their element size; host destinations are copied into, so need not be
    assert dev(_outs((p + 2, A.VOL_OPT, HWD, F32, 0)), 1) == 1 and b"aligned" in L.adc_last_error()
    assert dev(_outs((p + 1, A.VOL_OPT, HWD, A.COST_BF16, 0)), 1) == 1 and b"aligned" in L.adc_last_error()
    assert dev(_outs((p + 2, A.VOL_OPT, HWD, A.COST_BF16, 0)), 1) == 1 and b"engine is NULL" in L.adc_last_error()
    assert host(_outs((p + 2, A.VOL_OPT, HWD, F32, 0)), 1) == 1 and b"engine is NULL" in L.adc_last_error()


def test_volume_stage_names():
    import adcensus_b200 as A
    assert (A.VOL_COST, A.VOL_AGGR, A.VOL_OPT) == (0, 1, 2)
    assert A.engine.VOL_STAGES == {"cost": 0, "aggr": 1, "opt": 2}
    assert A.Engine.PROFILE_KERNELS["cost_export"] == 11
    assert ctypes.sizeof(A.engine.VolumeOut) == 24


def _bf16_rn_exact(u: int) -> int:
    """Round-to-nearest-even of one finite f32 (bit pattern u) to bfloat16, by exact rational arithmetic."""
    x = Fraction(float(np.uint32(u).view(np.float32)))
    lo = u >> 16
    hi = lo + 1
    val = lambda b: Fraction(float(np.uint32((b & 0xFFFF) << 16).view(np.float32))) if (b & 0x7F80) != 0x7F80 \
        else None
    vlo, vhi = val(lo), val(hi)
    if vhi is None:                       # rounding up would reach the infinity encoding: compare with 2^128
        s = -1 if u >> 31 else 1
        vhi = s * Fraction(2) ** 128
    dlo, dhi = abs(x - vlo), abs(x - vhi)
    if dlo != dhi:
        return lo if dlo < dhi else hi & 0xFFFF
    return lo if lo % 2 == 0 else hi & 0xFFFF


def test_bf16_rn_helper_exact():
    """XT.to_bf16_rn_bits against an exact restatement: ties both ways, subnormals, values around 65520 and the top of
    the f32 range, random patterns."""
    rng = np.random.default_rng(11)
    pats = []
    for hi in (0x3F80, 0x3F81, 0x4000, 0x477F, 0x4780, 0x0001, 0x0040, 0x8001, 0xBF81, 0x7F7F, 0x7F7E, 0x0000, 0x8000):
        for lo in (0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF):
            pats.append(hi << 16 | lo)
    pats += list(np.arange(1, 0x10000, 97, dtype=np.uint64))                                 # subnormals
    for v in (65504.0, 65519.0, 65519.99, 65520.0, 65535.0, 65536.0, 65536.5, 1e-40, 3e38):
        pats.append(int(np.float32(v).view(np.uint32)))
    r = rng.integers(0, 2 ** 32, 3000, dtype=np.uint64)
    r = r[(r & 0x7F800000) != 0x7F800000]                                                       # finite only
    pats += list(r)
    u = np.array(pats, np.uint64).astype(np.uint32)
    got = XT.to_bf16_rn_bits(u.view(np.float32))
    want = np.array([_bf16_rn_exact(int(x)) for x in u], np.uint16)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]
    # f16: numpy's conversion is the IEEE round-to-nearest-even the export matches; 65520 and above overflow to +inf
    with np.errstate(over="ignore"):
        assert np.isinf(np.float32([65520.0, 65535.0, 65536.0]).astype(np.float16)).all()
    assert np.float16(np.float32(65519.99)) == np.float16(65504.0)


# ---- GPU ------------------------------------------------------------------------------------------
def _parity_cases():
    pick = {"130x70x37": lambda c: c[:3] == (130, 70, 37),             # D % 4 != 0
            "33x21x5": lambda c: c[2] == 5,
            "300x24x256": lambda c: c[2] == 256,
            "dmin2": lambda c: c[3].get("min_disparity") == 2,
            "dmin-4": lambda c: c[3].get("min_disparity") == -4,
            "disc": lambda c: c[3].get("do_discontinuity_adjustment") == 1,
            "97x61x24-unfused": lambda c: c[:3] == (97, 61, 24)}     # COST in volA instead of volB
    out = []
    for k, f in pick.items():
        (case,) = [c for c in E.PARITY_CASES if f(c)]
        out.append((k, case, "DBG_UNFUSED_AGG" if k.endswith("unfused") else 0))
    return out


PARITY = _parity_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c[0] for c in PARITY] + ["cone"])
def test_export_stage_parity(case, cone):
    """All three stages x both layouts x all three element types from match_volumes: f32 bit-identical to the
    restatement's COST/VOL_INIT, AGG4/VOL_AGGR, SO4/VOL_AGGR (DHW: their transpose), f16 / bf16 the round-to-nearest-even
    conversion of those, the map of the same call the restatement's final map."""
    import adcensus_b200 as A
    flags = 0
    if case == "cone":
        left, right = cone
        opt = T.default_option()
    else:
        _, (w, h, D, over, seed), flag = next(c for c in PARITY if c[0] == case)
        opt = T.default_option(**{"max_disparity": D, **over})
        left, right = T.synthetic_pair(w, h, D, seed)
        flags = getattr(A.engine, flag) if flag else 0
    h, w, _ = left.shape
    want = E.oracle_outputs(w, h, opt, left, right)
    eng = E.engine(w, h, opt, debug_flags=flags)
    for layout in LAYOUTS:
        for dtype in DTYPES:
            disp, vols = eng.match_volumes(left, right, STAGES, layout, dtype)
            E.same(f"{layout}/{dtype} map", disp, want["final"])
            for name in STAGES:
                E.same(f"{layout}/{dtype} {name}", vols[name], XT.export_of(want[name], layout, dtype))
            if case == "cone":
                assert T.sha(disp).startswith("77d70a58d1aa5c71")
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cloth3", "kitti_s1", "p1080_s1"])
def test_export_large_shapes_vs_reference_goldens(name):
    """AGGR and OPT f32 exports of Cloth3, 1242x375x128 and 1920x1080x192 against the reference's AGG4/VOL_AGGR and
    SO4/VOL_AGGR hashes.  1080p goes through the batched device call with two pairs, so that the second pair's
    volumes (1.6 GB each) lie beyond 2^31 bytes of the destinations; its OPT volume is exported as DHW and transposed back
    on the host."""
    g = E.golden("golden_big.json")[name]
    if name == "cloth3":
        z = np.load(T.GOLDEN_DIR / "real_pairs.npz")
        left, right = z["cloth3_left"], z["cloth3_right"]
        D = g["max_disparity"]
    else:
        w, h, D = g["width"], g["height"], g["max_disparity"]
        left, right = T.synthetic_pair(w, h, D, int(name.rsplit("_s", 1)[1]))
    assert [T.sha(left), T.sha(right)] == g["input_sha"]
    h, w, _ = left.shape
    opt = T.default_option(max_disparity=D)
    if name != "p1080_s1":
        eng = E.engine(w, h, opt)
        disp, vols = eng.match_volumes(left, right, ["aggr", "opt"], "hwd", "f32")
        assert T.sha(vols["aggr"]) == g["hashes"]["AGG4/VOL_AGGR"]
        assert T.sha(vols["opt"]) == g["hashes"]["SO4/VOL_AGGR"]
        assert T.sha(disp) == g["hashes"]["MEDIAN/DISP_L"]
        eng.close()
        return
    import torch
    dev = torch.device("cuda", 0)
    n, ND = 2, h * w * D
    d_opt = torch.empty((n, D, h, w), dtype=torch.float32, device=dev)     # before the engine: its sizing sees them
    d_agg = torch.empty((n, h, w, D), dtype=torch.float32, device=dev)
    eng = E.engine(w, h, opt)
    d_l = torch.from_numpy(np.stack([left] * n)).to(dev)
    d_r = torch.from_numpy(np.stack([right] * n)).to(dev)
    d_disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream()
    eng.match_volumes_batch_device(n, d_l.data_ptr(), d_r.data_ptr(),
                                   [(d_opt.data_ptr(), "opt", "dhw", "f32"), (d_agg.data_ptr(), "aggr", "hwd", "f32")],
                                   d_disp=d_disp.data_ptr(), stream=st.cuda_stream)
    torch.cuda.synchronize()
    assert n * ND * 4 > 2 ** 31
    for i in range(n):
        assert T.sha(d_disp[i].cpu().numpy()) == g["hashes"]["MEDIAN/DISP_L"], f"pair {i} map"
        assert T.sha(d_agg[i].cpu().numpy()) == g["hashes"]["AGG4/VOL_AGGR"], f"pair {i} aggr"
        opt_hwd = d_opt[i].permute(1, 2, 0).contiguous().cpu().numpy()
        assert T.sha(opt_hwd) == g["hashes"]["SO4/VOL_AGGR"], f"pair {i} opt"
        del opt_hwd
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", GC.COST_CASES, ids=[GC.cost_case_id(c) for c in GC.COST_CASES])
def test_export_cost_input_round_trip(case):
    """A caller's cost in, the engine's volumes out: AGGR / OPT hash to the reference's AGG4 / SO4 volumes for that
    cost, COST is the cost itself, the map the reference's."""
    want = E.golden("golden_cost_cases.json")[GC.cost_case_id(case)]
    left, right, opt, cost = GC.cost_case_inputs(case)
    h, w, _ = left.shape
    eng = E.engine(w, h, opt)
    for cl in LAYOUTS:
        c = cost if cl == "hwd" else np.ascontiguousarray(cost.transpose(2, 0, 1))
        disp, vols = eng.match_volumes(left, right, STAGES, "hwd", "f32", cost=c, cost_layout=cl)
        E.same(f"{cl} cost", vols["cost"], CT.cost_domain(cost))
        assert T.sha(vols["aggr"]) == want["AGG4/VOL_AGGR"], cl
        assert T.sha(vols["opt"]) == want["SO4/VOL_AGGR"], cl
        assert T.sha(disp) == want["MEDIAN/DISP_L"], cl
        _, vo = eng.match_volumes(left, right, "opt", "dhw", "bf16", cost=c, cost_layout=cl, disparity=False)
        E.same(f"{cl} opt dhw bf16", vo["opt"], XT.export_of(vols["opt"], "dhw", "bf16"))
    eng.close()


@pytest.mark.gpu
def test_export_cost_value_domain():
    """COST export in cost-input mode = the ingested volume after the value domain, specials included."""
    w, h, D = 64, 40, 20
    opt = T.default_option(max_disparity=D)
    left, right = T.synthetic_pair(w, h, D, 51)
    cost = CT.synthetic_cost(w, h, D, 51) * np.float32(2000.0)
    rng = np.random.default_rng(5)
    specials = np.array([np.nan, np.inf, -np.inf, -0.0, -3.0, -1e-30, 65536.0, 70000.0, 1e38, 65535.5], np.float32)
    mask = rng.random(cost.shape) < 0.08
    cost[mask] = specials[rng.integers(0, len(specials), int(mask.sum()))]
    clamped = CT.cost_domain(cost)
    eng = E.engine(w, h, opt)
    want_disp = eng.match_cost(left, right, cost, "hwd")
    for layout in LAYOUTS:
        for dtype in DTYPES:
            disp, vols = eng.match_volumes(left, right, ["cost"], layout, dtype, cost=cost)
            E.same(f"{layout}/{dtype} cost", vols["cost"], XT.export_of(clamped, layout, dtype))
            E.same(f"{layout}/{dtype} map", disp, want_disp)
    eng.close()


@pytest.mark.gpu
def test_volumes_only_mode():
    """disparity=False: the same volumes as a call with a map, fewer launches, no map; a call with a map after it
    still gives the right map and right-view map."""
    w, h, D = 97, 61, 23
    opt = T.default_option(max_disparity=D)
    left, right = T.synthetic_pair(w, h, D, 2)
    eng = E.engine(w, h, opt)
    want = eng.match(left, right)
    want_r = eng.right_disparity()
    c0 = eng.launch_count
    eng.match(left, right)
    per_match = eng.launch_count - c0
    for stages in (["cost"], ["aggr"], ["opt"], ["cost", "opt"], STAGES):
        c0 = eng.launch_count
        disp, full = eng.match_volumes(left, right, stages, "dhw", "bf16")
        with_map = eng.launch_count - c0
        assert with_map == per_match + len(stages), stages
        E.same(f"{stages} map", disp, want)
        E.same(f"{stages} right map", eng.right_disparity(), want_r)
        c0 = eng.launch_count
        none, only = eng.match_volumes(left, right, stages, "dhw", "bf16", disparity=False)
        assert none is None
        assert eng.launch_count - c0 < with_map, stages
        for s in stages:
            E.same(f"{stages} {s}", only[s], full[s])
    eng.close()


def _export_batch_check(eng, pairs, n, specs, with_disp, pipelined):
    """n pairs (pair i = pairs[i % len(pairs)]) through match_volumes_batch_device with the volume requests `specs`
    [(stage, layout, dtype, skew)], each destination `skew` elements into a buffer with 4096 elements of 0xA5 bytes on
    either side; every volume and map equals the single-pair match_volumes result at its offset, and no element outside
    the n volumes changes."""
    torch, dev = E.cuda()
    H, W, D = eng.height, eng.width, eng.D
    ND = H * W * D
    k = len(pairs)
    singles = []
    for (l, r) in pairs:
        disp = None
        vols = {}
        for (stage, layout, dtype, _) in specs:
            disp, v = eng.match_volumes(l, r, [stage], layout, dtype)
            vols[stage] = v[stage]
        singles.append((disp, vols))
    d_l = torch.from_numpy(np.stack([pairs[i % k][0] for i in range(n)])).to(dev)
    d_r = torch.from_numpy(np.stack([pairs[i % k][1] for i in range(n)])).to(dev)
    d_out = torch.full((n, H, W), -1.0, dtype=torch.float32, device=dev) if with_disp else None
    es = {"f32": 4, "f16": 2, "bf16": 2}
    bufs = [E.guarded(n * ND * es[dtype], torch.uint8, (4096 + skew) * es[dtype], (4096 - skew) * es[dtype], 0xA5)
            for (_, _, dtype, skew) in specs]
    st = torch.cuda.current_stream()

    def issue(first, count):
        outs = [(data.data_ptr() + first * ND * es[dtype], stage, layout, dtype)
                for (data, _), (stage, layout, dtype, _) in zip(bufs, specs)]
        eng.match_volumes_batch_device(count, d_l[first:].data_ptr(), d_r[first:].data_ptr(), outs,
                                       d_disp=d_out[first:].data_ptr() if with_disp else 0, stream=st.cuda_stream)

    E.split_calls(eng, n, pipelined, issue)
    if with_disp:
        out = d_out.cpu().numpy()
        for i in range(n):
            E.same(f"pair {i} map", out[i], singles[i % k][0])
    for (data, intact), (stage, layout, dtype, _) in zip(bufs, specs):
        assert intact(), f"{stage}: bytes outside the volumes written"
        got = data.cpu().numpy()
        shape = (H, W, D) if layout == "hwd" else (D, H, W)
        for i in range(n):
            want = singles[i % k][1][stage]
            raw = got[i * ND * es[dtype]:(i + 1) * ND * es[dtype]]
            E.same(f"pair {i} {stage} {layout}/{dtype}", raw.view(want.dtype).reshape(shape), want)


# N = 71*47 and D = 23 are odd: pair i starts at an odd element, so every path of the kernels' alignment handling runs
BATCH_SPECS = [("cost", "hwd", "f16", 1), ("aggr", "dhw", "bf16", 1), ("opt", "dhw", "f32", 0)]
BATCH_SPECS_B = [("cost", "dhw", "f16", 0), ("aggr", "hwd", "f32", 1), ("opt", "hwd", "bf16", 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_export_batch_device_order_and_stride(pipelined):
    """Case A: n = 3 * wave_pairs + 2 distinct pairs, wave_pairs = 4, lanes = 3; every stage, mixed layouts / types, odd
    volume sizes and odd destination offsets."""
    w, h, D = 71, 47, 23
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt, wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    pairs = [T.synthetic_pair(w, h, D, 100 + s) for s in range(n)]
    _export_batch_check(eng, pairs, n, BATCH_SPECS, True, pipelined)
    _export_batch_check(eng, pairs, n, BATCH_SPECS_B, True, pipelined)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_export_batch_device_loaded_waves(pipelined):
    """Case B: default configuration with several waves per lane in flight, DHW bf16 OPT export plus the map."""
    w, h, D = 160, 120, 64
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt)
    n = 2 * eng.wave_pairs * eng.lanes + 5
    pairs = [T.synthetic_pair(w, h, D, 200 + s) for s in range(7)]
    _export_batch_check(eng, pairs, n, [("opt", "dhw", "bf16", 0)], True, pipelined)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_export_batch_device_volumes_only(pipelined):
    """Case C: no map output; the pipeline stops after the optimised volume."""
    w, h, D = 71, 47, 23
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt, wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    pairs = [T.synthetic_pair(w, h, D, 300 + s) for s in range(n)]
    _export_batch_check(eng, pairs, n, [("opt", "dhw", "bf16", 1), ("cost", "hwd", "f32", 0)], False, pipelined)
    eng.close()


@pytest.mark.gpu
def test_export_batch_device_cost_input():
    """The round trip on the device: a bf16 [N, D, H, W] cost in, the optimised volume out, with and without a map."""
    import torch
    dev = torch.device("cuda", 0)
    w, h, D = 72, 48, 24
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt, wave_pairs=4, lanes=2)
    n = 11
    ins = [T.synthetic_pair(w, h, D, 400 + s) for s in range(n)]
    costs = [np.ascontiguousarray(CT.synthetic_cost(w, h, D, 400 + s).transpose(2, 0, 1)) for s in range(n)]
    d_l = torch.from_numpy(np.stack([p[0] for p in ins])).to(dev)
    d_r = torch.from_numpy(np.stack([p[1] for p in ins])).to(dev)
    d_c = torch.from_numpy(np.stack([CT.to_bf16_bits(c) for c in costs])).to(dev)
    st = torch.cuda.current_stream()
    for with_disp in (True, False):
        d_opt = torch.empty((n, D, h, w), dtype=torch.bfloat16, device=dev)
        d_disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
        eng.match_volumes_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), [(d_opt.data_ptr(), "opt", "dhw", "bf16")],
                                       d_disp=d_disp.data_ptr() if with_disp else 0, d_cost=d_c.data_ptr(),
                                       cost_layout="dhw", cost_dtype="bf16", stream=st.cuda_stream)
        torch.cuda.synchronize()
        got = d_opt.view(torch.int16).cpu().numpy().view(np.uint16)
        for i in range(n):
            disp, v = eng.match_volumes(ins[i][0], ins[i][1], "opt", "dhw", "bf16", cost=CT.to_bf16_bits(costs[i]),
                                        cost_layout="dhw", cost_dtype="bf16")
            E.same(f"pair {i} opt", got[i], v["opt"])
            if with_disp:
                E.same(f"pair {i} map", d_disp[i].cpu().numpy(), disp)
    eng.close()


@pytest.mark.gpu
def test_no_export_path_unchanged(cone):
    """match_batch_device maps and launch count of a batch are the same before and after export calls on the engine."""
    import torch
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option(), wave_pairs=4, lanes=3)
    n = 9
    dev = torch.device("cuda", 0)
    d_l = torch.from_numpy(np.repeat(left[None], n, 0)).to(dev)
    d_r = torch.from_numpy(np.repeat(right[None], n, 0)).to(dev)
    st = torch.cuda.current_stream()

    def batch():
        d = torch.zeros((n, h, w), dtype=torch.float32, device=dev)
        c0 = eng.launch_count
        eng.match_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), d.data_ptr(), st.cuda_stream)
        torch.cuda.synchronize()
        return d.cpu().numpy(), eng.launch_count - c0

    maps0, launches0 = batch()
    d_v = torch.empty((n, 64, h, w), dtype=torch.bfloat16, device=dev)
    eng.match_volumes_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), [(d_v.data_ptr(), "opt", "dhw", "bf16")],
                                   stream=st.cuda_stream)
    eng.match_volumes(left, right, STAGES, "hwd", "f16")
    torch.cuda.synchronize()
    maps1, launches1 = batch()
    E.same("maps", maps1, maps0)
    assert launches1 == launches0
    hashes = E.golden_hashes("cone_full")
    assert all(T.sha(maps1[i]) == hashes["MEDIAN/DISP_L"] for i in range(n))
    eng.close()
