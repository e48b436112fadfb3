"""Dirty-engine parity: every entry point against the oracle with lane arenas poisoned before each wave and call, and
through one engine's long history of calls.

Most tests build a fresh engine, whose arena adc_create zeroes; a long-lived engine holds the previous wave's or
call's data instead, and other entry points use lane 0's buffers as scratch.  So a kernel that reads memory its own wave
did not write would pass them wherever zero ("no label", "no count", "cost 0") happens to be the right answer.
adc_config.debug_flags = ADC_DBG_POISON | ADC_DBG_POISON_BYTE(b) fills every byte of the arena (and the host calls'
device staging) with b before every wave and every one-pair call: 0xFF (NaN floats, -1 integers), 0x7F (3.4e38
floats, large positive integers) or 0x01 (every byte label a mismatch).

CPU: the flag constants of the header and the binding; the instantiation subset still reaches every template
instantiation in the library; the call script names every entry point of the header that matches, ingests or
post-processes.
GPU, every output bit for bit against each pair's oracle run, the reference's hashes or a numpy restatement:
  - poisoning takes effect (taps a COST run has not reached hold the pattern; zeros without the flag);
  - PARITY_CASES and Cone stage by stage and through match_outputs_batch_device (waves of 2 on 2 lanes, n odd);
  - a subset of the sweep cases that reaches every instantiation, and the option-space flag cases, through check_case,
    also with each other ADC_DBG_* flag;
  - every entry point on 72x48, dmin -3, with partial waves (CALLS);
  - 1242x375x128 with the default configuration and wave_pairs + 1 pairs against the reference's hashes;
  - the call script on one long-lived engine (poison off, pipelined off and on), forwards then backwards, each call
    against the same call on a fresh engine and against the oracle.
"""
import ctypes
import functools
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import adc_testlib as T
import bayer_testlib as B
import cloud_testlib as CL
import cost_testlib as CT
import engine_testlib as E  # puts tools/ on sys.path
import images_testlib as I
import make_golden_options as GO
import maps_testlib as MT
import rawdepth_testlib as RD
import rectify_testlib as R
import reproject_testlib as RP
import speckle_testlib as SP
import yuv_testlib as Y
from sweep_testlib import PLAN_CASES, Case, check_case, library_instantiations, plans, reached, sweep_case  # noqa: F401

POISON = 16
PATTERNS = (0xFF, 0x7F, 0x01)
HEADER = T.REPO / "include" / "adcensus_b200.h"


def flags(byte):
    import adcensus_b200 as A
    return A.engine.poison_flags(byte)


def test_poison_flag_constants():
    """ADC_DBG_POISON and ADC_DBG_POISON_BYTE in the header agree with the binding's DBG_POISON and poison_flags."""
    import adcensus_b200 as A
    h = HEADER.read_text()
    assert re.search(r"ADC_DBG_POISON = 16\b", h)
    assert re.search(r"#define ADC_DBG_POISON_BYTE\(b\) \(\(\(b\) & 0xff\) << 8\)", h)
    assert A.engine.DBG_POISON == POISON
    assert [A.engine.poison_flags(b) for b in (0xFF, 0x7F, 0x01, 0x100)] == [0xFF10, 0x7F10, 0x0110, 0x0010]


# ---- poisoning takes effect ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("byte", PATTERNS)
def test_poison_takes_effect(byte):
    """After debug_run(..., "COST") the buffers of later stages (DISP_L, DISP_R, ARMS, SUPCNT_H) hold the pattern bit for
    bit on a poisoned engine, and zeros on an unflagged fresh one: the fill reaches lane 0's arena before the run."""
    w, h, D = 64, 48, 16
    left, right = T.synthetic_pair(w, h, D, 1)
    for fl, want in ((flags(byte), byte), (0, 0)):
        eng = E.engine(w, h, T.default_option(max_disparity=D), debug_flags=fl)
        eng.debug_run(left, right, "COST")
        for tap in ("DISP_L", "DISP_R", "ARMS", "SUPCNT_H"):
            got = np.ascontiguousarray(eng.tap(tap)).view(np.uint8)
            assert (got == want).all(), f"{tap}: {int((got != want).sum())} bytes are not {want:#04x} (flags {fl:#x})"
        eng.close()


# ---- stage parity under poison ---------------------------------------------------------------------------------------
STAGE_CASES = [(f"{c[0]}x{c[1]}x{c[2]}-{i}", c) for i, c in enumerate(E.PARITY_CASES)] + [("cone", None)]
# the cases also run with 0x7F and 0x01: the defaults, no LR check, no filling, a negative dmin, D = 256
MORE_PATTERNS = {"64x48x16-0", "80x60x32-7", "80x60x32-8", "80x60x32-13", "300x24x256-15"}
STAGE_PARAMS = [pytest.param(name, c, 0xFF, id=f"{name}-ff") for name, c in STAGE_CASES] + \
    [pytest.param(name, c, b, id=f"{name}-{b:02x}") for name, c in STAGE_CASES if name in MORE_PATTERNS for b in (0x7F, 0x01)]


def _stage_inputs(c, cone):
    """(W, H, option, three distinct pairs) of a stage-parity case; Cone's other pairs are its mirror and its flip."""
    if c is None:
        l, r = cone
        h, w, _ = l.shape
        pairs = [(l, r), (np.ascontiguousarray(r[:, ::-1]), np.ascontiguousarray(l[:, ::-1])),
                 (np.ascontiguousarray(l[::-1]), np.ascontiguousarray(r[::-1]))]
        return w, h, T.default_option(), pairs
    w, h, D, over, seed = c
    return w, h, T.default_option(**{"max_disparity": D, **over}), [T.synthetic_pair(w, h, D, seed + 100 * i) for i in range(3)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,c,byte", STAGE_PARAMS)
def test_stage_parity_poisoned(name, c, byte, cone):
    """Every tap after every stage of the staged debug run, then one match_outputs_batch_device call over three pairs
    (waves of 2 on 2 lanes: the second wave's empty slot holds the pattern) exporting the three volumes, both WTA maps,
    the outlier map, both confidence maps and the final map, against each pair's oracle run."""
    torch, dev = E.cuda()
    w, h, opt, pairs = _stage_inputs(c, cone)
    with ThreadPoolExecutor(len(pairs)) as ex:
        futs = [ex.submit(E.oracle_outputs, w, h, opt, l, r) for l, r in pairs]
        eng = E.engine(w, h, opt, wave_pairs=2, lanes=2, debug_flags=flags(byte))
        left, right = pairs[0]
        orc = T.Oracle(w, h, opt)
        orc.begin(left, right)
        for st in T.STAGES:
            orc.step()
            eng.debug_run(left, right, st)
            for tap in T.STAGE_TAPS[st]:
                E.same(f"{name} {st}/{tap}", eng.tap(tap), orc.tap(tap))
        orc.close()
        d_l = torch.from_numpy(np.stack([p[0] for p in pairs])).to(dev)
        d_r = torch.from_numpy(np.stack([p[1] for p in pairs])).to(dev)
        got = E.batch_outputs(eng, eng.match_outputs_batch_device, len(pairs), d_l.data_ptr(), d_r.data_ptr(), 3 * w * h,
                              volumes=[(s, "hwd", "f32") for s in ("cost", "aggr", "opt")],
                              maps=["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"])
        eng.close()
        want = [f.result() for f in futs]
    for i, wi in enumerate(want):
        _same_outputs(f"{name} pair {i}", {k: v[i] for k, v in got.items()}, _oracle_maps(wi))


def _oracle_maps(w):
    """The outputs of match_outputs* for one pair, from its oracle run."""
    mc, pr = MT.confidence(w["opt"])
    return {"disp": w["final"], "cost": w["cost"], "aggr": w["aggr"], "opt": w["opt"], "wta_left": w["wta_left"],
            "wta_right": w["wta_right"], "outliers": (w["mismatches"].reshape(-1, 2), w["occlusions"].reshape(-1, 2)),
            "min_cost": mc, "peak_ratio": pr}


def _same_outputs(tag, got, want):
    """Every output named in `want` bit for bit; the outlier map against the one its mismatch / occlusion lists give,
    reprojected points and depths NaN-insensitively (their NaN payloads are not part of the contract)."""
    for k, wv in want.items():
        if k == "outliers":     # the whole map: 0 where neither list has the pixel
            want_map = np.zeros(np.shape(got[k]), np.uint8)
            for label, lst in ((1, wv[0]), (2, wv[1])):
                want_map[lst[:, 1], lst[:, 0]] = label
            E.same(f"{tag} {k}", np.asarray(got[k]), want_map)
        elif k.startswith("points") or k.startswith("depth"):
            assert RP.same_nan(got[k], wv), f"{tag} {k}: differs (NaN-insensitive)"
        else:
            E.same(f"{tag} {k}", np.asarray(got[k]), np.asarray(wv))


# ---- every instantiation under poison --------------------------------------------------------------------------------
# A subset of test_kernel_sweep's cases that together launch every instantiation of the seven templated kernels
# (sweep_testlib.reached); test_instantiation_subset_is_complete fails when a library change leaves one out.
INSTANTIATION_SUBSET = ["D1", "cost_volume_exact", "cost_volume_padded_ldg", "so_t2_lps16", "D8", "D40", "D12", "D18",
                        "D16", "D24", "D25", "D42", "D48", "D54", "D60", "D66", "D56", "D96", "D64", "D80", "D102",
                        "D114", "D132", "D128", "D112", "D162", "D192", "D198", "D160", "D228", "D224", "D256"]
# (case, other ADC_DBG_* flags, pattern): poison with each other test hook at least once, and the other patterns
COMBINED = [("D64", 1, 0xFF), ("D96", 2, 0xFF), ("D40", 4, 0xFF), ("D24", 8, 0xFF), ("D256", 8 | 2, 0x7F), ("D16", 0, 0x7F),
            ("D25", 0, 0x01), ("cost_volume_exact", 4, 0x01)]
OPTION_CASES = GO.cases()
FLAG_CASES = sorted(n for n in OPTION_CASES if n.startswith("flags_"))


def _subset_case(name):
    return PLAN_CASES[name][0] if name in PLAN_CASES else sweep_case(int(name[1:]))


def test_instantiation_subset_is_complete(plans):
    """The poisoned subset reaches every instantiation of the templated kernels in the library, and the flag cases are
    the eight flag combinations with dmin = 0 and dmin < 0."""
    lib = library_instantiations()
    union = set().union(*(reached(_subset_case(n), plans) for n in INSTANTIATION_SUBSET))
    assert union == lib, f"instantiations the poisoned subset does not reach: {sorted(lib - union)}"
    fl = {(o.do_lr_check, o.do_filling, o.do_discontinuity_adjustment, o.min_disparity < 0)
          for o in (GO.option(OPTION_CASES[n][2]) for n in FLAG_CASES)}
    assert len(fl) == 16 and len(FLAG_CASES) == 16
    for fl_other in (1, 2, 4, 8):
        assert any(f & fl_other for _, f, _ in COMBINED), fl_other


@pytest.mark.gpu
@pytest.mark.parametrize("name", INSTANTIATION_SUBSET)
def test_instantiation_poisoned(name):
    check_case(_subset_case(name), debug_flags=flags(0xFF))


@pytest.mark.gpu
@pytest.mark.parametrize("name,other,byte", COMBINED, ids=[f"{n}-dbg{f}-{b:02x}" for n, f, b in COMBINED])
def test_instantiation_poisoned_with_other_hooks(name, other, byte):
    check_case(_subset_case(name), debug_flags=flags(byte) | other)


@pytest.mark.gpu
@pytest.mark.parametrize("name", FLAG_CASES)
def test_option_flag_case_poisoned(name):
    W_, H_, over, seed = OPTION_CASES[name]
    check_case(Case(name, W_, H_, GO.option(over), seed), debug_flags=flags(0xFF))


# ---- every entry point (CALLS) ---------------------------------------------------------------------------------------
W, H, DMIN, DMAX = 72, 48, -3, 21
D = DMAX - DMIN
WAVE, LANES = 2, 2
N = 5                               # pairs of a batch call: waves of 2, 2 and 1, both lanes reused, the last wave partial
OPT = T.default_option(min_disparity=DMIN, max_disparity=DMAX)
RECT_SMALL, RECT_LARGE = (80, 56), (400, 300)   # raw frames: 2*80*56*3 bytes fit in a lane volume (2*N*Dp*4), 2*400*300*3 do not
SPECKLE = (30, 0.25)
IMAGE_FORMATS = ("gray", "rgb_planar", "nv12", "bayer_rggb", "bayer_rg12p")
DEBUG_STOPS = ("COST", "AGG2", "SO4", "WTA", "OUTLIER", "VOTE", "MEDIAN")


def _seed(k, i):
    return 1000 * k + i


def _pair(k, i, w=W, h=H):
    return T.synthetic_pair(w, h, D, _seed(k, i))


def _stack(k, n=N):
    ps = [_pair(k, i) for i in range(n)]
    return np.stack([p[0] for p in ps]), np.stack([p[1] for p in ps])


@functools.cache
def _oracle_views(left_bytes, right_bytes):
    l = np.frombuffer(left_bytes, np.uint8).reshape(H, W, 3)
    r = np.frombuffer(right_bytes, np.uint8).reshape(H, W, 3)
    return E.oracle_outputs(W, H, OPT, l, r)


def oracle(l, r):
    """The oracle outputs of one pair of packed BGR views (cached)."""
    return _oracle_views(np.ascontiguousarray(l).tobytes(), np.ascontiguousarray(r).tobytes())


def _oracles(pairs):
    with ThreadPoolExecutor(8) as ex:
        return list(ex.map(lambda p: oracle(*p), pairs))


@functools.cache
def _cost(k, i):
    return CT.synthetic_cost(W, H, D, _seed(k, i), DMIN)


@functools.cache
def _cost_final(k, i):
    l, r = _pair(k, i)
    return CT.CostOracle(W, H, OPT).match_cost(l, r, _cost(k, i))


def _q():
    return np.load(T.GOLDEN_DIR / "golden_reproject_cases.npz")["rig_zero_0/Q"]


def _dev(a):
    torch, dev = E.cuda()
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _done(eng):
    """Joins the engine's work onto the current stream (needed in pipelined mode) and waits for it."""
    torch, _ = E.cuda()
    eng.join(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def _st():
    torch, _ = E.cuda()
    return torch.cuda.current_stream().cuda_stream


def _lib_call(eng, fn, *args):
    import adcensus_b200 as A
    A.engine._check(getattr(eng._L, fn)(eng._h, *args))


# Each call: run(eng, k) -> {output: host array} and want(k) -> {output: expected}, k choosing the call's own pairs.
def c_match(eng, k):
    l, r = _pair(k, 0)
    return {"disp": eng.match(l, r), "right": eng.right_disparity()}


def w_match(k):
    o = oracle(*_pair(k, 0))
    return {"disp": o["final"], "right": o["wta_right"]}


def c_match_cost(eng, k):
    l, r = _pair(k, 0)
    return {"disp": eng.match_cost(l, r, _cost(k, 0), "hwd")}


def w_match_cost(k):
    return {"disp": _cost_final(k, 0)}


def w_finals(k, n=N):
    return {"disp": np.stack([o["final"] for o in _oracles([_pair(k, i) for i in range(n)])])}


def c_batch_pageable(eng, k):
    ls, rs = _stack(k)
    return {"disp": eng.match_batch(ls, rs)}


def c_batch_ptrs_pageable(eng, k):
    ls, rs = _stack(k)
    return {"disp": np.stack(eng.match_batch_ptrs(list(ls), list(rs)))}


def _pinned(a):
    torch, _ = E.cuda()
    t = torch.empty(a.shape, dtype=torch.uint8 if a.dtype == np.uint8 else torch.float32, pin_memory=True)
    t.numpy()[...] = a
    return t


def c_batch_pinned(eng, k):
    """adc_match_batch_strided and adc_match_batch on pinned buffers (one copy per view and wave, one per pair)."""
    ls, rs = _stack(k)
    pl, pr, pd = _pinned(ls), _pinned(rs), _pinned(np.full((N, H, W), -7.0, np.float32))
    _lib_call(eng, "adc_match_batch_strided", N, pl.data_ptr(), pr.data_ptr(), pd.data_ptr())
    out = {"strided": pd.numpy().copy()}
    pd.numpy()[...] = -7.0
    arr = ctypes.c_void_p * N
    _lib_call(eng, "adc_match_batch", N, arr(*[pl[i].data_ptr() for i in range(N)]),
              arr(*[pr[i].data_ptr() for i in range(N)]), arr(*[pd[i].data_ptr() for i in range(N)]))
    out["ptrs"] = pd.numpy().copy()
    return out


def w_batch_pinned(k):
    f = w_finals(k)["disp"]
    return {"strided": f, "ptrs": f}


def c_pinned_async(eng, k):
    ls, rs = _stack(k)
    pl, pr, pd = _pinned(ls), _pinned(rs), _pinned(np.full((N, H, W), -7.0, np.float32))
    eng.match_batch_pinned_async(N, pl.data_ptr(), pr.data_ptr(), pd.data_ptr(), _st())
    _done(eng)
    return {"disp": pd.numpy().copy()}


def c_batch_device(eng, k):
    torch, dev = E.cuda()
    ls, rs = _stack(k)
    dl, dr = _dev(ls), _dev(rs)
    dd = torch.full((N, H, W), -7.0, device=dev)
    eng.match_batch_device(N, dl.data_ptr(), dr.data_ptr(), dd.data_ptr(), _st())
    _done(eng)
    return {"disp": dd.cpu().numpy()}


def _cost_device(dtype, layout):
    def run(eng, k):
        torch, dev = E.cuda()
        ls, rs = _stack(k)
        c = np.stack([_cost(k, i) for i in range(N)])
        if layout == "dhw":
            c = c.transpose(0, 3, 1, 2)
        c = CT.to_bf16_bits(c).view(np.int16) if dtype == "bf16" else c.astype(np.float16 if dtype == "f16" else np.float32)
        dl, dr, dc = _dev(ls), _dev(rs), _dev(c)
        dd = torch.full((N, H, W), -7.0, device=dev)
        eng.match_cost_batch_device(N, dl.data_ptr(), dr.data_ptr(), dc.data_ptr(), dd.data_ptr(), layout, dtype, _st())
        _done(eng)
        return {"disp": dd.cpu().numpy()}
    return run


def w_cost_device(k):
    return {"disp": np.stack([_cost_final(k, i) for i in range(N)])}


def _volumes_only_device(stage):
    """adc_match_volumes_batch_device without a final map: the run stops after the stage of the one volume."""
    def run(eng, k):
        torch, dev = E.cuda()
        ls, rs = _stack(k, 3)
        dl, dr = _dev(ls), _dev(rs)
        v = torch.full((3, H, W, D), float("nan"), device=dev)
        eng.match_volumes_batch_device(3, dl.data_ptr(), dr.data_ptr(), [(v.data_ptr(), stage, "hwd", "f32")], stream=_st())
        _done(eng)
        return {stage: v.cpu().numpy()}
    return run


def _w_volume(stage):
    def want(k):
        return {stage: np.stack([o[stage] for o in _oracles([_pair(k, i) for i in range(3)])])}
    return want


def c_volumes_host(eng, k):
    l, r = _pair(k, 0)
    disp, v = eng.match_volumes(l, r, ["aggr"], disparity=False)
    assert disp is None
    return {"aggr": v["aggr"]}


def w_volumes_host(k):
    return {"aggr": oracle(*_pair(k, 0))["aggr"]}


MAPS = ["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"]
VOLS = ["cost", "aggr", "opt"]


def c_outputs_host(eng, k):
    l, r = _pair(k, 0)
    disp, out = eng.match_outputs(l, r, maps=MAPS, volumes=VOLS)
    return {"disp": disp, **out}


def w_outputs_host(k):
    return _oracle_maps(oracle(*_pair(k, 0)))


def c_outputs_batch(eng, k):
    ls, rs = _stack(k)
    dl, dr = _dev(ls), _dev(rs)     # held until the call has read them
    return E.batch_outputs(eng, eng.match_outputs_batch_device, N, dl.data_ptr(), dr.data_ptr(), 3 * W * H,
                           volumes=[(s, "hwd", "f32") for s in VOLS], maps=MAPS)


def w_outputs_batch(k):
    ws = [_oracle_maps(o) for o in _oracles([_pair(k, i) for i in range(N)])]
    out = {key: np.stack([w[key] for w in ws]) for key in ws[0] if key != "outliers"}
    out["outliers"] = [w["outliers"] for w in ws]
    return out


def _frame(fmt, bgr, seed):
    """(the frame of a packed BGR view in format fmt, the packed BGR view the engine matches for it)."""
    if fmt == "gray":
        g = I.from_bgr(bgr, "gray")
        return g, I.gray_to_bgr(g)
    if fmt == "rgb_planar":
        return I.from_bgr(bgr, fmt), bgr
    if fmt == "nv12":
        f = Y.encode(bgr, "nv12")
        return f, Y.decode(f, "nv12", W, H)
    if fmt in B.PATTERNS:
        f = B.mosaic(bgr, fmt)
        return f, B.demosaic(f, fmt)
    f = RD.encode(bgr, fmt, np.random.default_rng(seed))
    return f, RD.decode(f, fmt, W, H)


def _frames(fmt, k, n):
    out = []
    for i in range(n):
        l, r = _pair(k, i)
        (fl, vl), (fr, vr) = _frame(fmt, l, _seed(k, i)), _frame(fmt, r, _seed(k, i) + 1)
        out.append((fl, fr, vl, vr))
    return out


def _images_device(fmt):
    def run(eng, k):
        import adcensus_b200 as A
        torch, dev = E.cuda()
        fr = _frames(fmt, k, 3)
        dl, dr = _dev(np.stack([f[0] for f in fr])), _dev(np.stack([f[1] for f in fr]))
        dd = torch.full((3, H, W), -7.0, device=dev)
        eng.match_images_batch_device(3, dl.data_ptr(), dr.data_ptr(), image=A.image_desc(fmt), d_disp=dd.data_ptr(),
                                      stream=_st())
        _done(eng)
        return {"disp": dd.cpu().numpy()}
    return run


def _images_host(fmt):
    def run(eng, k):
        fl, fr, _, _ = _frames(fmt, k, 1)[0]
        disp, _ = eng.match_images(fl, fr, format=fmt)
        return {"disp": disp}
    return run


def _w_images(fmt, n):
    def want(k):
        return {"disp": np.stack([o["final"] for o in _oracles([(f[2], f[3]) for f in _frames(fmt, k, n)])])[:n]
                if n > 1 else oracle(*_frames(fmt, k, 1)[0][2:])["final"]}
    return want


def _raw(k, i, size):
    return T.synthetic_pair(size[0], size[1], D, _seed(k, i) + 7)


def _rect_maps(k, size):
    return tuple(R.warp_maps(W, H, size[0], size[1], _seed(k, 50 + v)) for v in range(2))


def _rectified(size, device):
    def run(eng, k):
        torch, dev = E.cuda()
        eng.set_rectification(*_rect_maps(k, size), src_size=size)
        if not device:
            l, r = _raw(k, 0, size)
            disp, _ = eng.match_rectified(l, r)
            return {"disp": disp}
        raws = [_raw(k, i, size) for i in range(3)]
        dl, dr = _dev(np.stack([p[0] for p in raws])), _dev(np.stack([p[1] for p in raws]))
        dd = torch.full((3, H, W), -7.0, device=dev)
        eng.match_rectified_batch_device(3, dl.data_ptr(), dr.data_ptr(), d_disp=dd.data_ptr(), stream=_st())
        _done(eng)
        return {"disp": dd.cpu().numpy()}
    return run


def _w_rectified(size, device):
    def want(k):
        maps = _rect_maps(k, size)
        views = [tuple(R.remap(v, *maps[j]) for j, v in enumerate(_raw(k, i, size))) for i in range(3 if device else 1)]
        f = np.stack([o["final"] for o in _oracles(views)])
        return {"disp": f if device else f[0]}
    return want


def c_ingest_downstream(eng, k):
    """The views of NV12 frames through adc_ingest_views and adc_ingest_views_batch_device, those views matched on the
    device, and the maps through reprojection, speckle removal and the point cloud, host and device."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    fr = _frames("nv12", k, 3)
    out = {"views_host": eng.ingest_views(fr[0][0], fr[0][1], format="nv12")}
    dl, dr = _dev(np.stack([f[0] for f in fr])), _dev(np.stack([f[1] for f in fr]))
    views = torch.full((3, 2, H, W, 3), 0x5a, dtype=torch.uint8, device=dev)
    eng.ingest_views_batch_device(3, dl.data_ptr(), dr.data_ptr(), views.data_ptr(), image=A.image_desc("nv12"), stream=_st())
    dd = torch.full((3, H, W), -7.0, device=dev)
    # pair i's views lie at views[i, 0] and views[i, 1]: packed BGR with an image stride of one pair's views
    eng.match_images_batch_device(3, views.data_ptr(), views[0, 1].data_ptr(), image=A.image_desc("bgr", image_stride=6 * W * H),
                                  d_disp=dd.data_ptr(), stream=_st())
    _done(eng)
    out["views"], out["disp"] = views.cpu().numpy(), dd.cpu().numpy()
    Q = _q()
    pts = torch.full((3, H, W, 3), -7.0, device=dev)
    dep = torch.full((3, H, W), -7.0, device=dev)
    s16 = torch.full((3, H, W), 0x5a5a, dtype=torch.int16, device=dev)
    eng.reproject_batch_device(3, dd.data_ptr(), Q, [(pts.data_ptr(), "points"), (dep.data_ptr(), "depth"),
                                                    (s16.data_ptr(), "disp_s16")], _st())
    sp = dd.clone()
    wb = eng.speckle_workspace_bytes(3)
    work = torch.empty(wb, dtype=torch.uint8, device=dev)
    eng.filter_speckles_batch_device(3, sp.data_ptr(), "f32", *SPECKLE, None, work.data_ptr(), wb, _st())
    cap = H * W
    cp = torch.full((3, cap, 3), -7.0, device=dev)
    cc = torch.full((3, cap, 3), 0x5a, dtype=torch.uint8, device=dev)
    cx = torch.full((3, cap), -7, dtype=torch.int32, device=dev)
    cn = torch.full((3,), -7, dtype=torch.int32, device=dev)
    cwb = eng.point_cloud_workspace_bytes(3)
    cwork = torch.empty(cwb, dtype=torch.uint8, device=dev)
    eng.point_cloud_batch_device(3, dd.data_ptr(), Q, cp.data_ptr(), cn.data_ptr(), cap, cwork.data_ptr(), cwb,
                                 d_bgr=views[:, 0].contiguous().data_ptr(), d_colors=cc.data_ptr(), d_pixels=cx.data_ptr(),
                                 stream=_st())
    torch.cuda.synchronize()
    out.update(points=pts.cpu().numpy(), depth=dep.cpu().numpy(), s16=s16.cpu().numpy(), speckled=sp.cpu().numpy())
    n = cn.cpu().numpy()
    out["cloud_counts"] = n
    for i in range(3):
        out[f"cloud{i}"] = cp[i, :n[i]].cpu().numpy()
        out[f"cloud_colors{i}"] = cc[i, :n[i]].cpu().numpy()
        out[f"cloud_pixels{i}"] = cx[i, :n[i]].cpu().numpy()
    m0 = out["disp"][0]
    host = eng.reproject(m0, Q, ("points", "depth", "disp_s16"))
    out.update(points_host=host["points"], depth_host=host["depth"], s16_host=host["disp_s16"])
    out["speckled_host"] = eng.filter_speckles(m0, *SPECKLE)
    hp, hc, hx = eng.point_cloud(m0, Q, bgr=out["views"][0, 0], pixels=True)
    out.update(cloud_host=hp, cloud_colors_host=hc, cloud_pixels_host=hx)
    return out


def w_ingest_downstream(k):
    fr = _frames("nv12", k, 3)
    finals = np.stack([o["final"] for o in _oracles([(f[2], f[3]) for f in fr])])
    views = np.stack([np.stack([f[2], f[3]]) for f in fr])
    Q = _q()
    out = {"views_host": views[0], "views": views, "disp": finals,
           "points": np.stack([RP.points(m, Q) for m in finals]), "depth": np.stack([RP.depth(m, Q) for m in finals]),
           "s16": np.stack([RP.disp_s16(m, DMIN) for m in finals]),
           "speckled": np.stack([SP.filter_f32(m, np.inf, *SPECKLE) for m in finals])}
    clouds = [CL.cloud(m, Q, views[i, 0]) for i, m in enumerate(finals)]
    out["cloud_counts"] = np.array([len(c[0]) for c in clouds], np.int32)
    for i, (p, c, x) in enumerate(clouds):
        out.update({f"cloud{i}": p, f"cloud_colors{i}": c, f"cloud_pixels{i}": x})
    out.update(points_host=out["points"][0], depth_host=out["depth"][0], s16_host=out["s16"][0],
               speckled_host=out["speckled"][0], cloud_host=clouds[0][0], cloud_colors_host=clouds[0][1],
               cloud_pixels_host=clouds[0][2])
    return out


def c_render_cloud(eng, k):
    """adc_render_disparity and adc_disparity_cloud on a final map (with invalid pixels) of the call's pair."""
    l, r = _pair(k, 0)
    m = oracle(l, r)["final"]
    gray, jet, mm = eng.render_disparity(m)
    return {"gray": gray, "jet": jet, "min_max": np.array(mm, np.float32), "cloud": eng.disparity_cloud(l, m)}


def w_render_cloud(k):
    import cv2
    l, r = _pair(k, 0)
    m = oracle(l, r)["final"]
    g, mn, mx = MT.gray8(m, W)
    ys, xs = np.nonzero(~np.isinf(m))
    cloud = np.stack([xs, ys, np.abs(m[ys, xs]), l[ys, xs, 2], l[ys, xs, 1], l[ys, xs, 0]], 1).astype(np.float32)
    return {"gray": g, "jet": cv2.applyColorMap(g, cv2.COLORMAP_JET), "min_max": np.array((mn, mx), np.float32),
            "cloud": cloud}


def _debug(stage):
    def run(eng, k):
        l, r = _pair(k, 0)
        eng.debug_run(l, r, stage)
        return {tap: eng.tap(tap) for tap in T.STAGE_TAPS[stage]}
    return run


@functools.cache
def _oracle_taps(k, stage):
    l, r = _pair(k, 0)
    orc = T.Oracle(W, H, OPT)
    orc.begin(l, r)
    orc.run_to(stage)
    out = {tap: orc.tap(tap).copy() for tap in T.STAGE_TAPS[stage]}
    orc.close()
    return out


def _w_debug(stage):
    return lambda k: _oracle_taps(k, stage)


CALLS = {
    "match+right": (c_match, w_match),
    "match_cost": (c_match_cost, w_match_cost),
    "batch_pageable": (c_batch_pageable, w_finals),
    "batch_ptrs_pageable": (c_batch_ptrs_pageable, w_finals),
    "batch_pinned": (c_batch_pinned, w_batch_pinned),
    "pinned_async": (c_pinned_async, w_finals),
    "batch_device": (c_batch_device, w_finals),
    "cost_f32_hwd": (_cost_device("f32", "hwd"), w_cost_device),
    "cost_f32_dhw": (_cost_device("f32", "dhw"), w_cost_device),
    "cost_f16_dhw": (_cost_device("f16", "dhw"), w_cost_device),
    "cost_bf16_hwd": (_cost_device("bf16", "hwd"), w_cost_device),
    **{f"volumes_only_{s}": (_volumes_only_device(s), _w_volume(s)) for s in VOLS},
    "volumes_host": (c_volumes_host, w_volumes_host),
    "outputs_host": (c_outputs_host, w_outputs_host),
    "outputs_batch": (c_outputs_batch, w_outputs_batch),
    **{f"images_{f}": (_images_device(f), _w_images(f, 3)) for f in IMAGE_FORMATS},
    **{f"images_host_{f}": (_images_host(f), _w_images(f, 1)) for f in ("gray", "bayer_rg12p")},
    "rectified_host_small": (_rectified(RECT_SMALL, False), _w_rectified(RECT_SMALL, False)),
    "rectified_host_large": (_rectified(RECT_LARGE, False), _w_rectified(RECT_LARGE, False)),
    "rectified_device_small": (_rectified(RECT_SMALL, True), _w_rectified(RECT_SMALL, True)),
    "rectified_device_large": (_rectified(RECT_LARGE, True), _w_rectified(RECT_LARGE, True)),
    "ingest_downstream": (c_ingest_downstream, w_ingest_downstream),
    "render_cloud": (c_render_cloud, w_render_cloud),
    **{f"debug_{s}": (_debug(s), _w_debug(s)) for s in DEBUG_STOPS},
}
# the C entry points each call reaches (the Python method's C function, and those a call invokes directly)
CALL_FUNCTIONS = {
    "adc_match", "adc_get_right_disparity", "adc_match_cost", "adc_match_batch", "adc_match_batch_strided",
    "adc_match_batch_pinned_async", "adc_match_batch_device", "adc_match_cost_batch_device",
    "adc_match_volumes_batch_device", "adc_match_volumes", "adc_match_outputs", "adc_match_outputs_batch_device",
    "adc_match_images_batch_device", "adc_match_images", "adc_set_rectification", "adc_match_rectified",
    "adc_match_rectified_batch_device", "adc_ingest_views", "adc_ingest_views_batch_device", "adc_reproject",
    "adc_reproject_batch_device", "adc_filter_speckles", "adc_filter_speckles_batch_device", "adc_point_cloud",
    "adc_point_cloud_batch_device", "adc_render_disparity", "adc_disparity_cloud", "adc_debug_run",
}
# header functions that take an engine and run no kernel on its arena, or run none of their own
NOT_CALLS = {"adc_destroy", "adc_synchronize", "adc_set_pipelined", "adc_join", "adc_launch_count", "adc_last_stage_ms",
             "adc_get_config", "adc_profile_kernel", "adc_debug_counters", "adc_debug_get", "adc_speckle_workspace_bytes",
             "adc_point_cloud_workspace_bytes", "adc_debug_run_cost"}


def test_call_script_covers_the_entry_points():
    """Every function of the header that takes an engine is in the call script or named as one that runs no pipeline
    work of its own; a new entry point fails here until it is placed."""
    h = HEADER.read_text()
    fns = set(re.findall(r"^\w[\w\s\*]*?\b(adc_\w+)\(\s*(?:const\s+)?adc_engine\s*\*", h, re.M))
    assert fns, "no engine functions found in the header"
    missing = fns - CALL_FUNCTIONS - NOT_CALLS
    assert not missing, f"entry points neither in CALLS nor in NOT_CALLS: {sorted(missing)}"
    assert CALL_FUNCTIONS <= fns, sorted(CALL_FUNCTIONS - fns)


def _run_call(eng, name, k):
    return CALLS[name][0](eng, k)


def _check_call(tag, got, want):
    assert set(want) <= set(got), (tag, sorted(set(want) - set(got)))
    if "outliers" in want and isinstance(want["outliers"], list):      # a batch: per pair
        for i, wv in enumerate(want["outliers"]):
            _same_outputs(f"{tag} pair {i}", {"outliers": got["outliers"][i]}, {"outliers": wv})
        want = {k: v for k, v in want.items() if k != "outliers"}
    _same_outputs(tag, got, want)


def _small_engine(debug_flags=0):
    return E.engine(W, H, OPT, wave_pairs=WAVE, lanes=LANES, debug_flags=debug_flags)


@pytest.mark.gpu
@pytest.mark.parametrize("byte", PATTERNS)
def test_entry_points_poisoned(byte):
    """Every call of CALLS on one poisoned engine, in order, against the oracle or a restatement."""
    eng = _small_engine(flags(byte))
    try:
        for k, name in enumerate(CALLS):
            _check_call(f"{name} (poison {byte:#04x})", _run_call(eng, name, k), CALLS[name][1](k))
    finally:
        E.cuda()[0].cuda.synchronize()
        eng.close()


# ---- one real shape --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_kitti_shape_poisoned():
    """1242x375x128 (seed 1) with the default configuration, wave_pairs + 1 copies of the pair through
    match_outputs_batch_device (the second wave partial): every final and WTA map against the reference's hashes."""
    torch, dev = E.cuda()
    g = E.golden("golden_big.json")["kitti_s1"]
    w, h, Dk = g["width"], g["height"], g["max_disparity"]
    left, right = T.synthetic_pair(w, h, Dk, 1)
    assert [T.sha(left), T.sha(right)] == g["input_sha"]
    eng = E.engine(w, h, T.default_option(max_disparity=Dk), debug_flags=flags(0xFF))
    n = eng.wave_pairs + 1
    dl = torch.from_numpy(left).to(dev).unsqueeze(0).repeat(n, 1, 1, 1).contiguous()
    dr = torch.from_numpy(right).to(dev).unsqueeze(0).repeat(n, 1, 1, 1).contiguous()
    got = E.batch_outputs(eng, eng.match_outputs_batch_device, n, dl.data_ptr(), dr.data_ptr(), 3 * w * h,
                          maps=["wta_left", "wta_right"])
    eng.close()
    for key, tap in (("disp", "MEDIAN/DISP_L"), ("wta_left", "WTA/DISP_L"), ("wta_right", "WTA/DISP_R")):
        bad = [i for i in range(n) if T.sha(got[key][i]) != g["hashes"][tap]]
        assert not bad, f"{key}: {len(bad)} of {n} maps differ from the reference ({tap}), pairs {bad[:8]}"


# ---- call history ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True], ids=["plain", "pipelined"])
def test_call_history(pipelined):
    """The call script on one long-lived engine without poison (what production sees: a real earlier call's data),
    forwards then backwards with new pairs for every call.  Each call's outputs must equal the same call on a fresh
    engine of the same configuration, and the oracle or restatement."""
    eng = _small_engine()
    names = list(CALLS)
    script = [(k, name) for k, name in enumerate(names)] + [(100 + k, name) for k, name in enumerate(reversed(names))]
    try:
        eng.set_pipelined(pipelined)
        for k, name in script:
            got = _run_call(eng, name, k)
            fresh = _small_engine()
            fresh.set_pipelined(pipelined)
            ref = _run_call(fresh, name, k)
            E.cuda()[0].cuda.synchronize()
            fresh.close()
            tag = f"{name} (call {k}, pipelined {pipelined})"
            assert set(got) == set(ref), tag
            for key in got:
                E.same(f"{tag} {key} vs fresh engine", np.asarray(got[key]), np.asarray(ref[key]))
            _check_call(tag, got, CALLS[name][1](k))
    finally:
        E.cuda()[0].cuda.synchronize()
        eng.close()
