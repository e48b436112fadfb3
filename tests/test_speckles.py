"""Speckle removal (adc_filter_speckles, adc_filter_speckles_batch_device): cv2.filterSpeckles on int16 maps (OpenCV's
plain C++ path) and the same rule on the engine's f32 maps, exact.

CPU: the numpy / scipy restatement (speckle_testlib) against the committed fixture of OpenCV's outputs (never skipped),
against live cv2 in random trials with IPP off and on (skipped without OpenCV), and its F32 rules against a per-pixel
flood fill; the argument rules on a NULL engine; the header's enum and struct against the ctypes mirror; k_speckle.cu's
local memory.
GPU: every fixture map through both entries; the F32 filter of the engine's final maps of Cone and of every
test_gpu_parity case, reprojection to S16 then the S16 filter, and the F32 == S16 cross-check on 1/16 multiples;
adversarial maps up to 1920 x 1080 and at width 9996 (the widest engine with a disparity range of 4); components of
exactly max_size and max_size + 1 pixels across tile borders; batched calls at odd offsets with guard elements around
maps and workspace, pipelined on a second stream after adc_join; a workspace past 2^31 bytes; four launches per call
and unchanged match calls around it.
"""
import ctypes
import re
from collections import deque

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E
import speckle_testlib as S

ROOT = T.REPO
GOLDEN = T.GOLDEN_DIR / "golden_speckle_cases.npz"
SRC = ROOT / "adcensus_b200" / "csrc" / "k_speckle.cu"
LAUNCHES = 4


def _fixture():
    z = np.load(GOLDEN)
    for name in sorted({k.split("/")[0] for k in z.files}):
        nv, ms, md = z[f"{name}/args"]
        ipp = z[f"{name}/want_ipp"] if f"{name}/want_ipp" in z.files else None
        yield name, z[f"{name}/map"], float(nv), int(ms), float(md), z[f"{name}/want"], ipp


# ---- CPU ------------------------------------------------------------------------------------------
def test_restatement_against_fixture():
    """The restatement reproduces every OpenCV output in the fixture (plain path), and IPP's output where it was
    recorded; the fixture holds the edge cases it claims."""
    seen, ipp_differs = set(), 0
    for name, img, nv, ms, md, want, want_ipp in _fixture():
        assert np.array_equal(S.filter_s16(img, nv, ms, md), want), name
        if want_ipp is not None:
            assert np.array_equal(S.filter_s16(img, nv, ms, md, ipp=True), want_ipp), name
            ipp_differs += not np.array_equal(want, want_ipp)
        seen.add(name.split("_")[0])
    assert seen == {"tie", "nv", "md", "size", "extreme", "line", "engine"}
    assert ipp_differs >= 5
    z = np.load(GOLDEN)
    shapes = {z[k].shape for k in z.files if k.endswith("/map")}
    assert {(1, 1), (1, 97), (89, 1)} <= shapes
    vals = np.concatenate([z[k].reshape(-1) for k in z.files if k.endswith("/map")])
    assert {32767, -32767, -32768} <= set(vals.tolist())
    args = np.stack([z[k] for k in z.files if k.endswith("/args")])
    assert {2.5, 3.5, 40000.0, -40000.0} <= set(args[:, 0].tolist())
    assert np.isnan(args[:, 2]).any() and {-1.0, 40000.0, 70000.0, 1e10} <= set(args[:, 2].tolist())
    assert {0, -3} <= set(args[:, 1].astype(int).tolist())


def test_cv_round():
    assert [S.cv_round(v) for v in (2.5, 3.5, -2.5, -0.5, 0.5, 1.5)] == [2, 4, -2, 0, 0, 2]
    assert [S.cv_round(v) for v in (float("nan"), 1e10, -1e10, 2.0 ** 31, 2.0 ** 31 - 1, -(2.0 ** 31))] == \
        [S.INT_MIN, S.INT_MIN, S.INT_MIN, S.INT_MIN, 2 ** 31 - 1, S.INT_MIN]
    assert [S.wrap16(v) for v in (40000, -40000, 65536, 70000, S.INT_MIN)] == [-25536, 25536, 0, 4464, 0]


def _random_trial(rng, i):
    """(map, new_val, max_size, max_diff) of trial i: maps 1..120 on a side with few distinct values, so that equal
    and close neighbours are common; the edge cases come up in turn."""
    H, W = (int(v) for v in rng.integers(1, 121, 2)) if i % 5 else (int(v) for v in rng.integers(1, 12, 2))
    scale = int(rng.choice([1, 3, 16, 2500]))
    img = (rng.integers(-4, 5, (H, W)) * scale).astype(np.int16)
    if i % 7 == 0:
        img[rng.random((H, W)) < 0.1] = rng.choice(np.array([32767, -32767, -32768, -25536, 25536], np.int16))
    nv = float(rng.choice([0.0, 2.5, 3.5, -16.0, float(scale), 40000.0, -40000.0, 1e10, float("nan")]))
    ms = int(rng.choice([-1, 0, 1, 2, 5, 20, H * W, H * W + 1]))
    md = float(rng.choice([-1.0, 0.0, 0.5, 1.5, float(scale), 2.0 * scale, 32767.0, 40000.0, 65536.0, 70000.0,
                           2.0 ** 31 - 1, 1e10, -1e10, float("nan")]))
    return img, nv, ms, md


def test_restatement_against_opencv():
    """240 random trials against cv2.filterSpeckles with IPP off (the plain path the engine follows), then 120 with IPP
    on against the restatement's IPP variant (cvRound(max_diff) and cvRound(new_val) wrapped to int16).  The trials
    cover cvRound ties, new_val and max_diff outside int16, max_diff negative and NaN, max_size <= 0 and >= H*W, values
    +-32767 / -32768, and maps from 1 x 1 to 120 x 120."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(16)
    was = cv2.ipp.useIPP()
    try:
        for ipp, trials in ((False, 240), (True, 120)):
            cv2.ipp.setUseIPP(ipp)
            for i in range(trials):
                img, nv, ms, md = _random_trial(rng, i)
                got = img.copy()
                cv2.filterSpeckles(got, nv, ms, md)
                assert np.array_equal(got, S.filter_s16(img, nv, ms, md, ipp=ipp)), (ipp, i, img.shape, nv, ms, md)
    finally:
        cv2.ipp.setUseIPP(was)


def _flood_f32(img, new_val, max_size, max_diff):
    """The F32 rules pixel by pixel: a breadth-first fill from every unvisited pixel that is not missing."""
    H, W = img.shape
    nv = np.float32(new_val)
    out = img.copy()
    seen = np.zeros((H, W), bool)
    with np.errstate(all="ignore"):
        for y0 in range(H):
            for x0 in range(W):
                if seen[y0, x0] or img[y0, x0] == nv:
                    continue
                comp, q = [], deque([(y0, x0)])
                seen[y0, x0] = True
                while q:
                    y, x = q.popleft()
                    comp.append((y, x))
                    for yy, xx in ((y - 1, x), (y + 1, x), (y, x - 1), (y, x + 1)):
                        if 0 <= yy < H and 0 <= xx < W and not seen[yy, xx] and img[yy, xx] != nv and \
                                float(abs(np.float32(img[y, x]) - np.float32(img[yy, xx]))) <= max_diff:
                            seen[yy, xx] = True
                            q.append((yy, xx))
                if len(comp) <= max_size:
                    for y, x in comp:
                        out[y, x] = nv
    return out


def test_f32_rules_against_flood_fill():
    """filter_f32 equals a per-pixel flood fill on 60 small maps with +-inf, NaN, +-0, huge values and quarter-pixel
    steps; new_val +inf, NaN, a value of the map and one that needs rounding to float; max_diff from -inf to +inf."""
    rng = np.random.default_rng(32)
    specials = np.array([np.inf, -np.inf, np.nan, 0.0, -0.0, 3e38, -3e38, 1e-40], np.float32)
    for i in range(60):
        H, W = (int(v) for v in rng.integers(1, 17, 2))
        img = (rng.integers(0, 12, (H, W)) / 4.0).astype(np.float32)
        m = rng.random((H, W)) < 0.15
        img[m] = rng.choice(specials, int(m.sum()))
        nv = [np.inf, np.nan, 1.0, 0.1 + 1e-12, -np.inf][i % 5]
        md = [0.25, 0.0, 1.0, -np.inf, np.inf, 0.2500000001, 1e300, -1.0][i % 8]
        ms = int(rng.integers(-1, 8))
        assert S.same_bits(S.filter_f32(img, nv, ms, md), _flood_f32(img, nv, ms, md)), (i, nv, md, ms)
    # the rules' corners: NaN never connects, -inf next to -inf gives NaN, a subtraction rounds in float
    a = np.array([[np.nan, np.nan, -np.inf, -np.inf, 1.0, 1.0 + 2 ** -23]], np.float32)
    got = S.filter_f32(a, np.inf, 1, 2.0 ** -23)
    assert np.isinf(got[0, :4]).all() and (got[0, 4:] == a[0, 4:]).all()
    b = np.array([[1e8, 1e8 + 8]], np.float32)   # the difference 8 is exact in float
    assert (S.filter_f32(b, np.inf, 1, 7.999) == np.inf).all() and (S.filter_f32(b, np.inf, 1, 8.0) == b).all()


def _lib():
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    return A, A.load_library()


def test_speckle_argument_errors_need_no_gpu():
    """Every rule that needs no engine fails with ADC_ERR_ARG naming the field before the engine is checked, on both
    entries and on adc_speckle_workspace_bytes; the alignment rules apply to the device entry only."""
    A, L = _lib()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data

    def prm(t=A.SPECKLE_S16, md=2.0, reserved=0):
        return ctypes.byref(A.SpeckleParams(t, 10, 0.0, md, reserved))

    def host(params, m=p):
        return L.adc_filter_speckles(None, m, params)

    def dev(params, m=p, n=1, work=p):
        return L.adc_filter_speckles_batch_device(None, n, m, params, work, 1 << 20, None)

    common = [(dict(params=None), b"params is NULL"),
              (dict(params=prm(t=2)), b"params.type 2 unknown"),
              (dict(params=prm(t=-1)), b"params.type -1 unknown"),
              (dict(params=prm(reserved=1)), b"params.reserved must be zero"),
              (dict(params=prm(t=A.SPECKLE_F32, md=float("nan"))), b"params.max_diff is NaN"),
              (dict(params=prm(), m=None), b"map is NULL")]
    for call, fn in ((host, b"adc_filter_speckles:"), (dev, b"adc_filter_speckles_batch_device:")):
        for kw, msg in common:
            assert call(**kw) == 1, (fn, msg)
            err = L.adc_last_error()
            assert msg in err and fn in err, err
    assert dev(prm(), n=-1) == 1 and b"n -1 is negative" in L.adc_last_error()
    for kw, msg in [(dict(params=prm(), m=p + 1), b"maps are not 2-byte aligned"),
                    (dict(params=prm(t=A.SPECKLE_F32), m=p + 2), b"maps are not 4-byte aligned"),
                    (dict(params=prm(), work=p + 2), b"work is not 4-byte aligned")]:
        assert dev(**kw) == 1 and msg in L.adc_last_error(), L.adc_last_error()
        if "work" not in kw:   # the host entry has no alignment rules: the same call gets as far as the engine check
            assert host(kw["params"], kw["m"]) == 1 and b"engine is NULL" in L.adc_last_error()
    # valid calls: a NaN max_diff on S16 (cvRound gives INT_MIN), minimum alignments, n = 0 reach the engine check
    for kw in (dict(params=prm(md=float("nan"))), dict(params=prm(), m=p + 2), dict(params=prm(t=A.SPECKLE_F32)),
               dict(params=prm(), n=0, work=None)):
        assert dev(**kw) == 1 and b"engine is NULL" in L.adc_last_error(), L.adc_last_error()
    assert host(prm(md=float("nan")), p + 1) == 1 and b"engine is NULL" in L.adc_last_error()
    out = ctypes.c_size_t()
    assert L.adc_speckle_workspace_bytes(None, 1, None) == 1 and b"out is NULL" in L.adc_last_error()
    assert L.adc_speckle_workspace_bytes(None, -2, ctypes.byref(out)) == 1 and b"n -2 is negative" in L.adc_last_error()
    assert L.adc_speckle_workspace_bytes(None, 1, ctypes.byref(out)) == 1 and b"engine is NULL" in L.adc_last_error()


def test_speckle_constants():
    """The header's enum and struct match the ctypes mirror."""
    import adcensus_b200 as A
    assert (A.SPECKLE_S16, A.SPECKLE_F32) == (0, 1) and A.SPECKLE_TYPES == {"s16": 0, "f32": 1}
    assert ctypes.sizeof(A.SpeckleParams) == 32
    assert [(n, getattr(A.SpeckleParams, n).offset) for n, _ in A.SpeckleParams._fields_] == [
        ("type", 0), ("max_size", 4), ("new_val", 8), ("max_diff", 16), ("reserved", 24)]
    h = (ROOT / "include" / "adcensus_b200.h").read_text()
    assert "enum { ADC_SPECKLE_S16 = 0, ADC_SPECKLE_F32 = 1 };" in h
    body = re.search(r"typedef struct adc_speckle_params \{(.*?)\} adc_speckle_params;", h, re.S).group(1)
    fields = re.findall(r"^\s*(\w+)\s+(\w+);", body, re.M)
    assert fields == [("int32_t", "type"), ("int32_t", "max_size"), ("double", "new_val"), ("double", "max_diff"),
                      ("int64_t", "reserved")]
    assert "k_speckle.cu" in (ROOT / "adcensus_b200" / "csrc" / "Makefile").read_text()


def test_speckle_kernel_uses_no_local_memory():
    """ptxas -v on k_speckle.cu: no stack frame and no spills in any of the seven kernels (local labelling, border
    merge and apply for each map type, and the count)."""
    report = E.ptxas_report(SRC)
    assert len(report) == 7 and all((f["stack"], f["spill_stores"], f["spill_loads"], f["lmem"]) == (0, 0, 0, 0)
                                    for f in report.values()), report
    assert sum(f["regs"] is not None and "k_speckle_" in name for name, f in report.items()) == 7, report


# ---- GPU ------------------------------------------------------------------------------------------
def _tname(a):
    return "s16" if a.dtype == np.int16 else "f32"


def _device_filter(eng, maps, max_size, max_diff, new_val):
    """maps [n][H][W] through the device entry on the current stream: the filtered maps (host)."""
    torch, dev = E.cuda()
    n = maps.shape[0]
    d = torch.from_numpy(np.ascontiguousarray(maps)).to(dev)
    wb = eng.speckle_workspace_bytes(n)
    work = torch.empty(max(wb, 4), dtype=torch.uint8, device=dev)
    eng.filter_speckles_batch_device(n, d.data_ptr(), _tname(maps), max_size, max_diff, new_val, work.data_ptr(), wb,
                                     torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d.cpu().numpy()


@pytest.mark.gpu
def test_fixture_through_both_entries():
    """Every fixture map, on an engine of its size, through the host entry and the device entry: equal to OpenCV's
    recorded output (the plain path)."""
    for name, img, nv, ms, md, want, _ in _fixture():
        H, W = img.shape
        eng = E.engine(W, H, T.default_option(max_disparity=4))
        assert np.array_equal(eng.filter_speckles(img, ms, md, nv), want), f"{name} host"
        assert np.array_equal(_device_filter(eng, img[None], ms, md, nv)[0], want), f"{name} device"
        eng.close()


def _final_map(case, cone):
    if case == "cone":
        left, right = cone
        h, w, _ = left.shape
        opt = dict(max_disparity=64)
    else:
        w, h, D, over, seed = E.PARITY_CASES[case]
        opt = {"max_disparity": D, **over}
        left, right = T.synthetic_pair(w, h, opt["max_disparity"] - opt.get("min_disparity", 0), seed)
    eng = E.engine(w, h, T.default_option(**opt))
    return eng, eng.match(left, right)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cone"] + list(range(len(E.PARITY_CASES))))
def test_engine_maps(case, cone):
    """The engine's final map of Cone and of every test_gpu_parity case: the F32 filter (+inf = missing) through both
    entries equals the restatement; its S16 reprojection through the S16 filter equals the restatement; and, on the
    map quantised to multiples of 1/16, F32 with max_diff k/16 equals S16 with max_diff k after reprojection."""
    eng, disp = _final_map(case, cone)
    dmin = eng.option.min_disparity
    s16_invalid = float((dmin - 1) * 16)
    s16 = eng.reproject(disp, np.eye(4), ["disp_s16"])["disp_s16"]
    assert (s16 != s16_invalid).sum() == np.isfinite(disp).sum()
    for ms, k in ((200, 32), (20, 4), (5000, 16), (1, 0)):
        want = S.filter_f32(disp, np.inf, ms, k / 16)
        got = eng.filter_speckles(disp, ms, k / 16)
        assert S.same_bits(got, want), (case, ms, k, "f32 host")
        assert S.same_bits(_device_filter(eng, disp[None], ms, k / 16, np.inf)[0], want), (case, ms, k, "f32 device")
        want16 = S.filter_s16(s16, s16_invalid, ms, k)
        got16 = eng.filter_speckles(s16, ms, k)
        assert np.array_equal(got16, want16), (case, ms, k, "s16 host")
        assert np.array_equal(_device_filter(eng, s16[None], ms, k, s16_invalid)[0], want16), (case, ms, k, "s16 dev")
        # the cross-check between the two types, on the map quantised to 1/16 (its S16 encoding over 16)
        q = np.where(s16 == s16_invalid, np.inf, s16 / 16.0).astype(np.float32)
        gotq = _device_filter(eng, q[None], ms, k / 16, np.inf)[0]
        assert S.same_bits(gotq, S.filter_f32(q, np.inf, ms, k / 16)), (case, ms, k, "f32 quantised")
        assert np.array_equal(eng.reproject(gotq, np.eye(4), ["disp_s16"])["disp_s16"], got16), (case, ms, k, "f32=s16")
    eng.close()


def _serpentine(H, W):
    """A one-pixel-wide path of 1s through the whole map on a background of 0s: every even row, joined at alternate
    ends by one pixel of the odd row between."""
    m = np.zeros((H, W), np.int16)
    m[0::2] = 1
    for y in range(1, H, 2):
        m[y, W - 1 if (y // 2) % 2 == 0 else 0] = 1
    return m


def _straddling(H, W, s, rng):
    """Horizontal and vertical bars of s and s + 1 pixels of distinct values on a background of 0s, placed across the
    tile borders (every 64 columns, every 32 rows) at offsets 1 .. s, one pixel of background between bars."""
    m = np.zeros((H, W), np.int16)
    v = 1
    y = 1
    for x0 in range(64, W - s - 2, 64):
        for off in range(1, s + 1):
            for ln in (s, s + 1):
                if y >= H - 1:
                    break
                xs = max(1, x0 - off)
                m[y, xs:xs + ln] = v
                v = v % 30000 + 1
                y += 2
    x = 1
    for y0 in range(32, H - s - 2, 32):
        for off in range(1, min(s, 31) + 1):
            for ln in (s, s + 1):
                if x >= W - 1:
                    break
                ys = max(1, y0 - off)
                if not m[ys - 1:ys + ln + 1, x - 1:x + 2].any():
                    m[ys:ys + ln, x] = v
                    v = v % 30000 + 1
                x += 2
    return m


def _adversarial(H, W, rng):
    """(name, int16 map, new_val, max_diff): serpentine, constant, checkerboard of singletons, white noise."""
    cb = np.where((np.arange(H)[:, None] + np.arange(W)[None]) % 2 == 0, 100, -100).astype(np.int16)
    return [("serpentine", _serpentine(H, W), 0.0, 0.0),
            ("constant", np.full((H, W), 7, np.int16), 0.0, 0.0),
            ("checkerboard", cb, 0.0, 1.0),
            ("noise", rng.integers(-40, 40, (H, W)).astype(np.int16), -41.0, 3.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1080, 1920), (64, 9996), (257, 333)])
def test_adversarial_maps(shape):
    """Serpentine (one component of about half the map), a constant map (one component of all of it), a checkerboard
    of singletons and white noise, as S16 and as F32, each with max_size just below and at the largest component's
    size: equal to the restatement."""
    H, W = shape
    rng = np.random.default_rng(H + W)
    eng = E.engine(W, H, T.default_option(max_disparity=4))
    for name, m, nv, md in _adversarial(H, W, rng):
        f = m.astype(np.float32)
        sizes = {"serpentine": int((m == 1).sum()), "constant": H * W, "checkerboard": 1, "noise": 3}
        for ms in (sizes[name] - 1, sizes[name], 200):
            want = S.filter_s16(m, nv, ms, md)
            assert np.array_equal(_device_filter(eng, m[None], ms, md, nv)[0], want), (shape, name, ms, "s16")
            wantf = S.filter_f32(f, nv, ms, md)
            assert S.same_bits(_device_filter(eng, f[None], ms, md, nv)[0], wantf), (shape, name, ms, "f32")
        if name in ("serpentine", "constant"):
            assert (want == m).all() and (S.filter_s16(m, nv, sizes[name], md) != m).any()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("s", [3, 40, 63, 64, 65, 100])
def test_components_straddling_tile_borders(s):
    """Bars of exactly max_size and max_size + 1 pixels across tile borders at every offset: the first are removed,
    the second kept, as the restatement says; S16 and F32, at 1080 x 1920."""
    H, W = 1080, 1920
    rng = np.random.default_rng(s)
    m = _straddling(H, W, s, rng)
    eng = E.engine(W, H, T.default_option(max_disparity=4))
    want = S.filter_s16(m, 0.0, s, 0.0)
    assert (want != m).any() and (want != 0).any()
    assert np.array_equal(_device_filter(eng, m[None], s, 0.0, 0.0)[0], want)
    f = m.astype(np.float32)
    assert S.same_bits(_device_filter(eng, f[None], s, 0.0, 0.0)[0], S.filter_f32(f, 0.0, s, 0.0))
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
@pytest.mark.parametrize("map_type", ["f32", "s16"])
def test_batched_device_calls(pipelined, map_type):
    """n = 9 maps of a 71 x 47 engine with min_disparity -3, at an odd element offset, the workspace at an odd 4-byte
    offset: guard elements before and after both untouched, each map equal to the host entry's result and to the
    restatement, four launches.  Pipelined: the maps come from a pipelined match batch and a second stream waits with
    adc_join before it filters them (S16: after a reprojection on that stream)."""
    torch, dev = E.cuda()
    w, h, dmin, D, n = 71, 47, -3, 20, 9
    N = w * h
    eng = E.engine(w, h, T.default_option(min_disparity=dmin, max_disparity=dmin + D))
    pairs = [T.synthetic_pair(w, h, D, 40 + i) for i in range(n)]
    st = torch.cuda.current_stream()
    # maps and workspace 1, 3 and 5 elements into buffers of -7 with 7 more after them
    f, f_intact = E.guarded(n * N, torch.float32, 1, 7, -7)
    if pipelined:
        dl = torch.from_numpy(np.stack([p[0] for p in pairs])).to(dev)
        dr = torch.from_numpy(np.stack([p[1] for p in pairs])).to(dev)
        eng.set_pipelined(True)
        eng.match_batch_device(n, dl.data_ptr(), dr.data_ptr(), f.data_ptr(), st.cuda_stream)
        stream = torch.cuda.Stream()
        eng.join(stream.cuda_stream)
    else:
        f.copy_(torch.from_numpy(np.stack([eng.match(*p) for p in pairs]).reshape(-1)))
        stream = st
    if map_type == "s16":
        maps, maps_intact = E.guarded(n * N, torch.int16, 3, 7, -7)
        with torch.cuda.stream(stream):
            eng.reproject_batch_device(n, f.data_ptr(), np.eye(4), [(maps.data_ptr(), "disp_s16")], stream.cuda_stream)
    else:
        maps, maps_intact = f, f_intact
    wb = eng.speckle_workspace_bytes(n)
    assert wb == 8 * n * N
    work, work_intact = E.guarded(wb // 4, torch.int32, 5, 7, -7)
    c0 = eng.launch_count
    with torch.cuda.stream(stream):
        src = maps.clone()
        eng.filter_speckles_batch_device(n, maps.data_ptr(), map_type, 30, 16 / 16 if map_type == "f32" else 16, None,
                                         work.data_ptr(), wb, stream.cuda_stream)
    assert eng.launch_count == c0 + LAUNCHES
    torch.cuda.synchronize()
    srcs = src.cpu().numpy().reshape(n, h, w)
    got = maps.cpu().numpy().reshape(n, h, w)
    for i in range(n):
        md = 1.0 if map_type == "f32" else 16
        assert S.same_bits(got[i], eng.filter_speckles(srcs[i], 30, md)), (map_type, pipelined, i)
        nv = np.inf if map_type == "f32" else (dmin - 1) * 16
        assert S.same_bits(got[i], S.filter_any(srcs[i], nv, 30, md)), (map_type, pipelined, i)
    assert maps_intact() and work_intact(), "guard overwritten"
    # a workspace one byte short is refused, naming the field
    import adcensus_b200 as A
    with pytest.raises(A.AdcError, match="work_bytes"):
        eng.filter_speckles_batch_device(n, maps.data_ptr(), map_type, 30, 1, None, work.data_ptr(), wb - 1,
                                         stream.cuda_stream)
    if pipelined:
        eng.set_pipelined(False)
    eng.close()


@pytest.mark.gpu
def test_workspace_past_2_31():
    """n = 8300 S16 maps of 256 x 128 (three distinct ones, repeated): the workspace spans 2.18e9 bytes, past 2^31.
    Every map equals the restatement of its source, and the element after the last map is untouched."""
    torch, dev = E.cuda()
    w, h, n = 256, 128, 8300
    N = w * h
    rng = np.random.default_rng(9)
    eng = E.engine(w, h, T.default_option(max_disparity=4))
    base = np.stack([rng.integers(-3, 4, (h, w)).astype(np.int16) * 16 for _ in range(3)])
    base[1] = 5
    wb = eng.speckle_workspace_bytes(n)
    assert wb > 2 ** 31
    src = torch.from_numpy(base).to(dev)
    buf = torch.full((n * N + 1,), -7, dtype=torch.int16, device=dev)
    buf[:-1].view(n, h, w).copy_(src[torch.arange(n, device=dev) % 3])
    work = torch.empty(wb, dtype=torch.uint8, device=dev)
    eng.filter_speckles_batch_device(n, buf.data_ptr(), "s16", 6, 16, 0.0, work.data_ptr(), wb,
                                     torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = buf[:-1].view(n, h, w)
    for r in range(3):
        want = torch.from_numpy(S.filter_s16(base[r], 0.0, 6, 16)).to(dev)
        assert torch.equal(got[r::3], want.expand_as(got[r::3])), f"maps {r} mod 3"
    assert int(buf[-1]) == -7
    del work, buf
    eng.close()


@pytest.mark.gpu
def test_launches_and_match_unchanged(cone):
    """Each call makes exactly four launches whatever the content (n = 0: none); a match batch gives the same maps
    with the same number of launches before and after speckle calls."""
    torch, dev = E.cuda()
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option(max_disparity=64))
    n = 3
    dl = torch.from_numpy(np.stack([left] * n)).to(dev)
    dr = torch.from_numpy(np.stack([right] * n)).to(dev)
    st = torch.cuda.current_stream().cuda_stream

    def batch():
        d = torch.empty((n, h, w), dtype=torch.float32, device=dev)
        c0 = eng.launch_count
        eng.match_batch_device(n, dl.data_ptr(), dr.data_ptr(), d.data_ptr(), st)
        torch.cuda.synchronize()
        return d, eng.launch_count - c0

    d0, l0 = batch()
    wb = eng.speckle_workspace_bytes(n)
    work = torch.empty(wb, dtype=torch.uint8, device=dev)
    maps = d0.clone()
    for content in (maps, torch.zeros_like(maps), torch.full_like(maps, float("inf"))):
        c0 = eng.launch_count
        eng.filter_speckles_batch_device(n, content.data_ptr(), "f32", 200, 2.0, None, work.data_ptr(), wb, st)
        assert eng.launch_count == c0 + LAUNCHES
    c0 = eng.launch_count
    eng.filter_speckles_batch_device(0, maps.data_ptr(), "f32", 200, 2.0, None, 0, 0, st)
    assert eng.launch_count == c0
    c0 = eng.launch_count
    host = eng.filter_speckles(d0[0].cpu().numpy(), 200, 2.0)
    assert eng.launch_count == c0 + LAUNCHES
    torch.cuda.synchronize()
    d1, l1 = batch()
    assert l1 == l0 and torch.equal(d0.view(torch.int32), d1.view(torch.int32))
    assert S.same_bits(host, maps[0].cpu().numpy())
    eng.close()
