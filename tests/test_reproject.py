"""Reprojection to 3-D (adc_reproject, adc_reproject_batch_device): disparity maps to the points of
cv2.reprojectImageTo3D, their depth and the StereoSGBM 16-bit encoding, bit for bit with OpenCV (NaN compared as NaN).

CPU: the numpy restatement (reproject_testlib) against the committed fixture of OpenCV's outputs (never skipped) and
against live cv2 in 60 random trials (skipped without OpenCV); the argument rules on a NULL engine; the constants, the
struct layout and the header's enum; k_reproject.cu's local memory, and its generated code free of contracted double
arithmetic.
GPU: every fixture map through both entries against OpenCV's recorded output; the engine's final maps of Cone and of
every test_gpu_parity case against the restatement; the camera path (raw frames -> match_rectified -> reprojection);
batched device calls at odd offsets with guard elements, each kind alone and all together, pipelined with adc_join on a
second stream, a points destination past 2^31 bytes; one launch per device call and unchanged match calls around it.
"""
import ctypes
import os
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E  # puts tools/ on sys.path
import rectify_testlib as R
import reproject_testlib as RP

ROOT = T.REPO
GOLDEN = T.GOLDEN_DIR / "golden_reproject_cases.npz"
KINDS = ["points", "depth", "disp_s16"]
SRC = ROOT / "adcensus_b200" / "csrc" / "k_reproject.cu"


def _fixture():
    z = np.load(GOLDEN)
    for name in sorted({k.split("/")[0] for k in z.files}):
        yield name, z[f"{name}/disp"], z[f"{name}/Q"], int(z[f"{name}/min_disparity"]), z[f"{name}/points"], z[f"{name}/s16"]


def _fixture_Q(name):
    return np.load(GOLDEN)[f"{name}/Q"]


# ---- CPU ------------------------------------------------------------------------------------------
def test_restatement_against_fixture():
    """The restatement reproduces every OpenCV output in the fixture: random Q at extreme scales with signed zeros,
    stereoRectify Q with and without CALIB_ZERO_DISPARITY, maps with specials, 1 x 1 / 1 x N / N x 1, S16 ties,
    saturation and int32 overflow."""
    seen = set()
    for name, disp, Q, dmin, pts, s16 in _fixture():
        assert RP.same_nan(RP.points(disp, Q), pts), name
        assert RP.same_nan(RP.depth(disp, Q), np.ascontiguousarray(pts[:, :, 2])), name
        assert np.array_equal(RP.disp_s16(disp, dmin), s16), name
        seen.add(name.split("_")[0])
    assert seen == {"rand", "rig", "line", "s16"}
    # the fixture holds what it claims: every special, a -0 first product, both S16 saturations and the overflow value
    z = np.load(GOLDEN)
    allv = np.concatenate([z[k].reshape(-1) for k in z.files if k.endswith("/disp")])
    for v in (np.inf, -np.inf, 1e-40, 3e38, -3e38, 2 ** 27):
        assert (allv == np.float32(v)).any(), v
    assert np.isnan(allv).any() and (np.signbit(allv) & (allv == 0)).any()
    s16 = np.concatenate([z[k].reshape(-1) for k in z.files if k.endswith("/s16")])
    assert {-32768, 32767} <= set(s16.tolist())


def test_restatement_against_opencv():
    """60 random trials against cv2.reprojectImageTo3D and cv2.multiply(d, 16, CV_16S): 40 with Q entries from 1e-30
    to 1e30 and +-0 entries, 20 with stereoRectify Q; maps up to 1600 wide with +-inf, NaN, +-0, f32 subnormals and
    +-3e38.  The two plausible alternatives (one division h_c / h_3; a sum that starts at the first product) differ
    from OpenCV on these trials, so the trials can tell them apart."""
    cv2 = pytest.importorskip("cv2")
    import make_golden_reproject as MG
    rng = np.random.default_rng(15)
    div_differs = start_differs = 0
    for i in range(60):
        H, W = (int(rng.integers(1, 5)), 1600) if i % 10 == 0 else (int(v) for v in rng.integers(1, 90, 2))
        Q = MG.random_Q(rng) if i < 40 else MG.rig_Q(int(rng.integers(40, 1700)), int(rng.integers(30, 1000)), i % 2 == 0)
        disp = MG.random_disp(rng, H, W) if i % 3 else MG.engine_disp(rng, H, W, int(rng.integers(-10, 10)))
        want = cv2.reprojectImageTo3D(disp, Q)
        assert RP.same_nan(RP.points(disp, Q), want), f"trial {i}"
        assert np.array_equal(RP.saturate_s16(disp), cv2.multiply(disp, 16.0, dtype=cv2.CV_16S).reshape(H, W)), i
        # the alternatives
        ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
        d = disp.astype(np.float64)
        with np.errstate(all="ignore"):
            h = [(((np.zeros_like(d) + Q[k, 0] * xs) + Q[k, 1] * ys) + Q[k, 2] * d) + Q[k, 3] for k in range(4)]
            h0 = [((Q[k, 0] * xs + Q[k, 1] * ys) + Q[k, 2] * d) + Q[k, 3] for k in range(4)]
            div = np.stack([(h[c] / h[3]).astype(np.float32) for c in range(3)], -1)
            start = np.stack([(h0[c].astype(np.float32).astype(np.float64) * (1.0 / h0[3])).astype(np.float32)
                              for c in range(3)], -1)
        div_differs += not RP.same_nan(div, want)
        start_differs += not RP.same_nan(start, want)
    assert div_differs > 0 and start_differs > 0, (div_differs, start_differs)
    # the examples of the S16 rule
    v = np.array([[2047.96875, 0.03125, 0.09375, 2 ** 27, 3e38]], np.float32)
    assert RP.saturate_s16(v).tolist() == [[32767, 0, 2, -32768, -32768]]


def _outs(*specs):
    import adcensus_b200 as A
    arr = (A.ReprojectOut * max(1, len(specs)))()
    for i, s in enumerate(specs):
        arr[i] = A.ReprojectOut(*s)
    return arr


def test_reproject_argument_errors_need_no_gpu():
    """Every rule fails with ADC_ERR_ARG naming the field before the engine is checked, on both entries; the
    alignment rules apply to the device entry only."""
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    Q = (ctypes.c_double * 16)()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    P, D, S = A.REPROJ_POINTS, A.REPROJ_DEPTH, A.REPROJ_DISP_S16

    def host(outs, n_outs, disp=p, q=Q, n=1):
        return L.adc_reproject(None, disp, q, outs, n_outs)

    def dev(outs, n_outs, disp=p, q=Q, n=1):
        return L.adc_reproject_batch_device(None, n, disp, q, outs, n_outs, None)

    common = [(dict(outs=_outs((p, P, 0)), n_outs=0), b"n_outs 0 outside 1..3"),
              (dict(outs=_outs((p, P, 0)), n_outs=4), b"n_outs 4 outside 1..3"),
              (dict(outs=None, n_outs=1), b"outs is NULL"),
              (dict(outs=_outs((p, 3, 0)), n_outs=1), b"outs[0].kind 3 unknown"),
              (dict(outs=_outs((p, -1, 0)), n_outs=1), b"outs[0].kind -1 unknown"),
              (dict(outs=_outs((p, D, 0), (p + 64, D, 0)), n_outs=2), b"outs[1].kind 1 requested twice"),
              (dict(outs=_outs((p, P, 0), (None, S, 0)), n_outs=2), b"outs[1].dst is NULL"),
              (dict(outs=_outs((p, S, 7)), n_outs=1), b"outs[0].reserved"),
              (dict(outs=_outs((p, P, 0)), n_outs=1, disp=None), b"disp is NULL"),
              (dict(outs=_outs((p, P, 0)), n_outs=1, q=None), b"Q is NULL")]
    for call in (host, dev):
        fn = b"adc_reproject_batch_device" if call is dev else b"adc_reproject:"
        for kw, msg in common:
            assert call(**kw) == 1, (call.__name__, msg)
            err = L.adc_last_error()
            assert msg in err and fn in err, err
    assert dev(_outs((p, P, 0)), 1, n=-1) == 1 and b"n -1 is negative" in L.adc_last_error()
    for kw, msg in [(dict(outs=_outs((p + 2, P, 0)), n_outs=1), b"outs[0].dst is not 4-byte aligned"),
                    (dict(outs=_outs((p, S, 0), (p + 1, D, 0)), n_outs=2), b"outs[1].dst is not 4-byte aligned"),
                    (dict(outs=_outs((p + 1, S, 0)), n_outs=1), b"outs[0].dst is not 2-byte aligned"),
                    (dict(outs=_outs((p, P, 0)), n_outs=1, disp=p + 2), b"disp is not 4-byte aligned")]:
        assert dev(**kw) == 1 and msg in L.adc_last_error(), L.adc_last_error()
        # the host entry has no alignment rules: the same call gets as far as the engine check
        assert host(**kw) == 1 and b"engine is NULL" in L.adc_last_error(), L.adc_last_error()
    # valid calls, the minimum alignments, all three kinds and n = 0 get as far as the engine check
    for call in (host, dev):
        for outs, k in [(_outs((p + 4, P, 0)), 1), (_outs((p + 2, S, 0), (p + 4, D, 0), (p + 8, P, 0)), 3)]:
            assert call(outs, k) == 1 and b"engine is NULL" in L.adc_last_error()
    assert dev(_outs((p, P, 0)), 1, n=0) == 1 and b"engine is NULL" in L.adc_last_error()


def test_reproject_constants():
    import adcensus_b200 as A
    assert (A.REPROJ_POINTS, A.REPROJ_DEPTH, A.REPROJ_DISP_S16) == (0, 1, 2)
    assert A.REPROJ_KINDS == {"points": 0, "depth": 1, "disp_s16": 2}
    assert ctypes.sizeof(A.ReprojectOut) == 16
    assert [(n, getattr(A.ReprojectOut, n).offset) for n, _ in A.ReprojectOut._fields_] == [
        ("dst", 0), ("kind", 8), ("reserved", 12)]
    h = (ROOT / "include" / "adcensus_b200.h").read_text()
    assert "enum { ADC_REPROJ_POINTS = 0, ADC_REPROJ_DEPTH = 1, ADC_REPROJ_DISP_S16 = 2 };" in h
    assert "k_reproject.cu" in (ROOT / "adcensus_b200" / "csrc" / "Makefile").read_text()
    with pytest.raises(ValueError):
        A.engine._q_matrix(np.eye(3))
    q = A.engine._q_matrix(np.arange(16, dtype=np.float32).reshape(4, 4))
    assert list(q) == [float(v) for v in range(16)]


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not Path(nvcc).exists():
        pytest.skip("nvcc not available")
    return nvcc


def test_reproject_kernel_uses_no_local_memory():
    """ptxas -v on k_reproject.cu: no stack frame and no spills in any of the seven instantiations (one per set of
    requested outputs)."""
    report = E.ptxas_report(SRC)
    assert len(report) == 7 and all((f["stack"], f["spill_stores"], f["spill_loads"], f["lmem"]) == (0, 0, 0, 0)
                                    for f in report.values()), report
    assert sum(f["regs"] is not None and "k_reproject" in name for name, f in report.items()) == 7, report


def test_reproject_arithmetic_is_not_contracted(tmp_path):
    """The double arithmetic reaches the machine code as written.  PTX: every double add and multiply is an explicit
    .rn operation and there is no double fma, so ptxas may not contract them; the reciprocal is rcp.rn.f64.  SASS
    (cuobjdump): each instantiation has exactly the DADDs of the formula, four pixels per thread, and among them the
    additions to +0.0 (DADD with RZ) that turn a -0 first product into +0.  The SASS does contain DFMAs: they are ptxas'
    correctly rounded expansion of rcp.rn.f64 (Newton steps after MUFU.RCP64H), not contracted formula steps."""
    nvcc = _nvcc()
    base = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-ffp-contract=off"]
    r = subprocess.run(base + ["-ptx", str(SRC), "-o", str(tmp_path / "k.ptx")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    ptx = (tmp_path / "k.ptx").read_text()
    assert "fma.rn.f64" not in ptx and not re.search(r"\bfma\.\w*\.?f64", ptx)
    assert not re.search(r"\b(add|mul|sub)\.f64", ptx), "a double add / mul without an explicit rounding mode"
    assert "rcp.rn.f64" in ptx and not re.search(r"\bdiv\.\w+\.f64", ptx)
    r = subprocess.run(base + ["-c", str(SRC), "-o", str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    cuobjdump = Path(nvcc).parent / "cuobjdump"
    sass = subprocess.run([str(cuobjdump), "-sass", str(tmp_path / "k.o")], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    seen = set()
    for f in funcs:
        m = re.match(r"_Z11k_reprojectILi(\d)EE", f)
        if not m:
            continue
        K = int(m.group(1))
        seen.add(K)
        per_pixel = 16 if K & 1 else 8 if K & 2 else 0          # rows 0..3 for points, rows 2..3 for depth only
        zero_start = 4 if K & 1 else 2 if K & 2 else 0
        assert len(re.findall(r"\bDADD\b", f)) == 4 * per_pixel, (K, len(re.findall(r"\bDADD\b", f)))
        assert len(re.findall(r"\bDADD R\d+, RZ, R\d+", f)) == 4 * zero_start, K
        if K == 4:
            assert not re.search(r"\bD(ADD|MUL|FMA)\b", f), "the S16-only kernel does no double arithmetic"
    assert seen == set(range(1, 8)), seen


# ---- GPU ------------------------------------------------------------------------------------------
def _host_all(eng, disp, Q):
    return eng.reproject(disp, Q, KINDS)


def _check_restated(name, got, disp, Q, dmin):
    assert RP.same_nan(got["points"], RP.points(disp, Q)), f"{name}: points"
    assert RP.same_nan(got["depth"], RP.depth(disp, Q)), f"{name}: depth"
    assert np.array_equal(got["disp_s16"], RP.disp_s16(disp, dmin)), f"{name}: disp_s16"
    # depth is the points' Z bit for bit, NaN payload included: both come from the same kernel
    assert np.array_equal(E.bits(got["depth"]), E.bits(np.ascontiguousarray(got["points"][:, :, 2]))), name


@pytest.mark.gpu
def test_fixture_through_both_entries():
    """Every fixture map, on an engine of its size and min_disparity, through the host entry (all three kinds) and the
    device entry (all three kinds in one call, then each alone): equal to OpenCV's recorded output, NaN as NaN."""
    torch, dev = E.cuda()
    st = torch.cuda.current_stream().cuda_stream
    for name, disp, Q, dmin, pts, s16 in _fixture():
        H, W = disp.shape
        eng = E.engine(W, H, T.default_option(min_disparity=dmin, max_disparity=dmin + 4))
        got = _host_all(eng, disp, Q)
        assert RP.same_nan(got["points"], pts), f"{name} host points"
        assert RP.same_nan(got["depth"], np.ascontiguousarray(pts[:, :, 2])), f"{name} host depth"
        assert np.array_equal(got["disp_s16"], s16), f"{name} host s16"
        d = torch.from_numpy(disp).to(dev)
        out = {"points": torch.empty((H, W, 3), dtype=torch.float32, device=dev),
               "depth": torch.empty((H, W), dtype=torch.float32, device=dev),
               "disp_s16": torch.empty((H, W), dtype=torch.int16, device=dev)}
        for kinds in (KINDS, ["points"], ["depth"], ["disp_s16"]):
            for t in out.values():
                t.fill_(0)
            eng.reproject_batch_device(1, d.data_ptr(), Q, [(out[k].data_ptr(), k) for k in kinds], st)
            torch.cuda.synchronize()
            for k in kinds:
                assert np.array_equal(E.bits(out[k].cpu().numpy()), E.bits(got[k])), f"{name} device {kinds}: {k}"
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cone"] + list(range(len(E.PARITY_CASES))))
def test_engine_maps(case, cone):
    """The engine's final map of Cone and of every test_gpu_parity case (min_disparity < 0 and > 0 included),
    reprojected with stereoRectify Q (CALIB_ZERO_DISPARITY on and off) through both entries: all three kinds equal the
    restatement on the same map."""
    torch, dev = E.cuda()
    if case == "cone":
        left, right = cone
        h, w, _ = left.shape
        opt = dict(max_disparity=64)
    else:
        w, h, D, over, seed = E.PARITY_CASES[case]
        opt = {"max_disparity": D, **over}
        left, right = T.synthetic_pair(w, h, opt["max_disparity"] - opt.get("min_disparity", 0), seed)
    eng = E.engine(w, h, T.default_option(**opt))
    disp = eng.match(left, right)
    dmin = eng.option.min_disparity
    d = torch.from_numpy(disp).to(dev)
    for qname in ("rig_zero_0", "rig_free_1"):
        Q = _fixture_Q(qname)
        got = _host_all(eng, disp, Q)
        _check_restated(f"{case} {qname} host", got, disp, Q, dmin)
        out = {"points": torch.empty((h, w, 3), dtype=torch.float32, device=dev),
               "depth": torch.empty((h, w), dtype=torch.float32, device=dev),
               "disp_s16": torch.empty((h, w), dtype=torch.int16, device=dev)}
        eng.reproject_batch_device(1, d.data_ptr(), Q, [(out[k].data_ptr(), k) for k in KINDS],
                                   torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        for k in KINDS:
            assert np.array_equal(E.bits(out[k].cpu().numpy()), E.bits(got[k])), f"{case} {qname} device {k}"
    eng.close()


@pytest.mark.gpu
def test_camera_path(cone):
    """Raw 640x480 frames of test_rectify's rig through match_rectified, then the reprojection: equal to the
    restatement and to cv2.reprojectImageTo3D of the same map."""
    cv2 = pytest.importorskip("cv2")
    left, right = cone
    h, w, _ = left.shape
    sw, sh = 640, 480
    raw = [cv2.resize(img, (sw, sh), interpolation=cv2.INTER_AREA) for img in (left, right)]
    eng = E.engine(w, h, T.default_option(max_disparity=64))
    for t in (cv2.CV_32FC1, cv2.CV_16SC2):
        maps = [R.cone_rig(cv2, sw, sh, w, h, t, s) for s in (1, -1)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        disp, _ = eng.match_rectified(raw[0], raw[1])
        assert np.isfinite(disp).mean() > 0.5
        Q = _fixture_Q("rig_zero_0")
        got = _host_all(eng, disp, Q)
        _check_restated(f"camera path {t}", got, disp, Q, 0)
        assert RP.same_nan(got["points"], cv2.reprojectImageTo3D(disp, Q)), t
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_batched_device_calls(pipelined):
    """n = 9 engine maps of a 71 x 47 engine with min_disparity -3 (plus specials), at an odd element offset; each kind
    alone and all three together, destinations at odd element offsets (4-byte, and 2-byte for S16, aligned), guard
    elements before and after untouched, each map equal to the host entry's result.  Pipelined: the maps come from a
    pipelined match batch, and a second stream waits with adc_join before it reprojects them.  Each device call is
    exactly one launch."""
    torch, dev = E.cuda()
    w, h, dmin, D, n = 71, 47, -3, 20, 9
    N = w * h
    eng = E.engine(w, h, T.default_option(min_disparity=dmin, max_disparity=dmin + D))
    rng = np.random.default_rng(3)
    pairs = [T.synthetic_pair(w, h, D, 40 + i) for i in range(n)]
    Q = _fixture_Q("rig_free_1")
    dbuf = torch.full((n * N + 8,), float("nan"), dtype=torch.float32, device=dev)
    d = dbuf[1:1 + n * N]
    st = torch.cuda.current_stream()
    if pipelined:
        dl = torch.from_numpy(np.stack([p[0] for p in pairs])).to(dev)
        dr = torch.from_numpy(np.stack([p[1] for p in pairs])).to(dev)
        eng.set_pipelined(True)
        eng.match_batch_device(n, dl.data_ptr(), dr.data_ptr(), d.data_ptr(), st.cuda_stream)
        s2 = torch.cuda.Stream()
        eng.join(s2.cuda_stream)
        stream = s2
    else:
        maps = np.stack([eng.match(*p) for p in pairs])
        specials = np.array([np.nan, -np.inf, -0.0, 0.0, 1e-40, 3e38, -3e38, 2047.96875, 2 ** 27], np.float32)
        flat = maps.reshape(-1)
        flat[rng.choice(flat.size, 200, replace=False)] = rng.choice(specials, 200)
        d.copy_(torch.from_numpy(flat))
        stream = st
    for kinds in (["points"], ["depth"], ["disp_s16"], KINDS):
        # destinations 1 (depth: 3) elements into buffers of -7 (int32 for f32 elements) with 7 more after them
        intact, views = {}, {}
        for k, (count, dt) in {"points": (3 * n * N, torch.float32), "depth": (n * N, torch.float32),
                               "disp_s16": (n * N, torch.int16)}.items():
            if k in kinds:
                data, intact[k] = E.guarded(count, torch.int32 if dt == torch.float32 else torch.int16,
                                            1 if k != "depth" else 3, 7, -7)
                views[k] = data.view(dt)
        c0 = eng.launch_count
        with torch.cuda.stream(stream):
            eng.reproject_batch_device(n, d.data_ptr(), Q, [(views[k].data_ptr(), k) for k in kinds],
                                       stream.cuda_stream)
        assert eng.launch_count == c0 + 1, kinds
        torch.cuda.synchronize()
        host_maps = d.cpu().numpy().reshape(n, h, w)
        for i in range(n):
            want = _host_all(eng, host_maps[i], Q)
            for k in kinds:
                got = views[k].cpu().numpy().reshape((n,) + want[k].shape)[i]
                assert np.array_equal(E.bits(got), E.bits(want[k])), f"pipelined={pipelined} {kinds} map {i}: {k}"
        for k, ok in intact.items():
            assert ok(), f"{kinds}: guard of {k} overwritten"
    if pipelined:
        eng.set_pipelined(False)
        for i in range(n):
            assert np.array_equal(E.bits(host_maps[i]), E.bits(eng.match(*pairs[i]))), f"pipelined map {i}"
    eng.close()


@pytest.mark.gpu
def test_points_past_2_31():
    """n = 5500 maps of 256 x 128 (three distinct ones, repeated): the points destination spans 2.16e9 bytes, past
    2^31.  Every map's points equal the host entry's for its source map, and the element after the last is untouched."""
    torch, dev = E.cuda()
    w, h, n = 256, 128, 5500
    N = w * h
    assert 12 * n * N > 2 ** 31
    rng = np.random.default_rng(8)
    eng = E.engine(w, h, T.default_option(max_disparity=64))
    base = np.stack([(rng.integers(0, 256, (h, w)) / 4.0).astype(np.float32) for _ in range(3)])
    base[0, 5, 7] = np.inf
    base[2, -1, -1] = np.nan
    Q = _fixture_Q("rig_zero_0")
    src = torch.from_numpy(base).to(dev)
    d = src[torch.arange(n, device=dev) % 3].contiguous()
    pts = torch.full((3 * n * N + 1,), -7, dtype=torch.int32, device=dev)
    eng.reproject_batch_device(n, d.data_ptr(), Q, [(pts.data_ptr(), "points")], torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    want = torch.from_numpy(np.stack([E.bits(eng.reproject(base[r], Q)["points"]).view(np.int32).reshape(-1)
                                      for r in range(3)])).to(dev)
    got = pts[:-1].view(n, 3 * N)
    for r in range(3):
        assert torch.equal(got[r::3], want[r].expand_as(got[r::3])), f"maps {r} mod 3"
    assert int(pts[-1]) == -7
    del d, pts
    eng.close()


@pytest.mark.gpu
def test_launches_and_match_unchanged(cone):
    """Each device call adds exactly one launch, the host entry one; a match batch gives the same maps with the same
    number of launches before and after reprojection calls."""
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
    Q = _fixture_Q("rig_zero_0")
    pts = torch.empty((n, h, w, 3), dtype=torch.float32, device=dev)
    s16 = torch.empty((n, h, w), dtype=torch.int16, device=dev)
    for outs in ([(pts.data_ptr(), "points")], [(s16.data_ptr(), "disp_s16"), (pts.data_ptr(), "points")]):
        c0 = eng.launch_count
        eng.reproject_batch_device(n, d0.data_ptr(), Q, outs, st)
        assert eng.launch_count == c0 + 1
    c0 = eng.launch_count
    eng.reproject_batch_device(0, d0.data_ptr(), Q, [(pts.data_ptr(), "points")], st)
    assert eng.launch_count == c0
    c0 = eng.launch_count
    host = eng.reproject(d0[0].cpu().numpy(), Q, ["depth"])
    assert eng.launch_count == c0 + 1
    torch.cuda.synchronize()
    d1, l1 = batch()
    assert l1 == l0 and torch.equal(d0.view(torch.int32), d1.view(torch.int32))
    assert np.array_equal(E.bits(host["depth"]), E.bits(np.ascontiguousarray(pts[0, :, :, 2].cpu().numpy())))
    eng.close()
