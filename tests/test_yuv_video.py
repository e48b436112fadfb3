"""Video-decoder YUV containers (ADC_IMG_I420, _YV12, _P016) and the colour encodings (ADC_IMG_YUV_BT709,
ADC_IMG_YUV_FULL_RANGE) of every YUV container: matched exactly as the restated conversion (yuv_video_testlib; OpenCV's
cvtColor where OpenCV has the rule) followed by the packed-BGR entry point, with or without rectification.

CPU: the restatement against the committed fixture (composed with rectify_testlib's remap) and against live cv2 (skipped
without OpenCV); every encoding on all 2^24 (Y, U, V) triples (BT.601 limited against yuv_testlib, full range against
cv2, BT.709 within +-1 of the floating-point matrix); the argument rules that need no engine; the header's, the
kernels' and the binding's constants; the view parser.
GPU: every container x encoding through the image, rectified and ingest-views entries, host and device (batches with
odd sizes, pitches and strides above their minimums, several waves, pipelined and not), side-by-side halves and
even-offset crops, guard bytes after each view, a poisoned engine, the size rules and launch counts.
"""
import ctypes
import re

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E
import rectify_testlib as R
import yuv_testlib as Y
import yuv_video_testlib as V

ROOT = T.REPO
CSRC = ROOT / "adcensus_b200" / "csrc"
MAPS = ["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"]
VOLS = ["cost", "aggr", "opt"]
GOLDEN = T.GOLDEN_DIR / "golden_yuv_video_cases.npz"
COMBOS = [(f, e) for f in V.ALL for e in V.ENC.values()]


def _triples():
    t = np.arange(1 << 24, dtype=np.uint32)
    return (t >> 16).astype(np.uint8), (t >> 8 & 255).astype(np.uint8), (t & 255).astype(np.uint8)


# ---- CPU ------------------------------------------------------------------------------------------
def test_restatement_against_fixture():
    """The restatement reproduces every OpenCV output in the fixture: I420, YV12 and P016 at BT.601 limited range and
    every container at BT.601 full range, at tiny, odd and even sizes with uniform samples and the rules' corner
    values, plain and followed by remap (both map types, the border BGR 0, 1 x N and 1 x 1 frames)."""
    z = np.load(GOLDEN)
    name_of = {v: k for k, v in V.ALL.items()}
    seen = set()
    for name in sorted({k.split("/")[0] for k in z.files}):
        fmt, enc = name_of[int(z[f"{name}/format"])], int(z[f"{name}/encoding"])
        w, h = (int(v) for v in z[f"{name}/size"])
        got = V.decode(z[f"{name}/frame"], fmt, w, h, enc)
        if f"{name}/map1" in z.files:
            got = R.remap(got, z[f"{name}/map1"], z[f"{name}/map2"])
        assert np.array_equal(got, z[f"{name}/out"]), name
        seen.add((name.split("_")[0], fmt, enc))
    want = {(f, 0) for f in V.NAMES} | {(f, V.FULL) for f in V.ALL}
    for kind in ("tiny", "odd", "rect"):
        assert {(f, e) for k, f, e in seen if k == kind} == want, kind


def test_restatement_against_opencv():
    """Live cv2 with the optimised paths on and off: I420 / YV12 cvtColor, P016 convertScaleAbs + cvtColor(NV12), and
    full range (nearest chroma, then COLOR_YCrCb2BGR) for every container, at 60 random sizes 1..160 each (a third from
    the corner values) and 1080 x 1920."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(41)
    opt = cv2.useOptimized()
    try:
        for use in (True, False):
            cv2.setUseOptimized(use)
            for i in range(60):
                w, h = (int(v) for v in rng.integers(1, 161, 2))
                for fmt in V.ALL:
                    frame = V.random_frame(rng, fmt, w, h, corners=i % 3 == 0)
                    for enc in ((0, V.FULL) if fmt in V.CODE else (V.FULL,)):
                        assert np.array_equal(V.decode(frame, fmt, w, h, enc), V.cv_decode(cv2, frame, fmt, w, h, enc)), \
                            (use, fmt, enc, w, h)
            for fmt in V.NAMES:
                frame = V.random_frame(rng, fmt, 1920, 1080)
                assert np.array_equal(V.decode(frame, fmt, 1920, 1080), V.cv_decode(cv2, frame, fmt, 1920, 1080)), fmt
    finally:
        cv2.setUseOptimized(opt)


def test_every_triple_of_every_encoding():
    """All 2^24 (Y, U, V): no flag is yuv_testlib's BT.601 limited rule bit for bit; BT.601 full range is
    cv2.cvtColor(COLOR_YCrCb2BGR) on (Y, V, U) (when OpenCV is present); BT.709 full range is within +-1 of the
    floating-point BT.709 matrix everywhere, BT.709 limited range for Y >= 16, and below 16 (where Y - 16 clamps at 0)
    within 19 levels; a grey pixel converts alike under both limited-range rules."""
    Yv, U, Vv = _triples()
    assert np.array_equal(V.convert(Yv, U, Vv, 0), Y.convert(Yv, U, Vv))
    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is not None:
        img = np.stack([Yv, Vv, U], -1).reshape(4096, 4096, 3)
        assert np.array_equal(cv2.cvtColor(img, cv2.COLOR_YCrCb2BGR).reshape(-1, 3), V.convert(Yv, U, Vv, V.FULL))
    for enc, lim in ((V.BT709 | V.FULL, 1), (V.BT709, 1)):
        d = np.abs(V.convert(Yv, U, Vv, enc).astype(np.int16) - V.float_convert(Yv, U, Vv, enc).astype(np.int16)).max(-1)
        hi = Yv >= 16 if not enc & V.FULL else np.ones_like(Yv, bool)
        assert d[hi].max() <= lim, enc
        if not enc & V.FULL:
            assert d[~hi].max() == 19
    g = np.arange(256, dtype=np.uint8)
    c = np.full(256, 128, np.uint8)
    assert np.array_equal(V.convert(g, c, c, 0), V.convert(g, c, c, V.BT709))


def test_rule_intermediates_fit_int32():
    """Every intermediate of every encoding's rule lies inside int32 (each is linear in Y', u and v, so its extremes
    lie at the corners of their ranges), and each constant is round(k * 2^shift) of its matrix coefficient."""
    ends = np.array([0, 16, 255], np.int64)
    yy, uu, vv = np.meshgrid(ends, ends, ends, indexing="ij")
    for enc, (rv, gu, gv, bu) in V.COEF.items():
        u, v = uu - 128, vv - 128
        y = yy if enc & V.FULL else np.maximum(0, yy - 16) * 1220542 + (1 << 19)
        for t in (y + rv * v, y + gu * u + gv * v, y + bu * u, rv * v + 8192, gu * u + gv * v + 8192):
            assert np.abs(t).max() < 2 ** 31, enc
    for enc in (V.BT709, V.BT709 | V.FULL):
        kr, kb = V.KR_KB[V.BT709]
        kg = 1 - kr - kb
        s, scale = (14, 1.0) if enc & V.FULL else (20, 255 / 224)
        k = [2 * (1 - kr), -2 * (1 - kb) * kb / kg, -2 * (1 - kr) * kr / kg, 2 * (1 - kb)]
        assert [round(c * scale * (1 << s)) for c in k] == list(V.COEF[enc]), enc


def test_view_helpers():
    """write_view lays only the view's own samples (W luma samples a row; ceil(W/2) bytes a row of each I420 chroma
    plane at half the pitch; 2*ceil(W/2) words a P016 chroma row) and samples() reads them back; encode() gives the
    host entries' shape; read_bytes counts exactly the samples written."""
    rng = np.random.default_rng(4)
    for fmt in V.NAMES:
        for w, h in ((7, 5), (8, 6), (1, 1)):
            frame = V.random_frame(rng, fmt, w, h)
            rp = V.tight_row(fmt, w) + 4
            pp = h * rp + 6
            buf = np.full(2 + V.footprint(fmt, h, rp, pp) + 4, 0xEE, np.uint8)
            mask = np.zeros_like(buf)
            V.write_view(buf, frame, fmt, w, h, rp, pp, 2)
            V.write_view(mask, np.full_like(frame, 0xFFFF if fmt == "p016" else 0xFF), fmt, w, h, rp, pp, 2)
            assert int((mask != 0).sum()) == V.read_bytes(fmt, w, h)
            assert buf[:2].tolist() == [0xEE, 0xEE] and (buf[-4:] == 0xEE).all()
            assert V.encode(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), fmt).shape == V.frame_shape(fmt, w, h)
    # encode() of I420 / YV12 / P016 carries NV12's samples
    bgr = rng.integers(0, 256, (6, 9, 3), dtype=np.uint8)
    want = Y.decode(Y.encode(bgr, "nv12"), "nv12", 9, 6)
    for fmt in V.NAMES:
        assert np.array_equal(V.decode(V.encode(bgr, fmt), fmt, 9, 6), want), fmt


def _entries(L, p):
    return {
        "adc_match_images:": lambda img, l=p, r=p: L.adc_match_images(None, l, r, img, None, 0, 0, p, None, 0, None, 0),
        "adc_match_images_batch_device": lambda img, l=p, r=p: L.adc_match_images_batch_device(
            None, 1, l, r, img, None, 0, 0, p, None, 0, None, 0, None),
        "adc_match_rectified:": lambda img, l=p, r=p: L.adc_match_rectified(None, l, r, img, None, 0, 0, p, None, 0, None,
                                                                           0),
        "adc_match_rectified_batch_device": lambda img, l=p, r=p: L.adc_match_rectified_batch_device(
            None, 1, l, r, img, None, 0, 0, p, None, 0, None, 0, None),
    }


def test_argument_rules_need_no_gpu():
    """Every container with every encoding passes the size-free rules and reaches the engine check on both image and
    both rectified entries; plane_pitch != 0 is accepted for the 4:2:0 containers; a flag on a format that is not YUV
    and any bit above 0x3ff fail naming img->format; an odd I420 / YV12 row_pitch fails on every entry; odd P016 base
    pointers, row_pitch, plane_pitch or image_stride fail on the device entries only; 37, 41, 63 stay unknown."""
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    D = A.ImageDesc
    for fn, call in _entries(L, p).items():
        dev = fn.endswith("device")
        for (name, base), enc in [(c, e) for c in V.ALL.items() for e in V.ENC.values()]:
            code = base | enc
            for d in (D(code, 0, 0, 0, 0), D(code, 0, 1002, 0, 1 << 33), D(code, 0, 0, 64, 0)):
                rc = call(ctypes.byref(d))
                err = L.adc_last_error()
                if d.plane_pitch and not V.is420(name):
                    assert rc == 1 and b"img->plane_pitch" in err and fn.encode() in err, (fn, code, err)
                else:
                    assert rc == 1 and b"engine is NULL" in err, (fn, code, err)
            assert call(ctypes.byref(D(code, 1, 0, 0, 0))) == 1 and b"img->reserved" in L.adc_last_error()
            rc = call(ctypes.byref(D(code, 0, 1001, 0, 0)))
            err = L.adc_last_error()
            if V.is_planar(name):
                assert rc == 1 and b"img->row_pitch 1001 must be even" in err and fn.encode() in err, err
            elif name == "p016" and dev:
                assert b"img->row_pitch 1001" in err and b"16-bit format" in err, err
            else:
                assert b"engine is NULL" in err, err
            if name == "p016":
                for what, kw, d in (("d_left", dict(l=p + 1), D(code, 0, 0, 0, 0)),
                                    ("d_right", dict(r=p + 1), D(code, 0, 0, 0, 0)),
                                    ("img->plane_pitch 8001", {}, D(code, 0, 0, 8001, 0)),
                                    ("img->image_stride 9001", {}, D(code, 0, 0, 0, 9001))):
                    assert call(ctypes.byref(d), **kw) == 1
                    err = L.adc_last_error()
                    if dev:
                        assert what.encode() in err and fn.encode() in err and b"16-bit format" in err, err
                    else:
                        assert b"engine is NULL" in err, err
        for code in (A.IMG_BGR | A.IMG_YUV_BT709, A.IMG_GRAY | A.IMG_YUV_FULL_RANGE, A.IMG_BAYER_RGGB | 0x300,
                     A.IMG_MONO12 | A.IMG_YUV_BT709):
            assert call(ctypes.byref(D(code, 0, 0, 0, 0))) == 1
            err = L.adc_last_error()
            assert f"img->format {code}:".encode() in err and b"YUV formats only" in err and fn.encode() in err, err
        for code in (37, 41, 63, A.IMG_NV12 | 0x400, A.IMG_I420 | 0x800, A.IMG_P016 | (1 << 30), 37 | 0x100, -1):
            assert call(ctypes.byref(D(code, 0, 0, 0, 0))) == 1
            err = L.adc_last_error()
            assert f"img->format {code} unknown".encode() in err and fn.encode() in err, err
    for bad in ("yuv", "mono14", "bgr/bt709", "i420/bt2020", "p010"):
        with pytest.raises(ValueError):
            A.image_desc(bad)


def test_constants():
    """The header's codes, flags and constant table, the kernels' constant rows and the binding's constants agree with
    the restatement; the binding's name dicts are disjoint; image_desc takes container and encoding names."""
    import adcensus_b200 as A
    h = (ROOT / "include" / "adcensus_b200.h").read_text()
    assert "enum { ADC_IMG_I420 = 38, ADC_IMG_YV12 = 39, ADC_IMG_P016 = 40 };" in h
    assert "enum { ADC_IMG_YUV_BT709 = 0x100, ADC_IMG_YUV_FULL_RANGE = 0x200 };" in h
    rows = {"BT.601 limited (no flag)": 0, "BT.709 limited": V.BT709, "BT.601 full range": V.FULL,
            "BT.709 full range": V.BT709 | V.FULL}
    for label, enc in rows.items():
        m = re.search(re.escape(label) + r"\s+(-?\d+)\s+(-?\d+)\s+(-?\d+)\s+(-?\d+)", h)
        assert m and tuple(int(v) for v in m.groups()) == V.COEF[enc], label
    k = (CSRC / "k_image.cuh").read_text()
    got = [tuple(int(v) for v in m.groups()) for m in re.finditer(r"YuvCoef\{(-?\d+), (-?\d+), (-?\d+), (-?\d+)\}", k)]
    assert got == [V.COEF[e] for e in (0, V.BT709, V.FULL, V.BT709 | V.FULL)]
    assert (A.IMG_I420, A.IMG_YV12, A.IMG_P016) == (38, 39, 40)
    assert (A.IMG_YUV_BT709, A.IMG_YUV_FULL_RANGE) == (V.BT709, V.FULL)
    assert A.YUV_VIDEO_FORMATS == V.CODE and A.YUV_ENCODINGS == V.ENC
    others = set(A.engine.IMG_FORMATS) | set(A.BAYER_FORMATS) | set(A.YUV_FORMATS) | set(A.RAW_DEPTH_FORMATS)
    assert not set(A.YUV_VIDEO_FORMATS) & others
    for (name, code), (en, enc) in [(c, e) for c in V.ALL.items() for e in V.ENC.items()]:
        d = A.image_desc(f"{name}/{en}", 80, 4000, 9000)
        assert (d.format, d.row_pitch, d.plane_pitch, d.image_stride) == (code | enc, 80, 4000, 9000)
    assert A.image_desc("i420").format == 38


def test_view_parser():
    """I420 / YV12: uint8 [H + ceil(H/2)][2*ceil(W/2)] with contiguous rows, plane pitch H * row pitch; P016: the same
    shape in uint16, pitched rows and side-by-side halves allowed; the encoding flags pass through."""
    import adcensus_b200 as A
    P = A.engine._image_view_desc
    for fmt in (A.IMG_I420, A.IMG_YV12 | A.IMG_YUV_BT709):
        d = P(np.zeros((9 + 5, 40), np.uint8), fmt, 9, 39)
        assert (d.format, d.row_pitch, d.plane_pitch, d.image_stride) == (fmt, 40, 360, 0)
        with pytest.raises(ValueError):
            P(np.zeros((14, 50), np.uint8)[:, :40], fmt, 9, 39)   # pitched rows: the chroma rows are not in the view
        with pytest.raises(ValueError):
            P(np.zeros((14, 40), np.uint16), fmt, 9, 39)
        with pytest.raises(ValueError):
            P(np.zeros((13, 40), np.uint8), fmt, 9, 39)
    frame = np.zeros((9 + 5, 2 * 40), np.uint16)
    for fmt in (A.IMG_P016, A.IMG_P016 | A.IMG_YUV_BT709 | A.IMG_YUV_FULL_RANGE):
        d = P(frame[:, 40:], fmt, 9, 40)
        assert (d.format, d.row_pitch, d.plane_pitch) == (fmt, 160, 9 * 160)
        assert P(frame[:, :38], fmt, 9, 37).row_pitch == 160
        with pytest.raises(ValueError):
            P(frame.view(np.uint8)[:, :80], fmt, 9, 40)
        with pytest.raises(ValueError):
            P(frame[:, :37], fmt, 9, 37)
    d = P(np.zeros((8, 50, 2), np.uint8)[1:8, 4:30], A.IMG_UYVY | A.IMG_YUV_FULL_RANGE, 7, 25)
    assert (d.format, d.row_pitch, d.plane_pitch) == (A.IMG_UYVY | A.IMG_YUV_FULL_RANGE, 100, 0)


# ---- GPU ------------------------------------------------------------------------------------------
def _batch(fmt, n, vw, vh, rng, extra_row, extra_plane, extra_stride, lead, guard=64):
    """n pairs of random frames with row pitch tight + extra_row, plane pitch H * row pitch + extra_plane (4:2:0),
    image stride footprint + extra_stride, `lead` bytes before the first view and random bytes everywhere else, one
    host buffer per view with `guard` bytes after the last view.  (host buffers, offset, desc args, left, right)."""
    rp = V.tight_row(fmt, vw) + extra_row
    pp = vh * rp + extra_plane if V.is420(fmt) else 0
    stride = V.footprint(fmt, vh, rp, pp) + extra_stride
    L = [V.random_frame(rng, fmt, vw, vh) for _ in range(n)]
    Rr = [V.random_frame(rng, fmt, vw, vh) for _ in range(n)]
    bufs = []
    for frames in (L, Rr):
        big = rng.integers(0, 256, size=lead + n * stride + guard, dtype=np.uint8)
        for i in range(n):
            V.write_view(big, frames[i], fmt, vw, vh, rp, pp, lead + i * stride)
        bufs.append(big)
    return bufs, lead, (rp, pp, stride), L, Rr


def _packed(frames, fmt, enc, w, h, maps=None):
    torch, dev = E.cuda()
    imgs = [V.decode(f, fmt, w, h, enc) for f in frames]
    if maps is not None:
        imgs = [R.remap(x, *maps) for x in imgs]
    return torch.from_numpy(np.stack(imgs)).to(dev)


def _equal_all(got, want, name):
    for k in want:
        assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), f"{name}: {k}"


def _pitches(k, fmt):
    """Row / plane / stride extras and the lead offset of case k: even where P016 or I420 need it."""
    ev = 2 if fmt == "p016" else 1
    row = (0, 6, 64, 2)[k % 4] if fmt in ("p016", "i420", "yv12") else (0, 7, 64, 1)[k % 4]
    return row, ev * (0, 5, 0, 3)[k % 4], ev * (5, 0, 3, 11)[k % 4], ev * (0, 3, 1, 6)[k % 4]


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_video_batched(pipelined):
    """wave_pairs = 4, lanes = 3, n = 14 (several waves per lane, a partial last one), odd W and H, every container in
    every encoding with row pitch, plane pitch and image stride above their minimums and views at offsets off the
    tight grid: every output equals adc_match_outputs_batch_device on the restated BGR views; the guard bytes after the
    last view are then changed and every output stays the same."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    rng = np.random.default_rng(8 + pipelined)
    outputs = dict(volumes=[(v, "hwd", "f32") for v in VOLS], maps=MAPS, pipelined=pipelined)
    for k, (fmt, enc) in enumerate(COMBOS):
        bufs, off, (rp, pp, stride), L, Rr = _batch(fmt, n, w, h, rng, *_pitches(k, fmt))
        views = [torch.from_numpy(b).to(dev) for b in bufs]
        desc = A.image_desc(V.ALL[fmt] | enc, rp, pp, stride)
        pl, pr = _packed(L, fmt, enc, w, h), _packed(Rr, fmt, enc, w, h)
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_images_batch_device, n, views[0].data_ptr() + off,
                              views[1].data_ptr() + off, stride, image=desc, **outputs)
        name = f"{fmt}|{enc:#x} rp {rp} pp {pp} stride {stride}"
        _equal_all(got, want, name)
        if k % 4 == 0:
            end = off + (n - 1) * stride + V.footprint(fmt, h, rp, pp)
            for v in views:
                v[end:] = 255 - v[end:]
            got = E.batch_outputs(eng, eng.match_images_batch_device, n, views[0].data_ptr() + off,
                                  views[1].data_ptr() + off, stride, image=desc, **outputs)
            _equal_all(got, want, name + " guard bytes changed")
    eng.close()


@pytest.mark.gpu
def test_video_side_by_side_and_crops():
    """Side-by-side NV12 (BT.709) and P016 (BT.709, full range) frames, the right view at base + W samples with one
    plane pitch for both, and crops at even offsets of larger NV21 (full range), P016 and YUYV (BT.709) frames, 3
    pairs a call: every output equals the packed-BGR call on the restated views."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 70, 45, 19
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=2)
    n = 3
    rng = np.random.default_rng(14)
    outputs = dict(volumes=[("opt", "hwd", "f32")], maps=MAPS)
    for fmt, enc in (("nv12", V.BT709), ("p016", V.BT709 | V.FULL), ("p016", 0)):
        frames = [V.random_frame(rng, fmt, 2 * w, h) for _ in range(n)]
        sample = frames[0].itemsize
        rp = 2 * w * sample
        stride = frames[0].nbytes + 2 * sample
        host = np.zeros(n * stride, np.uint8)
        for i, f in enumerate(frames):
            host[i * stride:i * stride + f.nbytes] = f.view(np.uint8).reshape(-1)
        d = torch.from_numpy(host).to(dev)
        halves = [[np.concatenate([f[:h, x:x + w], f[h:, x:x + w]]) for f in frames] for x in (0, w)]
        pl, pr = (_packed(hv, fmt, enc, w, h) for hv in halves)
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_images_batch_device, n, d.data_ptr(), d.data_ptr() + rp // 2, stride,
                              image=A.image_desc(V.ALL[fmt] | enc, rp, h * rp, stride), **outputs)
        _equal_all(got, want, f"side by side {fmt}|{enc:#x}")
    FW, FH, x0, y0, vh = w + 10, 52, 4, 6, 43
    eng.close()
    eng = E.engine(w, vh, T.default_option(max_disparity=D), wave_pairs=2)
    for fmt, enc in (("nv21", V.FULL), ("p016", V.BT709), ("yuyv", V.BT709)):
        frames = [[V.random_frame(rng, fmt, FW, FH) for _ in range(n)] for _ in range(2)]
        s = frames[0][0].itemsize
        rp = V.tight_row(fmt, FW)
        if V.is420(fmt):
            pp = (FH - y0 + y0 // 2) * rp
            crops = [[np.concatenate([f[y0:y0 + vh, x0:x0 + w], f[FH + y0 // 2:FH + y0 // 2 + V.half(vh), x0:x0 + w]])
                      for f in fs] for fs in frames]
            off = y0 * rp + x0 * s
        else:
            pp = 0
            crops = [[f[y0:y0 + vh, x0:x0 + w] for f in fs] for fs in frames]
            off = y0 * rp + 2 * x0
        stride = frames[0][0].nbytes
        d = [torch.from_numpy(np.concatenate([f.view(np.uint8).reshape(-1) for f in fs])).to(dev) for fs in frames]
        pl, pr = (_packed(c, fmt, enc, w, vh) for c in crops)
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * vh,
                               **outputs)
        got = E.batch_outputs(eng, eng.match_images_batch_device, n, d[0].data_ptr() + off, d[1].data_ptr() + off,
                              stride, image=A.image_desc(V.ALL[fmt] | enc, rp, pp, stride), **outputs)
        _equal_all(got, want, f"crop {fmt}|{enc:#x}")
    eng.close()


@pytest.mark.gpu
def test_video_host_entries_and_views():
    """Every container in every encoding through the single-pair host entries, odd W and H (P016 also as column
    slices of wider arrays): ingest_views is byte-equal to the restated decode, and match_images gives the final map,
    all three volumes and all five side maps of match_outputs on the restated views."""
    w, h, D = 61, 45, 20
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    rng = np.random.default_rng(21)
    for k, (fmt, enc) in enumerate(COMBOS):
        frames = [V.random_frame(rng, fmt, w, h) for _ in range(2)]
        if fmt == "p016" and k % 2:
            wide = []
            for f in frames:
                big = V.random_frame(rng, fmt, w + 9, h)[:, :f.shape[1] + 8].copy()
                big[:, :f.shape[1]] = f
                wide.append(big[:, :f.shape[1]])
            frames = wide
        name = f"{fmt}/{[n for n, e in V.ENC.items() if e == enc][0]}"
        want_views = np.stack([V.decode(f, fmt, w, h, enc) for f in frames])
        assert np.array_equal(eng.ingest_views(frames[0], frames[1], format=name), want_views), name
        if k % 4 == 1 or fmt in V.CODE:
            want_disp, want = eng.match_outputs(*want_views, maps=MAPS, volumes=VOLS)
            disp, got = eng.match_images(frames[0], frames[1], format=name, maps=MAPS, volumes=VOLS)
            E.same(f"{name} host disp", disp, want_disp)
            for key in want:
                E.same(f"{name} host {key}", got[key], want[key])
    eng.close()


@pytest.mark.gpu
def test_video_ingest_views_device():
    """adc_ingest_views_batch_device, plain and rectified, every container in every encoding, 5 pairs with pitches
    above their minimums: the packed views are byte-equal to the restated decode (rectified: followed by remap, the
    border BGR 0)."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 53, 37, 12
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=2)
    sw, sh = 59, 33
    maps = [R.warp_maps(w, h, sw, sh, 70 + v, True) for v in range(2)]
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    n = 5
    rng = np.random.default_rng(5)
    for k, (fmt, enc) in enumerate(COMBOS):
        for rect in (False, True):
            vw, vh = (sw, sh) if rect else (w, h)
            bufs, off, (rp, pp, stride), L, Rr = _batch(fmt, n, vw, vh, rng, *_pitches(k + rect, fmt))
            views = [torch.from_numpy(b).to(dev) for b in bufs]
            out = torch.full((n, 2, h, w, 3), 7, dtype=torch.uint8, device=dev)
            eng.ingest_views_batch_device(n, views[0].data_ptr() + off, views[1].data_ptr() + off, out.data_ptr(),
                                          image=A.image_desc(V.ALL[fmt] | enc, rp, pp, stride), rectified=rect,
                                          stream=torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            want = np.stack([_packed(L, fmt, enc, vw, vh, maps[0] if rect else None).cpu().numpy(),
                             _packed(Rr, fmt, enc, vw, vh, maps[1] if rect else None).cpu().numpy()], 1)
            assert np.array_equal(out.cpu().numpy(), want), (fmt, enc, rect)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_video_rectified(pipelined):
    """Raw frames through the rectified entries, every container in every encoding across the cases: both map types,
    frames larger and smaller than the engine, odd, 1 x 1 and 1 x N, pitches above their minimums: every output equals
    adc_match_outputs_batch_device on remap(decode(raw)); the host entry match_rectified agrees."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=3)
    n = 2 * eng.wave_pairs + 1
    rng = np.random.default_rng(12 + pipelined)
    sizes = [(83, 53), (64, 40), (1, 1), (57, 1), (3, 5), (90, 61), (1, 2), (33, 1)]
    for k, (fmt, enc) in enumerate(COMBOS):
        sw, sh = sizes[k % len(sizes)]
        fixed = k % 2 == 1
        maps = [R.warp_maps(w, h, sw, sh, 40 + 2 * k + v, fixed) for v in range(2)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        bufs, off, (rp, pp, stride), L, Rr = _batch(fmt, n, sw, sh, rng, *_pitches(k, fmt))
        views = [torch.from_numpy(b).to(dev) for b in bufs]
        outputs = dict(volumes=[(v, "hwd", "f32") for v in VOLS], maps=MAPS, pipelined=pipelined)
        pl, pr = _packed(L, fmt, enc, sw, sh, maps[0]), _packed(Rr, fmt, enc, sw, sh, maps[1])
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_rectified_batch_device, n, views[0].data_ptr() + off,
                              views[1].data_ptr() + off, stride, image=A.image_desc(V.ALL[fmt] | enc, rp, pp, stride),
                              **outputs)
        _equal_all(got, want, f"{sw}x{sh} {fmt}|{enc:#x} fixed={fixed}")
        if not pipelined and k % 3 == 0:
            disp, one = eng.match_rectified(L[1], Rr[1], format=V.ALL[fmt] | enc, maps=MAPS)
            E.same(f"{sw}x{sh} {fmt}|{enc:#x} host disp", disp, want["disp"][1])
            for m in MAPS:
                E.same(f"{sw}x{sh} {fmt}|{enc:#x} host {m}", one[m], want[m][1])
    eng.close()


@pytest.mark.gpu
def test_video_poisoned_engine():
    """With ADC_DBG_POISON (every lane arena and the host calls' staging filled with a pattern before each wave and
    call), I420 BT.709, YV12 full range and P016 BT.709 through the batched, host and rectified entries give the
    outputs of the packed-BGR call on the restated views."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 45, 31, 16
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=2, lanes=2, debug_flags=A.engine.poison_flags(0xA5))
    rng = np.random.default_rng(33)
    n = 5
    outputs = dict(volumes=[("cost", "hwd", "f32")], maps=MAPS)
    for k, (fmt, enc) in enumerate((("i420", V.BT709), ("yv12", V.FULL), ("p016", V.BT709))):
        bufs, off, (rp, pp, stride), L, Rr = _batch(fmt, n, w, h, rng, *_pitches(k + 1, fmt))
        views = [torch.from_numpy(b).to(dev) for b in bufs]
        pl, pr = _packed(L, fmt, enc, w, h), _packed(Rr, fmt, enc, w, h)
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_images_batch_device, n, views[0].data_ptr() + off,
                              views[1].data_ptr() + off, stride, image=A.image_desc(V.ALL[fmt] | enc, rp, pp, stride),
                              **outputs)
        _equal_all(got, want, f"poisoned {fmt}|{enc:#x}")
        disp, one = eng.match_images(L[2], Rr[2], format=V.ALL[fmt] | enc, maps=MAPS)
        E.same(f"poisoned {fmt} host disp", disp, want["disp"][2])
        maps = [R.warp_maps(w, h, w + 6, h + 4, 60 + v) for v in range(2)]
        eng.set_rectification(maps[0], maps[1], (w + 6, h + 4))
        fr = [V.random_frame(rng, fmt, w + 6, h + 4) for _ in range(2)]
        want_disp, _ = eng.match_outputs(*(R.remap(V.decode(fr[v], fmt, w + 6, h + 4, enc), *maps[v]) for v in range(2)))
        disp, _ = eng.match_rectified(fr[0], fr[1], format=V.ALL[fmt] | enc)
        E.same(f"poisoned {fmt} rectified disp", disp, want_disp)
        eng.set_rectification(None)
    eng.close()


@pytest.mark.gpu
def test_video_size_rules():
    """Each size-dependent rule violation fails with ADC_ERR_ARG naming its field, on the image and the rectified
    entries: I420 row_pitch below 2*ceil(W/2), an I420 plane_pitch one row pair short, a P016 row pitch of 2*W, an
    image stride short of the footprint; the minimums themselves are accepted."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 12
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    buf = torch.zeros(8 * (w + 1) * h * 2, dtype=torch.uint8, device=dev)
    d_o = torch.empty((2, h, w), dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def run(entry, code, rp=0, pp=0, stride=0):
        entry(2, buf.data_ptr(), buf.data_ptr(), image=A.image_desc(code, rp, pp, stride), d_disp=d_o.data_ptr(),
              stream=st)
        torch.cuda.synchronize()

    eng.set_rectification(*[R.warp_maps(w, h, w, h, 5)] * 2, (w, h))
    for entry in (eng.match_images_batch_device, eng.match_rectified_batch_device):
        bad = [(A.IMG_I420, dict(rp=70), r"img->row_pitch 70 is less than 2 \* ceil\(W / 2\) \(72\)"),
               (A.IMG_YV12 | A.IMG_YUV_BT709, dict(rp=72, pp=h * 72 - 2), r"img->plane_pitch 3382 is less than"),
               (A.IMG_P016, dict(rp=2 * w), r"img->row_pitch 142 is less than 4 \* ceil\(W / 2\) \(144\)"),
               (A.IMG_P016 | A.IMG_YUV_FULL_RANGE, dict(stride=144 * (h + 24) - 2),
                r"img->image_stride 10222 is less than the view's footprint \(10224\)"),
               (A.IMG_I420, dict(stride=72 * (h + 24) - 1), r"img->image_stride 5111 is less than")]
        for code, kw, msg in bad:
            with pytest.raises(A.AdcError, match=r"error 1: .*" + msg):
                run(entry, code, **kw)
        for code, kw in ((A.IMG_I420, dict(rp=72, pp=72 * h, stride=72 * (h + 24))),
                         (A.IMG_P016 | A.IMG_YUV_BT709, dict(rp=144, pp=144 * h, stride=144 * (h + 24)))):
            run(entry, code, **kw)
    eng.close()


@pytest.mark.gpu
def test_video_launch_counts():
    """A call in any new container or encoding issues exactly one launch per wave more than the tight packed-BGR call,
    through the image and the rectified entry; profile ids 13 / 14 replay the last format, encoding included, and
    report the algorithmic bytes (I420 / YV12: W*H + 2*ceil(W/2)*ceil(H/2) read, P016 twice that, plus 3*N written)."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=2)
    n = 3 * eng.wave_pairs + 1
    waves = -(-n // eng.wave_pairs)
    rng = np.random.default_rng(2)
    bgr = [torch.from_numpy(rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)).to(dev) for _ in range(2)]
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream()

    def count(call, *a, **kw):
        torch.cuda.synchronize()
        c0 = eng.launch_count
        call(*a, d_disp=d_o.data_ptr(), stream=st.cuda_stream, **kw)
        torch.cuda.synchronize()
        return eng.launch_count - c0

    def frames(fmt, vw, vh):
        return [torch.from_numpy(np.stack([V.random_frame(rng, fmt, vw, vh).view(np.uint8) for _ in range(n)])).to(dev)
                for _ in range(2)]

    base = count(eng.match_outputs_batch_device, n, bgr[0].data_ptr(), bgr[1].data_ptr())
    cases = [(f, e) for f in V.NAMES for e in V.ENC.values()] + [("nv12", V.FULL), ("uyvy", V.BT709 | V.FULL)]
    for fmt, enc in cases:
        yuv = frames(fmt, w, h)
        got = count(eng.match_images_batch_device, n, yuv[0].data_ptr(), yuv[1].data_ptr(),
                    image=A.image_desc(V.ALL[fmt] | enc))
        assert got == base + waves, (fmt, enc, got, base, waves)
        assert eng.profile_kernel("image_ingest", reps=2)[1] == 2 * eng.wave_pairs * (V.read_bytes(fmt, w, h) + 3 * h * w)
    sw, sh = 91, 61
    m = R.warp_maps(w, h, sw, sh, 3)
    eng.set_rectification(m, m, (sw, sh))
    for fmt, enc in cases:
        yuv = frames(fmt, sw, sh)
        got = count(eng.match_rectified_batch_device, n, yuv[0].data_ptr(), yuv[1].data_ptr(),
                    image=A.image_desc(V.ALL[fmt] | enc))
        assert got == base + waves, (fmt, enc, got, base, waves)
        ms, by = eng.profile_kernel("rectify", reps=2)
        assert ms > 0 and by == 2 * eng.wave_pairs * (V.read_bytes(fmt, sw, sh) + 3 * h * w) + 2 * 8 * h * w, fmt
    eng.close()
