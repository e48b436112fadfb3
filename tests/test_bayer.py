"""Bayer mosaics (ADC_IMG_BAYER_*): raw 8-bit colour-filter frames demosaiced on the way in, matched exactly as
cv2.cvtColor(raw, COLOR_Bayer*2BGR) followed by the packed-BGR entry point, with or without rectification.

CPU: the numpy restatement (bayer_testlib) against live cv2.cvtColor with IPP on and off (skipped without OpenCV) and
against the committed fixture, composed with rectify_testlib's cv2.remap (never skipped); the argument rules that need
no engine; the constants.
GPU: Cone mosaiced with every pattern against the CPU oracle on the restated demosaic; synthetic batches (odd sizes,
crops at even and odd offsets, row pitch > W, image stride > footprint, several waves with a partial last one, pipelined
and not) against adc_match_outputs_batch_device on the restated images, every output; the single-pair host entries;
raw frames through both map types, larger and smaller than the engine, 1 x 1 and 2 x N; launch counts.
"""
import ctypes

import numpy as np
import pytest

import adc_testlib as T
import bayer_testlib as B
import engine_testlib as E
import rectify_testlib as R

ROOT = T.REPO
MAPS = ["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"]
VOLS = ["cost", "aggr", "opt"]
GOLDEN = T.GOLDEN_DIR / "golden_bayer_cases.npz"


# ---- CPU ------------------------------------------------------------------------------------------
def _cases_from(npz):
    z = np.load(npz)
    code = {v: k for k, v in B.CODE.items()}
    for name in sorted({k.split("/")[0] for k in z.files}):
        maps = (z[f"{name}/map1"], z[f"{name}/map2"]) if f"{name}/map1" in z.files else None
        yield name, z[f"{name}/raw"], code[int(z[f"{name}/pattern"])], maps, z[f"{name}/out"]


def test_restatement_against_fixture():
    """The restatement reproduces every cvtColor output in the fixture (every pattern below 3 pixels, at 3 x N, N x 3,
    odd sizes and odd-offset crops) and, composed with the remap restatement, every cvtColor -> remap output (both map
    types, frames larger and smaller than the output, maps past the last row and column, 2 x N and 1 x 1 frames)."""
    seen = set()
    for name, raw, pat, maps, out in _cases_from(GOLDEN):
        got = B.demosaic(raw, pat)
        if maps is not None:
            got = R.remap(got, *maps)
        assert np.array_equal(got, out), name
        seen.add((name.split("_")[0], pat if maps is None else "rect"))
    assert {k for k, _ in seen} == {"tiny", "odd", "rect"}
    assert {p for k, p in seen if k != "rect"} == set(B.NAMES)


def test_restatement_against_opencv():
    """The restatement against live cv2.cvtColor, with IPP on and off: 200 random sizes 1..130 on a side per setting as
    crops at random offsets of larger frames, 3 x N, N x 3, 2 x N, N x 2, and 1080 x 1920, every pattern."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(17)
    ipp = cv2.ipp.useIPP()
    try:
        for use in (True, False):
            cv2.ipp.setUseIPP(use)
            shapes = [tuple(int(v) for v in rng.integers(1, 131, 2)) for _ in range(200)]
            shapes += [(3, 1), (3, 2), (3, 57), (57, 3), (2, 40), (40, 2), (2, 2), (1, 1), (1080, 1920)]
            for i, (h, w) in enumerate(shapes):
                big = rng.integers(0, 256, (h + 4, w + 9), dtype=np.uint8)
                y0, x0 = int(rng.integers(0, 5)), int(rng.integers(0, 10))
                raw = big[y0:y0 + h, x0:x0 + w]   # pitched view
                for pat in (B.NAMES if h * w < 10 ** 5 or i % 4 == 0 else B.NAMES[:1]):
                    assert np.array_equal(B.demosaic(raw, pat), B.cv_demosaic(cv2, raw, pat)), (use, h, w, pat)
            big = rng.integers(0, 256, (1080, 1920), dtype=np.uint8)
            for pat in B.NAMES:
                assert np.array_equal(B.demosaic(big, pat), B.cv_demosaic(cv2, big, pat)), (use, pat)
    finally:
        cv2.ipp.setUseIPP(ipp)


def test_mosaic_helper():
    """mosaic() samples each site's own colour: a demosaic of it keeps every raw value in its own channel."""
    rng = np.random.default_rng(3)
    bgr = rng.integers(0, 256, (7, 9, 3), dtype=np.uint8)
    ch = {"B": 0, "G": 1, "R": 2}
    for pat in B.NAMES:
        m = B.mosaic(bgr, pat)
        for y in range(7):
            for x in range(9):
                assert m[y, x] == bgr[y, x, ch[B.colour_at(pat, y, x)]]
        d = B.demosaic(m, pat)
        for y in range(1, 6):
            for x in range(1, 8):
                c = ch[B.colour_at(pat, y, x)]
                assert d[y, x, c] == m[y, x]


def test_bayer_argument_errors_need_no_gpu():
    """The four codes pass the size-free rules and reach the engine check on both image and both rectified entries;
    plane_pitch != 0 is refused for them; 6, 15 and 20 stay unknown; image_desc("yuv") still raises."""
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    entries = {
        "adc_match_images:": lambda img: L.adc_match_images(None, p, p, img, None, 0, 0, p, None, 0, None, 0),
        "adc_match_images_batch_device": lambda img: L.adc_match_images_batch_device(None, 1, p, p, img, None, 0, 0, p,
                                                                                      None, 0, None, 0, None),
        "adc_match_rectified:": lambda img: L.adc_match_rectified(None, p, p, img, None, 0, 0, p, None, 0, None, 0),
        "adc_match_rectified_batch_device": lambda img: L.adc_match_rectified_batch_device(None, 1, p, p, img, None, 0, 0,
                                                                                           p, None, 0, None, 0, None),
    }
    for fn, call in entries.items():
        for code in B.CODE.values():
            for d in (A.ImageDesc(code, 0, 0, 0, 0), A.ImageDesc(code, 0, 1001, 0, 1 << 33)):
                assert call(ctypes.byref(d)) == 1 and b"engine is NULL" in L.adc_last_error(), (fn, code)
            assert call(ctypes.byref(A.ImageDesc(code, 0, 0, 64, 0))) == 1
            err = L.adc_last_error()
            assert b"img->plane_pitch" in err and fn.encode() in err, err
            assert call(ctypes.byref(A.ImageDesc(code, 1, 0, 0, 0))) == 1 and b"img->reserved" in L.adc_last_error()
        for code in (6, 15, 20, -16):
            assert call(ctypes.byref(A.ImageDesc(code, 0, 0, 0, 0))) == 1
            err = L.adc_last_error()
            assert f"img->format {code} unknown".encode() in err and fn.encode() in err, err
    with pytest.raises(ValueError):
        A.image_desc("yuv")


def test_bayer_constants():
    import adcensus_b200 as A
    assert (A.IMG_BAYER_RGGB, A.IMG_BAYER_GRBG, A.IMG_BAYER_BGGR, A.IMG_BAYER_GBRG) == (16, 17, 18, 19)
    assert A.BAYER_FORMATS == B.CODE
    assert not set(A.BAYER_FORMATS) & set(A.engine.IMG_FORMATS)
    for name, code in B.CODE.items():
        d = A.image_desc(name, 77, 0, 9000)
        assert (d.format, d.row_pitch, d.plane_pitch, d.image_stride) == (code, 77, 0, 9000)
    h = (ROOT / "include" / "adcensus_b200.h").read_text()
    assert "enum { ADC_IMG_BAYER_RGGB = 16, ADC_IMG_BAYER_GRBG = 17, ADC_IMG_BAYER_BGGR = 18, ADC_IMG_BAYER_GBRG = 19 };" in h
    # the numpy view parser takes [H][W] uint8 views of any row pitch, as for gray
    frame = np.zeros((10, 40), np.uint8)
    d = A.engine._image_view_desc(frame[1:9, 3:30], A.IMG_BAYER_GRBG, 8, 27)
    assert (d.format, d.row_pitch, d.plane_pitch) == (A.IMG_BAYER_GRBG, 40, 0)
    with pytest.raises(ValueError):
        A.engine._image_view_desc(np.zeros((8, 27, 3), np.uint8), A.IMG_BAYER_RGGB, 8, 27)


# ---- GPU ------------------------------------------------------------------------------------------
def _mosaic_batch(n, vw, vh, rng, x0, y0, extra_row, extra_stride):
    """n pairs of random mosaics laid out as crops at (x0, y0) of frames with row pitch vw + x0 + extra_row and image
    stride footprint + extra_stride, random surroundings, one device buffer per view with guard bytes after the last
    view.  (views, offset of the first pixel, row pitch, image stride, left mosaics, right mosaics)."""
    torch, dev = E.cuda()
    rp = vw + x0 + extra_row
    stride = (vh + y0) * rp + extra_stride
    off = y0 * rp + x0
    L = [rng.integers(0, 256, (vh, vw), dtype=np.uint8) for _ in range(n)]
    Rr = [rng.integers(0, 256, (vh, vw), dtype=np.uint8) for _ in range(n)]
    views = []
    for imgs in (L, Rr):
        big = rng.integers(0, 256, size=n * stride + 64, dtype=np.uint8)
        for i in range(n):
            big[i * stride + off:i * stride + off + vh * rp].reshape(vh, rp)[:, :vw] = imgs[i]
        views.append(torch.from_numpy(big).to(dev))
    return views, off, rp, stride, L, Rr


def _equal_all(got, want, name):
    for k in want:
        assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), f"{name}: {k}"


@pytest.mark.gpu
def test_bayer_cone_against_oracle(cone):
    """Cone mosaiced with each pattern through adc_match_images_batch_device: the final map equals the CPU oracle run on
    the restated demosaic of the same mosaic, bit for bit."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option())
    oracle = T.Oracle(w, h, T.default_option())
    st = torch.cuda.current_stream()
    for pat in B.NAMES:
        ml, mr = B.mosaic(left, pat), B.mosaic(right, pat)
        d_l, d_r = (torch.from_numpy(np.stack([m, m])).to(dev) for m in (ml, mr))
        d_o = torch.empty((2, h, w), dtype=torch.float32, device=dev)
        eng.match_images_batch_device(2, d_l.data_ptr(), d_r.data_ptr(), image=A.image_desc(pat), d_disp=d_o.data_ptr(),
                                      stream=st.cuda_stream)
        torch.cuda.synchronize()
        want = oracle.match(B.demosaic(ml, pat), B.demosaic(mr, pat))
        got = d_o.cpu().numpy()
        E.same(f"cone {pat} pair 0", got[0], want)
        E.same(f"cone {pat} pair 1", got[1], want)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_bayer_batched(pipelined):
    """wave_pairs = 4, lanes = 3, n = 14 (several waves per lane, a partial last wave), odd W and H, every pattern as a
    crop at even and odd offsets with row pitch > W and image stride > footprint: every output equals
    adc_match_outputs_batch_device on the restated BGR images, and the source buffers are unchanged."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    rng = np.random.default_rng(8)
    for k, pat in enumerate(B.NAMES):
        x0, y0 = ((0, 0), (3, 1), (2, 5), (1, 2))[k]
        views, off, rp, stride, L, Rr = _mosaic_batch(n, w, h, rng, x0, y0, 7 * (k % 2), 5 * (k // 2))
        before = [t.clone() for t in views]
        packed_l = torch.from_numpy(np.stack([B.demosaic(x, pat) for x in L])).to(dev)
        packed_r = torch.from_numpy(np.stack([B.demosaic(x, pat) for x in Rr])).to(dev)
        outputs = dict(volumes=[(v, "hwd", "f32") for v in VOLS], maps=MAPS, pipelined=pipelined)
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, packed_l.data_ptr(), packed_r.data_ptr(),
                               3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_images_batch_device, n, views[0].data_ptr() + off,
                              views[1].data_ptr() + off, stride, image=A.image_desc(pat, rp, 0, stride), **outputs)
        _equal_all(got, want, f"{pat} crop ({x0}, {y0})")
        assert all(torch.equal(t, c) for t, c in zip(views, before)), f"{pat}: source buffer changed"
    eng.close()


@pytest.mark.gpu
def test_bayer_host_entry():
    """The single-pair host entry match_images on pitched numpy crops gives what match_outputs gives on the restated
    images: final map, all three volumes, all five side maps; also for a tight mosaic of an even-sized frame."""
    w, h, D = 61, 45, 20
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    rng = np.random.default_rng(21)
    for pat in B.NAMES:
        frame = [rng.integers(0, 256, (h + 3, w + 8), dtype=np.uint8) for _ in range(2)]
        views = [f[1:1 + h, 3:3 + w] for f in frame]
        want_disp, want = eng.match_outputs(*(B.demosaic(v, pat) for v in views), maps=MAPS, volumes=VOLS)
        disp, got = eng.match_images(views[0], views[1], format=pat, maps=MAPS, volumes=VOLS)
        E.same(f"{pat} host disp", disp, want_disp)
        for k in want:
            E.same(f"{pat} host {k}", got[k], want[k])
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_bayer_rectified(pipelined):
    """Raw mosaics through the rectified entries: both map types (with specials), frames larger and smaller than the
    engine, and 1 x 1 and 2 x N frames (all-zero views), as odd-offset crops with row pitch > W: every output equals
    adc_match_outputs_batch_device on remap(demosaic(raw)); the host entry match_rectified agrees."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=3)
    n = 2 * eng.wave_pairs + 1
    rng = np.random.default_rng(12)
    for k, (sw, sh) in enumerate(((83, 53), (64, 40), (1, 1), (57, 2), (3, 3))):
        pat = B.NAMES[k % 4]
        fixed = k % 2 == 1
        maps = [R.warp_maps(w, h, sw, sh, 40 + 2 * k + v, fixed) for v in range(2)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        views, off, rp, stride, L, Rr = _mosaic_batch(n, sw, sh, rng, 3, 1, 4, 0)
        packed_l = torch.from_numpy(np.stack([R.remap(B.demosaic(x, pat), *maps[0]) for x in L])).to(dev)
        packed_r = torch.from_numpy(np.stack([R.remap(B.demosaic(x, pat), *maps[1]) for x in Rr])).to(dev)
        if min(sw, sh) < 3:
            assert not packed_l.any() and not packed_r.any()
        outputs = dict(volumes=[(v, "hwd", "f32") for v in VOLS], maps=MAPS, pipelined=pipelined)
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, packed_l.data_ptr(), packed_r.data_ptr(),
                               3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_rectified_batch_device, n, views[0].data_ptr() + off,
                              views[1].data_ptr() + off, stride, image=A.image_desc(pat, rp, 0, stride), **outputs)
        _equal_all(got, want, f"{sw}x{sh} {pat} fixed={fixed}")
        if not pipelined:
            disp, one = eng.match_rectified(L[1], Rr[1], format=pat, maps=MAPS)
            E.same(f"{sw}x{sh} {pat} host disp", disp, want["disp"][1])
            for m in MAPS:
                E.same(f"{sw}x{sh} {pat} host {m}", one[m], want[m][1])
    eng.close()


@pytest.mark.gpu
def test_bayer_cone_rig(cone):
    """Cone mosaiced at 640x480 through initUndistortRectifyMap maps of a made-up rig (both map types): the final map
    equals the packed-BGR call on cv2.remap(cv2.cvtColor(raw)), computed by OpenCV itself."""
    cv2 = pytest.importorskip("cv2")
    import adcensus_b200 as A
    torch, dev = E.cuda()
    left, right = cone
    h, w, _ = left.shape
    sw, sh = 640, 480
    raw = [B.mosaic(cv2.resize(img, (sw, sh), interpolation=cv2.INTER_AREA), "bayer_rggb") for img in (left, right)]
    eng = E.engine(w, h, T.default_option())
    st = torch.cuda.current_stream()
    d = [torch.from_numpy(r).to(dev) for r in raw]
    for t in (cv2.CV_32FC1, cv2.CV_16SC2):
        maps = [R.cone_rig(cv2, sw, sh, w, h, t, s) for s in (1, -1)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        rect = [cv2.remap(B.cv_demosaic(cv2, raw[v], "bayer_rggb"), *maps[v], cv2.INTER_LINEAR,
                          borderMode=cv2.BORDER_CONSTANT, borderValue=0) for v in range(2)]
        want = eng.match(rect[0], rect[1])
        d_o = torch.empty((1, h, w), dtype=torch.float32, device=dev)
        eng.match_rectified_batch_device(1, d[0].data_ptr(), d[1].data_ptr(), image=A.image_desc("bayer_rggb"),
                                         d_disp=d_o.data_ptr(), stream=st.cuda_stream)
        torch.cuda.synchronize()
        E.same(f"rig {t}", d_o[0].cpu().numpy(), want)
    eng.close()


@pytest.mark.gpu
def test_bayer_launch_counts():
    """A Bayer call issues exactly one launch per wave more than the tight packed-BGR call of the same batch, through
    both the image and the rectified entry (where a packed-BGR call also takes one ingestion launch per wave); the
    ingestion profile ids replay the Bayer kernels after a Bayer call."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=2)
    n = 3 * eng.wave_pairs + 1
    waves = -(-n // eng.wave_pairs)
    rng = np.random.default_rng(2)
    mos = [torch.from_numpy(rng.integers(0, 256, (n, h, w), dtype=np.uint8)).to(dev) for _ in range(2)]
    bgr = [torch.from_numpy(rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)).to(dev) for _ in range(2)]
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream()

    def count(call, *a, **kw):
        torch.cuda.synchronize()
        c0 = eng.launch_count
        call(*a, d_disp=d_o.data_ptr(), stream=st.cuda_stream, **kw)
        torch.cuda.synchronize()
        return eng.launch_count - c0

    base = count(eng.match_outputs_batch_device, n, bgr[0].data_ptr(), bgr[1].data_ptr())
    for pat in B.NAMES:
        got = count(eng.match_images_batch_device, n, mos[0].data_ptr(), mos[1].data_ptr(), image=A.image_desc(pat))
        assert got == base + waves, (pat, got, base, waves)
    assert eng.profile_kernel("image_ingest", reps=2)[1] == 2 * eng.wave_pairs * (h * w + 3 * h * w)
    m = R.warp_maps(w, h, 90, 60, 3)
    eng.set_rectification(m, m, (90, 60))
    mos = [torch.from_numpy(rng.integers(0, 256, (n, 60, 90), dtype=np.uint8)).to(dev) for _ in range(2)]
    raw = [torch.from_numpy(rng.integers(0, 256, (n, 60, 90, 3), dtype=np.uint8)).to(dev) for _ in range(2)]
    rect_bgr = count(eng.match_rectified_batch_device, n, raw[0].data_ptr(), raw[1].data_ptr())
    assert rect_bgr == base + waves
    for pat in B.NAMES:
        got = count(eng.match_rectified_batch_device, n, mos[0].data_ptr(), mos[1].data_ptr(), image=A.image_desc(pat))
        assert got == base + waves, (pat, got, base, waves)
    ms, by = eng.profile_kernel("rectify", reps=2)
    assert ms > 0 and by == 2 * eng.wave_pairs * (90 * 60 + 3 * h * w) + 2 * 8 * h * w
    eng.close()
