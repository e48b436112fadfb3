"""Rectification on the way in (adc_set_rectification, adc_match_rectified*): raw frames resampled through per-view
remap tables while they are ingested, bit-exact with cv2.remap(INTER_LINEAR, BORDER_CONSTANT, 0) followed by the
packed-BGR entry point.

CPU: the numpy restatement (rectify_testlib) against cv2.remap on random, realistic and degenerate cases for both map
types (skipped without OpenCV) and against the committed fixture (never skipped); the argument rules that need no
engine; the structs' layout and the constants.
GPU: Cone through initUndistortRectifyMap maps of a made-up rig (both map types, sources smaller than, equal to and
larger than W x H, every format tight / pitched / cropped) against the restated images; identity maps against
adc_match_images; batches with several waves per lane, pipelined and not, with guard bytes; image strides past 2^31;
host, pinned and device maps, re-setting between pipelined calls, clearing; one ingestion launch per wave; the host
entry's staging fallback; the rules that need an engine.
"""
import ctypes

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E  # puts tools/ on sys.path
import images_testlib as IT
import rectify_testlib as R

MAPS = ["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"]
GOLDEN = T.GOLDEN_DIR / "golden_remap_cases.npz"


# ---- CPU ------------------------------------------------------------------------------------------
def _cases_from(npz):
    z = np.load(npz)
    for name in sorted({k.split("/")[0] for k in z.files}):
        yield name, z[f"{name}/src"], z[f"{name}/map1"], z[f"{name}/map2"], z[f"{name}/out"]


def test_restatement_against_fixture():
    """The restatement reproduces every cv2.remap output recorded in the fixture (random float and fixed maps with
    specials, initUndistortRectifyMap maps of both types, 1 x 1, 1 x N and N x 1 sources)."""
    seen = set()
    for name, src, m1, m2, out in _cases_from(GOLDEN):
        assert np.array_equal(R.remap(src, m1, m2), out), name
        seen.add(name.split("_")[0])
    assert seen == {"f32", "fixed", "rig", "line"}


def _cv_remap(cv2, src, m1, m2):
    out = cv2.remap(src, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    return out.reshape(np.shape(m2) + src.shape[2:])


def test_restatement_against_opencv():
    """The restatement against cv2.remap: 40 random float cases (1, 3, 4 channels, 5..90 pixels, ties at odd
    multiples of 1/64, NaN, +-inf, +-1e9, 70000, -0.0), 30 random fixed cases (saturated corners, junk high bits),
    initUndistortRectifyMap maps from 450x375, 640x480 and 1280x720 into 450x375 (both types), convertMaps of float maps,
    and 1 x 1, 1 x N, N x 1 sources."""
    cv2 = pytest.importorskip("cv2")
    import make_golden_remap as MG
    rng = np.random.default_rng(11)
    for i in range(40):
        h, w = (int(v) for v in rng.integers(5, 90, 2))
        H, W = (int(v) for v in rng.integers(5, 90, 2))
        src, mx, my = MG.random_f32(rng, h, w, H, W, [1, 3, 4][i % 3])
        want = _cv_remap(cv2, src, mx, my)
        assert np.array_equal(R.remap(src, mx, my), want), f"f32 case {i}"
        m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        assert np.array_equal(_cv_remap(cv2, src, m1, m2), want), f"convertMaps case {i}"
        r1, r2 = R.convert_maps(mx, my)
        assert np.array_equal(r1, m1) and np.array_equal(r2, m2), f"convert_maps case {i}"
    for i in range(30):
        h, w = (int(v) for v in rng.integers(3, 80, 2))
        H, W = (int(v) for v in rng.integers(3, 80, 2))
        src, m1, m2 = MG.random_fixed(rng, h, w, H, W, [1, 3, 4][i % 3])
        assert np.array_equal(R.remap(src, m1, m2), _cv_remap(cv2, src, m1, m2)), f"fixed case {i}"
    for sw, sh in ((450, 375), (640, 480), (1280, 720)):
        src = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        for t in (cv2.CV_32FC1, cv2.CV_16SC2):
            m1, m2 = MG.rig_maps(sw, sh, 450, 375, t)
            assert np.array_equal(R.remap(src, m1, m2), _cv_remap(cv2, src, m1, m2)), (sw, sh, t)
    for h, w in ((1, 1), (1, 17), (13, 1)):
        for c in (1, 3, 4):
            src, mx, my = MG.random_f32(rng, h, w, 7, 9, c)
            assert np.array_equal(R.remap(src, mx, my), _cv_remap(cv2, src, mx, my)), (h, w, c)
            m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
            assert np.array_equal(R.remap(src, m1, m2), _cv_remap(cv2, src, m1, m2)), (h, w, c, "fixed")
    # the builders the GPU tests use stand for what OpenCV does with their maps
    src = rng.integers(0, 256, (53, 83, 3), dtype=np.uint8)
    for fixed in (False, True):
        m1, m2 = R.warp_maps(71, 47, 83, 53, 5, fixed)
        assert np.array_equal(R.remap(src, m1, m2), _cv_remap(cv2, src, m1, m2)), fixed


def _remap_struct(m1=1024, m2=2048, p1=0, p2=0):
    import adcensus_b200 as A
    return A.Remap(m1, m2, p1, p2)


def _rect(sw=64, sh=48, t=0, reserved=0, views=None):
    import adcensus_b200 as A
    views = views or (_remap_struct(), _remap_struct())
    return A.Rectification(sw, sh, t, reserved, (A.Remap * 2)(*views))


def test_rectification_argument_errors_need_no_gpu():
    """Every rule that needs no output size fails with ADC_ERR_ARG naming the field, before the engine is checked; the
    rectified entries check the image entries' rules under their own names."""
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    cases = [
        (_rect(sw=0), b"r->src_width"), (_rect(sw=32768), b"r->src_width"), (_rect(sh=0), b"r->src_height"),
        (_rect(sh=-5), b"r->src_height"), (_rect(t=2), b"r->map_type"), (_rect(reserved=1), b"r->reserved"),
        (_rect(views=(_remap_struct(m1=0), _remap_struct())), b"r->view[0].map1 is NULL"),
        (_rect(views=(_remap_struct(), _remap_struct(m2=0))), b"r->view[1].map2 is NULL"),
        (_rect(views=(_remap_struct(p1=-4), _remap_struct())), b"r->view[0].map1_pitch"),
        (_rect(views=(_remap_struct(), _remap_struct(p2=-8))), b"r->view[1].map2_pitch"),
        (_rect(views=(_remap_struct(m1=1026), _remap_struct())), b"r->view[0].map1"),
        (_rect(views=(_remap_struct(), _remap_struct(p1=6))), b"r->view[1].map1"),
        (_rect(t=1, views=(_remap_struct(m2=1025), _remap_struct())), b"r->view[0].map2"),
        (_rect(t=1, views=(_remap_struct(), _remap_struct(p2=3))), b"r->view[1].map2"),
        (_rect(views=(_remap_struct(p2=2), _remap_struct())), b"r->view[0].map2"),
    ]
    for r, msg in cases:
        assert L.adc_set_rectification(None, ctypes.byref(r)) == 1, msg
        err = L.adc_last_error()
        assert msg in err and b"adc_set_rectification" in err, err
    # valid structs (fixed maps need only 2-byte alignment) and NULL get as far as the engine check
    for r in (None, _rect(), _rect(1, 1), _rect(32767, 32767, 1, views=(_remap_struct(m1=1026, p1=6, m2=1030, p2=2),) * 2)):
        assert L.adc_set_rectification(None, r if r is None else ctypes.byref(r)) == 1
        assert b"engine is NULL" in L.adc_last_error()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    maps1 = (A.engine.MapOut * 1)(A.engine.MapOut(p, A.MAP_PEAK_RATIO, 0))

    def host(img, maps=None, n_maps=0, disp=p, cost=None, cl=0):
        return L.adc_match_rectified(None, p, p, img, cost, cl, 0, disp, None, 0, maps, n_maps)

    def dev(img, maps=None, n_maps=0, disp=p, cost=None, cl=0):
        return L.adc_match_rectified_batch_device(None, 1, p, p, img, cost, cl, 0, disp, None, 0, maps, n_maps, None)

    for call in (host, dev):
        for kw, msg in [(dict(img=A.ImageDesc(6, 0, 0, 0, 0)), b"img->format"),
                        (dict(img=A.ImageDesc(1, 1, 0, 0, 0)), b"img->reserved"),
                        (dict(img=A.ImageDesc(2, 0, 0, 100, 0)), b"img->plane_pitch"),
                        (dict(img=A.ImageDesc(1, 0, -1, 0, 0)), b"img->row_pitch"),
                        (dict(img=None, maps=maps1, n_maps=6), b"n_maps"),
                        (dict(img=None, disp=None), b"no volume or map"),
                        (dict(img=None, cost=p, cl=2), b"cost_layout")]:
            assert call(**kw) == 1, (call.__name__, kw)
            err = L.adc_last_error()
            assert msg in err, err
            assert (b"adc_match_rectified_batch_device" if call is dev else b"adc_match_rectified:") in err, err
        assert call(A.image_desc("gray")) == 1 and b"engine is NULL" in L.adc_last_error()


def test_rectification_constants():
    import adcensus_b200 as A
    assert (A.REMAP_F32, A.REMAP_FIXED) == (0, 1)
    assert ctypes.sizeof(A.Remap) == 32 and ctypes.sizeof(A.Rectification) == 80
    assert [(n, getattr(A.Remap, n).offset) for n, _ in A.Remap._fields_] == [
        ("map1", 0), ("map2", 8), ("map1_pitch", 16), ("map2_pitch", 24)]
    assert [(n, getattr(A.Rectification, n).offset) for n, _ in A.Rectification._fields_] == [
        ("src_width", 0), ("src_height", 4), ("map_type", 8), ("reserved", 12), ("view", 16)]
    assert A.Engine.PROFILE_KERNELS["rectify"] == 14
    h = (T.REPO / "include" / "adcensus_b200.h").read_text()
    assert "enum { ADC_REMAP_F32 = 0, ADC_REMAP_FIXED = 1 };" in h


def test_map_builders_python():
    """The Python map parsing: dtype picks the map type, pitches come from strides, mismatches are refused."""
    from adcensus_b200.engine import _remap
    import adcensus_b200 as A
    mx, my = R.identity_maps(7, 5)
    t, r = _remap((mx, my), 5, 7)
    assert t == A.REMAP_F32 and (r.map1_pitch, r.map2_pitch) == (28, 28)
    big = np.zeros((5, 11, 2), np.int16)
    t, r = _remap((big[:, 2:9], np.zeros((5, 7), np.uint16)), 5, 7)
    assert t == A.REMAP_FIXED and (r.map1_pitch, r.map2_pitch) == (44, 14)
    with pytest.raises(ValueError):
        _remap((mx, my.astype(np.float64)), 5, 7)
    with pytest.raises(ValueError):
        _remap((mx[:, :6], my[:, :6]), 5, 7)
    with pytest.raises(ValueError):
        _remap((mx[:, ::2], my[:, ::2]), 5, 4)


# ---- GPU ------------------------------------------------------------------------------------------
def _frame_view(buf, fmt, h, w, rp, pp, off):
    """numpy view of one raw view in a flat buffer, as Engine.match_rectified takes it."""
    if fmt == "rgb_planar":
        return np.lib.stride_tricks.as_strided(buf[off:], (3, h, w), (pp, rp, 1))
    if fmt == "gray":
        return np.lib.stride_tricks.as_strided(buf[off:], (h, w), (rp, 1))
    C = IT.BPP[fmt]
    return np.lib.stride_tricks.as_strided(buf[off:], (h, w, C), (rp, C, 1))


def _layout(img, fmt, extra_row, lead, extra_plane=0):
    """(flat buffer with 0xEE padding, row pitch, plane pitch, offset) of a tight image in format fmt."""
    if fmt == "rgb_planar":
        _, h, w = img.shape
    else:
        h, w = img.shape[:2]
    rp = w * IT.BPP[fmt] + extra_row
    pp = h * rp + extra_plane if fmt == "rgb_planar" else 0
    buf = np.full(lead + IT.footprint(fmt, h, rp, pp) + 5, 0xEE, np.uint8)
    IT.write_view(buf, img, fmt, rp, pp, lead)
    return buf, rp, pp, lead


def _raw(bgr, fmt):
    """A raw BGR frame as the format stores it; gray frames take channel 1 and stand for (g, g, g)."""
    if fmt == "gray":
        return IT.from_bgr(IT.gray_to_bgr(bgr[:, :, 1]), "gray")
    return IT.from_bgr(bgr, fmt)


def _restated(bgr, fmt, maps):
    """The packed BGR image the rectified entries must match for raw frame bgr in format fmt."""
    src = IT.gray_to_bgr(bgr[:, :, 1]) if fmt == "gray" else bgr
    return R.remap(src, *maps)


@pytest.mark.gpu
@pytest.mark.parametrize("src_size", [(400, 330), (450, 375), (640, 480)])
def test_rectified_cone_rig(src_size, cone):
    """Cone frames resized to the source size, rectified through initUndistortRectifyMap maps of a made-up rig (both
    map types): the final map, the ADC_VOL_COST export and all five side maps equal adc_match_outputs on the restated
    images, through both entry points, for every format tight and pitched (the pitched frames are crops of larger
    ones)."""
    cv2 = pytest.importorskip("cv2")
    import adcensus_b200 as A
    torch, dev = E.cuda()
    left, right = cone
    h, w, _ = left.shape
    sw, sh = src_size
    raw = [cv2.resize(img, (sw, sh), interpolation=cv2.INTER_AREA) for img in (left, right)]
    eng = E.engine(w, h, T.default_option())
    st = torch.cuda.current_stream()
    for t in (cv2.CV_32FC1, cv2.CV_16SC2):
        maps = [R.cone_rig(cv2, sw, sh, w, h, t, s) for s in (1, -1)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        for fmt in IT.FORMATS:
            rect = [_restated(raw[v], fmt, maps[v]) for v in range(2)]
            want_disp, want = eng.match_outputs(rect[0], rect[1], maps=MAPS, volumes=["cost"])
            for extra, lead in ((0, 0), (13, 7)):
                name = f"{sw}x{sh} {t} {fmt} pad {extra}"
                lay = [_layout(_raw(raw[v], fmt), fmt, extra, lead, 3 if extra else 0) for v in range(2)]
                views = [_frame_view(b, fmt, sh, sw, rp, pp, off) for b, rp, pp, off in lay]
                disp, got = eng.match_rectified(views[0], views[1], format=fmt, maps=MAPS, volumes=["cost"])
                E.same(f"{name} host disp", disp, want_disp)
                for k in want:
                    E.same(f"{name} host {k}", got[k], want[k])
                if extra == 0 and fmt not in ("bgra", "gray"):
                    continue
                # device: both views in one buffer, the right one 1 byte after the left one's padding
                _, rp, pp, off = lay[0]
                size = lay[0][0].size
                d = torch.from_numpy(np.concatenate([lay[0][0], np.zeros(1, np.uint8), lay[1][0]])).to(dev)
                out = {m: torch.empty((1, h, w), dtype=torch.uint8 if m == "outliers" else torch.float32, device=dev)
                       for m in MAPS}
                d_disp = torch.empty((1, h, w), dtype=torch.float32, device=dev)
                d_cost = torch.empty((1, h, w, eng.D), dtype=torch.float32, device=dev)
                eng.match_rectified_batch_device(1, d.data_ptr() + off, d.data_ptr() + size + 1 + off,
                                                 image=A.image_desc(fmt, rp, pp, 0),
                                                 maps=[(b.data_ptr(), m) for m, b in out.items()],
                                                 volumes=[(d_cost.data_ptr(), "cost", "hwd", "f32")],
                                                 d_disp=d_disp.data_ptr(), stream=st.cuda_stream)
                torch.cuda.synchronize()
                E.same(f"{name} device disp", d_disp[0].cpu().numpy(), want_disp)
                E.same(f"{name} device cost", d_cost[0].cpu().numpy(), want["cost"])
                for m in MAPS:
                    E.same(f"{name} device {m}", out[m][0].cpu().numpy(), want[m])
    eng.close()


@pytest.mark.gpu
def test_identity_maps_match_images(cone):
    """Identity maps (both types) on a W x H source give exactly adc_match_images' map and cost volume for every
    format."""
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option())
    for fixed in (False, True):
        m = R.identity_maps(w, h, fixed)
        eng.set_rectification(m, m, (w, h))
        for fmt in IT.FORMATS:
            if fmt == "gray":
                l, r = (IT.from_bgr(IT.gray_to_bgr(x[:, :, 1]), "gray") for x in (left, right))
            else:
                l, r = IT.from_bgr(left, fmt), IT.from_bgr(right, fmt)
            want_disp, want = eng.match_images(l, r, format=fmt, volumes=["cost"])
            disp, got = eng.match_rectified(l, r, format=fmt, volumes=["cost"])
            E.same(f"identity {fixed} {fmt} disp", disp, want_disp)
            E.same(f"identity {fixed} {fmt} cost", got["cost"], want["cost"])
    eng.close()


def _raw_batch(fmt, n, sw, sh, rng, x0=5, y0=1):
    """n pairs of random raw frames (packed BGR; gray: (g, g, g)), laid out as odd-x crops of larger frames with
    random surroundings on the device, every view in its own buffer with guard bytes after the last view."""
    torch, dev = E.cuda()
    import adcensus_b200 as A
    L = [rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8) for _ in range(n)]
    Rr = [rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8) for _ in range(n)]
    if fmt == "gray":
        L = [IT.gray_to_bgr(x[:, :, 1]) for x in L]
        Rr = [IT.gray_to_bgr(x[:, :, 1]) for x in Rr]
    bpp, FH, FW = IT.BPP[fmt], sh + 3, sw + 11
    rp = FW * bpp
    pp = FH * rp if fmt == "rgb_planar" else 0
    stride = IT.footprint(fmt, FH, rp, pp)
    off = y0 * rp + x0 * bpp
    views = []
    for imgs in (L, Rr):
        big = rng.integers(0, 256, size=(n * stride + 64), dtype=np.uint8)
        for i in range(n):
            IT.write_view(big[i * stride:], IT.from_bgr(imgs[i], fmt), fmt, rp, pp, off)
        views.append(torch.from_numpy(big).to(dev))
    return views, off, A.image_desc(fmt, rp, pp, stride), stride, L, Rr


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_rectified_batched(pipelined):
    """wave_pairs = 4, lanes = 3, n = 14 (several waves per lane), odd W, sources larger and smaller than W x H, both
    map types with specials (NaN, inf, huge, ties, junk high bits), every format as odd-x crops with guard bytes: every
    output of a call with a cost volume, an exported volume and all five side maps equals the packed-BGR call's on the
    restated images, and the source buffers are unchanged."""
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    rng = np.random.default_rng(4)
    d_cost = torch.from_numpy(rng.random((n, D, h, w), dtype=np.float32) * np.float32(40)).to(dev)
    for k, fmt in enumerate(IT.FORMATS):
        sw, sh = ((83, 53), (64, 40), (71, 47))[k % 3]
        fixed = k % 2 == 1
        maps = [R.warp_maps(w, h, sw, sh, 30 + 2 * k + v, fixed) for v in range(2)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        views, off, desc, stride, L, Rr = _raw_batch(fmt, n, sw, sh, rng)
        before = [t.clone() for t in views]
        packed_l = torch.from_numpy(np.stack([R.remap(x, *maps[0]) for x in L])).to(dev)
        packed_r = torch.from_numpy(np.stack([R.remap(x, *maps[1]) for x in Rr])).to(dev)
        outputs = dict(volumes=[("opt", "dhw", "bf16")], maps=MAPS, d_cost=d_cost, cost_layout="dhw", cost_dtype="f32",
                       pipelined=pipelined)
        want = E.batch_outputs(eng, eng.match_images_batch_device, n, packed_l.data_ptr(), packed_r.data_ptr(), 3 * w * h,
                               **outputs)
        got = E.batch_outputs(eng, eng.match_rectified_batch_device, n, views[0].data_ptr() + off,
                              views[1].data_ptr() + off, stride, image=desc, **outputs)
        for key in want:
            assert np.array_equal(got[key].view(np.uint8), want[key].view(np.uint8)), f"{fmt} fixed={fixed}: {key}"
        assert all(torch.equal(t, c) for t, c in zip(views, before)), f"{fmt}: source buffer changed"
    eng.close()


@pytest.mark.gpu
def test_rectified_stride_past_2_31():
    """n = 2 gray raw pairs with an image stride above 2^31 bytes: the second pair is read from past 2^31."""
    torch, dev = E.cuda()
    import adcensus_b200 as A
    w, h, D = 97, 61, 24
    sw, sh = 120, 77
    rng = np.random.default_rng(9)
    grays = [(rng.integers(0, 256, (sh, sw), dtype=np.uint8), rng.integers(0, 256, (sh, sw), dtype=np.uint8))
             for _ in range(2)]
    stride = (1 << 31) + 4099
    N = sh * sw
    buf = torch.zeros(stride + 2 * N + 1, dtype=torch.uint8, device=dev)
    for i, (gl, gr) in enumerate(grays):
        buf[i * stride:i * stride + N] = torch.from_numpy(gl.reshape(-1)).to(dev)
        buf[i * stride + N + 1:i * stride + 2 * N + 1] = torch.from_numpy(gr.reshape(-1)).to(dev)
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    maps = [R.warp_maps(w, h, sw, sh, 60 + v) for v in range(2)]
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    d_disp = torch.empty((2, h, w), dtype=torch.float32, device=dev)
    eng.match_rectified_batch_device(2, buf.data_ptr(), buf.data_ptr() + N + 1, image=A.image_desc("gray", 0, 0, stride),
                                     d_disp=d_disp.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for i, (gl, gr) in enumerate(grays):
        want = eng.match(R.remap(IT.gray_to_bgr(gl), *maps[0]), R.remap(IT.gray_to_bgr(gr), *maps[1]))
        E.same(f"pair {i}", d_disp[i].cpu().numpy(), want)
    del buf
    eng.close()


@pytest.mark.gpu
def test_map_sources_and_updates():
    """Maps from pageable host memory, pinned host memory and (pitched) device memory give the same result; maps
    re-set between pipelined calls apply to the calls made after them only; clearing the maps makes the rectified
    entries fail with ADC_ERR_ARG; the rectified batch issues exactly one ingestion launch per wave more than the
    packed-BGR batch."""
    torch, dev = E.cuda()
    import adcensus_b200 as A
    w, h, D = 64, 40, 16
    sw, sh = 90, 58
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=3, lanes=2)
    rng = np.random.default_rng(12)
    n = 7
    waves = -(-n // eng.wave_pairs)
    views, off, desc, stride, L, Rr = _raw_batch("bgr", n, sw, sh, rng)
    st = torch.cuda.current_stream()

    def run(image=desc, pipelined=False):
        d = torch.empty((n, h, w), dtype=torch.float32, device=dev)
        eng.set_pipelined(pipelined)
        eng.match_rectified_batch_device(n, views[0].data_ptr() + off, views[1].data_ptr() + off, image=image,
                                         d_disp=d.data_ptr(), stream=st.cuda_stream)
        return d

    def want(maps):
        pl = torch.from_numpy(np.stack([R.remap(x, *maps[0]) for x in L])).to(dev)
        pr = torch.from_numpy(np.stack([R.remap(x, *maps[1]) for x in Rr])).to(dev)
        d = torch.empty((n, h, w), dtype=torch.float32, device=dev)
        eng.match_batch_device(n, pl.data_ptr(), pr.data_ptr(), d.data_ptr(), st.cuda_stream)
        torch.cuda.synchronize()
        return d.cpu().numpy()

    for fixed in (False, True):
        maps = [R.warp_maps(w, h, sw, sh, 80 + v + 2 * fixed, fixed) for v in range(2)]
        ref = want(maps)
        # pageable host
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        E.same(f"host maps {fixed}", run().cpu().numpy(), ref)
        # pinned host: the same bytes in adc_host_alloc memory
        pinned = []
        for mv in maps:
            pair = []
            for a in mv:
                p = eng._L.adc_host_alloc(a.nbytes)
                assert p
                ctypes.memmove(p, a.ctypes.data, a.nbytes)
                pair.append((p, np.ctypeslib.as_array((ctypes.c_uint8 * a.nbytes).from_address(p)).view(a.dtype).reshape(a.shape)))
            pinned.append(pair)
        eng.set_rectification(tuple(x for _, x in pinned[0]), tuple(x for _, x in pinned[1]), (sw, sh))
        for pair in pinned:
            for p, _ in pair:
                eng._L.adc_host_free(p)   # the engine holds its own copy
        E.same(f"pinned maps {fixed}", run().cpu().numpy(), ref)
        # device, pitched: the maps sit in wider tensors
        dmaps = []
        for mv in maps:
            pair = []
            for a in mv:
                big = torch.zeros((h, w + 5) + a.shape[2:], dtype=torch.int16 if a.dtype == np.uint16 else torch.from_numpy(a).dtype,
                                  device=dev)
                big[:, 3:3 + w] = torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).to(dev)
                pair.append(big[:, 3:3 + w])
            dmaps.append(tuple(pair))
        eng.set_rectification(dmaps[0], dmaps[1], (sw, sh))
        del dmaps
        torch.cuda.synchronize()
        E.same(f"device maps {fixed}", run().cpu().numpy(), ref)
    # re-setting between pipelined calls: each call uses the maps set when it was made
    m1 = [R.warp_maps(w, h, sw, sh, 90 + v) for v in range(2)]
    m2 = [R.warp_maps(w, h, sw, sh, 95 + v, True) for v in range(2)]
    w1, w2 = want(m1), want(m2)
    eng.set_rectification(m1[0], m1[1], (sw, sh))
    c0 = eng.launch_count
    a = run(pipelined=True)
    launches_rect = eng.launch_count - c0
    eng.set_rectification(m2[0], m2[1], (sw, sh))
    b = run(pipelined=True)
    eng.join(st.cuda_stream)
    torch.cuda.synchronize()
    eng.set_pipelined(False)
    E.same("pipelined call with the first maps", a.cpu().numpy(), w1)
    E.same("pipelined call with the second maps", b.cpu().numpy(), w2)
    # one ingestion launch per wave on top of the packed-BGR batch's launches
    pl = torch.from_numpy(np.stack(L)[:, :h, :w].copy()).to(dev)
    d = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    c0 = eng.launch_count
    eng.match_batch_device(n, pl.data_ptr(), pl.data_ptr(), d.data_ptr(), st.cuda_stream)
    torch.cuda.synchronize()
    assert launches_rect == eng.launch_count - c0 + waves
    # clearing
    eng.set_rectification(None)
    c0 = eng.launch_count
    with pytest.raises(A.AdcError, match="no rectification"):
        run()
    with pytest.raises(A.AdcError, match="no rectification"):
        eng.match_rectified(L[0], Rr[0])
    host = np.zeros(1 << 16, np.uint8)
    disp = np.zeros((h, w), np.float32)
    assert eng._L.adc_match_rectified(eng._h, host.ctypes.data, host.ctypes.data, None, None, 0, 0, disp.ctypes.data,
                                      None, 0, None, 0) == 1
    assert b"no rectification" in eng._L.adc_last_error()
    assert eng.launch_count == c0
    eng.close()


@pytest.mark.gpu
def test_host_entry_staging_fallback():
    """The host entry runs for raw frames that fit in the lane volume and for frames far larger than it (device
    staging), for every format, and equals the packed-BGR call on the restated images."""
    w, h, D = 24, 16, 4
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=1, lanes=1)
    vol_bytes = w * h * 4 * 4
    rng = np.random.default_rng(21)
    for sw, sh in ((20, 12), (300, 200)):
        maps = [R.warp_maps(w, h, sw, sh, 40 + v, sw > 100) for v in range(2)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        for fmt in IT.FORMATS:
            raw = [rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8) for _ in range(2)]
            frames = [_raw(x, fmt) for x in raw]
            assert (2 * frames[0].nbytes > vol_bytes) == (sw > 100), (sw, fmt)
            rect = [_restated(raw[v], fmt, maps[v]) for v in range(2)]
            want_disp, want = eng.match_outputs(rect[0], rect[1], maps=["peak_ratio"], volumes=["cost"])
            disp, got = eng.match_rectified(frames[0], frames[1], format=fmt, maps=["peak_ratio"], volumes=["cost"])
            E.same(f"{sw}x{sh} {fmt} disp", disp, want_disp)
            E.same(f"{sw}x{sh} {fmt} cost", got["cost"], want["cost"])
            E.same(f"{sw}x{sh} {fmt} peak ratio", got["peak_ratio"], want["peak_ratio"])
    eng.close()


@pytest.mark.gpu
def test_rules_that_need_an_engine():
    """Map pitches shorter than a row, and image descriptors checked against the raw frame size (not W x H), fail with
    ADC_ERR_ARG naming the field, before any device work."""
    torch, dev = E.cuda()
    import adcensus_b200 as A
    w, h, D = 33, 20, 16
    sw, sh = 50, 30
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    L = A.load_library()
    mx, my = R.identity_maps(w, h)
    m1, m2 = R.identity_maps(w, h, True)
    for r, msg in [(_rect(sw, sh, 0, views=(_remap_struct(mx.ctypes.data, my.ctypes.data, 4 * w - 4), _remap_struct(mx.ctypes.data, my.ctypes.data))), b"r->view[0].map1_pitch"),
                   (_rect(sw, sh, 1, views=(_remap_struct(m1.ctypes.data, m2.ctypes.data), _remap_struct(m1.ctypes.data, m2.ctypes.data, 0, 2 * w - 2))), b"r->view[1].map2_pitch"),
                   (_rect(sw, sh, 0, views=(_remap_struct(mx.ctypes.data, my.ctypes.data, 1 << 62), _remap_struct(mx.ctypes.data, my.ctypes.data))), b"r->view[0].map1_pitch")]:
        assert L.adc_set_rectification(eng._h, ctypes.byref(r)) == 1 and msg in L.adc_last_error(), L.adc_last_error()
    eng.set_rectification((mx, my), (mx, my), (sw, sh))
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device=dev)
    out = torch.zeros((1, h, w), dtype=torch.float32, device=dev)
    p = buf.data_ptr()
    cases = [(A.ImageDesc(A.IMG_RGB, 0, 3 * sw - 1, 0, 0), b"img->row_pitch"),
             (A.ImageDesc(A.IMG_GRAY, 0, sw - 1, 0, 0), b"img->row_pitch"),
             (A.ImageDesc(A.IMG_RGB_PLANAR, 0, sw + 2, sh * (sw + 2) - 1, 0), b"img->plane_pitch"),
             (A.ImageDesc(A.IMG_GRAY, 0, 0, 0, sh * sw - 1), b"img->image_stride"),
             (A.ImageDesc(A.IMG_BGR, 0, 3 * w, 0, 0), b"img->row_pitch")]   # W x H would pass
    for img, msg in cases:
        c0 = eng.launch_count
        rc = L.adc_match_rectified_batch_device(eng._h, 1, p, p, ctypes.byref(img), None, 0, 0, out.data_ptr(), None, 0,
                                                None, 0, None)
        assert rc == 1 and msg in L.adc_last_error(), (img.format, L.adc_last_error())
        host = np.zeros(1 << 16, np.uint8)
        disp = np.zeros((h, w), np.float32)
        rc = L.adc_match_rectified(eng._h, host.ctypes.data, host.ctypes.data, ctypes.byref(img), None, 0, 0,
                                   disp.ctypes.data, None, 0, None, 0)
        assert rc == 1 and msg in L.adc_last_error(), (img.format, L.adc_last_error())
        assert eng.launch_count == c0
    # the raw frame size, not W x H, is what a tight descriptor resolves to: a tight gray frame of sw x sh runs
    frame = np.random.default_rng(1).integers(0, 256, (sh, sw), dtype=np.uint8)
    disp, _ = eng.match_rectified(frame, frame, format="gray")
    want = eng.match(R.remap(IT.gray_to_bgr(frame), mx, my), R.remap(IT.gray_to_bgr(frame), mx, my))
    E.same("tight gray raw frame", disp, want)
    eng.close()
