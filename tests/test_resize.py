"""Resizing on the way in (adc_set_rectification with ADC_RESIZE_AREA / ADC_RESIZE_LINEAR_EXACT): raw frames of another
size than the engine's, converted with their format's rule and resized as cv::resize does, then matched as packed BGR.

CPU: the numpy restatement (resize_testlib) against live cv2.resize (every AREA factor 1..10 x 1..10 and the largest
accepted, every accepted 1-D AREA factor 1..4096 on half-way samples, every 1-D LINEAR_EXACT size pair 1..512, random 2-D sizes, the BASELINE shapes, 1 / 3 / 4 channels) and
against the committed fixture; the argument rules that need no engine; the header's and the binding's constants.
GPU: Cone through the full pipeline from larger and smaller frames against the packed-BGR call on the restated
images; adc_ingest_views_batch_device for every ADC_IMG_* code and encoding under both rules (tight, pitched,
side-by-side, odd sizes, one-pixel-wide and -high sources, other bytes of the buffer changed); batched device and host
entries, pipelined and not, the host staging fallback, a poisoned engine, geometries switched between pipelined calls;
the rules that need an engine; profile id 14.
"""
import ctypes

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E
import rectify_testlib as R
import resize_testlib as RS

ROOT = T.REPO
MAPS = ["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"]
VOLS = ["cost", "aggr", "opt"]
GOLDEN = T.GOLDEN_DIR / "golden_resize_cases.npz"
INTERPS = {"area": RS.AREA, "linear_exact": RS.LINEAR_EXACT}
# every code a kernel is instantiated for: each format, and each YUV container with each encoding flag
CODES = [(f, 0) for f in RS.CODE] + [(f, e) for f in RS.V.ALL for e in RS.ENC.values() if e]


# ---- CPU ------------------------------------------------------------------------------------------
def test_restatement_against_fixture():
    """The restatement reproduces every cv2.resize output in the committed fixture."""
    z = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in z.files})
    assert len(names) >= 60
    for name in names:
        src, t = z[f"{name}/src"], int(z[f"{name}/interp"])
        W, H = (int(v) for v in z[f"{name}/size"])
        assert np.array_equal(RS.resize(src, W, H, t), z[f"{name}/out"]), name


def _channels(rng, shape, c):
    return rng.integers(0, 256, shape + ((c,) if c > 1 else ()), dtype=np.uint8)


def test_area_against_opencv():
    """INTER_AREA at every factor kx, ky in 1..10 and at the largest accepted (64 x 64, 4096 x 1, 1 x 4096), on 1, 3
    and 4 channels, with uniform samples and with samples of 127 / 128 only (sums at the rounding points)."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    factors = [(kx, ky) for kx in range(1, 11) for ky in range(1, 11)] + [(64, 64), (4096, 1), (1, 4096)]
    for kx, ky in factors:
        W, H = (1, 1) if kx * ky >= 4096 else (9, 7)
        for c in (1, 3, 4):
            for half_way in (False, True):
                src = _channels(rng, (H * ky, W * kx), c)
                if half_way:
                    src = (127 + (src & 1)).astype(np.uint8)
                want = cv2.resize(src, (W, H), interpolation=cv2.INTER_AREA).reshape((H, W) + src.shape[2:])
                assert np.array_equal(RS.area(src, kx, ky), want), (kx, ky, c, half_way)


def test_area_every_accepted_factor_against_opencv():
    """Every 1-D factor 1..4096 that the engine accepts (area_exact), along x and along y, on 1 and 3 channels, against
    cv2.resize: three output pixels, one block of 128s then 127s (its mean at or next to a half-way point), one of
    random 127s and 128s, one of uniform samples.  The rule does not depend on the output size; and for the rejected
    factors (640 of 4096), where OpenCV takes its general area path, the rule disagrees with cv2 on most."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for W in (1, 7, 450, 640):
        assert all(RS.area_exact(k, W) == RS.area_exact(k) for k in range(1, 32767 // W + 1)), W
    rejected = [k for k in range(1, 4097) if not RS.area_exact(k)]
    assert len(rejected) == 640 and rejected[:6] == [49, 93, 98, 99, 103, 105]
    differs = 0
    for k in range(1, 4097):
        for c in (1, 3):
            half = np.where(np.arange(k) < k // 2, 128, 127).astype(np.uint8)
            mixed = (127 + rng.integers(0, 2, k)).astype(np.uint8)
            line = np.concatenate([half, mixed, rng.integers(0, 256, k, dtype=np.uint8)])
            line = np.repeat(line[:, None], c, 1) if c > 1 else line
            for src, W, H, kx, ky in ((line[None], 3, 1, k, 1), (line[:, None], 1, 3, 1, k)):
                want = cv2.resize(src, (W, H), interpolation=cv2.INTER_AREA).reshape((H, W) + src.shape[2:])
                same = np.array_equal(RS.area(src, kx, ky), want)
                if RS.area_exact(k):
                    assert same, (k, c, kx, ky)
                else:
                    differs += not same
    assert differs > len(rejected), differs


def test_linear_exact_against_opencv():
    """INTER_LINEAR_EXACT for every 1-D size pair (n_src, n_dst) in 1..512 along x and a sample of them along y, 200
    random 2-D sizes 1..200 up and down on 1, 3 and 4 channels, and the BASELINE shapes (1080p, 900 x 750 and 320 x 240
    to 450 x 375, 640 x 480 to 1242 x 375, 450 x 375 to 1920 x 1080, 3000 x 17 to 1 x 1)."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(4)
    n = 512
    rows = rng.integers(0, 256, (2, n), dtype=np.uint8)
    for ns in range(1, n + 1):
        src = rows[:, :ns]
        for nd in range(1, n + 1):
            got = RS.linear_exact(src, nd, 2)
            assert np.array_equal(got, cv2.resize(src, (nd, 2), interpolation=cv2.INTER_LINEAR_EXACT)), (ns, nd)
    col = rng.integers(0, 256, (n, 1), dtype=np.uint8)
    for ns in range(1, n + 1, 7):
        for nd in range(1, n + 1, 5):
            got = RS.linear_exact(col[:ns], 1, nd)
            assert np.array_equal(got, cv2.resize(col[:ns], (1, nd), interpolation=cv2.INTER_LINEAR_EXACT)), (ns, nd)
    cases = [tuple(int(v) for v in rng.integers(1, 201, 4)) for _ in range(200)]
    cases += [(1920, 1080, 450, 375), (900, 750, 450, 375), (320, 240, 450, 375), (640, 480, 1242, 375),
              (450, 375, 1920, 1080), (3000, 17, 1, 1), (1, 1, 7, 5), (1, 9, 4, 3), (9, 1, 3, 4)]
    for k, (sw, sh, W, H) in enumerate(cases):
        c = (1, 3, 4)[k % 3]
        src = _channels(rng, (sh, sw), c)
        want = cv2.resize(src, (W, H), interpolation=cv2.INTER_LINEAR_EXACT).reshape((H, W) + src.shape[2:])
        assert np.array_equal(RS.linear_exact(src, W, H), want), (sw, sh, W, H, c)


def test_linear_exact_taps():
    """Both borders replicate: every index lies in the frame, c1 is 0 wherever the tap is clamped, and the weights
    sum to 256."""
    for ns, nd in ((1, 9), (5, 17), (17, 5), (1080, 375), (375, 1080), (32767, 1)):
        i0, i1, c1 = RS.taps(ns, nd)
        assert i0.min() >= 0 and i1.max() <= ns - 1 and ((c1 >= 0) & (c1 <= 256)).all()
        assert (c1[i0 == i1] == 0).all()


def _rect(sw, sh, t, views=None, reserved=0):
    import adcensus_b200 as A
    return A.Rectification(sw, sh, t, reserved, (A.Remap * 2)(*(views or (A.Remap(), A.Remap()))))


def test_resize_argument_errors_need_no_gpu():
    """A resize with any map pointer or pitch fails with ADC_ERR_ARG naming the field before the engine is checked;
    the size range and reserved rules apply as for maps; 2..15 and 18 are unknown; valid resizes reach the engine
    check."""
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    for t in (RS.AREA, RS.LINEAR_EXACT):
        for v in (0, 1):
            for field, remap in (("map1", A.Remap(1024, 0, 0, 0)), ("map2", A.Remap(0, 2048, 0, 0)),
                                 ("map1_pitch", A.Remap(0, 0, 64, 0)), ("map2_pitch", A.Remap(0, 0, 0, 64))):
                views = [A.Remap(), A.Remap()]
                views[v] = remap
                assert L.adc_set_rectification(None, ctypes.byref(_rect(64, 48, t, views))) == 1
                err = L.adc_last_error()
                assert f"r->view[{v}].{field} must be".encode() in err and b"adc_set_rectification" in err, err
        for r, msg in ((_rect(0, 48, t), b"r->src_width"), (_rect(32768, 48, t), b"r->src_width"),
                       (_rect(64, 0, t), b"r->src_height"), (_rect(64, 48, t, reserved=1), b"r->reserved")):
            assert L.adc_set_rectification(None, ctypes.byref(r)) == 1 and msg in L.adc_last_error()
        for sw, sh in ((64, 48), (1, 1), (32767, 32767), (7, 3)):
            assert L.adc_set_rectification(None, ctypes.byref(_rect(sw, sh, t))) == 1
            assert b"engine is NULL" in L.adc_last_error()
    for t in (2, 3, 15, 18, -1, 1 << 20):
        assert L.adc_set_rectification(None, ctypes.byref(_rect(64, 48, t))) == 1
        assert f"r->map_type {t} unknown".encode() in L.adc_last_error()


def test_resize_constants():
    """The header's enum line, the binding's names and the unchanged struct layout."""
    import adcensus_b200 as A
    h = (ROOT / "include" / "adcensus_b200.h").read_text()
    assert "enum { ADC_RESIZE_AREA = 16, ADC_RESIZE_LINEAR_EXACT = 17 };" in h
    assert "enum { ADC_REMAP_F32 = 0, ADC_REMAP_FIXED = 1 };" in h
    assert (A.RESIZE_AREA, A.RESIZE_LINEAR_EXACT) == (RS.AREA, RS.LINEAR_EXACT) == (16, 17)
    assert A.RESIZE_INTERPOLATIONS == INTERPS
    assert ctypes.sizeof(A.Rectification) == 80 and A.Rectification.map_type.offset == 8
    r = A.Rectification(900, 750, A.RESIZE_AREA, 0)
    assert (r.view[0].map1, r.view[1].map2, r.view[0].map1_pitch) == (None, None, 0)


# ---- GPU ------------------------------------------------------------------------------------------
def _dev(a):
    torch, dev = E.cuda()
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _bgr_source(rng, base, sw, sh):
    """A plausible sw x sh BGR frame of the scene in `base`: base scaled by the restated LINEAR_EXACT rule, plus
    noise in the low bits."""
    big = RS.linear_exact(base, sw, sh).astype(np.int16) + rng.integers(-2, 3, (sh, sw, 3))
    return np.clip(big, 0, 255).astype(np.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("src_size,interp", [((900, 750), "area"), ((1350, 1125), "area"), ((900, 375), "area"),
                                             ((1920, 1080), "linear_exact"), ((320, 240), "linear_exact")])
def test_resize_cone(src_size, interp, cone):
    """Cone (450 x 375, 64 disparities) from frames 2x, 3x and 2 x 1 its size (AREA) and from 1920 x 1080 and 320 x 240
    (LINEAR_EXACT), three pairs a batch: the final map, the cost volume and all five side maps equal the packed-BGR
    call on the restated images, through the device and the host entries."""
    import adcensus_b200 as A
    left, right = cone
    H, W = left.shape[:2]
    sw, sh = src_size
    rng = np.random.default_rng(sw + sh)
    eng = E.engine(W, H, T.default_option(max_disparity=64), wave_pairs=2)
    eng.set_resize(src_size, interp)
    n = 3
    raw = [np.stack([_bgr_source(rng, img, sw, sh) for _ in range(n)]) for img in (left, right)]
    small = [np.stack([RS.resize(f, W, H, INTERPS[interp]) for f in r]) for r in raw]
    pl, pr = _dev(small[0]), _dev(small[1])
    outputs = dict(volumes=[("cost", "hwd", "f32")], maps=MAPS)
    want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * W * H, **outputs)
    rl, rr = _dev(raw[0]), _dev(raw[1])
    got = E.batch_outputs(eng, eng.match_rectified_batch_device, n, rl.data_ptr(), rr.data_ptr(), 3 * sw * sh,
                          image=A.image_desc("bgr"), **outputs)
    for k in want:
        E.same(f"{sw}x{sh} {interp} {k}", got[k], want[k])
    disp, one = eng.match_rectified(raw[0][1], raw[1][1], maps=MAPS, volumes=["cost"])
    E.same(f"{sw}x{sh} {interp} host disp", disp, want["disp"][1])
    for k in MAPS + ["cost"]:
        E.same(f"{sw}x{sh} {interp} host {k}", one[k], want[k][1])
    eng.close()


def _word(fmt):
    """Formats whose device views need even pointers and pitches (16-bit samples), or an even row pitch (I420 / YV12)."""
    return fmt == "p016" or (fmt in RS.RD.CODE and not fmt.endswith("p")) or fmt in ("i420", "yv12")


def _layout(fmt, sw, sh, n, k, fill, frames_l, frames_r):
    """Two flat buffers (left, right) of `fill` bytes holding n views each, laid per case k: 0 tight, 1 pitched with an
    image stride above the footprint and an odd (even for 16-bit formats) lead, 2 side by side (right view of pair i
    in the left buffer, one row pitch holding both) for formats with one plane.  (buffers, left offset, right offset,
    desc args)."""
    ev = 2 if _word(fmt) else 1
    tight = RS.tight_row(fmt, sw)
    sbs = k == 2 and not RS.planes(fmt)
    rp = 2 * tight + ev * 4 if sbs else tight + (ev * 3 if k else 0)
    pp = sh * rp + (ev * 5 if k else 0) if RS.planes(fmt) else 0
    foot = RS.footprint(fmt, sh, rp, pp)
    stride = foot + (ev * 7 if k else 0)
    lead = ev if k else 0
    right_off = lead + tight + ev * 2 if sbs else lead
    bufs = [np.full(lead + n * stride + 32, fill, np.uint8) for _ in range(2)]
    for i in range(n):
        RS.write_view(bufs[0], frames_l[i], fmt, sw, sh, rp, pp, lead + i * stride)
        RS.write_view(bufs[0] if sbs else bufs[1], frames_r[i], fmt, sw, sh, rp, pp, right_off + i * stride)
    return bufs, lead, right_off, (rp, pp, stride), sbs


@pytest.mark.gpu
@pytest.mark.parametrize("interp", ["area", "linear_exact"])
def test_ingest_views_every_code(interp):
    """adc_ingest_views_batch_device(rectified = 1) under a resize, for every ADC_IMG_* code and YUV encoding, 3 pairs:
    the views are byte-equal to the restated conversion followed by the restated resize.  Layouts cycle through tight,
    pitched and side-by-side; sources cycle through sizes (AREA 2 x 2, 3 x 1, 1 x 3, 4 x 4 of a 23 x 17 engine;
    LINEAR_EXACT larger, smaller, odd, one pixel wide and one pixel high); every buffer is filled with 0xEE around the
    views, and filling it with 0x11 instead changes nothing."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h = 23, 17
    eng = E.engine(w, h, T.default_option(max_disparity=8), wave_pairs=2)
    t = INTERPS[interp]
    sizes = [(46, 34), (69, 17), (23, 51), (92, 68)] if t == RS.AREA else \
        [(61, 45), (13, 9), (1, 30), (40, 1), (300, 11), (23, 17), (1, 1)]
    n = 3
    rng = np.random.default_rng(t)
    for k, (fmt, enc) in enumerate(CODES):
        sw, sh = sizes[k % len(sizes)]
        eng.set_resize((sw, sh), interp)
        L = [RS.random_frame(rng, fmt, sw, sh) for _ in range(n)]
        Rr = [RS.random_frame(rng, fmt, sw, sh) for _ in range(n)]
        want = np.stack([np.stack([RS.resize(RS.decode(f, fmt, sw, sh, enc), w, h, t) for f in fr]) for fr in (L, Rr)], 1)
        results = []
        for fill in (0xEE, 0x11):
            bufs, lo, ro, (rp, pp, stride), sbs = _layout(fmt, sw, sh, n, k % 3, fill, L, Rr)
            d = [_dev(b) for b in bufs]
            out = torch.full((n, 2, h, w, 3), 7, dtype=torch.uint8, device=dev)
            eng.ingest_views_batch_device(n, d[0].data_ptr() + lo, (d[0] if sbs else d[1]).data_ptr() + ro,
                                          out.data_ptr(), image=A.image_desc(RS.CODE[fmt] | enc, rp, pp, stride),
                                          rectified=True, stream=torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            results.append(out.cpu().numpy())
        name = f"{fmt}|{enc:#x} {sw}x{sh} layout {k % 3}"
        assert np.array_equal(results[0], want), name
        assert np.array_equal(results[1], want), name + " other bytes changed"
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_resize_batched(pipelined):
    """wave_pairs = 3, lanes = 2, n = 7 (several waves, a partial last one): packed BGR (AREA 2 x 2), NV12 BT.709
    (LINEAR_EXACT down), BayerRG12p (AREA 3 x 2) and RGBA (LINEAR_EXACT up) through match_rectified_batch_device give
    every output of match_outputs_batch_device on the restated views; the host entry agrees on one pair."""
    import adcensus_b200 as A
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=3, lanes=2)
    n = 7
    rng = np.random.default_rng(30 + pipelined)
    outputs = dict(volumes=[(v, "hwd", "f32") for v in VOLS], maps=MAPS, pipelined=pipelined)
    for fmt, enc, interp, (sw, sh) in (("bgr", 0, "area", (142, 94)), ("nv12", RS.V.BT709, "linear_exact", (160, 90)),
                                       ("bayer_rg12p", 0, "area", (213, 94)), ("rgba", 0, "linear_exact", (50, 30))):
        eng.set_resize((sw, sh), interp)
        L = [RS.random_frame(rng, fmt, sw, sh) for _ in range(n)]
        Rr = [RS.random_frame(rng, fmt, sw, sh) for _ in range(n)]
        pl, pr = (_dev(np.stack([RS.resize(RS.decode(f, fmt, sw, sh, enc), w, h, INTERPS[interp]) for f in fr]))
                  for fr in (L, Rr))
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h,
                               **outputs)
        bufs, lo, ro, (rp, pp, stride), _ = _layout(fmt, sw, sh, n, 1, 0xEE, L, Rr)
        d = [_dev(b) for b in bufs]
        got = E.batch_outputs(eng, eng.match_rectified_batch_device, n, d[0].data_ptr() + lo, d[1].data_ptr() + ro,
                              stride, image=A.image_desc(RS.CODE[fmt] | enc, rp, pp, stride), **outputs)
        for key in want:
            E.same(f"{fmt} {interp} {key}", got[key], want[key])
        if not pipelined:
            disp, one = eng.match_rectified(L[4], Rr[4], format=RS.CODE[fmt] | enc, maps=MAPS)
            E.same(f"{fmt} {interp} host disp", disp, want["disp"][4])
            for m in MAPS:
                E.same(f"{fmt} {interp} host {m}", one[m], want[m][4])
    eng.close()


@pytest.mark.gpu
def test_resize_host_staging_and_poison():
    """The host entry runs for raw frames that fit in the lane volume and for frames far larger (device staging), on a
    plain engine and on one with ADC_DBG_POISON, and equals the packed-BGR call on the restated images."""
    import adcensus_b200 as A
    w, h, D = 24, 16, 4
    rng = np.random.default_rng(44)
    vol_bytes = w * h * 4 * 4
    for flags in (0, A.engine.poison_flags(0x5A)):
        eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=1, lanes=1, debug_flags=flags)
        for fmt, interp, (sw, sh) in (("bgr", "area", (48, 16)), ("gray", "linear_exact", (30, 20)),
                                      ("bgra", "area", (240, 160)), ("p016", "linear_exact", (400, 300)),
                                      ("bayer_gr10", "area", (72, 48))):
            eng.set_resize((sw, sh), interp)
            frames = [RS.random_frame(rng, fmt, sw, sh) for _ in range(2)]
            fits = 2 * frames[0].nbytes <= vol_bytes
            assert fits == (sw * sh < 1000), (fmt, sw, sh)
            small = [RS.resize(RS.decode(f, fmt, sw, sh), w, h, INTERPS[interp]) for f in frames]
            want_disp, want = eng.match_outputs(small[0], small[1], maps=["peak_ratio"], volumes=["cost"])
            assert np.array_equal(eng.ingest_views(frames[0], frames[1], format=fmt, rectified=True), np.stack(small))
            disp, got = eng.match_rectified(frames[0], frames[1], format=fmt, maps=["peak_ratio"], volumes=["cost"])
            name = f"flags {flags:#x} {fmt} {sw}x{sh}"
            E.same(f"{name} disp", disp, want_disp)
            E.same(f"{name} cost", got["cost"], want["cost"])
            E.same(f"{name} peak ratio", got["peak_ratio"], want["peak_ratio"])
        eng.close()


@pytest.mark.gpu
def test_geometry_switches_between_pipelined_calls():
    """In pipelined mode, with no join in between: a call under an AREA resize, one under remap maps, one under a
    LINEAR_EXACT resize and one under the AREA resize again (each geometry set between the calls) each give what the
    geometry set when it was made gives."""
    torch, dev = E.cuda()
    w, h, D = 40, 30, 12
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=2, lanes=2)
    rng = np.random.default_rng(9)
    n = 3
    sw, sh = 80, 60
    raw = [np.stack([RS.random_frame(rng, "bgr", sw, sh) for _ in range(n)]) for _ in range(2)]
    maps = [R.warp_maps(w, h, sw, sh, 90 + v) for v in range(2)]
    geoms = [("area", None), ("maps", maps), ("linear_exact", None), ("area", None)]

    def restated(kind, m):
        if kind == "maps":
            return [np.stack([R.remap(f, *m[v]) for f in raw[v]]) for v in range(2)]
        return [np.stack([RS.resize(f, w, h, INTERPS[kind]) for f in raw[v]]) for v in range(2)]

    wants = []
    for kind, m in geoms:
        pl, pr = (_dev(x) for x in restated(kind, m))
        wants.append(E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h,
                                     maps=["wta_left"]))
    rl, rr = _dev(raw[0]), _dev(raw[1])
    st = torch.cuda.current_stream().cuda_stream
    outs = [(torch.full((n, h, w), -7.0, device=dev), torch.full((n, h, w), -7.0, device=dev)) for _ in geoms]
    eng.set_pipelined(True)
    for (kind, m), (disp, wl) in zip(geoms, outs):
        if kind == "maps":
            eng.set_rectification(m[0], m[1], (sw, sh))
        else:
            eng.set_resize((sw, sh), kind)
        eng.match_rectified_batch_device(n, rl.data_ptr(), rr.data_ptr(), maps=[(wl.data_ptr(), "wta_left")],
                                         d_disp=disp.data_ptr(), stream=st)
    eng.join(st)
    torch.cuda.synchronize()
    eng.set_pipelined(False)
    for (kind, _), (disp, wl), want in zip(geoms, outs, wants):
        E.same(f"{kind} disp", disp.cpu().numpy(), want["disp"])
        E.same(f"{kind} wta_left", wl.cpu().numpy(), want["wta_left"])
    eng.close()


@pytest.mark.gpu
def test_resize_rules_that_need_an_engine_and_profile():
    """AREA sources that are not whole multiples of W x H, upscales, and blocks of more than 4096 pixels fail naming
    r->src_width / r->src_height, as do factors that are not exact in double (49, 93, 98); the largest accepted blocks
    pass; LINEAR_EXACT takes any size; clearing
    works; profile id 14 reports both raw frames + 2*3*N per pair (no maps) while a resize is set, and the map bytes
    again after maps are set."""
    import adcensus_b200 as A
    w, h, D = 40, 30, 12
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=2)
    L = A.load_library()
    eng.set_resize((80, 60), "area")
    for (sw, sh), msg in (((81, 60), b"r->src_width 81 is not a multiple of W (40)"),
                          ((80, 61), b"r->src_height 61 is not a multiple of H (30)"),
                          ((20, 60), b"r->src_width 20 is not a multiple"), ((80, 15), b"r->src_height 15"),
                          ((40 * 65, 30 * 64), b"more than 4096"), ((40 * 4097, 30), b"r->src_width"),
                          ((40 * 49, 30), b"r->src_width 1960: the factor 49 is not exact in double"),
                          ((40 * 2, 30 * 93), b"r->src_height 2790: the factor 93 is not exact in double"),
                          ((40 * 98, 30 * 2), b"r->src_width 3920: the factor 98")):
        r = A.Rectification(min(sw, 32767), sh, A.RESIZE_AREA, 0)
        assert L.adc_set_rectification(eng._h, ctypes.byref(r)) == 1 and msg in L.adc_last_error(), L.adc_last_error()
    for sw, sh in ((40 * 64, 30 * 64), (40 * 819, 30 * 5), (40, 30), (40, 30 * 64)):
        eng.set_resize((sw, sh), "area")
    eng.set_resize((80, 60), "area")
    N = w * h
    by = eng.profile_kernel("rectify", reps=2)[1]
    assert by == 2 * eng.wave_pairs * (80 * 60 * 3 + 3 * N), by
    for sw, sh in ((1, 1), (32767, 2), (17, 5)):
        eng.set_resize((sw, sh), "linear_exact")
    assert eng.profile_kernel("rectify", reps=2)[1] == 2 * eng.wave_pairs * (17 * 5 * 3 + 3 * N)
    m = R.warp_maps(w, h, 80, 60, 1)
    eng.set_rectification(m, m, (80, 60))
    assert eng.profile_kernel("rectify", reps=2)[1] == 2 * eng.wave_pairs * (80 * 60 * 3 + 3 * N) + 2 * 8 * N
    eng.set_rectification(None)
    with pytest.raises(A.AdcError, match="no rectification"):
        eng.profile_kernel("rectify", reps=1)
    eng.close()
