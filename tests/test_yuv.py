"""YUV frames (ADC_IMG_NV12, _NV21, _YUYV, _UYVY, _YVYU): video-decoder and camera frames converted on the way in,
matched exactly as cv2.cvtColor(frame, COLOR_YUV2BGR_*) (cropped to the view) followed by the packed-BGR entry point,
with or without rectification.

CPU: the numpy restatement (yuv_testlib) against live cv2.cvtColor with the optimised paths on and off (skipped without
OpenCV) and against the committed fixture, composed with rectify_testlib's cv2.remap (never skipped); the argument
rules that need no engine; the constants and the view parser.
GPU: Cone in every format through a 450 x 376 surface against the CPU oracle on the restated decode; synthetic batches
(odd sizes, row pitch, plane pitch and image stride above their minimums, several waves with a partial last one,
pipelined and not), even-offset crops and side-by-side frames against adc_match_outputs_batch_device on the restated
images, every output; the single-pair host entries; raw frames through both map types, larger and smaller than the
engine, odd, 1 x 1 and 1 x N; the size-dependent rule violations; launch counts.
"""
import ctypes

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E
import rectify_testlib as R
import yuv_testlib as Y

ROOT = T.REPO
MAPS = ["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"]
VOLS = ["cost", "aggr", "opt"]
GOLDEN = T.GOLDEN_DIR / "golden_yuv_cases.npz"


# ---- CPU ------------------------------------------------------------------------------------------
def _cases_from(npz):
    z = np.load(npz)
    name_of = {v: k for k, v in Y.CODE.items()}
    for name in sorted({k.split("/")[0] for k in z.files}):
        maps = (z[f"{name}/map1"], z[f"{name}/map2"]) if f"{name}/map1" in z.files else None
        w, h = (int(v) for v in z[f"{name}/size"])
        yield name, z[f"{name}/frame"], name_of[int(z[f"{name}/format"])], w, h, maps, z[f"{name}/out"]


def test_restatement_against_fixture():
    """The restatement reproduces every cvtColor output in the fixture (every format at tiny, odd and even sizes, with
    uniform bytes and the rule's corner values) and, composed with the remap restatement, every cvtColor -> remap
    output (both map types, frames larger and smaller than the output, maps past the last row and column, whose border
    is BGR 0, odd source sizes, 1 x N and 1 x 1 frames)."""
    seen = set()
    for name, frame, fmt, w, h, maps, out in _cases_from(GOLDEN):
        got = Y.decode(frame, fmt, w, h)
        if maps is not None:
            got = R.remap(got, *maps)
        assert np.array_equal(got, out), name
        seen.add((name.split("_")[0], fmt))
    assert {k for k, _ in seen} == {"tiny", "odd", "rect"}
    for kind in ("tiny", "odd", "rect"):
        assert {f for k, f in seen if k == kind} == set(Y.NAMES), kind


def test_restatement_against_opencv():
    """The restatement against live cv2.cvtColor with the optimised paths on and off: every format at 150 random sizes
    1..160 per setting (a third drawn from the rule's corner values; odd views as crops of cvtColor on their even
    enclosing frame), exhaustive Y x U x V planes through 4:2:2 macropixels, and 1080 x 1920."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(31)
    opt = cv2.useOptimized()
    try:
        for use in (True, False):
            cv2.setUseOptimized(use)
            for i in range(150):
                w, h = (int(v) for v in rng.integers(1, 161, 2))
                for fmt in Y.NAMES:
                    frame = Y.random_frame(rng, fmt, w, h, corners=i % 3 == 0)
                    assert np.array_equal(Y.decode(frame, fmt, w, h), Y.cv_decode(cv2, frame, fmt, w, h)), \
                        (use, fmt, w, h)
            # every (Y, U, V) with Y in 0..255 and U, V on a 17-step grid: YUYV macropixels Y U Y V
            yy, uu, vv = np.meshgrid(np.arange(256), np.arange(0, 256, 15), np.arange(0, 256, 15), indexing="ij")
            m = np.stack([yy, uu, yy, vv], -1).reshape(-1, 4).astype(np.uint8)
            frame = m.reshape(1, -1, 2)
            wpx = frame.shape[1]
            assert np.array_equal(Y.decode(frame, "yuyv", wpx, 1), Y.cv_decode(cv2, frame, "yuyv", wpx, 1)), use
            for fmt in Y.NAMES:
                frame = Y.random_frame(rng, fmt, 1920, 1080)
                assert np.array_equal(Y.decode(frame, fmt, 1920, 1080), Y.cv_decode(cv2, frame, fmt, 1920, 1080)), \
                    (use, fmt)
    finally:
        cv2.setUseOptimized(opt)


def test_rule_corners():
    """The stated anchors of the limited-range rule: Y = U = V = 128 gives (130, 130, 130), zero samples give
    (0, 154, 0) (the reason the rectified border is BGR 0 rather than converted zeros), and every intermediate of the
    rule stays inside int32 (each is linear in Y', U and V, so its extremes lie at the corners of their ranges)."""
    v = np.array([128], np.uint8)
    assert Y.convert(v, v, v).tolist() == [[130, 130, 130]]
    z = np.array([0], np.uint8)
    assert Y.convert(z, z, z).tolist() == [[0, 154, 0]]
    ends = np.array([0, 16, 255], np.int64)
    yy, uu, vv = np.meshgrid(ends, ends, ends, indexing="ij")
    y = np.maximum(0, yy - 16) * 1220542 + (1 << 19)
    u, w = uu - 128, vv - 128
    for t in (y + 1673527 * w, y - 852492 * w - 409993 * u, y + 2116026 * u):
        assert np.abs(t).max() < 5.7e8


def test_view_helpers():
    """write_view lays only the view's own samples (W luma bytes, 2*ceil(W/2) chroma bytes, 4*ceil(W/2) packed bytes a
    row) and samples() reads them back from the host entries' array shape; encode() gives that shape."""
    rng = np.random.default_rng(4)
    for fmt in Y.NAMES:
        for w, h in ((7, 5), (8, 6), (1, 1)):
            frame = Y.random_frame(rng, fmt, w, h)
            rp = Y.tight_row(fmt, w) + 3
            pp = h * rp + 5 if Y.is420(fmt) else 0
            buf = np.full(2 + Y.footprint(fmt, h, rp, pp) + 4, 0xEE, np.uint8)
            Y.write_view(buf, frame, fmt, w, h, rp, pp, 2)
            written = int((buf != 0xEE).sum())
            own = w * h + 2 * Y.half(w) * Y.half(h) if Y.is420(fmt) else 4 * Y.half(w) * h
            assert written <= own and buf[:2].tolist() == [0xEE, 0xEE] and (buf[-4:] == 0xEE).all()
            assert Y.encode(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), fmt).shape == Y.frame_shape(fmt, w, h)


def test_yuv_argument_errors_need_no_gpu():
    """The five codes pass the size-free rules and reach the engine check on both image and both rectified entries;
    plane_pitch != 0 is accepted for NV12 / NV21 and refused for 4:2:2; 6, 15, 20, 31 and 37 stay unknown;
    image_desc("yuv") still raises."""
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
        for name, code in Y.CODE.items():
            for d in (A.ImageDesc(code, 0, 0, 0, 0), A.ImageDesc(code, 0, 1001, 0, 1 << 33)):
                assert call(ctypes.byref(d)) == 1 and b"engine is NULL" in L.adc_last_error(), (fn, code)
            assert call(ctypes.byref(A.ImageDesc(code, 0, 0, 64, 0))) == 1
            err = L.adc_last_error()
            if Y.is420(name):
                assert b"engine is NULL" in err, err
            else:
                assert b"img->plane_pitch" in err and fn.encode() in err, err
            assert call(ctypes.byref(A.ImageDesc(code, 0, 0, -1, 0))) == 1 and b"img->plane_pitch" in L.adc_last_error()
            assert call(ctypes.byref(A.ImageDesc(code, 1, 0, 0, 0))) == 1 and b"img->reserved" in L.adc_last_error()
        for code in (6, 15, 20, 31, 37):
            assert call(ctypes.byref(A.ImageDesc(code, 0, 0, 0, 0))) == 1
            err = L.adc_last_error()
            assert f"img->format {code} unknown".encode() in err and fn.encode() in err, err
    with pytest.raises(ValueError):
        A.image_desc("yuv")


def test_yuv_constants():
    import adcensus_b200 as A
    assert (A.IMG_NV12, A.IMG_NV21, A.IMG_YUYV, A.IMG_UYVY, A.IMG_YVYU) == (32, 33, 34, 35, 36)
    assert A.YUV_FORMATS == Y.CODE
    assert not set(A.YUV_FORMATS) & (set(A.engine.IMG_FORMATS) | set(A.BAYER_FORMATS))
    for name, code in Y.CODE.items():
        d = A.image_desc(name, 78, 4000 if Y.is420(name) else 0, 9000)
        assert (d.format, d.row_pitch, d.plane_pitch, d.image_stride) == (code, 78, 4000 if Y.is420(name) else 0, 9000)
    h = (ROOT / "include" / "adcensus_b200.h").read_text()
    assert "enum { ADC_IMG_NV12 = 32, ADC_IMG_NV21 = 33, ADC_IMG_YUYV = 34, ADC_IMG_UYVY = 35, ADC_IMG_YVYU = 36 };" in h
    P = A.engine._image_view_desc
    # NV12 / NV21: [H + ceil(H/2)][2*ceil(W/2)], plane pitch H * row stride: the halves of a side-by-side frame, an odd W
    frame = np.zeros((9 + 5, 2 * 40), np.uint8)
    for fmt in (A.IMG_NV12, A.IMG_NV21):
        d = P(frame[:, 40:], fmt, 9, 40)
        assert (d.format, d.row_pitch, d.plane_pitch) == (fmt, 80, 9 * 80)
        d = P(frame[:, :38], fmt, 9, 37)
        assert (d.row_pitch, d.plane_pitch) == (80, 720)
        with pytest.raises(ValueError):
            P(frame[:, :37], fmt, 9, 37)   # a chroma row of an odd-width view is 2*ceil(W/2) bytes
        with pytest.raises(ValueError):
            P(frame[:13], fmt, 9, 40)
    # 4:2:2: [H][2*ceil(W/2)][2] (CV_8UC2), crops at even x of a wider frame
    frame = np.zeros((8, 50, 2), np.uint8)
    for fmt in (A.IMG_YUYV, A.IMG_UYVY, A.IMG_YVYU):
        d = P(frame[1:8, 4:30], fmt, 7, 25)
        assert (d.format, d.row_pitch, d.plane_pitch) == (fmt, 100, 0)
        with pytest.raises(ValueError):
            P(frame[1:8, 4:29], fmt, 7, 25)
        with pytest.raises(ValueError):
            P(np.zeros((7, 26), np.uint8), fmt, 7, 26)


# ---- GPU ------------------------------------------------------------------------------------------
def _yuv_batch(fmt, n, vw, vh, rng, extra_row, extra_plane, extra_stride, lead):
    """n pairs of random frames laid out with row pitch tight + extra_row, plane pitch H * row pitch + extra_plane
    (4:2:0), image stride footprint + extra_stride, `lead` bytes before the first view, random bytes everywhere else,
    one device buffer per view with guard bytes after the last view.  (views, offset of the first view, desc, left
    frames, right frames)."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    rp = Y.tight_row(fmt, vw) + extra_row
    pp = vh * rp + extra_plane if Y.is420(fmt) else 0
    stride = Y.footprint(fmt, vh, rp, pp) + extra_stride
    L = [Y.random_frame(rng, fmt, vw, vh) for _ in range(n)]
    Rr = [Y.random_frame(rng, fmt, vw, vh) for _ in range(n)]
    views = []
    for frames in (L, Rr):
        big = rng.integers(0, 256, size=lead + n * stride + 64, dtype=np.uint8)
        for i in range(n):
            Y.write_view(big, frames[i], fmt, vw, vh, rp, pp, lead + i * stride)
        views.append(torch.from_numpy(big).to(dev))
    return views, lead, A.image_desc(fmt, rp, pp, stride), L, Rr


def _packed(frames, fmt, w, h, maps=None):
    torch, dev = E.cuda()
    imgs = [Y.decode(f, fmt, w, h) for f in frames]
    if maps is not None:
        imgs = [R.remap(x, *maps) for x in imgs]
    return torch.from_numpy(np.stack(imgs)).to(dev)


def _equal_all(got, want, name):
    for k in want:
        assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), f"{name}: {k}"


@pytest.mark.gpu
def test_yuv_cone_against_oracle(cone):
    """Cone (450 x 375) encoded in each format and held in a 450 x 376 decoder surface (row pitch 512, NV12 / NV21
    chroma at 376 * pitch) through adc_match_images_batch_device: the final map equals the CPU oracle run on the restated
    decode of the same frames, bit for bit."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option())
    oracle = T.Oracle(w, h, T.default_option())
    st = torch.cuda.current_stream()
    for fmt in Y.NAMES:
        frames = [Y.encode(img, fmt) for img in (left, right)]
        rp = 512 if Y.is420(fmt) else 1024
        pp = 376 * rp if Y.is420(fmt) else 0
        stride = Y.footprint(fmt, 376, rp, pp)
        bufs = []
        for f in frames:
            host = np.zeros(2 * stride, np.uint8)
            for i in range(2):
                Y.write_view(host, f, fmt, w, h, rp, pp, i * stride)
            bufs.append(torch.from_numpy(host).to(dev))
        d_o = torch.empty((2, h, w), dtype=torch.float32, device=dev)
        eng.match_images_batch_device(2, bufs[0].data_ptr(), bufs[1].data_ptr(), image=A.image_desc(fmt, rp, pp, stride),
                                      d_disp=d_o.data_ptr(), stream=st.cuda_stream)
        torch.cuda.synchronize()
        want = oracle.match(Y.decode(frames[0], fmt, w, h), Y.decode(frames[1], fmt, w, h))
        got = d_o.cpu().numpy()
        E.same(f"cone {fmt} pair 0", got[0], want)
        E.same(f"cone {fmt} pair 1", got[1], want)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_yuv_batched(pipelined):
    """wave_pairs = 4, lanes = 3, n = 14 (several waves per lane, a partial last wave), odd W and H, every format with
    row pitch, plane pitch and image stride above their minimums and views at odd byte offsets: every output equals
    adc_match_outputs_batch_device on the restated BGR images, and the source buffers are unchanged."""
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    rng = np.random.default_rng(8)
    for k, fmt in enumerate(Y.NAMES):
        views, off, desc, L, Rr = _yuv_batch(fmt, n, w, h, rng, (0, 7, 64, 1, 3)[k], (0, 5, 0, 0, 0)[k] + 3 * k,
                                             (5, 0, 3, 11, 0)[k], (0, 3, 1, 6, 13)[k])
        before = [t.clone() for t in views]
        outputs = dict(volumes=[(v, "hwd", "f32") for v in VOLS], maps=MAPS, pipelined=pipelined)
        pl, pr = _packed(L, fmt, w, h), _packed(Rr, fmt, w, h)
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_images_batch_device, n, views[0].data_ptr() + off,
                              views[1].data_ptr() + off, desc.image_stride, image=desc, **outputs)
        _equal_all(got, want, f"{fmt} rp {desc.row_pitch} pp {desc.plane_pitch} stride {desc.image_stride}")
        assert all(torch.equal(t, c) for t, c in zip(views, before)), f"{fmt}: source buffer changed"
    eng.close()


@pytest.mark.gpu
def test_yuv_side_by_side_and_crops():
    """Side-by-side NV12 and YUYV frames (the right view at base + W, resp. 2 * W bytes, one plane pitch for both) and
    crops at even offsets of a larger frame in every format, 3 pairs a call: every output equals the packed-BGR call on
    the restated views (NV12 chroma of a crop taken from the crop's own even position)."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 70, 45, 19
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=2)
    n = 3
    rng = np.random.default_rng(14)
    outputs = dict(volumes=[("opt", "hwd", "f32")], maps=MAPS)

    def crop(big, fmt, FH, x0, y0, vw, vh):
        """The host-entry array of the vw x vh view at even (x0, y0) of a frame of FH rows."""
        wp = 2 * Y.half(vw)
        if Y.is420(fmt):
            return np.concatenate([big[y0:y0 + vh, x0:x0 + wp], big[FH + y0 // 2:FH + y0 // 2 + Y.half(vh), x0:x0 + wp]])
        return big[y0:y0 + vh, x0:x0 + wp]

    # side by side: one frame of 2W x H per pair
    for fmt in ("nv12", "yuyv"):
        frames = [Y.random_frame(rng, fmt, 2 * w, h) for _ in range(n)]
        rp = 2 * w if fmt == "nv12" else 4 * w
        pp = h * rp if fmt == "nv12" else 0
        stride = frames[0].nbytes + 6
        host = np.zeros(n * stride, np.uint8)
        for i, f in enumerate(frames):
            host[i * stride:i * stride + f.nbytes] = f.reshape(-1)
        d = torch.from_numpy(host).to(dev)
        pl, pr = (_packed([crop(f, fmt, h, x, 0, w, h) for f in frames], fmt, w, h) for x in (0, w))
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h,
                               **outputs)
        got = E.batch_outputs(eng, eng.match_images_batch_device, n, d.data_ptr(), d.data_ptr() + rp // 2, stride,
                              image=A.image_desc(fmt, rp, pp, stride), **outputs)
        _equal_all(got, want, f"side by side {fmt}")
    # crops at even offsets of a larger frame (FW x FH), odd view height
    FW, FH, x0, y0, vh = w + 10, 52, 4, 6, 43
    eng.close()
    eng = E.engine(w, vh, T.default_option(max_disparity=D), wave_pairs=2)
    for fmt in Y.NAMES:
        frames = [[Y.random_frame(rng, fmt, FW, FH) for _ in range(n)] for _ in range(2)]
        rp = Y.tight_row(fmt, FW)
        pp = (FH - y0 + y0 // 2) * rp if Y.is420(fmt) else 0   # chroma of the crop from the crop's own base
        off = y0 * rp + (x0 if Y.is420(fmt) else 2 * x0)
        stride = frames[0][0].nbytes
        d = [torch.from_numpy(np.concatenate([f.reshape(-1) for f in fs])).to(dev) for fs in frames]
        pl, pr = (_packed([crop(f, fmt, FH, x0, y0, w, vh) for f in fs], fmt, w, vh) for fs in frames)
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * vh,
                               **outputs)
        got = E.batch_outputs(eng, eng.match_images_batch_device, n, d[0].data_ptr() + off, d[1].data_ptr() + off,
                              stride, image=A.image_desc(fmt, rp, pp, stride), **outputs)
        _equal_all(got, want, f"crop {fmt}")
    eng.close()


@pytest.mark.gpu
def test_yuv_host_entry():
    """The single-pair host entry match_images, odd W and H, on tight frames and on column slices of wider arrays (a
    larger row pitch): final map, all three volumes and all five side maps equal match_outputs on the restated images."""
    w, h, D = 61, 45, 20
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    rng = np.random.default_rng(21)
    for k, fmt in enumerate(Y.NAMES):
        frames = [Y.random_frame(rng, fmt, w, h) for _ in range(2)]
        if k % 2:   # the same samples in arrays 8 pixels wider
            wide = []
            for f in frames:
                shape = list(f.shape)
                shape[1] += 8
                big = rng.integers(0, 256, shape, dtype=np.uint8)
                big[:, :f.shape[1]] = f
                wide.append(big[:, :f.shape[1]])
            frames = wide
        want_disp, want = eng.match_outputs(*(Y.decode(f, fmt, w, h) for f in frames), maps=MAPS, volumes=VOLS)
        disp, got = eng.match_images(frames[0], frames[1], format=fmt, maps=MAPS, volumes=VOLS)
        E.same(f"{fmt} host disp", disp, want_disp)
        for key in want:
            E.same(f"{fmt} host {key}", got[key], want[key])
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_yuv_rectified(pipelined):
    """Raw YUV frames through the rectified entries: both map types (with specials), frames larger and smaller than the
    engine, odd, 1 x 1 and 1 x N, with row pitch and plane pitch above their minimums: every output equals
    adc_match_outputs_batch_device on remap(decode(raw)) (the border BGR 0); the host entry match_rectified agrees."""
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=3)
    n = 2 * eng.wave_pairs + 1
    rng = np.random.default_rng(12)
    cases = [((83, 53), "nv12"), ((64, 40), "nv21"), ((1, 1), "yuyv"), ((57, 1), "uyvy"), ((3, 5), "yvyu"),
             ((90, 61), "nv12"), ((1, 1), "nv21"), ((33, 1), "nv12")]
    for k, ((sw, sh), fmt) in enumerate(cases):
        fixed = k % 2 == 1
        maps = [R.warp_maps(w, h, sw, sh, 40 + 2 * k + v, fixed) for v in range(2)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        views, off, desc, L, Rr = _yuv_batch(fmt, n, sw, sh, rng, 4, 2, 0, 1)
        outputs = dict(volumes=[(v, "hwd", "f32") for v in VOLS], maps=MAPS, pipelined=pipelined)
        pl, pr = _packed(L, fmt, sw, sh, maps[0]), _packed(Rr, fmt, sw, sh, maps[1])
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_rectified_batch_device, n, views[0].data_ptr() + off,
                              views[1].data_ptr() + off, desc.image_stride, image=desc, **outputs)
        _equal_all(got, want, f"{sw}x{sh} {fmt} fixed={fixed}")
        if not pipelined:
            disp, one = eng.match_rectified(L[1], Rr[1], format=fmt, maps=MAPS)
            E.same(f"{sw}x{sh} {fmt} host disp", disp, want["disp"][1])
            for m in MAPS:
                E.same(f"{sw}x{sh} {fmt} host {m}", one[m], want[m][1])
    eng.close()


@pytest.mark.gpu
def test_yuv_rectified_host_large_frames():
    """The host entry match_rectified with 1280 x 720 NV12 and 1279 x 719 UYVY raw frames, larger than the lane volume
    the staging otherwise uses (so the grown device staging takes them): the result equals match_outputs on
    remap(decode(raw))."""
    w, h, D = 71, 47, 12
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    rng = np.random.default_rng(30)
    for fmt, (sw, sh) in (("nv12", (1280, 720)), ("uyvy", (1279, 719))):
        maps = [R.warp_maps(w, h, sw, sh, 90 + v) for v in range(2)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        frames = [Y.random_frame(rng, fmt, sw, sh) for _ in range(2)]
        want_disp, want = eng.match_outputs(*(R.remap(Y.decode(frames[v], fmt, sw, sh), *maps[v]) for v in range(2)),
                                            maps=MAPS)
        disp, got = eng.match_rectified(frames[0], frames[1], format=fmt, maps=MAPS)
        E.same(f"{fmt} {sw}x{sh} disp", disp, want_disp)
        for m in MAPS:
            E.same(f"{fmt} {sw}x{sh} {m}", got[m], want[m])
    eng.close()


@pytest.mark.gpu
def test_yuv_size_rules():
    """Each size-dependent rule violation fails with ADC_ERR_ARG naming its field, on the image and the rectified
    entries: an odd-W NV12 view with row_pitch = W, plane_pitch = H * row_pitch - 1, a 4:2:2 row pitch of 2 * W for odd
    W, an image stride one byte short of the footprint (chroma rows included); the minimums themselves are accepted."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 12
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    buf = torch.zeros(4 * (w + 1) * h * 2 * 2, dtype=torch.uint8, device=dev)
    d_o = torch.empty((2, h, w), dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def run(entry, fmt, rp=0, pp=0, stride=0):
        entry(2, buf.data_ptr(), buf.data_ptr(), image=A.image_desc(fmt, rp, pp, stride), d_disp=d_o.data_ptr(),
              stream=st)
        torch.cuda.synchronize()

    eng.set_rectification(*[R.warp_maps(w, h, w, h, 5)] * 2, (w, h))
    for entry in (eng.match_images_batch_device, eng.match_rectified_batch_device):
        bad = [("nv12", dict(rp=w), r"img->row_pitch 71 is less than 2 \* ceil\(W / 2\) \(72\)"),
               ("nv21", dict(rp=72, pp=h * 72 - 1), r"img->plane_pitch 3383 is less than H \* row_pitch \(3384\)"),
               ("yuyv", dict(rp=2 * w), r"img->row_pitch 142 is less than 4 \* ceil\(W / 2\) \(144\)"),
               ("uyvy", dict(rp=143), r"img->row_pitch 143"),
               ("nv12", dict(stride=72 * (h + 24) - 1), r"img->image_stride 5111 is less than the view's footprint \(5112\)"),
               ("yvyu", dict(stride=144 * h - 1), r"img->image_stride"),
               ("nv12", dict(rp=1 << 62), r"img->row_pitch .* is too large"),
               ("nv21", dict(rp=72, pp=(1 << 63) - 72), r"img->plane_pitch .* is too large")]
        for fmt, kw, msg in bad:
            with pytest.raises(A.AdcError, match=r"error 1: .*" + msg):
                run(entry, fmt, **kw)
        for fmt, kw in (("nv12", dict(rp=72, pp=72 * h, stride=72 * (h + 24))), ("yuyv", dict(rp=144, stride=144 * h))):
            run(entry, fmt, **kw)
    eng.close()


@pytest.mark.gpu
def test_yuv_launch_counts():
    """A YUV call issues exactly one launch per wave more than the tight packed-BGR call of the same batch, through both
    the image and the rectified entry; the ingestion profile ids replay the YUV kernels after a YUV call and report
    the algorithmic bytes (4:2:0: W*H + 2*ceil(W/2)*ceil(H/2) read, 4:2:2: 4*ceil(W/2)*H, plus 3*N written)."""
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

    def read_bytes(fmt, vw, vh):
        return vw * vh + 2 * Y.half(vw) * Y.half(vh) if Y.is420(fmt) else 4 * Y.half(vw) * vh

    base = count(eng.match_outputs_batch_device, n, bgr[0].data_ptr(), bgr[1].data_ptr())
    for fmt in Y.NAMES:
        yuv = [torch.from_numpy(np.stack([Y.random_frame(rng, fmt, w, h) for _ in range(n)])).to(dev) for _ in range(2)]
        got = count(eng.match_images_batch_device, n, yuv[0].data_ptr(), yuv[1].data_ptr(), image=A.image_desc(fmt))
        assert got == base + waves, (fmt, got, base, waves)
        assert eng.profile_kernel("image_ingest", reps=2)[1] == 2 * eng.wave_pairs * (read_bytes(fmt, w, h) + 3 * h * w)
    sw, sh = 91, 61
    m = R.warp_maps(w, h, sw, sh, 3)
    eng.set_rectification(m, m, (sw, sh))
    raw = [torch.from_numpy(rng.integers(0, 256, (n, sh, sw, 3), dtype=np.uint8)).to(dev) for _ in range(2)]
    rect_bgr = count(eng.match_rectified_batch_device, n, raw[0].data_ptr(), raw[1].data_ptr())
    assert rect_bgr == base + waves
    for fmt in Y.NAMES:
        yuv = [torch.from_numpy(np.stack([Y.random_frame(rng, fmt, sw, sh) for _ in range(n)])).to(dev) for _ in range(2)]
        got = count(eng.match_rectified_batch_device, n, yuv[0].data_ptr(), yuv[1].data_ptr(), image=A.image_desc(fmt))
        assert got == base + waves, (fmt, got, base, waves)
        ms, by = eng.profile_kernel("rectify", reps=2)
        assert ms > 0 and by == 2 * eng.wave_pairs * (read_bytes(fmt, sw, sh) + 3 * h * w) + 2 * 8 * h * w, fmt
    eng.close()
