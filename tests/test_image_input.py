"""Image input formats (adc_match_images*): RGB, BGRA / RGBA, gray and planar images with row, plane and image pitch,
read in place and matched exactly as the same pixels packed as BGR.

CPU: the argument rules (on a NULL engine, before any device work), the descriptor's layout and the constants, the numpy
packing helper against hand-built images, the gray golden cases (recorded from the unmodified reference) against the C
restatement.
GPU: every colour format on Cone through both entry points (the reference's map, the packed-BGR call's matching cost);
the gray golden cases; side-by-side, stacked, cropped and gray batches through the batched entry with several waves per
lane; image strides past 2^31 bytes; the unchanged default path; the size-dependent argument rules.
"""
import ctypes

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E  # puts tools/ on sys.path
import images_testlib as IT
import make_golden as G
import make_golden_gray as GG

MAPS = ["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"]
COLOUR = ["bgr", "rgb", "bgra", "rgba", "rgb_planar"]
CONE_SHA = "77d70a58d1aa5c71"


# ---- CPU ------------------------------------------------------------------------------------------
def _desc(fmt=0, reserved=0, row=0, plane=0, stride=0):
    import adcensus_b200 as A
    return A.ImageDesc(fmt, reserved, row, plane, stride)


def test_image_argument_errors_need_no_gpu():
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    maps1 = (A.engine.MapOut * 1)(A.engine.MapOut(p, A.MAP_PEAK_RATIO, 0))
    vol_bad = (A.engine.VolumeOut * 1)(A.engine.VolumeOut(p, 3, A.COST_HWD, A.COST_F32, 0))

    def host(img, maps=None, n_maps=0, vols=None, n_vols=0, disp=p, cost=None, cl=0, cd=0):
        return L.adc_match_images(None, p, p, img, cost, cl, cd, disp, vols, n_vols, maps, n_maps)

    def dev(img, maps=None, n_maps=0, vols=None, n_vols=0, disp=p, cost=None, cl=0, cd=0):
        return L.adc_match_images_batch_device(None, 1, p, p, img, cost, cl, cd, disp, vols, n_vols, maps, n_maps, None)

    for call in (host, dev):
        cases = [
            (dict(img=_desc(6)), b"img->format"),
            (dict(img=_desc(-1)), b"img->format"),
            (dict(img=_desc(A.IMG_RGB, reserved=1)), b"img->reserved"),
            (dict(img=_desc(A.IMG_BGRA, plane=100)), b"img->plane_pitch"),
            (dict(img=_desc(A.IMG_GRAY, plane=1)), b"img->plane_pitch"),
            (dict(img=_desc(A.IMG_RGB, row=-1)), b"img->row_pitch"),
            (dict(img=_desc(A.IMG_RGB_PLANAR, plane=-3)), b"img->plane_pitch"),
            (dict(img=_desc(A.IMG_GRAY, stride=-(1 << 40))), b"img->image_stride"),
            # the output / cost rules of adc_match_outputs*, under this entry's names
            (dict(img=None, maps=maps1, n_maps=6), b"n_maps"),
            (dict(img=None, maps=None, n_maps=1), b"maps is NULL"),
            (dict(img=None, vols=vol_bad, n_vols=1), b"vols[0].stage"),
            (dict(img=None, vols=None, n_vols=4), b"n_vols"),
            (dict(img=None, disp=None), b"no volume or map"),
            (dict(img=None, cost=p, cl=2), b"cost_layout"),
            (dict(img=None, cost=p, cd=5), b"cost_dtype"),
        ]
        for kw, msg in cases:
            assert call(**kw) == 1, (call.__name__, kw)
            err = L.adc_last_error()
            assert msg in err, (call.__name__, kw, err)
            assert (b"adc_match_images_batch_device" if call is dev else b"adc_match_images:") in err, err
        # valid descriptors get as far as the engine check
        valid = [None, _desc(), _desc(A.IMG_BGR, row=3001, stride=1 << 33), _desc(A.IMG_RGB, row=7),
                 _desc(A.IMG_BGRA, row=1 << 20), _desc(A.IMG_RGBA), _desc(A.IMG_GRAY, row=13, stride=5),
                 _desc(A.IMG_RGB_PLANAR), _desc(A.IMG_RGB_PLANAR, row=9, plane=1001, stride=3003)]
        for img in valid:
            assert call(img) == 1 and b"engine is NULL" in L.adc_last_error(), (call.__name__, img and img.format)
        assert call(_desc(A.IMG_GRAY), maps=maps1, n_maps=1, disp=None) == 1 and b"engine is NULL" in L.adc_last_error()


def test_image_constants():
    import adcensus_b200 as A
    D = A.ImageDesc
    assert ctypes.sizeof(D) == 32
    assert [(n, getattr(D, n).offset) for n, _ in D._fields_] == [
        ("format", 0), ("reserved", 4), ("row_pitch", 8), ("plane_pitch", 16), ("image_stride", 24)]
    assert (A.IMG_BGR, A.IMG_RGB, A.IMG_BGRA, A.IMG_RGBA, A.IMG_GRAY, A.IMG_RGB_PLANAR) == (0, 1, 2, 3, 4, 5)
    assert A.engine.IMG_FORMATS == IT.CODE
    assert A.Engine.PROFILE_KERNELS["image_ingest"] == 13
    d = A.image_desc("rgb_planar", 5, 100, 400)
    assert (d.format, d.reserved, d.row_pitch, d.plane_pitch, d.image_stride) == (5, 0, 5, 100, 400)
    with pytest.raises(ValueError):
        A.image_desc("yuv")


def test_to_bgr_helper_hand_built():
    """to_bgr against images written byte by byte: W = 3 (odd), H = 2, pitch > tight, a non-zero offset, junk around."""
    H, W = 2, 3
    px = [[(10, 20, 30), (11, 21, 31), (12, 22, 32)], [(13, 23, 33), (14, 24, 34), (15, 25, 35)]]   # (B, G, R)
    want = np.array(px, np.uint8)
    for fmt in IT.FORMATS:
        bpp = IT.BPP[fmt]
        rp, off = W * bpp + 5, 7
        pp = H * rp + 3 if fmt == "rgb_planar" else 0
        buf = np.full(off + max(IT.footprint(fmt, H, rp, pp), H * rp) + 9, 0xEE, np.uint8)
        for y in range(H):
            for x in range(W):
                b, g, r = px[y][x]
                o = off + y * rp + x * bpp
                if fmt in ("bgr", "bgra"):
                    buf[o:o + 3] = (b, g, r)
                elif fmt in ("rgb", "rgba"):
                    buf[o:o + 3] = (r, g, b)
                elif fmt == "gray":
                    buf[o] = g
                else:
                    for c, v in enumerate((r, g, b)):
                        buf[off + c * pp + y * rp + x] = v
                if bpp == 4:
                    buf[o + 3] = 0x77
        got = IT.to_bgr(buf, fmt, H, W, rp, pp, off)
        if fmt == "gray":
            assert got.tolist() == np.repeat(want[:, :, 1:2], 3, axis=2).tolist(), fmt
        else:
            assert got.tolist() == want.tolist(), fmt
        # from_bgr / write_view lay the same pixels out again
        src = want if fmt != "gray" else np.repeat(want[:, :, 1:2], 3, axis=2)
        buf2 = np.full_like(buf, 0xEE)
        IT.write_view(buf2, IT.from_bgr(src, fmt, alpha=np.full((H, W), 0x77, np.uint8)), fmt, rp, pp, off)
        assert np.array_equal(buf2, buf), fmt


def test_gray_golden_restatement():
    """The C restatement reproduces every tap the unmodified reference recorded for the gray golden cases, and the
    replicated input's GRAY tap is not the input: gray(128, 128, 128) = 127."""
    golden = E.golden("golden_gray_cases.json")
    assert set(golden) == set(GG.GRAY_CASES)
    for name, g in golden.items():
        gl, gr, opt = GG.gray_case_inputs(name)
        assert [T.sha(gl), T.sha(gr)] == g["input_sha"], name
        h, w = gl.shape
        orc = T.Oracle(w, h, opt)
        orc.begin(IT.gray_to_bgr(gl), IT.gray_to_bgr(gr))
        for st in T.STAGES:
            orc.step()
            for tap in T.STAGE_TAPS[st]:
                a = orc.tap(tap)
                assert T.sha(G.ref_case_tap(opt, tap, a)) == g["hashes"][f"{st}/{tap}"], f"{name} {st}/{tap}"
                if st == "COST" and tap == "GRAY_L" and name == "synth_gray_odd":
                    m = gl == 128
                    assert m.sum() >= 4 * w and (a[m] == 127).all(), name
        orc.close()
    assert golden["synth_gray_odd"]["width"] % 2 == 1


# ---- GPU ------------------------------------------------------------------------------------------
def _padded(img, fmt, extra_row, extra_plane=0, extra_stride=0, lead=0):
    """(flat buffer, row_pitch, plane_pitch, offset) of a tight image laid out with padded pitches and `lead` bytes
    before it; every padding byte is 0xEE."""
    if fmt == "rgb_planar":
        _, H, W = img.shape
    else:
        H, W = img.shape[:2]
    rp = W * IT.BPP[fmt] + extra_row
    pp = H * rp + extra_plane if fmt == "rgb_planar" else 0
    buf = np.full(lead + IT.footprint(fmt, H, rp, pp) + extra_stride, 0xEE, np.uint8)
    IT.write_view(buf, img, fmt, rp, pp, lead)
    return buf, rp, pp, lead


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", COLOUR)
def test_colour_formats_cone(fmt, cone):
    """Cone in each colour format, tight and with a padded odd row pitch (and plane pitch), through both entry points:
    the final map is the reference's and the f32 ADC_VOL_COST export -- the earliest output that depends on every
    converted byte of both views -- is bit-identical to the packed-BGR call's."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option())
    want_disp, want = eng.match_outputs(left, right, volumes=["cost"])
    assert T.sha(want_disp).startswith(CONE_SHA)
    st = torch.cuda.current_stream()
    for extra in (0, 7):
        views = []
        for img in (left, right):
            buf, rp, pp, off = _padded(IT.from_bgr(img, fmt), fmt, extra, 5 if extra else 0)
            views.append((buf, off))
        name = f"{fmt} pad {extra}"
        # host entry: numpy views of the padded buffers
        if fmt == "rgb_planar":
            mk = lambda b, o: np.lib.stride_tricks.as_strided(b[o:], (3, h, w), (pp, rp, 1))
        else:
            C = IT.BPP[fmt]
            mk = lambda b, o: np.lib.stride_tricks.as_strided(b[o:], (h, w, C), (rp, C, 1))
        disp, got = eng.match_images(mk(*views[0]), mk(*views[1]), format=fmt, volumes=["cost"])
        assert T.sha(disp).startswith(CONE_SHA), name
        E.same(f"{name} host cost volume", got["cost"], want["cost"])
        # batched device entry: two pairs per call, image stride = footprint + 3 (odd), the right view in its own buffer
        n = 2
        stride = views[0][0].size + 3
        d = [torch.full((n * stride,), 0xEE, dtype=torch.uint8, device=dev) for _ in range(2)]
        for i in range(n):
            for v in range(2):
                d[v][i * stride:i * stride + views[v][0].size] = torch.from_numpy(views[v][0]).to(dev)
        desc = A.image_desc(fmt, rp, pp, stride)
        d_disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
        d_cost = torch.empty((n, h, w, eng.D), dtype=torch.float32, device=dev)
        eng.match_images_batch_device(n, d[0].data_ptr() + views[0][1], d[1].data_ptr() + views[1][1], image=desc,
                                      volumes=[(d_cost.data_ptr(), "cost", "hwd", "f32")], d_disp=d_disp.data_ptr(),
                                      stream=st.cuda_stream)
        torch.cuda.synchronize()
        for i in range(n):
            assert T.sha(d_disp[i].cpu().numpy()).startswith(CONE_SHA), f"{name} pair {i}"
            E.same(f"{name} device cost volume pair {i}", d_cost[i].cpu().numpy(), want["cost"])
    eng.close()


def _check_gray(name, g, opt, disp, got):
    hs = g["hashes"]
    assert T.sha(disp) == hs["MEDIAN/DISP_L"], f"{name}: final map"
    assert T.sha(got["cost"]) == hs["COST/VOL_INIT"], f"{name}: cost volume"
    assert T.sha(got["aggr"]) == hs["AGG4/VOL_AGGR"], f"{name}: aggregated volume"
    assert T.sha(got["opt"]) == hs["SO4/VOL_AGGR"], f"{name}: optimised volume"
    assert T.sha(got["wta_left"]) == hs["WTA/DISP_L"], f"{name}: wta_left"
    assert T.sha(G.ref_case_tap(opt, "DISP_R", got["wta_right"])) == hs["WTA/DISP_R"], f"{name}: wta_right"
    import maps_testlib as MT
    mis, occ = MT.outlier_lists(got["outliers"])
    assert T.sha(mis) == hs["OUTLIER/MISMATCHES"] and T.sha(occ) == hs["OUTLIER/OCCLUSIONS"], f"{name}: outliers"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GG.GRAY_CASES))
def test_gray_golden(name):
    """The gray golden cases through both entry points: every exported volume (f32 [H][W][D]), the WTA maps, the
    outlier lists and the final map hash to what the unmodified reference gives for the replicated images."""
    torch, dev = E.cuda()
    import adcensus_b200 as A
    g = E.golden("golden_gray_cases.json")[name]
    gl, gr, opt = GG.gray_case_inputs(name)
    assert [T.sha(gl), T.sha(gr)] == g["input_sha"]
    h, w = gl.shape
    eng = E.engine(w, h, opt)
    disp, got = eng.match_images(gl, gr, format="gray", maps=MAPS, volumes=["cost", "aggr", "opt"])
    _check_gray(f"{name} host", g, opt, disp, got)
    n, D = 3, eng.D
    d_l = torch.from_numpy(np.stack([gl] * n)).to(dev)
    d_r = torch.from_numpy(np.stack([gr] * n)).to(dev)
    d_disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    vols = {s: torch.empty((n, h, w, D), dtype=torch.float32, device=dev) for s in ("cost", "aggr", "opt")}
    maps = {m: torch.empty((n, h, w), dtype=torch.uint8 if m == "outliers" else torch.float32, device=dev) for m in MAPS}
    eng.match_images_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), image=A.image_desc("gray"),
                                  maps=[(b.data_ptr(), m) for m, b in maps.items()],
                                  volumes=[(b.data_ptr(), s, "hwd", "f32") for s, b in vols.items()],
                                  d_disp=d_disp.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for i in range(n):
        got_i = {k: b[i].cpu().numpy() for k, b in {**vols, **maps}.items()}
        _check_gray(f"{name} device pair {i}", g, opt, d_disp[i].cpu().numpy(), got_i)
    eng.close()


class _Batch:
    """n pairs of one geometry on the device: for each view the source tensor and the byte offset of pair 0's view in
    it, the descriptor, and the packed BGR images the views were built from."""

    def __init__(self, views, desc, bgr_l, bgr_r):
        self.views, self.desc, self.bgr_l, self.bgr_r = views, desc, bgr_l, bgr_r
        self.bases = [t.data_ptr() + off for t, off in views]


def _geometry(kind, fmt, n, h, w, D, rng):
    """A batch of n pairs of distinct synthetic images in geometry `kind`: "sbs" (side-by-side BGRA frames
    [n][H][2W][4], right view at +4W bytes), "stacked" (planar pairs [n][2][3][H][W] in one buffer), "crop" (odd-x crops
    of larger frames with random surroundings, any format), "gray" ([n][H][W])."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    pairs = [T.synthetic_pair(w, h, D, 900 + s) for s in range(n)]
    if fmt == "gray":
        pairs = [(IT.gray_to_bgr(l[:, :, 1]), IT.gray_to_bgr(r[:, :, 1])) for l, r in pairs]
    L, R = [p[0] for p in pairs], [p[1] for p in pairs]
    if kind == "sbs":
        frame = np.stack([np.concatenate([IT.from_bgr(l, "bgra"), IT.from_bgr(r, "bgra")], axis=1) for l, r in pairs])
        buf = torch.from_numpy(frame.reshape(-1)).to(dev)
        return _Batch([(buf, 0), (buf, 4 * w)], A.image_desc("bgra", 8 * w, 0, h * 8 * w), L, R)
    if kind == "stacked":
        arr = np.stack([np.stack([IT.from_bgr(l, "rgb_planar"), IT.from_bgr(r, "rgb_planar")]) for l, r in pairs])
        buf = torch.from_numpy(arr.reshape(-1)).to(dev)
        return _Batch([(buf, 0), (buf, 3 * h * w)], A.image_desc("rgb_planar", w, h * w, 6 * h * w), L, R)
    if kind == "gray":
        bl = torch.from_numpy(np.stack([IT.from_bgr(x, "gray") for x in L]).reshape(-1)).to(dev)
        br = torch.from_numpy(np.stack([IT.from_bgr(x, "gray") for x in R]).reshape(-1)).to(dev)
        return _Batch([(bl, 0), (br, 0)], A.image_desc("gray"), L, R)
    # crop: (x0, y0) = (5, 1) in frames of (H + 3) x (W + 11) pixels
    bpp, x0, y0, FH, FW = IT.BPP[fmt], 5, 1, h + 3, w + 11
    rp = FW * bpp
    pp = FH * rp if fmt == "rgb_planar" else 0
    stride = IT.footprint(fmt, FH, rp, pp)
    off = y0 * rp + x0 * bpp
    views = []
    for imgs in (L, R):
        big = rng.integers(0, 256, size=(n, stride), dtype=np.uint8)
        for i in range(n):
            IT.write_view(big[i], IT.from_bgr(imgs[i], fmt), fmt, rp, pp, off)
        views.append((torch.from_numpy(big.reshape(-1)).to(dev), off))
    return _Batch(views, A.image_desc(fmt, rp, pp, stride), L, R)


def _resolved(desc, fmt, h, w):
    """(row_pitch, plane_pitch, image_stride) of a descriptor with its zero defaults replaced, as the header defines."""
    rp = desc.row_pitch or w * IT.BPP[fmt]
    pp = (desc.plane_pitch or h * rp) if fmt == "rgb_planar" else 0
    return rp, pp, desc.image_stride or IT.footprint(fmt, h, rp, pp)


GEOMETRIES = [("sbs", "bgra"), ("stacked", "rgb_planar"), ("gray", "gray")] + [("crop", f) for f in IT.FORMATS]


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_geometry_batched(pipelined):
    """wave_pairs = 4, lanes = 3, n = 14 (several waves per lane, n not a multiple of the wave), odd W: side-by-side BGRA
    (the right view's base is not word-aligned), stacked planar pairs, odd-x crops of larger frames in every format, and
    gray.  Every output of a call with a cost volume, an exported volume and all five side maps equals the same call's on
    the packed BGR images (to_bgr of the same bytes), and the source buffers are unchanged."""
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    opt = T.default_option(max_disparity=D)
    eng = E.engine(w, h, opt, wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    rng = np.random.default_rng(3)
    d_cost = torch.from_numpy(rng.random((n, D, h, w), dtype=np.float32) * np.float32(40)).to(dev)
    for kind, fmt in GEOMETRIES:
        b = _geometry(kind, fmt, n, h, w, D, rng)
        before = [t.clone() for t, _ in b.views]
        # the views stand for the packed BGR images they were built from (numpy restatement of the descriptor)
        rp, pp, stride = _resolved(b.desc, fmt, h, w)
        for (t, off), imgs in zip(b.views, (b.bgr_l, b.bgr_r)):
            raw = t.cpu().numpy()
            for i in range(n):
                assert np.array_equal(IT.to_bgr(raw, fmt, h, w, rp, pp, off + i * stride), imgs[i]), (kind, fmt, i)
        packed_l = torch.from_numpy(np.stack(b.bgr_l)).to(dev)
        packed_r = torch.from_numpy(np.stack(b.bgr_r)).to(dev)
        outputs = dict(volumes=[("opt", "dhw", "bf16")], maps=MAPS, d_cost=d_cost, cost_layout="dhw", cost_dtype="f32",
                       pipelined=pipelined)
        entry = eng.match_images_batch_device
        want = E.batch_outputs(eng, entry, n, packed_l.data_ptr(), packed_r.data_ptr(), 3 * h * w, **outputs)
        got = E.batch_outputs(eng, entry, n, b.bases[0], b.bases[1], stride, image=b.desc, **outputs)
        for k in want:
            assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), f"{kind} {fmt}: {k}"
        assert all(torch.equal(t, c) for (t, _), c in zip(b.views, before)), f"{kind} {fmt}: source buffer changed"
    eng.close()


@pytest.mark.gpu
def test_image_stride_past_2_31():
    """n = 2 gray pairs with an image stride above 2^31 bytes: the second pair's views are read from past 2^31."""
    torch, dev = E.cuda()
    import adcensus_b200 as A
    w, h, D = 97, 61, 24
    opt = T.default_option(max_disparity=D)
    pairs = [T.synthetic_pair(w, h, D, s) for s in (71, 72)]
    grays = [(l[:, :, 2].copy(), r[:, :, 0].copy()) for l, r in pairs]
    stride = (1 << 31) + 4099
    N = h * w
    buf = torch.zeros(stride + 2 * N + 1, dtype=torch.uint8, device=dev)   # pair i: left at i*stride, right at +N+1
    for i, (gl, gr) in enumerate(grays):
        buf[i * stride:i * stride + N] = torch.from_numpy(gl.reshape(-1)).to(dev)
        buf[i * stride + N + 1:i * stride + 2 * N + 1] = torch.from_numpy(gr.reshape(-1)).to(dev)
    eng = E.engine(w, h, opt)
    d_disp = torch.empty((2, h, w), dtype=torch.float32, device=dev)
    eng.match_images_batch_device(2, buf.data_ptr(), buf.data_ptr() + N + 1, image=A.image_desc("gray", 0, 0, stride),
                                  d_disp=d_disp.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for i, (gl, gr) in enumerate(grays):
        want = eng.match(IT.gray_to_bgr(gl), IT.gray_to_bgr(gr))
        E.same(f"pair {i}", d_disp[i].cpu().numpy(), want)
    del buf
    eng.close()


@pytest.mark.gpu
def test_default_path_unchanged(cone):
    """A NULL descriptor and a tight packed-BGR descriptor issue exactly the launches of adc_match_outputs_batch_device
    and give identical maps; any other format adds one launch per wave."""
    torch, dev = E.cuda()
    import adcensus_b200 as A
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option(), wave_pairs=4, lanes=3)
    n = 9
    waves = -(-n // eng.wave_pairs)
    d_l = torch.from_numpy(np.repeat(left[None], n, 0)).to(dev)
    d_r = torch.from_numpy(np.repeat(right[None], n, 0)).to(dev)
    rgb_l = torch.from_numpy(np.repeat(IT.from_bgr(left, "rgb")[None], n, 0)).to(dev)
    rgb_r = torch.from_numpy(np.repeat(IT.from_bgr(right, "rgb")[None], n, 0)).to(dev)
    st = torch.cuda.current_stream()
    side = {m: torch.empty((n, h, w), dtype=torch.uint8 if m == "outliers" else torch.float32, device=dev)
            for m in ("outliers", "peak_ratio")}
    maps = [(b.data_ptr(), m) for m, b in side.items()]

    def run(fn):
        d = torch.zeros((n, h, w), dtype=torch.float32, device=dev)
        c0 = eng.launch_count
        fn(d)
        torch.cuda.synchronize()
        return d.cpu().numpy(), {m: b.cpu().numpy() for m, b in side.items()}, eng.launch_count - c0

    m0, s0, l0 = run(lambda d: eng.match_outputs_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), maps=maps,
                                                              d_disp=d.data_ptr(), stream=st.cuda_stream))
    for image in (None, A.image_desc("bgr"), A.image_desc("bgr", 3 * w, 0, 3 * w * h)):
        m1, s1, l1 = run(lambda d: eng.match_images_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), image=image, maps=maps,
                                                                 d_disp=d.data_ptr(), stream=st.cuda_stream))
        assert l1 == l0
        E.same("map", m1, m0)
        for m in side:
            E.same(m, s1[m], s0[m])
    m2, s2, l2 = run(lambda d: eng.match_images_batch_device(n, rgb_l.data_ptr(), rgb_r.data_ptr(), image=A.image_desc("rgb"),
                                                             maps=maps, d_disp=d.data_ptr(), stream=st.cuda_stream))
    assert l2 == l0 + waves
    E.same("rgb map", m2, m0)
    m3, _, l3 = run(lambda d: eng.match_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), d.data_ptr(), st.cuda_stream))
    hashes = E.golden_hashes("cone_full")
    assert all(T.sha(m2[i]) == hashes["MEDIAN/DISP_L"] for i in range(n))
    E.same("plain batch", m3, m0)
    # the host entry: NULL descriptor = adc_match_outputs, launch for launch; gray / planar add one launch
    c0 = eng.launch_count
    d_a, _ = eng.match_outputs(left, right)
    la = eng.launch_count - c0
    c0 = eng.launch_count
    d_b, _ = eng.match_images(left, right, format="bgr")
    assert eng.launch_count - c0 == la
    E.same("host bgr", d_b, d_a)
    c0 = eng.launch_count
    d_c, _ = eng.match_images(IT.from_bgr(left, "rgb_planar"), IT.from_bgr(right, "rgb_planar"), format="rgb_planar")
    assert eng.launch_count - c0 == la + 1
    E.same("host planar", d_c, d_a)
    eng.close()


@pytest.mark.gpu
def test_size_dependent_image_rules():
    """Rules that need the image size fail after the engine check, with ADC_ERR_ARG naming the field, before any device
    work (no launch)."""
    torch, dev = E.cuda()
    import adcensus_b200 as A
    w, h, D = 33, 20, 16
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    L = A.load_library()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device=dev)
    out = torch.zeros((1, h, w), dtype=torch.float32, device=dev)
    p = buf.data_ptr()
    cases = [(_desc(A.IMG_RGB, row=3 * w - 1), b"img->row_pitch"), (_desc(A.IMG_BGRA, row=4 * w - 3), b"img->row_pitch"),
             (_desc(A.IMG_GRAY, row=w - 1), b"img->row_pitch"),
             (_desc(A.IMG_RGB_PLANAR, row=w + 2, plane=h * (w + 2) - 1), b"img->plane_pitch"),
             (_desc(A.IMG_GRAY, stride=h * w - 1), b"img->image_stride"),
             (_desc(A.IMG_RGB_PLANAR, stride=3 * h * w - 1), b"img->image_stride"),
             (_desc(A.IMG_BGR, row=3 * w + 4, stride=h * (3 * w + 4) - 1), b"img->image_stride"),
             (_desc(A.IMG_RGBA, row=1 << 62), b"img->row_pitch")]
    for img, msg in cases:
        c0 = eng.launch_count
        rc = L.adc_match_images_batch_device(eng._h, 1, p, p, ctypes.byref(img), None, 0, 0, out.data_ptr(), None, 0,
                                             None, 0, None)
        assert rc == 1 and msg in L.adc_last_error(), (img.format, L.adc_last_error())
        host = np.zeros(1 << 16, np.uint8)
        disp = np.zeros((h, w), np.float32)
        rc = L.adc_match_images(eng._h, host.ctypes.data, host.ctypes.data, ctypes.byref(img), None, 0, 0,
                                disp.ctypes.data, None, 0, None, 0)
        assert rc == 1 and msg in L.adc_last_error(), (img.format, L.adc_last_error())
        assert eng.launch_count == c0
    eng.close()
