"""The views as the engine matches them (adc_ingest_views, adc_ingest_views_batch_device): the packed BGR views stage 1
reads, for every format family, plain and through the rectification, handed to the caller; and the camera path from raw
frames to a coloured point cloud; and the ingestion kernel itself.

CPU: ptxas -v on every file that instantiates the ingestion kernel: each family file holds k_view_ingest for its own
codes x the four source geometries, every ADC_IMG_* code once per geometry across them, none with a stack frame, spills
or local memory; k_rectify.cu only its two map conversions.
GPU: views of BGRA side-by-side frames, planar RGB, NV12, YUYV, BayerRG8, Mono12 and BayerRG12p, plain and rectified,
with row pitches and image strides above tight and odd offsets, against the numpy restatements of the formats and of
cv::remap; the same views fed back as packed BGR match to the same final maps as the raw-format call; the host entry;
the rectified call without a rectification; launch counts; batches of more pairs than one launch takes, plain and
resized, against the restatements; raw BayerRG12p frames through ingest_views, the rectified match and a point cloud
coloured by the left views, against the host chain restated in numpy.
"""
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import adc_testlib as T
import bayer_testlib as B
import cloud_testlib as C
import engine_testlib as E
import images_testlib as IT
import rawdepth_testlib as RD
import rectify_testlib as R
import resize_testlib as RS
import yuv_testlib as Y
import yuv_video_testlib as V

FORMATS = ["bgra", "rgb_planar", "nv12", "yuyv", "bayer_rggb", "mono12", "bayer_rg12p"]
CSRC = T.REPO / "adcensus_b200" / "csrc"
GEOMETRIES = 4   # k_view_ingest's G: plain, remap, area, linear-exact

# The file that instantiates k_view_ingest for each code: the family files of img_format.h.
FAMILY_FILES = {
    "k_image.cu": sorted(IT.CODE.values()),
    "k_bayer.cu": sorted(B.CODE.values()),
    "k_yuv.cu": sorted(Y.CODE.values()),
    "k_yuv_encodings.cu": sorted(c | e for c in Y.CODE.values() for e in V.ENC.values() if e),
    "k_yuv_video.cu": sorted(c | e for c in V.CODE.values() for e in V.ENC.values()),
    "k_rawdepth.cu": sorted(RD.CODE.values()),
}


def test_ingestion_kernels_use_no_local_memory():
    """ptxas -v on each file that instantiates k_view_ingest<F, G> and on k_rectify.cu: no function has a stack frame,
    spills or local memory; each family file holds exactly its own codes x the four geometries, so that every code of
    ADC_IMG_CODES is instantiated once per geometry (268 kernels); k_rectify.cu holds its two map conversions only."""
    mk = (CSRC / "Makefile").read_text()
    files = [*FAMILY_FILES, "k_rectify.cu"]
    assert all(f in mk for f in files)
    with ThreadPoolExecutor(len(files)) as ex:
        reports = dict(zip(files, ex.map(lambda f: E.ptxas_report(CSRC / f), files)))
    for f, report in reports.items():
        assert all((k["stack"], k["spill_stores"], k["spill_loads"], k["lmem"]) == (0, 0, 0, 0)
                   for k in report.values()), (f, report)
    conv = reports.pop("k_rectify.cu")
    assert sorted(n for n, k in conv.items() if k["regs"] is not None) == sorted(conv) and len(conv) == 2
    assert all("k_remap_convert_" in n for n in conv), sorted(conv)
    every = []
    for f, codes in FAMILY_FILES.items():
        kernels = [n for n, k in reports[f].items() if k["regs"] is not None]
        got = [re.fullmatch(r"_Z\d+k_view_ingestILi(\d+)ELi(\d+)E.*", n) for n in kernels]
        assert all(got), (f, kernels)
        got = sorted((int(m.group(1)), int(m.group(2))) for m in got)
        assert got == sorted((c, g) for c in codes for g in range(GEOMETRIES)), f
        every += got
    want = sorted((RS.CODE[f] | e, g) for f in RS.CODE for e in ([0] + [e for e in V.ENC.values() if e]
                                                                  if f in V.ALL else [0]) for g in range(GEOMETRIES))
    assert sorted(every) == want and len(every) == 268


def _frame(rng, fmt, W, H):
    """A random raw view of `fmt` in the shape the host entries take."""
    if fmt == "bgra":
        return rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    if fmt == "rgb_planar":
        return rng.integers(0, 256, (3, H, W), dtype=np.uint8)
    if fmt == "bayer_rggb":
        return rng.integers(0, 256, (H, W), dtype=np.uint8)
    if fmt in Y.CODE:
        return Y.random_frame(rng, fmt, W, H)
    return RD.random_frame(rng, fmt, W, H)


def _decode(f, fmt, W, H):
    """The packed BGR [H][W][3] of one raw view (the restatements of each format family)."""
    if fmt == "bgra":
        return f[..., :3]
    if fmt == "rgb_planar":
        return np.stack([f[2], f[1], f[0]], -1)
    if fmt == "bayer_rggb":
        return B.demosaic(f, fmt)
    if fmt in Y.CODE:
        return Y.decode(f, fmt, W, H)
    return RD.decode(f, fmt, W, H)


def _rows(f, fmt):
    """The view's bytes as rows: planar planes one after the other, every other format row by row."""
    b = np.ascontiguousarray(f).view(np.uint8)
    return b.reshape(-1, b.shape[-1]) if fmt == "rgb_planar" else b.reshape(b.shape[0], -1)


def _device_frames(fmt, lefts, rights, H):
    """(buffer tensor, left offset, right offset, ImageDesc) holding the pairs at a row pitch and an image stride above
    tight, from an odd byte (even for the 16-bit container); BGRA pairs as side-by-side frames."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    even = fmt == "mono12"
    lead = 2 if even else 1
    rl = [_rows(f, fmt) for f in lefts]
    nrows, rb = rl[0].shape
    sbs = fmt == "bgra"
    pitch = (2 * rb if sbs else rb) + 6
    plane = H * pitch if fmt in ("rgb_planar", "nv12") else 0
    stride = (nrows * pitch + 10) if sbs else 2 * (nrows * pitch + 10)
    buf = np.full(lead + len(lefts) * stride + 16, 0x5a, np.uint8)
    for i, (l, r) in enumerate(zip(rl, [_rows(f, fmt) for f in rights])):
        for k, rows in enumerate((l, r)):
            base = lead + i * stride + (k * rb if sbs else k * (nrows * pitch + 10))
            for y in range(nrows):
                buf[base + y * pitch:base + y * pitch + rb] = rows[y]
    right_off = lead + (rb if sbs else nrows * pitch + 10)
    return torch.from_numpy(buf).to(dev), lead, right_off, A.image_desc(fmt, pitch, plane, stride)


def _device_views(eng, n, d, lo, ro, desc, rectified):
    torch, dev = E.cuda()
    N = eng.width * eng.height
    views, intact = E.guarded(6 * n * N, torch.uint8, 3, 5, 0xee)
    c0 = eng.launch_count
    eng.ingest_views_batch_device(n, d.data_ptr() + lo, d.data_ptr() + ro, views.data_ptr(), desc, rectified,
                                  torch.cuda.current_stream().cuda_stream)
    assert eng.launch_count == c0 + 1
    torch.cuda.synchronize()
    assert intact(), "a guard of the views was overwritten"
    return views


@pytest.mark.gpu
@pytest.mark.parametrize("rectified", [False, True])
@pytest.mark.parametrize("fmt", FORMATS)
def test_views_and_what_was_matched(fmt, rectified):
    """Three pairs of each format through the device entry, pitched: every view equals the format's restatement
    (rectified: then cv::remap restated).  The host entry gives pair 0's views.  Fed back as packed BGR, the views match
    to the final maps of the raw-format call bit for bit."""
    torch, dev = E.cuda()
    W, H, n, D = 64, 48, 3, 16
    sw, sh = (82, 61) if rectified else (W, H)
    rng = np.random.default_rng(len(fmt) + 10 * rectified)
    eng = E.engine(W, H, T.default_option(max_disparity=D))
    if rectified:
        maps = [R.warp_maps(W, H, sw, sh, s, specials=False) for s in (1, 2)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
    lefts = [_frame(rng, fmt, sw, sh) for _ in range(n)]
    rights = [_frame(rng, fmt, sw, sh) for _ in range(n)]
    d, lo, ro, desc = _device_frames(fmt, lefts, rights, sh)
    views = _device_views(eng, n, d, lo, ro, desc, rectified)
    got = views.cpu().numpy().reshape(n, 2, H, W, 3)
    for i in range(n):
        for k, f in enumerate((lefts[i], rights[i])):
            want = _decode(f, fmt, sw, sh)
            if rectified:
                want = R.remap(want, *maps[k])
            assert np.array_equal(got[i, k], want), f"{fmt} pair {i} view {k}"
    host = eng.ingest_views(lefts[0], rights[0], fmt, rectified)
    assert np.array_equal(host, got[0])
    # what was matched: the views as tight packed BGR give the raw-format call's maps
    import adcensus_b200 as A
    N = W * H
    raw_disp = torch.full((n, H, W), -7.0, device=dev)
    bgr_disp = torch.full((n, H, W), -7.0, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    call = eng.match_rectified_batch_device if rectified else eng.match_images_batch_device
    call(n, d.data_ptr() + lo, d.data_ptr() + ro, image=desc, d_disp=raw_disp.data_ptr(), stream=st)
    eng.match_images_batch_device(n, views.data_ptr(), views.data_ptr() + 3 * N, image=A.image_desc("bgr", 0, 0, 6 * N),
                                  d_disp=bgr_disp.data_ptr(), stream=st)
    torch.cuda.synchronize()
    assert np.isfinite(raw_disp.cpu().numpy()).mean() > 0.2
    assert torch.equal(raw_disp.view(torch.int32), bgr_disp.view(torch.int32)), fmt
    eng.close()


@pytest.mark.gpu
def test_errors_and_launch_counts():
    """The rectified entries without a rectification fail with ADC_ERR_ARG; a plain call of n pairs is one launch, the
    host entry one, n = 0 none; rectified not 0 / 1 and a NULL destination fail before the engine is used."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    W, H = 40, 30
    eng = E.engine(W, H, T.default_option(max_disparity=8))
    img = torch.zeros((5, 2, H, W, 3), dtype=torch.uint8, device=dev)
    out = torch.empty_like(img)
    st = torch.cuda.current_stream().cuda_stream
    with pytest.raises(A.AdcError, match="no rectification is set"):
        eng.ingest_views_batch_device(5, img.data_ptr(), img.data_ptr() + 3 * W * H, out.data_ptr(),
                                      A.image_desc("bgr", 0, 0, 6 * W * H), True, st)
    L = A.load_library()
    assert L.adc_ingest_views_batch_device(eng._h, 1, img.data_ptr(), img.data_ptr(), None, 2, out.data_ptr(), st) == 1
    assert b"rectified 2 is not 0 or 1" in L.adc_last_error()
    assert L.adc_ingest_views_batch_device(eng._h, 1, img.data_ptr(), img.data_ptr(), None, 0, None, st) == 1
    assert b"views is NULL" in L.adc_last_error()
    c0 = eng.launch_count
    eng.ingest_views_batch_device(5, img.data_ptr(), img.data_ptr() + 3 * W * H, out.data_ptr(),
                                  A.image_desc("bgr", 0, 0, 6 * W * H), False, st)
    eng.ingest_views_batch_device(0, img.data_ptr(), img.data_ptr(), out.data_ptr(), None, False, st)
    assert eng.launch_count == c0 + 1
    torch.cuda.synchronize()
    assert torch.equal(out, img)
    with pytest.raises(A.AdcError, match="no rectification is set"):
        eng.ingest_views(np.zeros((H, W, 3), np.uint8), np.zeros((H, W, 3), np.uint8), "bgr", rectified=True)
    c0 = eng.launch_count
    eng.ingest_views(np.zeros((H, W, 3), np.uint8), np.zeros((H, W, 3), np.uint8), "bgr")
    assert eng.launch_count == c0 + 1
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("geometry", ["plain", "area", "linear_exact"])
@pytest.mark.parametrize("fmt", ["bgr", "bayer_rggb"])
def test_more_pairs_than_one_launch(fmt, geometry):
    """65535 + 9 pairs of 8 x 4 views through adc_ingest_views_batch_device, plain and resized (2 x 2 AREA, 13 x 7
    LINEAR_EXACT): two launches, and every pair equals the restatement of its frames (the format's conversion, then the
    resize).  Pair i takes frames i mod 509 and (i + 254) mod 509 of 509 distinct random frames, so a pair read from or
    written to another pair's place fewer than 509 pairs away, in either launch, shows."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    W, H, n, P = 8, 4, 65535 + 9, 509
    sw, sh = {"plain": (W, H), "area": (2 * W, 2 * H), "linear_exact": (13, 7)}[geometry]
    rng = np.random.default_rng(len(fmt) + len(geometry))
    eng = E.engine(W, H, T.default_option(max_disparity=4), wave_pairs=2, lanes=1)
    if geometry != "plain":
        eng.set_resize((sw, sh), geometry)
    frames = [RS.random_frame(rng, fmt, sw, sh) for _ in range(P)]
    want = [RS.decode(f, fmt, sw, sh) for f in frames]
    if geometry != "plain":
        want = [RS.resize(b, W, H, RS.AREA if geometry == "area" else RS.LINEAR_EXACT) for b in want]
    want = np.stack(want)
    raw = np.stack([np.ascontiguousarray(f).reshape(-1) for f in frames])   # tight frames, one per row
    li = np.arange(n) % P
    ri = (li + P // 2) % P
    left, right = (torch.from_numpy(raw[k]).to(dev) for k in (li, ri))
    views, intact = E.guarded(6 * n * W * H, torch.uint8, 3, 5, 0xee)
    c0 = eng.launch_count
    eng.ingest_views_batch_device(n, left.data_ptr(), right.data_ptr(), views.data_ptr(),
                                  A.image_desc(fmt, 0, 0, raw.shape[1]), geometry != "plain",
                                  torch.cuda.current_stream().cuda_stream)
    assert eng.launch_count == c0 + 2
    torch.cuda.synchronize()
    assert intact(), "a guard of the views was overwritten"
    got = views.cpu().numpy().reshape(n, 2, H, W, 3)
    assert np.array_equal(got[:, 0], want[li]) and np.array_equal(got[:, 1], want[ri])
    eng.close()


@pytest.mark.gpu
def test_camera_path_to_coloured_cloud(cone):
    """Raw BayerRG12p 640 x 480 frames of Cone through the rig's maps: ingest_views, the rectified match and a point
    cloud coloured by the left views (stride 6*H*W), against the host chain restated in numpy (unpack, demosaic at full
    depth, reduce, remap; reproject and mask)."""
    cv2 = pytest.importorskip("cv2")
    torch, dev = E.cuda()
    left, right = cone
    h, w, _ = left.shape
    sw, sh, n = 640, 480, 2
    fmt = "bayer_rg12p"
    rng = np.random.default_rng(12)
    frames = [RD.encode(cv2.resize(img, (sw, sh), interpolation=cv2.INTER_AREA), fmt, rng) for img in (left, right)]
    eng = E.engine(w, h, T.default_option(max_disparity=64))
    maps = [R.cone_rig(cv2, sw, sh, w, h, cv2.CV_16SC2, s) for s in (1, -1)]
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    views = eng.ingest_views(frames[0], frames[1], fmt, rectified=True)
    want = [R.remap(RD.decode(f, fmt, sw, sh), *maps[k]) for k, f in enumerate(frames)]
    assert np.array_equal(views[0], want[0]) and np.array_equal(views[1], want[1])
    N = w * h
    d, lo, ro, desc = _device_frames(fmt, [frames[0]] * n, [frames[1]] * n, sh)
    dv = _device_views(eng, n, d, lo, ro, desc, True)
    disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    eng.match_rectified_batch_device(n, d.data_ptr() + lo, d.data_ptr() + ro, image=desc, d_disp=disp.data_ptr(),
                                     stream=st)
    Q = np.load(T.GOLDEN_DIR / "golden_reproject_cases.npz")["rig_zero_0/Q"]
    pts = torch.empty((n, N, 3), dtype=torch.float32, device=dev)
    cols = torch.empty((n, N, 3), dtype=torch.uint8, device=dev)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    wb = eng.point_cloud_workspace_bytes(n)
    work = torch.empty(wb // 8 + 1, dtype=torch.int64, device=dev)
    eng.point_cloud_batch_device(n, disp.data_ptr(), Q, pts.data_ptr(), counts.data_ptr(), N, work.data_ptr(), wb,
                                 d_bgr=dv.data_ptr(), bgr_stride=6 * N, d_colors=cols.data_ptr(), stream=st)
    torch.cuda.synchronize()
    host_disp, _ = eng.match_rectified(frames[0], frames[1], fmt)
    assert np.array_equal(E.bits(host_disp), E.bits(disp[0].cpu().numpy()))
    assert np.array_equal(E.bits(eng.match(views[0], views[1])), E.bits(host_disp))
    wp, wc, _ = C.cloud(host_disp, Q, want[0])
    assert len(wp) > N // 2
    for i in range(n):
        k = int(counts[i])
        assert k == len(wp)
        assert np.array_equal(E.bits(pts[i, :k].cpu().numpy()), E.bits(wp))
        assert np.array_equal(cols[i, :k].cpu().numpy(), wc)
    eng.close()
