"""SURVEY.md 8(f) ranks 3 and 4: the output side of the reference's demo (main.cpp:147-230) and an accuracy harness
against the Middlebury ground truth of the bundled Cone pair.

The CPU restatement of the demo's arithmetic is maps_testlib.gray8 (a dozen lines of float32 numpy, each citing main.cpp);
the JET table is compared with the OpenCV build in this image (`cv2.applyColorMap`)."""
import numpy as np
import pytest

import adc_testlib as T
import maps_testlib as MT


def _bad_pixel_rates(disp: np.ndarray, gt_u8: np.ndarray):
    """Middlebury quarter-size set: true disparity = value / 4, 0 = unknown.  Invalid pixels count as bad."""
    known = gt_u8 > 0
    truth = gt_u8.astype(np.float32) / 4.0
    err = np.abs(np.where(np.isinf(disp), np.float32(1e9), disp) - truth)
    return {t: float((err[known] > t).mean()) for t in (1.0, 2.0)}


def test_cone_accuracy_of_the_reference_map():
    """Guards against being bit-exact to a mis-built oracle: the reference's own Cone map (golden fixture generated
    from the unmodified sources) must be a reasonable stereo result, and the numbers are pinned."""
    gt = np.load(T.GOLDEN_DIR / "cone_gt.npz")["disp2"]
    ref = np.load(T.GOLDEN_DIR / "golden_cone_full.npz")["MEDIAN__DISP_L"]
    r = _bad_pixel_rates(ref, gt)
    assert 0.05 < r[1.0] < 0.15 and r[2.0] < r[1.0], r     # SURVEY 8f: about 10 % bad > 1 px on Cone
    want = T.Oracle(450, 375).match(*T.load_cone())
    assert _bad_pixel_rates(want, gt) == r                  # the C restatement gives the very same map


@pytest.mark.gpu
def test_cone_accuracy_on_gpu(cone):
    import adcensus_b200 as A
    left, right = cone
    gt = np.load(T.GOLDEN_DIR / "cone_gt.npz")["disp2"]
    ref = np.load(T.GOLDEN_DIR / "golden_cone_full.npz")["MEDIAN__DISP_L"]
    eng = A.Engine(450, 375, A.ADCensusOption())
    got = eng.match(left, right)
    assert _bad_pixel_rates(got, gt) == _bad_pixel_rates(ref, gt)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cone", "synthetic_with_invalid", "constant"])
def test_render_and_cloud(case, cone):
    import cv2
    import adcensus_b200 as A
    if case == "cone":
        left, _ = cone
        disp = np.load(T.GOLDEN_DIR / "golden_cone_full.npz")["WTA__DISP_L"].copy()   # has invalid pixels and sub-pixel values
    elif case == "synthetic_with_invalid":
        rng = np.random.default_rng(5)
        left = rng.integers(0, 256, (61, 97, 3), dtype=np.uint8)
        disp = (rng.random((61, 97), dtype=np.float32) * 40 - 3).astype(np.float32)    # some negative: the demo takes abs()
        disp[rng.random((61, 97)) < 0.2] = np.inf
    else:
        left = np.full((40, 50, 3), 7, np.uint8)
        disp = np.full((40, 50), 12.5, np.float32)
    h, w = disp.shape
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=64))
    gray, jet, (mn, mx) = eng.render_disparity(disp)
    want_gray, wmn, wmx = MT.gray8(disp, w)
    assert (mn, mx) == (wmn, wmx)
    assert np.array_equal(gray, want_gray)
    assert np.array_equal(jet, cv2.applyColorMap(want_gray, cv2.COLORMAP_JET))
    cloud = eng.disparity_cloud(left, disp)
    ys, xs = np.nonzero(~np.isinf(disp))                    # raster order
    want = np.stack([xs, ys, np.abs(disp[ys, xs]), left[ys, xs, 2], left[ys, xs, 1], left[ys, xs, 0]], 1).astype(np.float32)
    assert cloud.shape == want.shape and np.array_equal(cloud, want)
    eng.close()


# ---- the author's published result images (doc/exp/res/*-d.png): the only known-answer data the reference holds -----
# SaveDisparityMap's 8-bit normalisation (main.cpp:180-206) of the author's own MSVC run.  Weak pins (8-bit, min/max
# normalised, another libm): SURVEY.md 4.2 measured 99.4 % of the Cone pixels within +-1 grey level for the glibc build of
# the reference.  The Piano image was evidently produced with other settings than the bundled d_range.txt (85 %); it is
# kept as a loose sanity bound only.
_DOC_PINS = {"cone": ("doc_cone_d", 0.99), "cloth3": ("doc_cloth_d", 0.98), "piano": ("doc_piano_d", 0.80)}
# Middlebury 2006 half-size ground truth of the bundled Cloth3 / Wood2 pairs: true disparity = value / 2, 0 = unknown
_GT_SCALE = {"cone": 4.0, "cloth3": 2.0, "wood2": 2.0}


def _reference_map(name):
    if name == "cone":
        return np.load(T.GOLDEN_DIR / "golden_cone_full.npz")["MEDIAN__DISP_L"]
    return np.load(T.GOLDEN_DIR / "real_pairs.npz")[f"{name}_final"]


def _bad_rates(disp, gt_u8, scale):
    known = gt_u8 > 0
    truth = gt_u8.astype(np.float32) / np.float32(scale)
    err = np.abs(np.where(np.isinf(disp), np.float32(1e9), disp) - truth)
    return {t: float((err[known] > t).mean()) for t in (1.0, 2.0)}


@pytest.mark.parametrize("name", ["cone", "cloth3", "piano"])
def test_reference_maps_match_the_authors_published_images(name):
    """CPU side of the pin: the unmodified reference's maps (golden fixtures), normalised as main.cpp does."""
    key, thr = _DOC_PINS[name]
    doc = np.load(T.GOLDEN_DIR / "real_pairs.npz")[key]
    ref = _reference_map(name)
    g, _, _ = MT.gray8(ref, ref.shape[1])
    within1 = float((np.abs(g.astype(np.int32) - doc.astype(np.int32)) <= 1).mean())
    assert within1 >= thr, f"{name}: only {within1:.4f} of the pixels within +-1 grey level of the author's image"


@pytest.mark.parametrize("name", ["cloth3", "wood2"])
def test_reference_accuracy_on_the_other_ground_truths(name):
    gt = np.load(T.GOLDEN_DIR / "real_pairs.npz")[f"{name}_gt"]
    r = _bad_rates(_reference_map(name), gt, _GT_SCALE[name])
    assert r[2.0] < r[1.0] < 0.25, r          # Cloth3 9.3 % / 3.7 %, Wood2 20.1 % / 7.1 % bad pixels (> 1 px / > 2 px)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cone", "cloth3", "piano", "wood2"])
def test_gpu_maps_through_the_demo_output_path(name):
    """SURVEY.md 8(f) ranks 3 and 4 pinned to what the reference holds: the GPU map of each bundled pair goes through
    adc_render_disparity (the demo's 8-bit normalisation, on the device) and must (a) equal the numpy restatement of
    main.cpp:180-206, (b) match the author's published image as well as the reference's own map does, (c) have the
    reference's bad-pixel rates against the Middlebury ground truth."""
    import adcensus_b200 as A
    z = np.load(T.GOLDEN_DIR / "real_pairs.npz")
    if name == "cone":
        left, right = T.load_cone()
        dmax, gt = 64, np.load(T.GOLDEN_DIR / "cone_gt.npz")["disp2"]
    else:
        left, right = z[f"{name}_left"], z[f"{name}_right"]
        dmax, gt = (64 if name == "piano" else 128), (z[f"{name}_gt"] if f"{name}_gt" in z else None)
    h, w, _ = left.shape
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=dmax))
    got = eng.match(left, right)
    ref = _reference_map(name)
    assert got.view(np.uint32).tobytes() == ref.view(np.uint32).tobytes()
    gray, jet, (mn, mx) = eng.render_disparity(got)
    want, wmn, wmx = MT.gray8(ref, w)
    assert np.array_equal(gray, want) and (mn, mx) == (wmn, wmx)
    if name in _DOC_PINS:
        key, thr = _DOC_PINS[name]
        within1 = float((np.abs(gray.astype(np.int32) - z[key].astype(np.int32)) <= 1).mean())
        assert within1 >= thr, f"{name}: {within1:.4f}"
    if gt is not None:
        assert _bad_rates(got, gt, _GT_SCALE[name]) == _bad_rates(ref, gt, _GT_SCALE[name])
    eng.close()
