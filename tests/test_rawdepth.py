"""High-bit-depth mono and Bayer frames (ADC_IMG_MONO10 ... ADC_IMG_BAYER_GB12P): 10-, 12- and 16-bit samples in 16-bit
words or in the PFNC 10p / 12p bit streams, matched exactly as the unpacked CV_16UC1 frame through cv2.cvtColor (Bayer)
and convertTo(CV_8U, 2^-s) followed by the packed-BGR entry point, with or without rectification.

CPU: the numpy restatement (rawdepth_testlib) against live OpenCV with the optimised paths on and off (skipped without
OpenCV) and against the committed fixture, composed with rectify_testlib's cv2.remap (never skipped); the bit streams
against byte vectors written out from the PFNC definition; the corners of the depth reduction; the argument rules that
need no engine; the constants and the view parser.
GPU: Cone synthesised at 12 bits in all five containers, as a mosaic and as mono, against the CPU oracle on the restated
8-bit image; batches (odd sizes, pitches and strides above tight, a leading offset, pipelined and not), side-by-side
frames and crops at the allowed offsets, the host entries, raw frames through both map types down to 1 x 1, the
size-dependent rules and launch counts, every output against adc_match_outputs_batch_device on the restated images.
"""
import ctypes
import re

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E
import rawdepth_testlib as X
import rectify_testlib as R

ROOT = T.REPO
MAPS = ["wta_left", "wta_right", "outliers", "min_cost", "peak_ratio"]
VOLS = ["cost", "aggr", "opt"]
GOLDEN = T.GOLDEN_DIR / "golden_rawdepth_cases.npz"
CONTAINERS = [s for s, _, _ in X.CONTAINERS]


# ---- CPU ------------------------------------------------------------------------------------------
def test_restatement_against_fixture():
    """The restatement reproduces every OpenCV output in the fixture: every format at 1 x 1, 2 x 5, 3 x 3, 5 x 7 and
    random sizes (uniform samples and the reduction's corner values), and, composed with the remap restatement, decode
    -> remap for both map types, down to 1 x N, 2 x 2 and 1 x 1 frames."""
    z = np.load(GOLDEN)
    name_of = {v: k for k, v in X.CODE.items()}
    seen = set()
    for name in sorted({k.split("/")[0] for k in z.files}):
        w, h = (int(v) for v in z[f"{name}/size"])
        fmt = name_of[int(z[f"{name}/format"])]
        got = X.decode(z[f"{name}/frame"], fmt, w, h)
        if f"{name}/map1" in z.files:
            got = R.remap(got, z[f"{name}/map1"], z[f"{name}/map2"])
        assert np.array_equal(got, z[f"{name}/out"]), name
        seen.add((name.split("_")[0], fmt))
    for kind in ("tiny", "odd"):
        assert {f for k, f in seen if k == kind} == set(X.NAMES), kind
    assert len({f for k, f in seen if k == "rect"}) == 10


def test_restatement_against_opencv():
    """The restatement against live cv2.cvtColor on uint16 + cv2.convertScaleAbs with the optimised paths on and off:
    every format at 1 x 1, 2 x 5, 3 x 3, odd x odd and 40 random sizes per setting, a third of them drawn from the
    reduction's corner values; every 16-bit value through the mono reduction; 1080 x 1920 BayerRG12p."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(33)
    opt = cv2.useOptimized()
    try:
        for use in (True, False):
            cv2.setUseOptimized(use)
            sizes = [(1, 1), (5, 2), (3, 3), (7, 5), (33, 21)] + [tuple(int(v) for v in rng.integers(1, 120, 2))
                                                                  for _ in range(40)]
            for i, (w, h) in enumerate(sizes):
                for fmt in X.NAMES:
                    frame = X.random_frame(rng, fmt, w, h, corners=i % 3 == 2)
                    assert np.array_equal(X.decode(frame, fmt, w, h), X.cv_decode(cv2, frame, fmt, w, h)), (use, fmt, w, h)
            every = np.arange(65536, dtype=np.uint16).reshape(256, 256)
            for fmt in ("mono10", "mono12", "mono16"):
                assert np.array_equal(X.decode(every, fmt, 256, 256), X.cv_decode(cv2, every, fmt, 256, 256)), (use, fmt)
            frame = X.random_frame(rng, "bayer_rg12p", 1920, 1080)
            assert np.array_equal(X.decode(frame, "bayer_rg12p", 1920, 1080),
                                  X.cv_decode(cv2, frame, "bayer_rg12p", 1920, 1080)), use
    finally:
        cv2.setUseOptimized(opt)


def test_demosaic_then_reduce_is_not_reduce_then_demosaic():
    """The order the header fixes matters: reducing the mosaic first and demosaicing at 8 bits differs in the last bit."""
    raw = np.array([[0, 0, 0], [16, 0, 0], [0, 0, 0]], np.uint16)   # GB mosaic: the centre is a G site between two R sites
    assert X.decode(raw, "bayer_gb12", 3, 3)[1, 1, 2] == 0           # R = (16 + 0 + 1) >> 1 = 8, to8(8) = 0 (0.5 to even)
    assert (int(X.to8(16, 4)) + int(X.to8(0, 4)) + 1) >> 1 == 1      # to8(16) = 1, to8(0) = 0: (1 + 0 + 1) >> 1 = 1


def test_bit_streams_by_hand():
    """A 12p and a 10p row whose bytes are written out from the PFNC definition (W not a multiple of the group),
    unpack(pack(v)) == v, and the last-byte property: sample W - 1 ends in the last byte of the tight row, so that
    nothing past ceil(b * W / 8) bytes is read."""
    # Mono12p, W = 3: p0 = 0xABC, p1 = 0x123, p2 = 0xFED.  byte0 = p0[7:0], byte1 = p0[11:8] | p1[3:0] << 4,
    # byte2 = p1[11:4], byte3 = p2[7:0], byte4 = p2[11:8] (high nibble unused)
    v12 = np.array([[0xABC, 0x123, 0xFED]])
    b12 = np.array([[0xBC, 0x3A, 0x12, 0xED, 0x0F]], np.uint8)
    assert np.array_equal(X.pack(v12, 12), b12) and np.array_equal(X.unpack(b12, 12, 3), v12)
    b12[0, 4] |= 0xF0   # the unused bits are ignored
    assert np.array_equal(X.unpack(b12, 12, 3), v12)
    # Mono10p, W = 6: p = 0x3FF, 0x000, 0x2AA, 0x155, 0x201, 0x1FE.  Bits are laid LSB first:
    # byte0 = p0[7:0]; byte1 = p0[9:8] | p1[5:0] << 2; byte2 = p1[9:6] | p2[3:0] << 4; byte3 = p2[9:4] | p3[1:0] << 6;
    # byte4 = p3[9:2]; byte5 = p4[7:0]; byte6 = p4[9:8] | p5[5:0] << 2; byte7 = p5[9:6]
    v10 = np.array([[0x3FF, 0x000, 0x2AA, 0x155, 0x201, 0x1FE]])
    b10 = np.array([[0xFF, 0x03, 0xA0, 0x6A, 0x55, 0x01, 0xFA, 0x07]], np.uint8)
    assert np.array_equal(X.pack(v10, 10), b10) and np.array_equal(X.unpack(b10, 10, 6), v10)
    rng = np.random.default_rng(5)
    for bits in (10, 12):
        for w in range(1, 19):
            v = rng.integers(0, 1 << bits, (3, w))
            rows = X.pack(v, bits)
            assert rows.shape == (3, (bits * w + 7) // 8)
            assert np.array_equal(X.unpack(rows, bits, w), v)
            assert ((w - 1) * bits >> 3) + 1 == rows.shape[1] - 1   # row[k + 1] of the last sample is the last byte


def test_to8_corners():
    """Every half-way value of the reduction for s = 2, 4 and 8 rounds to the even neighbour (both parities), the
    depth's largest values give 255, and words above the nominal depth saturate."""
    for s in (2, 4, 8):
        q = np.arange(0, 255)
        halfway = (q << s) + (1 << (s - 1))
        assert np.array_equal(X.to8(halfway, s), q + (q & 1)), s
        assert np.array_equal(X.to8(halfway - 1, s), q) and np.array_equal(X.to8(halfway + 1, s), q + 1), s
        assert X.to8((255 << s) + (1 << (s - 1)), s) == 255
    assert X.to8(1023, 2) == 255 and X.to8(4095, 4) == 255 and X.to8(65535, 8) == 255
    assert X.to8(1021, 2) == 255 and X.to8(1018, 2) == 254          # 254.5 -> 254 (even)
    assert X.to8(1024, 2) == 255 and X.to8(4096, 4) == 255 and X.to8(65535, 2) == 255 and X.to8(65535, 4) == 255
    assert X.to8(0, 8) == 0 and X.to8(128, 8) == 0 and X.to8(129, 8) == 1 and X.to8(384, 8) == 2


def test_rawdepth_argument_errors_need_no_gpu():
    """The twenty-five codes pass the size-free rules and reach the engine check on both image and both rectified
    entries; plane_pitch and reserved must be zero; on the device entries an odd pointer, row pitch or image stride is
    refused for the 16-bit containers and accepted for the packed ones, and the host entries take odd pointers; 63 and 89
    stay unknown."""
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    L = A.load_library()
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data

    def host(fn):
        return lambda img, l=p, r=p: getattr(L, fn)(None, l, r, img, None, 0, 0, p, None, 0, None, 0)

    def device(fn):
        return lambda img, l=p, r=p: getattr(L, fn)(None, 1, l, r, img, None, 0, 0, p, None, 0, None, 0, None)

    entries = {"adc_match_images:": host("adc_match_images"), "adc_match_rectified:": host("adc_match_rectified"),
               "adc_match_images_batch_device": device("adc_match_images_batch_device"),
               "adc_match_rectified_batch_device": device("adc_match_rectified_batch_device")}
    for fn, call in entries.items():
        dev = fn.endswith("device")
        for name, code in X.CODE.items():
            words = not X.info(name)[2]
            for d in (A.ImageDesc(code, 0, 0, 0, 0), A.ImageDesc(code, 0, 1002, 0, 1 << 33)):
                assert call(ctypes.byref(d)) == 1 and b"engine is NULL" in L.adc_last_error(), (fn, code)
            assert call(ctypes.byref(A.ImageDesc(code, 0, 0, 64, 0))) == 1
            assert b"img->plane_pitch must be 0" in L.adc_last_error() and fn.encode() in L.adc_last_error()
            assert call(ctypes.byref(A.ImageDesc(code, 1, 0, 0, 0))) == 1 and b"img->reserved" in L.adc_last_error()
            odd = [("d_left", dict(l=p + 1), A.ImageDesc(code, 0, 0, 0, 0)),
                   ("d_right", dict(r=p + 1), A.ImageDesc(code, 0, 0, 0, 0)),
                   ("img->row_pitch 1001", {}, A.ImageDesc(code, 0, 1001, 0, 0)),
                   ("img->image_stride 8001", {}, A.ImageDesc(code, 0, 0, 0, 8001))]
            for what, kw, d in odd:
                assert call(ctypes.byref(d), **kw) == 1
                err = L.adc_last_error()
                if dev and words:
                    assert what.encode() in err and fn.encode() in err and b"16-bit format" in err, err
                else:
                    assert b"engine is NULL" in err, err
        for code in (63, 89, -64):
            assert call(ctypes.byref(A.ImageDesc(code, 0, 0, 0, 0))) == 1
            err = L.adc_last_error()
            assert f"img->format {code} unknown".encode() in err and fn.encode() in err, err
    with pytest.raises(ValueError):
        A.image_desc("mono14")


def test_rawdepth_constants():
    import adcensus_b200 as A
    assert {k: v[0] for k, v in A.RAW_DEPTH_FORMATS.items()} == X.CODE
    for name, (code, bits, container) in A.RAW_DEPTH_FORMATS.items():
        colour, b, packed = X.info(name)
        assert (bits, container) == (b, "p" if packed else "u16")
        assert getattr(A, "IMG_" + name.upper()) == code
        c_name = "ADC_IMG_" + name.upper()
        assert re.search(rf"\b{c_name} = {code}\b", (ROOT / "include" / "adcensus_b200.h").read_text()), c_name
        assert A.image_desc(name, 200, 0, 9000).format == code
    assert not set(A.RAW_DEPTH_FORMATS) & (set(A.engine.IMG_FORMATS) | set(A.BAYER_FORMATS) | set(A.YUV_FORMATS))
    P = A.engine._image_view_desc
    frame = np.zeros((9, 80), np.uint16)
    for fmt in (A.IMG_MONO12, A.IMG_BAYER_RG10, A.IMG_BAYER_GB16):
        d = P(frame[:, 40:], fmt, 9, 40)   # the right half of a side-by-side frame
        assert (d.format, d.row_pitch, d.plane_pitch) == (fmt, 160, 0)
        with pytest.raises(ValueError):
            P(frame.view(np.uint8)[:, :80], fmt, 9, 40)
        with pytest.raises(ValueError):
            P(frame[:, ::2], fmt, 9, 40)
    rows = np.zeros((9, 120), np.uint8)
    assert P(rows[:, 60:], A.IMG_BAYER_RG12P, 9, 40).row_pitch == 120          # 40 samples = 60 bytes
    assert P(rows[:, 50:97], A.IMG_MONO10P, 9, 37).row_pitch == 120            # ceil(370 / 8) = 47 bytes
    with pytest.raises(ValueError):
        P(rows[:, :46], A.IMG_MONO10P, 9, 37)
    with pytest.raises(ValueError):
        P(frame[:, :40], A.IMG_MONO12P, 9, 40)


# ---- GPU ------------------------------------------------------------------------------------------
def _batch(fmt, n, vw, vh, rng, extra_row, extra_stride, lead, corners=False):
    """n pairs of random frames laid out with row pitch tight + extra_row, image stride H * row pitch + extra_stride,
    `lead` bytes before the first view, random bytes everywhere else, one device buffer per view whose last view's last
    row ends the buffer.  (views, desc, left frames, right frames)."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    rp = X.tight_row(fmt, vw) + extra_row
    stride = vh * rp + extra_stride
    L = [X.random_frame(rng, fmt, vw, vh, corners) for _ in range(n)]
    Rr = [X.random_frame(rng, fmt, vw, vh, corners) for _ in range(n)]
    views = []
    for frames in (L, Rr):
        big = rng.integers(0, 256, size=lead + (n - 1) * stride + (vh - 1) * rp + X.tight_row(fmt, vw), dtype=np.uint8)
        for i in range(n):
            X.write_view(big, frames[i], fmt, vw, vh, rp, lead + i * stride)
        views.append(torch.from_numpy(big).to(dev))
    return views, A.image_desc(fmt, rp, 0, stride), L, Rr


def _packed(frames, fmt, w, h, maps=None):
    torch, dev = E.cuda()
    imgs = [X.decode(f, fmt, w, h) for f in frames]
    if maps is not None:
        imgs = [R.remap(x, *maps) for x in imgs]
    return torch.from_numpy(np.stack(imgs)).to(dev)


def _equal_all(got, want, name):
    for k in want:
        assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), f"{name}: {k}"


@pytest.mark.gpu
def test_rawdepth_cone_against_oracle(cone):
    """Cone (450 x 375) synthesised at 12 bits (the 8-bit image x 16 plus seeded low bits), as an RG mosaic and as mono,
    in all five containers (10-bit containers take the samples >> 2, the 16-bit one the samples << 4, MSB-aligned) with a
    row pitch above tight: the final map equals the CPU oracle run on the restated 8-bit images, bit for bit."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option())
    oracle = T.Oracle(w, h, T.default_option())
    st = torch.cuda.current_stream()
    wants = {}
    for colour in ("bayer_rg", "mono"):
        rng = np.random.default_rng(12)
        v12 = [X.samples(X.encode(img, colour + "12", rng), colour + "12", w, h) for img in (left, right)]
        for suffix, bits, packed in X.CONTAINERS:
            fmt = colour + suffix
            frames = [X.from_samples(v >> 2 if bits == 10 else v << 4 if bits == 16 else v, fmt) for v in v12]
            rp = X.tight_row(fmt, w) + 10
            bufs = []
            for f in frames:
                host = np.zeros(2 * h * rp, np.uint8)
                for i in range(2):
                    X.write_view(host, f, fmt, w, h, rp, i * h * rp)
                bufs.append(torch.from_numpy(host).to(dev))
            d_o = torch.empty((2, h, w), dtype=torch.float32, device=dev)
            eng.match_images_batch_device(2, bufs[0].data_ptr(), bufs[1].data_ptr(), image=A.image_desc(fmt, rp),
                                          d_disp=d_o.data_ptr(), stream=st.cuda_stream)
            torch.cuda.synchronize()
            imgs = [X.decode(f, fmt, w, h) for f in frames]
            key = b"".join(x.tobytes() for x in imgs)
            if key not in wants:
                wants[key] = oracle.match(*imgs)
            got = d_o.cpu().numpy()
            E.same(f"cone {fmt} pair 0", got[0], wants[key])
            E.same(f"cone {fmt} pair 1", got[1], wants[key])
    assert len(wants) == 5   # mono 12 = 12p = 16, mono 10 = 10p; mosaic 12 = 12p, 10 = 10p, 16 on its own
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_rawdepth_batched(pipelined):
    """wave_pairs = 4, lanes = 3, n = 14 (several waves per lane, a partial last wave), odd W and H, every format with
    row pitch and image stride above tight and a leading offset (odd for the packed containers), corner-valued samples
    in every third format: every output equals adc_match_outputs_batch_device on the restated BGR images, and the source
    buffers are unchanged."""
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=3)
    n = 3 * eng.wave_pairs + 2
    rng = np.random.default_rng(9)
    for k, fmt in enumerate(X.NAMES):
        packed = X.info(fmt)[2]
        lead = (0, 3, 1, 6, 13)[k % 5] if packed else (0, 2, 6, 14, 4)[k % 5]
        views, desc, L, Rr = _batch(fmt, n, w, h, rng, (0, 7, 64, 1, 3)[k % 5] * (1 if packed else 2),
                                    (5, 0, 3, 11, 0)[k % 5] * (1 if packed else 2), lead, corners=k % 3 == 1)
        before = [t.clone() for t in views]
        full = k % 5 in (0, 1)   # every volume for mono and RG of each container, the optimised one elsewhere
        outputs = dict(volumes=[(v, "hwd", "f32") for v in (VOLS if full else ["opt"])], maps=MAPS, pipelined=pipelined)
        pl, pr = _packed(L, fmt, w, h), _packed(Rr, fmt, w, h)
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_images_batch_device, n, views[0].data_ptr() + lead,
                              views[1].data_ptr() + lead, desc.image_stride, image=desc, **outputs)
        _equal_all(got, want, f"{fmt} rp {desc.row_pitch} stride {desc.image_stride} lead {lead}")
        assert all(torch.equal(t, c) for t, c in zip(views, before)), f"{fmt}: source buffer changed"
    eng.close()


@pytest.mark.gpu
def test_rawdepth_side_by_side_and_crops():
    """Side-by-side frames (the right view W samples into each row: 2 * W bytes for a 16-bit container, 10 * W / 8 or
    12 * W / 8 for a packed one with W a multiple of 4) and crops of a larger frame at even (x, y) on a byte boundary of
    the stream, in every container, mono and GB mosaic, 3 pairs a call: every output equals the packed-BGR call on the
    restated views."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 68, 45, 19
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=2)
    n = 3
    rng = np.random.default_rng(15)
    outputs = dict(volumes=[("opt", "hwd", "f32")], maps=MAPS)
    FW, FH, x0, y0 = 2 * w + 8, h + 6, 2 * w - w + 4, 4   # frames of FW x FH; the crop starts at x0 = 72, a multiple of 4
    for suffix in CONTAINERS:
        for colour in ("mono", "bayer_gb"):
            fmt = colour + suffix
            _, bits, packed = X.info(fmt)
            frames = [X.samples(X.random_frame(rng, fmt, FW, FH), fmt, FW, FH) for _ in range(n)]
            host = np.stack([X.from_samples(f, fmt).view(np.uint8).reshape(FH, -1) for f in frames])
            rp, stride = host.shape[2], host.shape[1] * host.shape[2]
            d = torch.from_numpy(host).to(dev)
            bytes_at = (lambda x: x * bits // 8) if packed else (lambda x: 2 * x)
            # side by side: left = columns [0, w), right = [w, 2w) of the frame's first h rows
            views = [[X.from_samples(f[:h, x:x + w], fmt) for f in frames] for x in (0, w)]
            pl, pr = (_packed(v, fmt, w, h) for v in views)
            want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h,
                                   **outputs)
            got = E.batch_outputs(eng, eng.match_images_batch_device, n, d.data_ptr(), d.data_ptr() + bytes_at(w), stride,
                                  image=A.image_desc(fmt, rp, 0, stride), **outputs)
            _equal_all(got, want, f"side by side {fmt}")
            # crops: left at (4, y0), right at (x0, y0): even positions, multiples of 4
            views = [[X.from_samples(f[y0:y0 + h, x:x + w], fmt) for f in frames] for x in (4, x0)]
            pl, pr = (_packed(v, fmt, w, h) for v in views)
            want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h,
                                   **outputs)
            got = E.batch_outputs(eng, eng.match_images_batch_device, n, d.data_ptr() + y0 * rp + bytes_at(4),
                                  d.data_ptr() + y0 * rp + bytes_at(x0), stride, image=A.image_desc(fmt, rp, 0, stride),
                                  **outputs)
            _equal_all(got, want, f"crop {fmt}")
    eng.close()


@pytest.mark.gpu
def test_rawdepth_host_entry():
    """The single-pair host entry match_images, odd W and H, on tight frames, on column slices of wider arrays (a larger
    row pitch) and, for a 16-bit format, on frames at an odd host address: final map, all three volumes and all five
    side maps equal match_outputs on the restated images."""
    w, h, D = 61, 45, 20
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    rng = np.random.default_rng(22)
    for k, fmt in enumerate(["mono12", "bayer_rg12", "bayer_gr16", "bayer_bg10", "mono10p", "bayer_gb10p", "mono12p",
                             "bayer_rg12p"]):
        frames = [X.random_frame(rng, fmt, w, h) for _ in range(2)]
        if k % 2:   # the same samples in arrays 8 elements wider
            wide = []
            for f in frames:
                big = rng.integers(0, 256, (h, f.shape[1] + 8)).astype(f.dtype)
                big[:, :f.shape[1]] = f
                wide.append(big[:, :f.shape[1]])
            frames = wide
        if fmt == "bayer_gr16":   # uint16 views at odd addresses
            odd = []
            for f in frames:
                raw = np.zeros(f.nbytes + 1, np.uint8)
                v = raw[1:].view(np.uint16).reshape(f.shape)
                v[:] = f
                assert v.ctypes.data % 2 == 1
                odd.append(v)
            frames = odd
        want_disp, want = eng.match_outputs(*(X.decode(f, fmt, w, h) for f in frames), maps=MAPS, volumes=VOLS)
        disp, got = eng.match_images(frames[0], frames[1], format=fmt, maps=MAPS, volumes=VOLS)
        E.same(f"{fmt} host disp", disp, want_disp)
        for key in want:
            E.same(f"{fmt} host {key}", got[key], want[key])
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True])
def test_rawdepth_rectified(pipelined):
    """Raw frames through the rectified entries: both map types (with specials, reaching outside the frame), frames from
    640 x 480 down to 2 x 2, 1 x N and 1 x 1, every container, pitched rows: every output equals
    adc_match_outputs_batch_device on remap(decode(raw)); the host entry match_rectified agrees."""
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=3)
    n = 2 * eng.wave_pairs + 1
    rng = np.random.default_rng(13)
    cases = [((640, 480), "bayer_rg12p"), ((83, 53), "bayer_gr10p"), ((64, 40), "bayer_bg12"), ((1, 1), "bayer_gb12p"),
             ((57, 1), "mono12p"), ((2, 2), "bayer_rg10"), ((3, 5), "bayer_gb16"), ((90, 61), "mono10p"),
             ((1, 1), "mono16"), ((33, 1), "bayer_rg10p"), ((45, 38), "mono10"), ((4, 3), "bayer_bg12p")]
    for k, ((sw, sh), fmt) in enumerate(cases):
        fixed = k % 2 == 1
        packed = X.info(fmt)[2]
        maps = [R.warp_maps(w, h, sw, sh, 60 + 2 * k + v, fixed) for v in range(2)]
        eng.set_rectification(maps[0], maps[1], (sw, sh))
        lead = 1 if packed else 2
        views, desc, L, Rr = _batch(fmt, n, sw, sh, rng, 4, 0 if k % 3 else 6, lead, corners=k % 4 == 3)
        full = k < 2
        outputs = dict(volumes=[(v, "hwd", "f32") for v in (VOLS if full else ["opt"])], maps=MAPS, pipelined=pipelined)
        pl, pr = _packed(L, fmt, sw, sh, maps[0]), _packed(Rr, fmt, sw, sh, maps[1])
        want = E.batch_outputs(eng, eng.match_outputs_batch_device, n, pl.data_ptr(), pr.data_ptr(), 3 * w * h, **outputs)
        got = E.batch_outputs(eng, eng.match_rectified_batch_device, n, views[0].data_ptr() + lead,
                              views[1].data_ptr() + lead, desc.image_stride, image=desc, **outputs)
        _equal_all(got, want, f"{sw}x{sh} {fmt} fixed={fixed}")
        if not pipelined:
            disp, one = eng.match_rectified(L[1], Rr[1], format=fmt, maps=MAPS)
            E.same(f"{sw}x{sh} {fmt} host disp", disp, want["disp"][1])
            for m in MAPS:
                E.same(f"{sw}x{sh} {fmt} host {m}", one[m], want[m][1])
    eng.close()


@pytest.mark.gpu
def test_rawdepth_size_rules():
    """Each size-dependent rule violation fails with ADC_ERR_ARG naming its field, on the image and the rectified
    entries, before any device work (the output keeps its sentinel): a row pitch below the tight row of each container,
    an image stride below H * row_pitch, overflowing pitches; the minimums themselves are accepted."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 12
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    buf = torch.zeros(2 * w * h * 2 * 2, dtype=torch.uint8, device=dev)
    d_o = torch.full((2, h, w), -7.0, dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def run(entry, fmt, rp=0, stride=0):
        entry(2, buf.data_ptr(), buf.data_ptr(), image=A.image_desc(fmt, rp, 0, stride), d_disp=d_o.data_ptr(), stream=st)
        torch.cuda.synchronize()

    eng.set_rectification(*[R.warp_maps(w, h, w, h, 5)] * 2, (w, h))
    for entry in (eng.match_images_batch_device, eng.match_rectified_batch_device):
        d_o.fill_(-7.0)
        bad = [("mono12", dict(rp=140), r"img->row_pitch 140 is less than 2 \* W \(142\)"),
               ("bayer_rg16", dict(rp=72), r"img->row_pitch 72 is less than 2 \* W \(142\)"),
               ("bayer_gb10p", dict(rp=88), r"img->row_pitch 88 is less than ceil\(10 \* W / 8\) \(89\)"),
               ("mono12p", dict(rp=106), r"img->row_pitch 106 is less than ceil\(12 \* W / 8\) \(107\)"),
               ("bayer_rg12", dict(stride=142 * h - 2), r"img->image_stride 6672 is less than the view's footprint \(6674\)"),
               ("bayer_rg12p", dict(rp=110, stride=110 * h - 1), r"img->image_stride 5169 is less than the view's footprint \(5170\)"),
               ("mono10p", dict(rp=1 << 62), r"img->row_pitch .* is too large"),
               ("mono10", dict(rp=1 << 62), r"img->row_pitch .* is too large")]
        for fmt, kw, msg in bad:
            with pytest.raises(A.AdcError, match=r"error 1: .*" + msg):
                run(entry, fmt, **kw)
        assert bool((d_o == -7.0).all())
        for fmt, kw in (("mono12", dict(rp=142, stride=142 * h)), ("bayer_gb10p", dict(rp=89, stride=89 * h)),
                        ("bayer_rg12p", dict(rp=107))):
            run(entry, fmt, **kw)
    eng.close()


@pytest.mark.gpu
def test_rawdepth_launch_counts():
    """A call in a high-bit-depth format issues exactly one launch per wave more than the tight packed-BGR call of the
    same batch, through both the image and the rectified entry; the ingestion profile ids replay the format's kernels
    and report the algorithmic bytes (both views' tight rows read plus 3 * N written)."""
    import adcensus_b200 as A
    torch, dev = E.cuda()
    w, h, D = 71, 47, 23
    eng = E.engine(w, h, T.default_option(max_disparity=D), wave_pairs=4, lanes=2)
    n = 3 * eng.wave_pairs + 1
    waves = -(-n // eng.wave_pairs)
    rng = np.random.default_rng(3)
    bgr = [torch.from_numpy(rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)).to(dev) for _ in range(2)]
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream()
    fmts = ["mono12", "bayer_rg10", "bayer_gb16", "mono10p", "bayer_rg12p"]

    def count(call, *a, **kw):
        torch.cuda.synchronize()
        c0 = eng.launch_count
        call(*a, d_disp=d_o.data_ptr(), stream=st.cuda_stream, **kw)
        torch.cuda.synchronize()
        return eng.launch_count - c0

    def device_frames(fmt, vw, vh):
        return [torch.from_numpy(np.stack([X.random_frame(rng, fmt, vw, vh) for _ in range(n)]).view(np.uint8)).to(dev)
                for _ in range(2)]

    base = count(eng.match_outputs_batch_device, n, bgr[0].data_ptr(), bgr[1].data_ptr())
    for fmt in fmts:
        raw = device_frames(fmt, w, h)
        got = count(eng.match_images_batch_device, n, raw[0].data_ptr(), raw[1].data_ptr(), image=A.image_desc(fmt))
        assert got == base + waves, (fmt, got, base, waves)
        assert eng.profile_kernel("image_ingest", reps=2)[1] == 2 * eng.wave_pairs * (X.tight_row(fmt, w) * h + 3 * h * w)
    sw, sh = 91, 61
    m = R.warp_maps(w, h, sw, sh, 3)
    eng.set_rectification(m, m, (sw, sh))
    for fmt in fmts:
        raw = device_frames(fmt, sw, sh)
        got = count(eng.match_rectified_batch_device, n, raw[0].data_ptr(), raw[1].data_ptr(), image=A.image_desc(fmt))
        assert got == base + waves, (fmt, got, base, waves)
        ms, by = eng.profile_kernel("rectify", reps=2)
        assert ms > 0 and by == 2 * eng.wave_pairs * (X.tight_row(fmt, sw) * sh + 3 * h * w) + 2 * 8 * h * w, fmt
    eng.close()
