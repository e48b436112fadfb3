"""Small end-to-end cases for compute-sanitizer (memcheck / racecheck are 10-100x slower than a plain run):
two small pairs through Match, the batched entry point, the voting fallbacks' sizes and the render calls."""
import sys
from pathlib import Path
import numpy as np
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import adcensus_b200 as A
import adc_testlib as T

cases = [(97, 61, 24, 2, {}), (130, 70, 37, 3, {}), (80, 60, 32, 10, {"do_discontinuity_adjustment": 1}),
         (80, 60, 32, 31, {"min_disparity": 2, "max_disparity": 34}),
         (70, 44, 64, 4, {}),        # D = 64: eight quads per CTA (compile-time strides), 8 lanes per scanline
         (150, 40, 130, 12, {}),     # 16 lanes per scanline, padded disparity stride
         (600, 16, 12, 18, {}),      # a row cut into segments by the fused horizontal double pass
         (64, 40, 255, 15, {}),      # D = 255: the WIDE voting kernels (16-bit votes, one count per histogram word)
         (60, 300, 16, 17, {"cross_L1": 130, "cross_L2": 17, "cross_t1": 300, "cross_t2": 300})]   # L1 > 127: WIDE, enumerating
for (w, h, D, seed, over) in cases:
    left, right = T.synthetic_pair(w, h, D, seed)
    kw = dict(max_disparity=D); kw.update(over)
    eng = A.Engine(w, h, A.ADCensusOption(**kw), wave_pairs=2, lanes=2)
    a = eng.match(left, right)
    b = eng.match_batch(np.stack([left] * 5), np.stack([right] * 5))
    assert (b.view(np.uint32) == a.view(np.uint32)[None]).all()
    want = T.Oracle(w, h, T.default_option(**kw)).match(left, right)
    assert a.tobytes() == want.tobytes(), (w, h, D)
    g, j, mm = eng.render_disparity(a)
    c = eng.disparity_cloud(left, a)
    eng.close()
    print("ok", w, h, D, mm, c.shape, flush=True)

# cost-input mode: both layouts, a bf16 volume and the batched device entry point
import cost_testlib as CT
for (w, h, D, seed, over) in [(97, 61, 22, 2, {}), (80, 60, 32, 42, {"min_disparity": -4, "max_disparity": 28})]:
    kw = dict(max_disparity=D); kw.update(over)
    dmin = kw.get("min_disparity", 0)
    D = kw["max_disparity"] - dmin
    left, right = T.synthetic_pair(w, h, D, seed)
    cost = CT.synthetic_cost(w, h, D, seed, dmin)
    eng = A.Engine(w, h, A.ADCensusOption(**kw), wave_pairs=2, lanes=2)
    a = eng.match_cost(left, right, cost, "hwd")
    dhw = np.ascontiguousarray(cost.transpose(2, 0, 1))
    assert eng.match_cost(left, right, dhw, "dhw").tobytes() == a.tobytes()
    assert eng.match_cost(left, right, CT.to_bf16_bits(cost), "hwd", dtype="bf16").tobytes() == a.tobytes()
    import torch
    dev = torch.device("cuda", 0)
    n = 5
    d_l = torch.from_numpy(np.stack([left] * n)).to(dev)
    d_r = torch.from_numpy(np.stack([right] * n)).to(dev)
    d_c = torch.from_numpy(np.stack([CT.to_bf16_bits(dhw)] * n)).to(dev)
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    eng.match_cost_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), d_c.data_ptr(), d_o.data_ptr(), "dhw", "bf16",
                                torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert (d_o.cpu().numpy().view(np.uint32) == a.view(np.uint32)[None]).all()
    eng.close()
    print("cost ok", w, h, D, flush=True)

# volume export: every stage, both layouts, 2-byte types, D % 4 != 0 and odd H*W (odd pair offsets), volumes only,
# the batched device entry point at an odd destination offset
for (w, h, D, seed) in [(97, 61, 22, 2), (71, 47, 23, 5)]:
    left, right = T.synthetic_pair(w, h, D, seed)
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D), wave_pairs=2, lanes=2)
    a = eng.match(left, right)
    for layout in ("hwd", "dhw"):
        for dtype in ("f32", "bf16", "f16"):
            disp, vols = eng.match_volumes(left, right, ["cost", "aggr", "opt"], layout, dtype)
            assert disp.tobytes() == a.tobytes()
            none, only = eng.match_volumes(left, right, ["opt"], layout, dtype, disparity=False)
            assert none is None and only["opt"].tobytes() == vols["opt"].tobytes()
    import torch
    dev = torch.device("cuda", 0)
    n, ND = 5, h * w * D
    d_l = torch.from_numpy(np.stack([left] * n)).to(dev)
    d_r = torch.from_numpy(np.stack([right] * n)).to(dev)
    d_v = torch.empty(n * ND + 1, dtype=torch.bfloat16, device=dev)
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    eng.match_volumes_batch_device(n, d_l.data_ptr(), d_r.data_ptr(), [(d_v[1:].data_ptr(), "aggr", "dhw", "bf16")],
                                   d_disp=d_o.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert (d_o.cpu().numpy().view(np.uint32) == a.view(np.uint32)[None]).all()
    _, want = eng.match_volumes(left, right, "aggr", "dhw", "bf16")
    got = d_v[1:].view(torch.int16).cpu().numpy().view(np.uint16).reshape(n, -1)
    assert (got == want["aggr"].reshape(1, -1)).all()
    eng.close()
    print("export ok", w, h, D, flush=True)

# image input: odd-x crops in every format, the right view of each ending exactly at the end of its own cudaMalloc
# allocation (torch's caching allocator would hide an over-read inside a larger block), through the batched entry
import ctypes
import images_testlib as IT
cudart = ctypes.CDLL("libcudart.so.12")       # already loaded by the engine library
cudart.cudaMalloc.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_size_t]
cudart.cudaMemcpy.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
cudart.cudaFree.argtypes = [ctypes.c_void_p]
w, h, D, n = 71, 47, 23, 3
left, right = T.synthetic_pair(w, h, D, 8)
eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D), wave_pairs=2, lanes=2)
want = eng.match(left, right)
for fmt in IT.FORMATS:
    l, r = (IT.gray_to_bgr(left[:, :, 1]), IT.gray_to_bgr(right[:, :, 1])) if fmt == "gray" else (left, right)
    bpp, x0 = IT.BPP[fmt], 3
    rp = (w + x0) * bpp
    pp = h * rp if fmt == "rgb_planar" else 0
    stride = IT.footprint(fmt, h, rp, pp)
    ptrs = []
    for img in (l, r):
        host = np.zeros(n * stride, np.uint8)
        for i in range(n):
            IT.write_view(host[i * stride:], IT.from_bgr(img, fmt), fmt, rp, pp, x0 * bpp)
        # the allocation ends with the last pixel of the last row of the last view: drop the row's unused tail
        size = n * stride - (rp - (x0 + w) * bpp)
        p = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(p), size) == 0
        assert cudart.cudaMemcpy(p, host.ctypes.data, size, 1) == 0
        ptrs.append(p.value)
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    eng.match_images_batch_device(n, ptrs[0] + x0 * bpp, ptrs[1] + x0 * bpp, image=A.image_desc(fmt, rp, pp, stride),
                                  d_disp=d_o.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    single = eng.match(l, r)
    assert (d_o.cpu().numpy().view(np.uint32) == single.view(np.uint32)[None]).all(), fmt
    if fmt != "gray":
        assert single.tobytes() == want.tobytes(), fmt
    for p in ptrs:
        cudart.cudaFree(p)
    print("images ok", fmt, flush=True)
eng.close()

# rectified input: raw odd-x crops in every format, the right view of each ending exactly at the end of its own
# cudaMalloc allocation, with maps that sample the last row and column, half a pixel and more beyond them
import rectify_testlib as R
w, h, D, n, sw, sh = 71, 47, 23, 3, 83, 53
eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D), wave_pairs=2, lanes=2)
rng = np.random.default_rng(5)
edge = np.array([sw - 1, sw - 1.5, sw - 0.5, sw - 1 / 64, sw, sw + 0.5, -0.5, -1 / 64], np.float32)
for k, fmt in enumerate(IT.FORMATS):
    maps = []
    for v in range(2):
        mx, my = R.warp_maps(w, h, sw, sh, 70 + v, specials=False)
        mx[:, -8:] = edge
        my[-8:, :] = (edge * sh / sw).astype(np.float32)[:, None]
        my[-1, :] = sh - 1
        mx[-1, ::2] = sw - 1
        maps.append(R.convert_maps(mx, my) if k % 2 else (mx, my))
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    raw = [rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8) for _ in range(2)]
    if fmt == "gray":
        raw = [IT.gray_to_bgr(x[:, :, 1]) for x in raw]
    bpp, x0 = IT.BPP[fmt], 3
    rp = (sw + x0) * bpp
    pp = sh * rp if fmt == "rgb_planar" else 0
    stride = IT.footprint(fmt, sh, rp, pp)
    ptrs = []
    for img in raw:
        host = np.zeros(n * stride, np.uint8)
        for i in range(n):
            IT.write_view(host[i * stride:], IT.from_bgr(img, fmt), fmt, rp, pp, x0 * bpp)
        size = n * stride - (rp - (x0 + sw) * bpp)
        p = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(p), size) == 0
        assert cudart.cudaMemcpy(p, host.ctypes.data, size, 1) == 0
        ptrs.append(p.value)
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    eng.match_rectified_batch_device(n, ptrs[0] + x0 * bpp, ptrs[1] + x0 * bpp, image=A.image_desc(fmt, rp, pp, stride),
                                     d_disp=d_o.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    single = eng.match(R.remap(raw[0], *maps[0]), R.remap(raw[1], *maps[1]))
    assert (d_o.cpu().numpy().view(np.uint32) == single.view(np.uint32)[None]).all(), fmt
    for p in ptrs:
        cudart.cudaFree(p)
    print("rectified ok", fmt, flush=True)
eng.close()

# reprojection: n maps and every output, each in its own cudaMalloc allocation that ends exactly with its last element,
# the S16 output at a 2-byte offset, one kind at a time and all three together
import reproject_testlib as RP
w, h, n = 71, 47, 3
N = w * h
eng = A.Engine(w, h, A.ADCensusOption(min_disparity=-2, max_disparity=21), wave_pairs=2, lanes=2)
maps = np.stack([eng.match(*T.synthetic_pair(w, h, 23, 60 + i)) for i in range(n)])
Q = np.array([[1, 0, 0, -35.2], [0, 1, 0, -23.9], [0, 0, 0, 60.0], [0, 0, 8.3, -0.0]])
sizes = {"points": 12 * n * N, "depth": 4 * n * N, "disp_s16": 2 * n * N + 2}
for kinds in (["points"], ["depth"], ["disp_s16"], ["points", "depth", "disp_s16"]):
    p = ctypes.c_void_p()
    assert cudart.cudaMalloc(ctypes.byref(p), maps.nbytes) == 0
    assert cudart.cudaMemcpy(p, maps.ctypes.data, maps.nbytes, 1) == 0
    ptrs = {"disp": p.value}
    for k in kinds:
        q = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(q), sizes[k]) == 0
        ptrs[k] = q.value + (2 if k == "disp_s16" else 0)
    eng.reproject_batch_device(n, ptrs["disp"], Q, [(ptrs[k], k) for k in kinds], torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for k in kinds:
        got = np.empty(sizes[k] - (2 if k == "disp_s16" else 0), np.uint8)
        assert cudart.cudaMemcpy(got.ctypes.data, ptrs[k], got.nbytes, 2) == 0
        for i in range(n):
            want = eng.reproject(maps[i], Q, [k])[k]
            assert got.reshape(n, -1)[i].tobytes() == want.tobytes(), (kinds, k, i)
        cudart.cudaFree(ptrs[k] - (2 if k == "disp_s16" else 0))
    cudart.cudaFree(ptrs["disp"])
    assert RP.same_nan(eng.reproject(maps[0], Q)["points"], RP.points(maps[0], Q))
    print("reprojection ok", kinds, flush=True)
eng.close()

# speckle removal: n maps of each type and the workspace, each in its own cudaMalloc allocation that ends exactly with
# its last element (the S16 maps start 2 bytes in), serpentine and noise content
import speckle_testlib as SP
w, h, n = 131, 67, 3
N = w * h
eng = A.Engine(w, h, A.ADCensusOption(max_disparity=8), wave_pairs=2, lanes=2)
rng = np.random.default_rng(5)
s16 = rng.integers(-3, 4, (n, h, w)).astype(np.int16)
s16[0, 0::2] = 1
s16[0, 1::2] = 0
for t, maps, lead in (("s16", s16, 2), ("f32", (s16 / 4.0).astype(np.float32), 0)):
    p, q = ctypes.c_void_p(), ctypes.c_void_p()
    assert cudart.cudaMalloc(ctypes.byref(p), maps.nbytes + lead) == 0
    wb = eng.speckle_workspace_bytes(n)
    assert cudart.cudaMalloc(ctypes.byref(q), wb) == 0
    assert cudart.cudaMemcpy(p.value + lead, maps.ctypes.data, maps.nbytes, 1) == 0
    md = 1 if t == "s16" else 0.25
    eng.filter_speckles_batch_device(n, p.value + lead, t, 5, md, 0.0, q.value, wb, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = np.empty_like(maps)
    assert cudart.cudaMemcpy(got.ctypes.data, p.value + lead, maps.nbytes, 2) == 0
    for i in range(n):
        assert got[i].tobytes() == SP.filter_any(maps[i], 0.0, 5, md).tobytes(), (t, i)
        assert got[i].tobytes() == eng.filter_speckles(maps[i], 5, md, 0.0).tobytes(), (t, i)
    cudart.cudaFree(p)
    cudart.cudaFree(q)
    print("speckles ok", t, flush=True)
eng.close()

# Bayer mosaics: raw odd-x crops, the right view of each ending exactly at the end of its own cudaMalloc allocation,
# plain (every pattern) and rectified (maps sampling the last row and column and beyond, and a 2-row frame)
import bayer_testlib as BT


def bayer_views(raws, n, vw, vh, x0):
    rp = vw + x0
    stride = vh * rp
    ptrs = []
    for img in raws:
        host = np.zeros(n * stride, np.uint8)
        for i in range(n):
            host[i * stride:(i + 1) * stride].reshape(vh, rp)[:, x0:] = img
        size = n * stride
        p = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(p), size) == 0
        assert cudart.cudaMemcpy(p, host.ctypes.data, size, 1) == 0
        ptrs.append(p.value)
    return ptrs, rp, stride


w, h, D, n, x0 = 71, 47, 23, 3, 3
eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D), wave_pairs=2, lanes=2)
rng = np.random.default_rng(9)
for pat in BT.NAMES:
    raws = [rng.integers(0, 256, (h, w), dtype=np.uint8) for _ in range(2)]
    ptrs, rp, stride = bayer_views(raws, n, w, h, x0)
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    eng.match_images_batch_device(n, ptrs[0] + x0, ptrs[1] + x0, image=A.image_desc(pat, rp, 0, stride),
                                  d_disp=d_o.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    single = eng.match(BT.demosaic(raws[0], pat), BT.demosaic(raws[1], pat))
    assert (d_o.cpu().numpy().view(np.uint32) == single.view(np.uint32)[None]).all(), pat
    for p in ptrs:
        cudart.cudaFree(p)
    print("bayer ok", pat, flush=True)
for k, (sw, sh) in enumerate(((83, 53), (40, 2))):
    pat = BT.NAMES[k + 1]
    edge = np.array([sw - 1, sw - 1.5, sw - 0.5, sw - 1 / 64, sw, sw + 0.5, -0.5, -1 / 64], np.float32)
    maps = []
    for v in range(2):
        mx, my = R.warp_maps(w, h, sw, sh, 80 + v, specials=False)
        mx[:, -8:] = edge
        my[-8:, :] = (edge * sh / sw).astype(np.float32)[:, None]
        my[-1, :] = sh - 1
        mx[-1, ::2] = sw - 1
        maps.append(R.convert_maps(mx, my) if k % 2 else (mx, my))
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    raws = [rng.integers(0, 256, (sh, sw), dtype=np.uint8) for _ in range(2)]
    ptrs, rp, stride = bayer_views(raws, n, sw, sh, x0)
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    eng.match_rectified_batch_device(n, ptrs[0] + x0, ptrs[1] + x0, image=A.image_desc(pat, rp, 0, stride),
                                     d_disp=d_o.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    single = eng.match(*(R.remap(BT.demosaic(raws[v], pat), *maps[v]) for v in range(2)))
    assert (d_o.cpu().numpy().view(np.uint32) == single.view(np.uint32)[None]).all(), (sw, sh)
    for p in ptrs:
        cudart.cudaFree(p)
    print("bayer rectified ok", sw, sh, flush=True)
eng.close()

# YUV frames: odd-size views at even-x offsets with row and plane pitch above their minimums, the right view of each
# ending with its last read byte (the last chroma byte of NV12 / NV21, byte 4*ceil(W/2) of the last 4:2:2 row) at the
# end of its own cudaMalloc allocation; plain (every format) and rectified (maps sampling the last row and column and
# beyond, a 1-row frame)
import yuv_testlib as YT


def yuv_views(frames, fmt, n, vw, vh, lead):
    rp = YT.tight_row(fmt, vw) + lead + 4
    pp = vh * rp + 6 if YT.is420(fmt) else 0
    stride = YT.footprint(fmt, vh, rp, pp)
    last = pp + (YT.half(vh) - 1) * rp if YT.is420(fmt) else (vh - 1) * rp
    size = lead + (n - 1) * stride + last + YT.tight_row(fmt, vw)
    ptrs = []
    for f in frames:
        host = np.zeros(size, np.uint8)
        for i in range(n):
            YT.write_view(host, f, fmt, vw, vh, rp, pp, lead + i * stride)
        p = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(p), size) == 0
        assert cudart.cudaMemcpy(p, host.ctypes.data, size, 1) == 0
        ptrs.append(p.value)
    return ptrs, A.image_desc(fmt, rp, pp, stride)


w, h, D, n = 71, 47, 23, 3
eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D), wave_pairs=2, lanes=2)
rng = np.random.default_rng(10)
for fmt in YT.NAMES:
    frames = [YT.random_frame(rng, fmt, w, h) for _ in range(2)]
    ptrs, desc = yuv_views(frames, fmt, n, w, h, 4)
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    eng.match_images_batch_device(n, ptrs[0] + 4, ptrs[1] + 4, image=desc, d_disp=d_o.data_ptr(),
                                  stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    single = eng.match(YT.decode(frames[0], fmt, w, h), YT.decode(frames[1], fmt, w, h))
    assert (d_o.cpu().numpy().view(np.uint32) == single.view(np.uint32)[None]).all(), fmt
    for p in ptrs:
        cudart.cudaFree(p)
    print("yuv ok", fmt, flush=True)
for k, (sw, sh, fmt) in enumerate(((83, 53, "nv12"), (40, 1, "nv21"), (57, 9, "uyvy"))):
    edge = np.array([sw - 1, sw - 1.5, sw - 0.5, sw - 1 / 64, sw, sw + 0.5, -0.5, -1 / 64], np.float32)
    maps = []
    for v in range(2):
        mx, my = R.warp_maps(w, h, sw, sh, 90 + v, specials=False)
        mx[:, -8:] = edge
        my[-8:, :] = (edge * sh / sw).astype(np.float32)[:, None]
        my[-1, :] = sh - 1
        mx[-1, ::2] = sw - 1
        maps.append(R.convert_maps(mx, my) if k % 2 else (mx, my))
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    frames = [YT.random_frame(rng, fmt, sw, sh) for _ in range(2)]
    ptrs, desc = yuv_views(frames, fmt, n, sw, sh, 2)
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    eng.match_rectified_batch_device(n, ptrs[0] + 2, ptrs[1] + 2, image=desc, d_disp=d_o.data_ptr(),
                                     stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    single = eng.match(*(R.remap(YT.decode(frames[v], fmt, sw, sh), *maps[v]) for v in range(2)))
    assert (d_o.cpu().numpy().view(np.uint32) == single.view(np.uint32)[None]).all(), (sw, sh, fmt)
    for p in ptrs:
        cudart.cudaFree(p)
    print("yuv rectified ok", fmt, sw, sh, flush=True)
eng.close()

# High-bit-depth frames: views a few samples into wider rows, the right view of each ending with its last sample (the
# last 16-bit word, or byte ceil(b*W/8) of the last packed row, which the last field's second byte is) at the end of
# its own cudaMalloc allocation; plain (every container, mono and a mosaic) and rectified (one format per container,
# maps sampling the last row and column and beyond, a 2-row frame)
import rawdepth_testlib as XT


def rawdepth_views(frames, fmt, n, vw, vh, lead):
    rp = XT.tight_row(fmt, vw) + lead + 4
    stride = vh * rp + 6
    size = lead + (n - 1) * stride + (vh - 1) * rp + XT.tight_row(fmt, vw)
    ptrs = []
    for f in frames:
        host = np.zeros(size, np.uint8)
        for i in range(n):
            XT.write_view(host, f, fmt, vw, vh, rp, lead + i * stride)
        p = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(p), size) == 0
        assert cudart.cudaMemcpy(p, host.ctypes.data, size, 1) == 0
        ptrs.append(p.value)
    return ptrs, A.image_desc(fmt, rp, 0, stride)


w, h, D, n = 71, 47, 23, 3
eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D), wave_pairs=2, lanes=2)
rng = np.random.default_rng(11)
for suffix, bits, packed in XT.CONTAINERS:
    for colour in ("mono", "bayer_gr"):
        fmt = colour + suffix
        lead = bits // 2 if packed else 4   # 4 samples into the row: 5 or 6 bytes of a stream, 2 words
        frames = [XT.random_frame(rng, fmt, w, h) for _ in range(2)]
        ptrs, desc = rawdepth_views(frames, fmt, n, w, h, lead)
        d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
        eng.match_images_batch_device(n, ptrs[0] + lead, ptrs[1] + lead, image=desc, d_disp=d_o.data_ptr(),
                                      stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        single = eng.match(XT.decode(frames[0], fmt, w, h), XT.decode(frames[1], fmt, w, h))
        assert (d_o.cpu().numpy().view(np.uint32) == single.view(np.uint32)[None]).all(), fmt
        for p in ptrs:
            cudart.cudaFree(p)
        print("rawdepth ok", fmt, flush=True)
for k, (sw, sh, fmt) in enumerate(((83, 53, "bayer_rg12p"), (40, 2, "bayer_gb10p"), (57, 9, "mono12"), (31, 33, "bayer_bg10"),
                                   (45, 3, "bayer_gr16"))):
    edge = np.array([sw - 1, sw - 1.5, sw - 0.5, sw - 1 / 64, sw, sw + 0.5, -0.5, -1 / 64], np.float32)
    maps = []
    for v in range(2):
        mx, my = R.warp_maps(w, h, sw, sh, 100 + v, specials=False)
        mx[:, -8:] = edge
        my[-8:, :] = (edge * sh / sw).astype(np.float32)[:, None]
        my[-1, :] = sh - 1
        mx[-1, ::2] = sw - 1
        maps.append(R.convert_maps(mx, my) if k % 2 else (mx, my))
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    frames = [XT.random_frame(rng, fmt, sw, sh) for _ in range(2)]
    ptrs, desc = rawdepth_views(frames, fmt, n, sw, sh, 2)
    d_o = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    eng.match_rectified_batch_device(n, ptrs[0] + 2, ptrs[1] + 2, image=desc, d_disp=d_o.data_ptr(),
                                     stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    single = eng.match(*(R.remap(XT.decode(frames[v], fmt, sw, sh), *maps[v]) for v in range(2)))
    assert (d_o.cpu().numpy().view(np.uint32) == single.view(np.uint32)[None]).all(), (sw, sh, fmt)
    for p in ptrs:
        cudart.cudaFree(p)
    print("rawdepth rectified ok", fmt, sw, sh, flush=True)
eng.close()
print("all ok")
