#!/usr/bin/env python
"""Video-decoder YUV containers and colour encodings on the way in, on bench.py's workload (Cone 450x375x64, batch 256,
device-resident, pipelined), in one process so that every figure comes from the same run:

  python tools/bench_yuv_video.py [--steps 5 --warmup 3 --rounds 3]

* i420            : adc_match_images_batch_device on Cone as tight I420 frames (FFmpeg yuv420p, BT.601 limited)
* i420_bgr        : adc_match_images_batch_device (packed BGR, no descriptor) on the same frames converted beforehand:
                    the yardstick for `i420`, whose image content differs from Cone's
* p016_bt709      : the same entry on Cone as P016 | ADC_IMG_YUV_BT709 in 450 x 376 decoder surfaces (row pitch 1024
                    bytes, chroma plane at 376 * 1024, as NVDEC writes a 10-bit surface)
* p016_bt709_bgr  : packed BGR of the same frames converted beforehand
* nv12_full       : the same entry on tight NV12 | ADC_IMG_YUV_FULL_RANGE frames
* nv12_full_bgr   : packed BGR of the same frames converted beforehand
* rect_p016_bt709 : adc_match_rectified_batch_device on raw 640 x 480 P016 | BT.709 frames (Cone resized and encoded)
                    through initUndistortRectifyMap maps (CV_16SC2) of rectify_testlib's made-up rig
* rect_bgr_raw    : adc_match_rectified_batch_device on the same raw frames converted beforehand, [N, 480, 640, 3]
  The eight are timed in alternating windows (`--rounds`); the medians are reported.
* host            : the tight I420 frames through cv2.cvtColor(COLOR_YUV2BGR_I420) on the host (both views of every pair,
                    all OpenCV threads; Cone's odd height is converted as the even frame holding it, then cropped)
                    followed by adc_match_batch: wall clock over one batch, after a warm-up batch.
* kernels         : the plain ingestion kernel (adc_profile_kernel id 13) for I420 and P016 | BT.709 and the rectified
                    one (id 14) for P016 | BT.709 over one wave (CUDA events), each next to a device-to-device
                    cudaMemcpyAsync that moves as many bytes (read + write) as the kernel's algorithmic bytes (per view
                    W*H + 2*ceil(W/2)*ceil(H/2) samples read, 1 or 2 bytes each, and 3N written; plus both views' maps
                    once per wave for id 14).
Every YUV map is checked bit for bit against the packed-BGR maps of the converted images (and the host path's).  The
card's name and power limit are recorded beside the numbers.  Prints one JSON line; writes nothing.
"""
import os
import statistics
import sys

import cv2
import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import rectify_testlib as R
import yuv_video_testlib as V


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    rep16 = B.cone(n, raw=True)[2]
    h, w, _ = left.shape
    sw, sh = 640, 480
    D = 64
    BT709, FULL = A.IMG_YUV_BT709, A.IMG_YUV_FULL_RANGE

    # tight I420 frames
    i420 = [V.encode(img, "i420") for img in (left, right)]
    i420_bgr = [V.decode(f, "i420", w, h) for f in i420]
    # P016 in 450 x 376 surfaces of pitch 1024
    p16 = [V.encode(img, "p016") for img in (left, right)]
    p16_bgr = [V.decode(f, "p016", w, h, BT709) for f in p16]
    rp, SH = 1024, 376
    pp = SH * rp
    surf = V.footprint("p016", SH, rp, pp)
    p16_d = [rep(V.write_view(np.zeros(surf, np.uint8), f, "p016", w, h, rp, pp)) for f in p16]
    p16_desc = A.image_desc(A.IMG_P016 | BT709, rp, pp, surf)
    # tight full-range NV12
    nv = [V.encode(img, "nv12") for img in (left, right)]
    nv_bgr = [V.decode(f, "nv12", w, h, FULL) for f in nv]
    # raw 640 x 480 P016
    raw = [V.encode(cv2.resize(img, (sw, sh), interpolation=cv2.INTER_LINEAR), "p016") for img in (left, right)]
    raw_bgr = [V.decode(r, "p016", sw, sh, BT709) for r in raw]
    maps = [R.cone_rig(cv2, sw, sh, w, h, cv2.CV_16SC2, s) for s in (1, -1)]

    yuv_d = {"i420": [rep(x) for x in i420], "p016_bt709": p16_d, "nv12_full": [rep(x) for x in nv],
             "rect_p016_bt709": [rep16(x) for x in raw]}
    bgr_d = {"i420_bgr": [rep(x) for x in i420_bgr], "p016_bt709_bgr": [rep(x) for x in p16_bgr],
             "nv12_full_bgr": [rep(x) for x in nv_bgr], "rect_bgr_raw": [rep(x) for x in raw_bgr]}
    descs = {"i420": A.image_desc("i420"), "p016_bt709": p16_desc, "nv12_full": A.image_desc(A.IMG_NV12 | FULL),
             "rect_p016_bt709": A.image_desc(A.IMG_P016 | BT709)}
    names = ("i420", "i420_bgr", "p016_bt709", "p016_bt709_bgr", "nv12_full", "nv12_full_bgr", "rect_p016_bt709",
             "rect_bgr_raw")
    out = {k: torch.empty((n, h, w), dtype=torch.float32, device=dev) for k in names}
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()

    def path(name):
        rect = name.startswith("rect_")
        entry = eng.match_rectified_batch_device if rect else eng.match_images_batch_device
        bufs, desc = (yuv_d[name], descs[name]) if name in yuv_d else (bgr_d[name], None)

        def run(_):
            entry(n, bufs[0].data_ptr(), bufs[1].data_ptr(), image=desc, d_disp=out[name].data_ptr(),
                  stream=st.cuda_stream)
        run.__name__ = name
        return run

    ms = B.windows(eng, st, tuple(path(k) for k in names), args.steps, args.warmup, args.rounds)
    eng.set_pipelined(False)

    # host path: cv2.cvtColor of every I420 view on all cores (Cone's odd height: on the even frame holding the view,
    # then cropped, as OpenCV's I420 Mat needs an even height), then adc_match_batch (pointer-array form)
    lefts, rights = [i420[0]] * n, [i420[1]] * n

    def host():
        return eng.match_batch_ptrs([V.cv_decode(cv2, x, "i420", w, h) for x in lefts],
                                    [V.cv_decode(cv2, x, "i420", w, h) for x in rights])

    threads = os.cpu_count()
    host_s, host_maps = B.host_seconds(host, args.rounds, threads=threads)
    got = {k: v.cpu().numpy() for k, v in out.items()}
    checks = {f"{k}_vs_{k}_bgr": got[k].tobytes() == got[k + "_bgr"].tobytes()
              for k in ("i420", "p016_bt709", "nv12_full")}
    checks["rect_p016_bt709_vs_rect_bgr_raw"] = got["rect_p016_bt709"].tobytes() == got["rect_bgr_raw"].tobytes()
    checks["i420_vs_host"] = all(got["i420"][i].tobytes() == host_maps[i].tobytes() for i in range(n))
    checks["i420_bgr_is_cv2"] = all(np.array_equal(V.cv_decode(cv2, f, "i420", w, h), b) for f, b in zip(i420, i420_bgr))

    kernels = B.kernels_vs_copy(eng, (
        ("image_ingest_i420", "image_ingest", lambda: eng.match_images(i420[0], i420[1], format="i420")),
        ("image_ingest_p016_bt709", "image_ingest", lambda: eng.match_images(p16[0], p16[1], format="p016/bt709")),
        ("rectify_p016_bt709", "rectify", lambda: eng.match_rectified(raw[0], raw[1], format="p016/bt709")),
        ("rectify_bgr", "rectify", lambda: eng.match_rectified(raw_bgr[0], raw_bgr[1]))), reps=50, dev=dev)
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    host_rate = round(n / statistics.median(host_s), 2)
    calls = {"i420": "adc_match_images_batch_device (tight I420)",
             "p016_bt709": "adc_match_images_batch_device (P016 | BT709, 450x376 surfaces, pitch 1024)",
             "nv12_full": "adc_match_images_batch_device (tight NV12 | FULL_RANGE)",
             "rect_p016_bt709": "adc_match_rectified_batch_device (640x480 raw P016 | BT709, CV_16SC2 maps)",
             "rect_bgr_raw": "adc_match_rectified_batch_device (the same raw frames converted beforehand, BGR)"}
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s"}
    for k in names:
        line[k] = {"value": rate[k], "call": calls.get(k, "adc_match_images_batch_device (the same frames converted "
                                                          "beforehand, packed BGR)")}
    line.update({
        "host_cvtcolor": {"value": host_rate, "threads": threads, "opencv": cv2.__version__,
                          "call": "cv2.cvtColor(COLOR_YUV2BGR_I420) on the host (both views) + adc_match_batch"},
        "i420_vs_i420_bgr": round(rate["i420"] / rate["i420_bgr"], 4),
        "p016_bt709_vs_p016_bt709_bgr": round(rate["p016_bt709"] / rate["p016_bt709_bgr"], 4),
        "nv12_full_vs_nv12_full_bgr": round(rate["nv12_full"] / rate["nv12_full_bgr"], 4),
        "rect_p016_bt709_vs_rect_bgr_raw": round(rate["rect_p016_bt709"] / rate["rect_bgr_raw"], 4),
        "i420_vs_host": round(rate["i420"] / host_rate, 2),
        "windows_ms": {k: [round(x, 2) for x in v] for k, v in ms.items()},
        "checks": checks,
        "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
        "kernels": kernels,
        "card": B.card()})
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
