#!/usr/bin/env python
"""YUV frames on the way in, on bench.py's workload (Cone 450x375x64, batch 256, device-resident, pipelined), in one
process so that every figure comes from the same run:

  python tools/bench_yuv.py [--steps 5 --warmup 3 --rounds 3]

* nv12         : adc_match_images_batch_device on Cone encoded as NV12 in 450 x 376 decoder surfaces (row pitch 512,
                 chroma plane at 376 * 512, as a video decoder writes them) (ADC_IMG_NV12)
* nv12_bgr     : adc_match_batch_device on the same frames decoded beforehand (cv2.cvtColor), packed BGR on the device:
                 the yardstick for `nv12`, whose image content differs from Cone's
* yuyv_sbs     : adc_match_images_batch_device on side-by-side YUYV frames (900 x 375, the right view at 2 * 450 bytes
                 into each row) (ADC_IMG_YUYV)
* yuyv_bgr     : adc_match_batch_device on the same views decoded beforehand, packed BGR
* rect_nv12    : adc_match_rectified_batch_device on raw 640 x 480 NV12 frames (Cone resized and encoded), rectified
                 through initUndistortRectifyMap maps (CV_16SC2) of rectify_testlib's made-up rig
* rect_bgr_raw : adc_match_rectified_batch_device on the same raw frames decoded beforehand, [N, 480, 640, 3]
  The six are timed in alternating windows (`--rounds`); the medians are reported.
* host         : the same raw NV12 frames through cv2.cvtColor and cv2.remap on the host (both views of every pair, 16
                 OpenCV threads) followed by adc_match_batch on the rectified images: wall clock over one batch, after a
                 warm-up batch.
* kernels      : the plain ingestion kernel (adc_profile_kernel id 13) for NV12 and YUYV and the rectified one (id 14)
                 for NV12 alone over one wave (CUDA events), each next to a device-to-device cudaMemcpyAsync (torch copy_)
                 that moves as many bytes (read + write) as the kernel's algorithmic bytes (per view W*H +
                 2*ceil(W/2)*ceil(H/2) (4:2:0) or 4*ceil(W/2)*H (4:2:2) read and 3N written; plus both views' maps once
                 per wave for id 14).
Every YUV map is checked bit for bit against the packed-BGR maps of the decoded images (and the host path's).  The
card's name and power limit are recorded beside the numbers.  Prints one JSON line; writes nothing.
"""
import statistics
import sys

import cv2
import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import rectify_testlib as R
import yuv_testlib as Y


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    sw, sh = 640, 480
    D = 64

    # NV12 in 450 x 376 surfaces
    nv = [Y.encode(img, "nv12") for img in (left, right)]
    nv_dec = [Y.cv_decode(cv2, f, "nv12", w, h) for f in nv]
    rp, SH = 512, 376
    pp = SH * rp
    surf = Y.footprint("nv12", SH, rp, pp)
    nv_d = [rep(Y.write_view(np.zeros(surf, np.uint8), f, "nv12", w, h, rp, pp)) for f in nv]
    nv_desc = A.image_desc("nv12", rp, pp, surf)
    # side-by-side YUYV: one 900 x 375 frame a pair
    sbs = Y.encode(np.concatenate([left, right], 1), "yuyv")
    yu_dec = [Y.cv_decode(cv2, sbs[:, x:x + w], "yuyv", w, h) for x in (0, w)]
    sbs_d = rep(sbs)
    yu_desc = A.image_desc("yuyv", 4 * w, 0, sbs.nbytes)   # 2 bytes a pixel, 2 * w pixels a row
    # raw 640 x 480 NV12 frames
    raw = [Y.encode(cv2.resize(img, (sw, sh), interpolation=cv2.INTER_LINEAR), "nv12") for img in (left, right)]
    raw_bgr = [Y.cv_decode(cv2, r, "nv12", sw, sh) for r in raw]
    maps = [R.cone_rig(cv2, sw, sh, w, h, cv2.CV_16SC2, s) for s in (1, -1)]
    b_nv = [rep(x) for x in nv_dec]
    b_yu = [rep(x) for x in yu_dec]
    r_nv = [rep(x) for x in raw]
    r_bgr = [rep(x) for x in raw_bgr]
    names = ("nv12", "nv12_bgr", "yuyv_sbs", "yuyv_bgr", "rect_nv12", "rect_bgr_raw")
    out = {k: torch.empty((n, h, w), dtype=torch.float32, device=dev) for k in names}
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    nv_raw_desc = A.image_desc("nv12")

    def nv12(_):
        eng.match_images_batch_device(n, nv_d[0].data_ptr(), nv_d[1].data_ptr(), image=nv_desc,
                                      d_disp=out["nv12"].data_ptr(), stream=st.cuda_stream)

    def nv12_bgr(_):
        eng.match_batch_device(n, b_nv[0].data_ptr(), b_nv[1].data_ptr(), out["nv12_bgr"].data_ptr(), st.cuda_stream)

    def yuyv_sbs(_):
        eng.match_images_batch_device(n, sbs_d.data_ptr(), sbs_d.data_ptr() + 2 * w, image=yu_desc,
                                      d_disp=out["yuyv_sbs"].data_ptr(), stream=st.cuda_stream)

    def yuyv_bgr(_):
        eng.match_batch_device(n, b_yu[0].data_ptr(), b_yu[1].data_ptr(), out["yuyv_bgr"].data_ptr(), st.cuda_stream)

    def rect_nv12(_):
        eng.match_rectified_batch_device(n, r_nv[0].data_ptr(), r_nv[1].data_ptr(), image=nv_raw_desc,
                                         d_disp=out["rect_nv12"].data_ptr(), stream=st.cuda_stream)

    def rect_bgr_raw(_):
        eng.match_rectified_batch_device(n, r_bgr[0].data_ptr(), r_bgr[1].data_ptr(),
                                         d_disp=out["rect_bgr_raw"].data_ptr(), stream=st.cuda_stream)

    ms = B.windows(eng, st, (nv12, nv12_bgr, yuyv_sbs, yuyv_bgr, rect_nv12, rect_bgr_raw), args.steps, args.warmup,
                   args.rounds)
    eng.set_pipelined(False)

    # host path: cv2.cvtColor + cv2.remap of every view on 16 threads, then adc_match_batch (pointer-array form)
    code = cv2.COLOR_YUV2BGR_NV12
    lefts, rights = [raw[0]] * n, [raw[1]] * n

    def host():
        return eng.match_batch_ptrs([B.remap(cv2.cvtColor(x, code), maps[0]) for x in lefts],
                                    [B.remap(cv2.cvtColor(x, code), maps[1]) for x in rights])

    host_s, host_maps = B.host_seconds(host, args.rounds, threads=16)
    got = {k: v.cpu().numpy() for k, v in out.items()}
    checks = {"nv12_vs_nv12_bgr": got["nv12"].tobytes() == got["nv12_bgr"].tobytes(),
              "yuyv_sbs_vs_yuyv_bgr": got["yuyv_sbs"].tobytes() == got["yuyv_bgr"].tobytes(),
              "rect_nv12_vs_rect_bgr_raw": got["rect_nv12"].tobytes() == got["rect_bgr_raw"].tobytes(),
              "rect_nv12_vs_host": all(got["rect_nv12"][i].tobytes() == host_maps[i].tobytes() for i in range(n)),
              "nv12_vs_single_pair": all(got["nv12"][i].tobytes() == eng.match(nv_dec[0], nv_dec[1]).tobytes()
                                         for i in (0, n - 1))}

    sbs_views = [np.ascontiguousarray(sbs[:, x:x + w]) for x in (0, w)]
    kernels = B.kernels_vs_copy(eng, (
        ("image_ingest_nv12", "image_ingest", lambda: eng.match_images(nv[0], nv[1], format="nv12")),
        ("image_ingest_yuyv", "image_ingest", lambda: eng.match_images(sbs_views[0], sbs_views[1], format="yuyv")),
        ("rectify_nv12", "rectify", lambda: eng.match_rectified(raw[0], raw[1], format="nv12")),
        ("rectify_bgr", "rectify", lambda: eng.match_rectified(raw_bgr[0], raw_bgr[1]))), reps=50, dev=dev)
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    host_rate = round(n / statistics.median(host_s), 2)
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "nv12": {"value": rate["nv12"], "call": "adc_match_images_batch_device (NV12, 450x376 surfaces, pitch 512)"},
            "nv12_bgr": {"value": rate["nv12_bgr"],
                         "call": "adc_match_batch_device (the same frames decoded beforehand, packed BGR)"},
            "yuyv_sbs": {"value": rate["yuyv_sbs"], "call": "adc_match_images_batch_device (side-by-side YUYV 900x375)"},
            "yuyv_bgr": {"value": rate["yuyv_bgr"],
                         "call": "adc_match_batch_device (the same views decoded beforehand, packed BGR)"},
            "rect_nv12": {"value": rate["rect_nv12"],
                          "call": "adc_match_rectified_batch_device (640x480 raw NV12, CV_16SC2 maps)"},
            "rect_bgr_raw": {"value": rate["rect_bgr_raw"],
                             "call": "adc_match_rectified_batch_device (the same raw frames decoded beforehand, BGR)"},
            "host_cvtcolor_remap": {"value": host_rate,
                                    "call": "cv2.cvtColor + cv2.remap on the host (both views, 16 threads) + adc_match_batch",
                                    "opencv": cv2.__version__},
            "nv12_vs_nv12_bgr": round(rate["nv12"] / rate["nv12_bgr"], 4),
            "yuyv_sbs_vs_yuyv_bgr": round(rate["yuyv_sbs"] / rate["yuyv_bgr"], 4),
            "rect_nv12_vs_rect_bgr_raw": round(rate["rect_nv12"] / rate["rect_bgr_raw"], 4),
            "rect_nv12_vs_host": round(rate["rect_nv12"] / host_rate, 2),
            "windows_ms": {k: [round(x, 2) for x in v] for k, v in ms.items()},
            "checks": checks,
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "kernels": kernels,
            "card": B.card()}
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
