#!/usr/bin/env python
"""Bayer mosaics on the way in, on bench.py's workload (Cone 450x375x64, batch 256, device-resident, pipelined), in one
process so that every figure comes from the same run:

  python tools/bench_bayer.py [--steps 5 --warmup 3 --rounds 3]

* bayer        : adc_match_images_batch_device on Cone mosaiced as BayerRG8 [N, 375, 450] (ADC_IMG_BAYER_RGGB)
* bayer_bgr    : adc_match_batch_device on the same mosaics demosaiced beforehand (cv2.cvtColor), packed BGR on the
                 device: the yardstick for `bayer`, whose image content differs from Cone's
* rect_bayer   : adc_match_rectified_batch_device on raw BayerRG8 frames [N, 480, 640]: Cone resized to 640x480 and
                 mosaiced, rectified through initUndistortRectifyMap maps (CV_16SC2) of rectify_testlib's made-up rig
* rect_bgr_raw : adc_match_rectified_batch_device on the same raw frames demosaiced beforehand, [N, 480, 640, 3]
  The four are timed in alternating windows (`--rounds`); the medians are reported.
* host         : the same raw frames through cv2.cvtColor and cv2.remap on the host (both views of every pair, OpenCV's
                 own threading) followed by adc_match_batch on the rectified images: wall clock over one batch, after a
                 warm-up batch.
* kernels      : the plain and the rectified ingestion kernel alone over one wave (adc_profile_kernel ids 13 and 14, CUDA
                 events) for Bayer input, the rectified one also for the demosaiced BGR frames, each next to a
                 device-to-device cudaMemcpyAsync (torch copy_) that moves as many bytes (read + write) as the kernel's
                 algorithmic bytes (per view N read + 3N written; plus both views' maps once per wave for id 14).
Every Bayer map is checked bit for bit against the packed-BGR maps of the demosaiced images (and the host path's).  The
card's name and power limit are recorded beside the numbers.  Prints one JSON line; writes nothing.
"""
import statistics
import sys

import cv2
import torch

import benchlib as B
import adcensus_b200 as A
import bayer_testlib as BT
import rectify_testlib as R

PAT = "bayer_rggb"


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    sw, sh = 640, 480
    D = 64
    mos = [BT.mosaic(img, PAT) for img in (left, right)]
    demo = [BT.cv_demosaic(cv2, m, PAT) for m in mos]
    raw = [BT.mosaic(cv2.resize(img, (sw, sh), interpolation=cv2.INTER_LINEAR), PAT) for img in (left, right)]
    raw_bgr = [BT.cv_demosaic(cv2, r, PAT) for r in raw]
    maps = [R.cone_rig(cv2, sw, sh, w, h, cv2.CV_16SC2, s) for s in (1, -1)]
    m_left, m_right = rep(mos[0]), rep(mos[1])
    b_left, b_right = rep(demo[0]), rep(demo[1])
    r_left, r_right = rep(raw[0]), rep(raw[1])
    rb_left, rb_right = rep(raw_bgr[0]), rep(raw_bgr[1])
    out = {k: torch.empty((n, h, w), dtype=torch.float32, device=dev)
           for k in ("bayer", "bayer_bgr", "rect_bayer", "rect_bgr_raw")}
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    desc = A.image_desc(PAT)

    def bayer(_):
        eng.match_images_batch_device(n, m_left.data_ptr(), m_right.data_ptr(), image=desc,
                                      d_disp=out["bayer"].data_ptr(), stream=st.cuda_stream)

    def bayer_bgr(_):
        eng.match_batch_device(n, b_left.data_ptr(), b_right.data_ptr(), out["bayer_bgr"].data_ptr(), st.cuda_stream)

    def rect_bayer(_):
        eng.match_rectified_batch_device(n, r_left.data_ptr(), r_right.data_ptr(), image=desc,
                                         d_disp=out["rect_bayer"].data_ptr(), stream=st.cuda_stream)

    def rect_bgr_raw(_):
        eng.match_rectified_batch_device(n, rb_left.data_ptr(), rb_right.data_ptr(),
                                         d_disp=out["rect_bgr_raw"].data_ptr(), stream=st.cuda_stream)

    ms = B.windows(eng, st, (bayer, bayer_bgr, rect_bayer, rect_bgr_raw), args.steps, args.warmup, args.rounds)
    eng.set_pipelined(False)

    # host path: cv2.cvtColor + cv2.remap of every view, then adc_match_batch (pointer-array form)
    code = getattr(cv2, BT.CV_NAME[PAT])
    lefts, rights = [raw[0]] * n, [raw[1]] * n

    def host():
        return eng.match_batch_ptrs([B.remap(cv2.cvtColor(x, code), maps[0]) for x in lefts],
                                    [B.remap(cv2.cvtColor(x, code), maps[1]) for x in rights])

    host_s, host_maps = B.host_seconds(host, args.rounds)
    got = {k: v.cpu().numpy() for k, v in out.items()}
    checks = {"bayer_vs_bayer_bgr": got["bayer"].tobytes() == got["bayer_bgr"].tobytes(),
              "rect_bayer_vs_rect_bgr_raw": got["rect_bayer"].tobytes() == got["rect_bgr_raw"].tobytes(),
              "rect_bayer_vs_host": all(got["rect_bayer"][i].tobytes() == host_maps[i].tobytes() for i in range(n)),
              "bayer_vs_single_pair": all(got["bayer"][i].tobytes() == eng.match(demo[0], demo[1]).tobytes()
                                          for i in (0, n - 1))}

    kernels = B.kernels_vs_copy(eng, (
        ("image_ingest_bayer", "image_ingest", lambda: eng.match_images(mos[0], mos[1], format=PAT)),
        ("rectify_bayer", "rectify", lambda: eng.match_rectified(raw[0], raw[1], format=PAT)),
        ("rectify_bgr", "rectify", lambda: eng.match_rectified(raw_bgr[0], raw_bgr[1]))), reps=50, dev=dev)
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    host_rate = round(n / statistics.median(host_s), 2)
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "bayer": {"value": rate["bayer"], "call": "adc_match_images_batch_device ([N, H, W] BayerRG8)"},
            "bayer_bgr": {"value": rate["bayer_bgr"],
                          "call": "adc_match_batch_device (the same mosaics demosaiced beforehand, packed BGR)"},
            "rect_bayer": {"value": rate["rect_bayer"],
                           "call": "adc_match_rectified_batch_device (640x480 raw BayerRG8, CV_16SC2 maps)"},
            "rect_bgr_raw": {"value": rate["rect_bgr_raw"],
                             "call": "adc_match_rectified_batch_device (the same raw frames demosaiced beforehand, BGR)"},
            "host_cvtcolor_remap": {"value": host_rate,
                                    "call": "cv2.cvtColor + cv2.remap on the host (both views) + adc_match_batch",
                                    "cv2_threads": cv2.getNumThreads(), "opencv": cv2.__version__},
            "bayer_vs_bayer_bgr": round(rate["bayer"] / rate["bayer_bgr"], 4),
            "rect_bayer_vs_rect_bgr_raw": round(rate["rect_bayer"] / rate["rect_bgr_raw"], 4),
            "rect_bayer_vs_host": round(rate["rect_bayer"] / host_rate, 2),
            "windows_ms": {k: [round(x, 2) for x in v] for k, v in ms.items()},
            "checks": checks,
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "kernels": kernels,
            "card": B.card()}
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
