#!/usr/bin/env python
"""Rectification on the way in, on bench.py's workload (Cone 450x375x64, batch 256, device-resident, pipelined) fed
from 640x480 raw BGR frames, in one process so that every figure comes from the same run:

  python tools/bench_rectify.py [--steps 5 --warmup 3 --rounds 3]

* bgr       : adc_match_batch_device on packed BGR Cone [N, 375, 450, 3] (what bench.py's "value" times)
* rectified : adc_match_rectified_batch_device on raw frames [N, 480, 640, 3]: Cone resized to 640x480, rectified
              through initUndistortRectifyMap maps (CV_16SC2) of a made-up rig into 450x375
* rect_bgr  : adc_match_batch_device on the same frames rectified by cv2.remap beforehand, packed BGR on the device: the
              yardstick for `rectified`, whose image content (black borders, resampled texture, and so the work of the
              data-dependent refinement) differs from Cone's
  The three are timed in alternating windows (`--rounds`); the medians are reported.
* host      : the same raw frames through cv2.remap on the host (both views of every pair, OpenCV's own threading)
              followed by adc_match_batch on the rectified images: wall clock over one batch, after a warm-up batch.
* kernel    : the rectified ingestion kernel alone over one wave (adc_profile_kernel id 14, CUDA events), next to a
              device-to-device cudaMemcpyAsync (torch copy_) that moves as many bytes (read + write) as the kernel's
              algorithmic bytes, timed in the same process.
Every map of the rectified batch is checked bit for bit against the host path's and rect_bgr's.  The card's name and power limit are
recorded beside the numbers.  Prints one JSON line; writes nothing.
"""
import statistics
import sys

import cv2
import torch

import benchlib as B
import adcensus_b200 as A
import adc_testlib as T
import rectify_testlib as R


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    sw, sh = 640, 480
    D = 64
    raw = [cv2.resize(img, (sw, sh), interpolation=cv2.INTER_LINEAR) for img in (left, right)]
    maps = [R.cone_rig(cv2, sw, sh, w, h, cv2.CV_16SC2, s) for s in (1, -1)]
    d_left, d_right = rep(left), rep(right)
    r_left, r_right = rep(raw[0]), rep(raw[1])
    b_left, b_right = rep(B.remap(raw[0], maps[0])), rep(B.remap(raw[1], maps[1]))
    out = {k: torch.empty((n, h, w), dtype=torch.float32, device=dev) for k in ("bgr", "rectified", "rect_bgr")}
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()

    def bgr(_):
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), out["bgr"].data_ptr(), st.cuda_stream)

    def rectified(_):
        eng.match_rectified_batch_device(n, r_left.data_ptr(), r_right.data_ptr(), d_disp=out["rectified"].data_ptr(),
                                         stream=st.cuda_stream)

    def rect_bgr(_):
        eng.match_batch_device(n, b_left.data_ptr(), b_right.data_ptr(), out["rect_bgr"].data_ptr(), st.cuda_stream)

    ms = B.windows(eng, st, (bgr, rectified, rect_bgr), args.steps, args.warmup, args.rounds)
    eng.set_pipelined(False)

    # host path: cv2.remap of every view, then adc_match_batch (pointer-array form) on the rectified images
    lefts, rights = [raw[0]] * n, [raw[1]] * n

    def host():
        return eng.match_batch_ptrs([B.remap(x, maps[0]) for x in lefts], [B.remap(x, maps[1]) for x in rights])

    host_s, host_maps = B.host_seconds(host, args.rounds)
    got = out["rectified"].cpu().numpy()
    got_b = out["rect_bgr"].cpu().numpy()
    golden = B.golden()
    checks = {"rectified_vs_host": all(got[i].tobytes() == host_maps[i].tobytes() for i in range(n)),
              "rectified_vs_rect_bgr": got.tobytes() == got_b.tobytes(),
              "bgr_vs_reference": all(T.sha(m) == golden for m in out["bgr"].cpu().numpy())}

    reps = 50
    k_ms, k_bytes, cp_ms, cp_gbs = B.kernel_vs_copy(eng, "rectify", reps, dev)
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    host_rate = round(n / statistics.median(host_s), 2)
    line = {"workload": "cone_450x375_d64_batch256_from_640x480", "unit": "maps/s",
            "bgr": {"value": rate["bgr"], "call": "adc_match_batch_device (packed BGR, already rectified)"},
            "rectified": {"value": rate["rectified"],
                          "call": "adc_match_rectified_batch_device (640x480 raw BGR, CV_16SC2 maps)"},
            "host_remap": {"value": host_rate,
                           "call": "cv2.remap on the host (both views) + adc_match_batch on the rectified images",
                           "cv2_threads": cv2.getNumThreads(), "opencv": cv2.__version__},
            "rect_bgr": {"value": rate["rect_bgr"],
                         "call": "adc_match_batch_device (the same frames rectified beforehand, packed BGR)"},
            "rectified_vs_bgr": round(rate["rectified"] / rate["bgr"], 4),
            "rectified_vs_rect_bgr": round(rate["rectified"] / rate["rect_bgr"], 4),
            "rectified_vs_host_remap": round(rate["rectified"] / host_rate, 2),
            "checks": checks,
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "rectify_kernel": {"ms_per_wave": round(k_ms, 4), "algorithmic_bytes": k_bytes,
                               "achieved_gbs": round(k_bytes / (k_ms * 1e-3) / 1e9, 1),
                               "note": f"one wave; per pair both raw frames + 2*3*N written, plus both views' maps "
                                       f"(2*8*N) once per wave; CUDA events over {reps} launches"},
            "d2d_copy_same_bytes": {"ms": round(cp_ms, 4), "achieved_gbs": round(cp_gbs, 1),
                                    "note": "one cudaMemcpyAsync of algorithmic_bytes / 2, read + write counted"},
            "kernel_vs_copy": round(cp_ms / k_ms, 4),
            "card": B.card()}
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
