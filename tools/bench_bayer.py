#!/usr/bin/env python
"""Bayer mosaics on the way in, on bench.py's workload (Cone 450x375x64, batch 256, device-resident, pipelined), in one
process so that every figure comes from the same run:

  python tools/bench_bayer.py [--steps 5 --warmup 3 --rounds 3]

* bayer        : adc_match_images_batch_device on Cone mosaiced as BayerRG8 [N, 375, 450] (ADC_IMG_BAYER_RGGB)
* bayer_bgr    : adc_match_batch_device on the same mosaics demosaiced beforehand (cv2.cvtColor), packed BGR on the
                 device: the yardstick for `bayer`, whose image content differs from Cone's
* rect_bayer   : adc_match_rectified_batch_device on raw BayerRG8 frames [N, 480, 640]: Cone resized to 640x480 and
                 mosaiced, rectified through initUndistortRectifyMap maps (CV_16SC2) of bench_rectify's made-up rig
* rect_bgr_raw : adc_match_rectified_batch_device on the same raw frames demosaiced beforehand, [N, 480, 640, 3]
  The four are timed in alternating windows (`--rounds`, bench_volume_export's timing); the medians are reported.
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
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import cv2
import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import adcensus_b200 as A  # noqa: E402
import adc_testlib as T  # noqa: E402
import bayer_testlib as B  # noqa: E402
from bench_cost_input import card  # noqa: E402
from bench_rectify import rig_maps  # noqa: E402
from bench_volume_export import alternating_windows, d2d_copy  # noqa: E402

PAT = "bayer_rggb"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timed windows of each path")
    ap.add_argument("--pairs", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bayer.py: no CUDA device (there is no CPU fallback)")
    dev = torch.device("cuda", 0)
    left, right = T.load_cone()
    h, w, _ = left.shape
    sw, sh = 640, 480
    D, n = 64, args.pairs
    mos = [B.mosaic(img, PAT) for img in (left, right)]
    demo = [B.cv_demosaic(cv2, m, PAT) for m in mos]
    raw = [B.mosaic(cv2.resize(img, (sw, sh), interpolation=cv2.INTER_LINEAR), PAT) for img in (left, right)]
    raw_bgr = [B.cv_demosaic(cv2, r, PAT) for r in raw]
    maps = [rig_maps(sw, sh, w, h, s) for s in (1, -1)]
    rep = lambda a: torch.from_numpy(np.repeat(a[None], n, 0)).to(dev)
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

    def bayer():
        eng.match_images_batch_device(n, m_left.data_ptr(), m_right.data_ptr(), image=desc,
                                      d_disp=out["bayer"].data_ptr(), stream=st.cuda_stream)

    def bayer_bgr():
        eng.match_batch_device(n, b_left.data_ptr(), b_right.data_ptr(), out["bayer_bgr"].data_ptr(), st.cuda_stream)

    def rect_bayer():
        eng.match_rectified_batch_device(n, r_left.data_ptr(), r_right.data_ptr(), image=desc,
                                         d_disp=out["rect_bayer"].data_ptr(), stream=st.cuda_stream)

    def rect_bgr_raw():
        eng.match_rectified_batch_device(n, rb_left.data_ptr(), rb_right.data_ptr(),
                                         d_disp=out["rect_bgr_raw"].data_ptr(), stream=st.cuda_stream)

    ms = alternating_windows(eng, st, (bayer, bayer_bgr, rect_bayer, rect_bgr_raw), args.steps, args.warmup, args.rounds)
    eng.set_pipelined(False)

    # host path: cv2.cvtColor + cv2.remap of every view, then adc_match_batch (pointer-array form)
    remap = lambda img, m: cv2.remap(img, *m, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    code = getattr(cv2, B.CV_NAME[PAT])
    lefts, rights = [raw[0]] * n, [raw[1]] * n

    def host():
        return eng.match_batch_ptrs([remap(cv2.cvtColor(x, code), maps[0]) for x in lefts],
                                    [remap(cv2.cvtColor(x, code), maps[1]) for x in rights])

    host()
    host_s = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        host_maps = host()
        host_s.append(time.perf_counter() - t0)
    got = {k: v.cpu().numpy() for k, v in out.items()}
    checks = {"bayer_vs_bayer_bgr": got["bayer"].tobytes() == got["bayer_bgr"].tobytes(),
              "rect_bayer_vs_rect_bgr_raw": got["rect_bayer"].tobytes() == got["rect_bgr_raw"].tobytes(),
              "rect_bayer_vs_host": all(got["rect_bayer"][i].tobytes() == host_maps[i].tobytes() for i in range(n)),
              "bayer_vs_single_pair": all(got["bayer"][i].tobytes() == eng.match(demo[0], demo[1]).tobytes()
                                          for i in (0, n - 1))}

    reps = 50
    kernels = {}
    # the profile ids replay the format of the engine's last images / rectified call: make one of each first
    for name, pid, call in (("image_ingest_bayer", "image_ingest",
                             lambda: eng.match_images(mos[0], mos[1], format=PAT)),
                            ("rectify_bayer", "rectify", lambda: eng.match_rectified(raw[0], raw[1], format=PAT)),
                            ("rectify_bgr", "rectify", lambda: eng.match_rectified(raw_bgr[0], raw_bgr[1]))):
        call()
        k_ms, k_bytes = eng.profile_kernel(pid, reps=reps)
        cp_bytes = int(k_bytes // 2)
        cp_ms, cp_gbs = d2d_copy(torch.zeros(cp_bytes, dtype=torch.uint8, device=dev), cp_bytes, reps)
        kernels[name] = {"ms_per_wave": round(k_ms, 4), "algorithmic_bytes": k_bytes,
                         "achieved_gbs": round(k_bytes / (k_ms * 1e-3) / 1e9, 1),
                         "d2d_copy_same_bytes_ms": round(cp_ms, 4), "d2d_copy_gbs": round(cp_gbs, 1),
                         "kernel_vs_copy": round(cp_ms / k_ms, 4)}
    rate = lambda v: round(n * args.steps / (statistics.median(v) * 1e-3), 2)
    host_rate = round(n / statistics.median(host_s), 2)
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "bayer": {"value": rate(ms["bayer"]), "call": "adc_match_images_batch_device ([N, H, W] BayerRG8)"},
            "bayer_bgr": {"value": rate(ms["bayer_bgr"]),
                          "call": "adc_match_batch_device (the same mosaics demosaiced beforehand, packed BGR)"},
            "rect_bayer": {"value": rate(ms["rect_bayer"]),
                           "call": "adc_match_rectified_batch_device (640x480 raw BayerRG8, CV_16SC2 maps)"},
            "rect_bgr_raw": {"value": rate(ms["rect_bgr_raw"]),
                             "call": "adc_match_rectified_batch_device (the same raw frames demosaiced beforehand, BGR)"},
            "host_cvtcolor_remap": {"value": host_rate,
                                    "call": "cv2.cvtColor + cv2.remap on the host (both views) + adc_match_batch",
                                    "cv2_threads": cv2.getNumThreads(), "opencv": cv2.__version__},
            "bayer_vs_bayer_bgr": round(rate(ms["bayer"]) / rate(ms["bayer_bgr"]), 4),
            "rect_bayer_vs_rect_bgr_raw": round(rate(ms["rect_bayer"]) / rate(ms["rect_bgr_raw"]), 4),
            "rect_bayer_vs_host": round(rate(ms["rect_bayer"]) / host_rate, 2),
            "windows_ms": {k: [round(x, 2) for x in v] for k, v in ms.items()},
            "checks": checks,
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "kernels": {**kernels, "note": f"one wave; CUDA events over {reps} launches; the copy is one cudaMemcpyAsync "
                                           f"of algorithmic_bytes / 2, read + write counted"},
            "card": card()}
    eng.close()
    print(json.dumps(line), flush=True)
    return 0 if all(checks.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
