#!/usr/bin/env python
"""Reprojection to 3-D on bench.py's workload (Cone 450x375x64, batch 256, device-resident, pipelined), in one process
so that every figure comes from the same run:

  python tools/bench_reproject.py [--steps 5 --warmup 3 --rounds 3]

* plain        : adc_match_batch_device on packed BGR Cone (what bench.py's "value" times)
* reproj       : the same batch, then, on a second stream that waits with adc_join, adc_reproject_batch_device of its
                 256 maps to all three kinds (points, depth, disp_s16)
* rect         : adc_match_rectified_batch_device on 640x480 raw BGR frames (Cone resized, CV_16SC2 rig maps): the
                 camera path
* rect_points  : the camera path, then the points of its maps on the second stream
  Each path is timed in `rounds` alternating windows of `steps` steps (CUDA events on the first stream, which waits for
  the second at the end of a window); the medians are reported.  Consecutive steps alternate between two map buffers
  so that a step's batch does not overwrite the maps the previous step's reprojection reads.
* kernel       : adc_reproject_batch_device alone over 256 Cone maps (all three kinds, and points alone), CUDA events,
                 next to a device-to-device cudaMemcpyAsync (torch copy_) that moves as many bytes (read + write) in the
                 same process.
Every timed output is checked against the numpy restatement (tests/reproject_testlib.py) of a map whose sha256 is the
reference's Cone MEDIAN/DISP_L, and of the camera path's map.  The card's name and power limit are recorded beside the
numbers.  Prints one JSON line; writes nothing.
"""
import sys

import cv2
import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import adc_testlib as T
import reproject_testlib as RP
import rectify_testlib as R
from make_golden_reproject import rig_Q

KINDS = ["points", "depth", "disp_s16"]


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    N, D = w * h, 64
    sw, sh = 640, 480
    raw = [cv2.resize(img, (sw, sh), interpolation=cv2.INTER_LINEAR) for img in (left, right)]
    d_left, d_right = rep(left), rep(right)
    r_left, r_right = rep(raw[0]), rep(raw[1])
    Q = rig_Q(w, h, True)
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    maps = [R.cone_rig(cv2, sw, sh, w, h, cv2.CV_16SC2, s) for s in (1, -1)]
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    s2 = torch.cuda.Stream()
    disp = {k: [torch.empty((n, h, w), dtype=torch.float32, device=dev) for _ in range(2)]
            for k in ("plain", "reproj", "rect", "rect_points")}
    outs = {"points": torch.empty((n, h, w, 3), dtype=torch.float32, device=dev),
            "depth": torch.empty((n, h, w), dtype=torch.float32, device=dev),
            "disp_s16": torch.empty((n, h, w), dtype=torch.int16, device=dev)}
    cam_points = torch.empty((n, h, w, 3), dtype=torch.float32, device=dev)

    def reproject_on_s2(d, o):
        eng.join(s2.cuda_stream)
        eng.reproject_batch_device(n, d.data_ptr(), Q, o, s2.cuda_stream)

    def plain(i):
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), disp["plain"][i % 2].data_ptr(), st.cuda_stream)

    def reproj(i):
        d = disp["reproj"][i % 2]
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d.data_ptr(), st.cuda_stream)
        reproject_on_s2(d, [(outs[k].data_ptr(), k) for k in KINDS])

    def rect(i):
        eng.match_rectified_batch_device(n, r_left.data_ptr(), r_right.data_ptr(), d_disp=disp["rect"][i % 2].data_ptr(),
                                         stream=st.cuda_stream)

    def rect_points(i):
        d = disp["rect_points"][i % 2]
        eng.match_rectified_batch_device(n, r_left.data_ptr(), r_right.data_ptr(), d_disp=d.data_ptr(),
                                         stream=st.cuda_stream)
        reproject_on_s2(d, [(cam_points.data_ptr(), "points")])

    ms = B.windows(eng, st, (plain, reproj, rect, rect_points), args.steps, args.warmup, args.rounds, side=s2)
    eng.set_pipelined(False)

    # checks: the maps are the reference's, and every output of the timed reprojections is the restatement's
    golden = B.golden()
    m0 = disp["reproj"][0][0].cpu().numpy()
    cam = disp["rect_points"][0][0].cpu().numpy()
    same_all = lambda t: bool((t.view(torch.int32 if t.element_size() == 4 else torch.int16) ==
                               t[:1].view(torch.int32 if t.element_size() == 4 else torch.int16)).all())
    checks = {"maps_are_reference_cone": all(T.sha(m) == golden for k in ("plain", "reproj") for b in disp[k]
                                             for m in b.cpu().numpy()),
              "points_vs_restatement": RP.same_nan(outs["points"][0].cpu().numpy(), RP.points(m0, Q)),
              "depth_vs_restatement": RP.same_nan(outs["depth"][0].cpu().numpy(), RP.depth(m0, Q)),
              "disp_s16_vs_restatement": bool(np.array_equal(outs["disp_s16"][0].cpu().numpy(), RP.disp_s16(m0, 0))),
              "every_map_the_same": all(same_all(t) for t in list(outs.values()) + [cam_points]),
              "camera_maps_same": all(same_all(b) for b in disp["rect_points"] + disp["rect"]) and
                                  disp["rect"][0][0].cpu().numpy().tobytes() == cam.tobytes(),
              "camera_points_vs_restatement": RP.same_nan(cam_points[0].cpu().numpy(), RP.points(cam, Q))}

    reps = 20
    d0 = disp["reproj"][0]
    kinds_all, kinds_pts = [(outs[k].data_ptr(), k) for k in KINDS], [(outs["points"].data_ptr(), "points")]
    k_all = B.events_ms(lambda: eng.reproject_batch_device(n, d0.data_ptr(), Q, kinds_all, st.cuda_stream), reps, st)
    k_pts = B.events_ms(lambda: eng.reproject_batch_device(n, d0.data_ptr(), Q, kinds_pts, st.cuda_stream), reps, st)
    checks["kernel_outputs_vs_restatement"] = RP.same_nan(outs["points"][-1].cpu().numpy(), RP.points(m0, Q))
    bytes_all, bytes_pts = n * N * (4 + 12 + 4 + 2), n * N * (4 + 12)
    cp = torch.empty(bytes_all // 2, dtype=torch.uint8, device=dev)
    cp_all_ms, cp_all_gbs = B.d2d_copy(cp, bytes_all // 2, reps)
    cp_pts_ms, cp_pts_gbs = B.d2d_copy(cp, bytes_pts // 2, reps)
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "plain": {"value": rate["plain"], "call": "adc_match_batch_device"},
            "reproj": {"value": rate["reproj"],
                       "call": "adc_match_batch_device + adc_reproject_batch_device (points, depth, disp_s16) on a "
                               "second stream after adc_join"},
            "reproj_vs_plain": round(rate["reproj"] / rate["plain"], 4),
            "rect": {"value": rate["rect"], "call": "adc_match_rectified_batch_device (640x480 raw BGR)"},
            "rect_points": {"value": rate["rect_points"],
                            "call": "adc_match_rectified_batch_device + adc_reproject_batch_device (points)"},
            "rect_points_vs_rect": round(rate["rect_points"] / rate["rect"], 4),
            "kernel_all_kinds": {"ms_per_256_maps": round(k_all, 4), "bytes": bytes_all,
                                 "achieved_gbs": round(bytes_all / (k_all * 1e-3) / 1e9, 1),
                                 "d2d_copy_same_bytes_ms": round(cp_all_ms, 4), "d2d_copy_gbs": round(cp_all_gbs, 1),
                                 "kernel_vs_copy": round(cp_all_ms / k_all, 4)},
            "kernel_points": {"ms_per_256_maps": round(k_pts, 4), "bytes": bytes_pts,
                              "achieved_gbs": round(bytes_pts / (k_pts * 1e-3) / 1e9, 1),
                              "d2d_copy_same_bytes_ms": round(cp_pts_ms, 4), "d2d_copy_gbs": round(cp_pts_gbs, 1),
                              "kernel_vs_copy": round(cp_pts_ms / k_pts, 4)},
            "checks": checks,
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "card": B.card()}
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
