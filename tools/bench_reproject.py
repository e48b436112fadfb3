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
import argparse
import json
import statistics
import sys
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
import reproject_testlib as RP  # noqa: E402
from bench_cost_input import card  # noqa: E402
from bench_rectify import rig_maps  # noqa: E402
from bench_volume_export import d2d_copy  # noqa: E402
from make_golden_reproject import rig_Q  # noqa: E402

KINDS = ["points", "depth", "disp_s16"]


def windows(eng, st, s2, paths, steps, warmup, rounds):
    """{path name: [ms per window]}: like bench_volume_export.alternating_windows, but a window ends only when both
    the engine (adc_join) and the second stream are done."""
    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for i in range(steps):
            fn(i)
        eng.join(st.cuda_stream)
        st.wait_stream(s2)
        e1.record(st)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for fn in paths:
        for i in range(max(2, warmup)):
            fn(i)
        eng.join(st.cuda_stream)
        torch.cuda.synchronize()
    ms = {fn.__name__: [] for fn in paths}
    for _ in range(rounds):
        for fn in paths:
            ms[fn.__name__].append(timed(fn))
    return ms


def kernel_ms(eng, n, d_disp, Q, outs, reps, st):
    eng.reproject_batch_device(n, d_disp, Q, outs, st.cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(reps):
        eng.reproject_batch_device(n, d_disp, Q, outs, st.cuda_stream)
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timed windows of each path")
    ap.add_argument("--pairs", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reproject.py: no CUDA device (there is no CPU fallback)")
    dev = torch.device("cuda", 0)
    left, right = T.load_cone()
    h, w, _ = left.shape
    N, D, n = w * h, 64, args.pairs
    sw, sh = 640, 480
    raw = [cv2.resize(img, (sw, sh), interpolation=cv2.INTER_LINEAR) for img in (left, right)]
    rep = lambda a: torch.from_numpy(np.repeat(a[None], n, 0)).to(dev)
    d_left, d_right = rep(left), rep(right)
    r_left, r_right = rep(raw[0]), rep(raw[1])
    Q = rig_Q(w, h, True)
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_rectification(rig_maps(sw, sh, w, h, 1), rig_maps(sw, sh, w, h, -1), (sw, sh))
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

    ms = windows(eng, st, s2, (plain, reproj, rect, rect_points), args.steps, args.warmup, args.rounds)
    eng.set_pipelined(False)

    # checks: the maps are the reference's, and every output of the timed reprojections is the restatement's
    golden = json.loads(str(np.load(T.GOLDEN_DIR / "golden_cone_full.npz")["hashes"]))["MEDIAN/DISP_L"]
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
    k_all = kernel_ms(eng, n, d0.data_ptr(), Q, [(outs[k].data_ptr(), k) for k in KINDS], reps, st)
    k_pts = kernel_ms(eng, n, d0.data_ptr(), Q, [(outs["points"].data_ptr(), "points")], reps, st)
    checks["kernel_outputs_vs_restatement"] = RP.same_nan(outs["points"][-1].cpu().numpy(), RP.points(m0, Q))
    bytes_all, bytes_pts = n * N * (4 + 12 + 4 + 2), n * N * (4 + 12)
    cp = torch.empty(bytes_all // 2, dtype=torch.uint8, device=dev)
    cp_all_ms, cp_all_gbs = d2d_copy(cp, bytes_all // 2, reps)
    cp_pts_ms, cp_pts_gbs = d2d_copy(cp, bytes_pts // 2, reps)
    rate = lambda v: round(n * args.steps / (statistics.median(v) * 1e-3), 2)
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "plain": {"value": rate(ms["plain"]), "call": "adc_match_batch_device"},
            "reproj": {"value": rate(ms["reproj"]),
                       "call": "adc_match_batch_device + adc_reproject_batch_device (points, depth, disp_s16) on a "
                               "second stream after adc_join"},
            "reproj_vs_plain": round(rate(ms["reproj"]) / rate(ms["plain"]), 4),
            "rect": {"value": rate(ms["rect"]), "call": "adc_match_rectified_batch_device (640x480 raw BGR)"},
            "rect_points": {"value": rate(ms["rect_points"]),
                            "call": "adc_match_rectified_batch_device + adc_reproject_batch_device (points)"},
            "rect_points_vs_rect": round(rate(ms["rect_points"]) / rate(ms["rect"]), 4),
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
            "card": card()}
    eng.close()
    print(json.dumps(line), flush=True)
    return 0 if all(checks.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
