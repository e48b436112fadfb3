#!/usr/bin/env python
"""Point clouds on bench.py's workload (Cone 450x375x64, batch 256, device-resident, pipelined), in one process so that
every figure comes from the same run:

  python tools/bench_point_cloud.py [--steps 5 --warmup 3 --rounds 3]

* plain        : adc_match_batch_device on packed BGR Cone (what bench.py's "value" times)
* cloud        : the same batch, then, on a second stream that waits with adc_join, adc_point_cloud_batch_device of its
                 256 maps coloured by the left images, with pixel indices
* rect         : adc_match_rectified_batch_device on 640x480 raw BayerRG12p frames (Cone resized and mosaiced, CV_16SC2
                 rig maps): the camera path
* rect_cloud   : the camera path, then on the second stream adc_ingest_views_batch_device of the raw frames and the
                 coloured cloud of the maps by the left views
  Each path is timed in `rounds` alternating windows of `steps` steps (CUDA events on the first stream, which waits for
  the second at the end of a window); medians reported.
* kernel       : adc_point_cloud_batch_device alone over 256 Cone maps (coloured, with pixels), next to
                 adc_reproject_batch_device (points) on the same maps and a device-to-device copy of as many bytes
                 (read + write) as the cloud moves; and reprojection followed by torch boolean indexing (a host sync
                 for the output size), the way a caller without the cloud entry would do it.
Every timed output is checked against the numpy restatement (tests/cloud_testlib.py).  The card's name and power limit
are recorded beside the numbers.  Prints one JSON line; writes nothing.
"""
import sys

import cv2
import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import cloud_testlib as C
import rawdepth_testlib as RD
import rectify_testlib as R
from make_golden_reproject import rig_Q


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    N, D = w * h, 64
    sw, sh = 640, 480
    fmt = "bayer_rg12p"
    rng = np.random.default_rng(0)
    raw = [RD.encode(cv2.resize(img, (sw, sh), interpolation=cv2.INTER_LINEAR), fmt, rng) for img in (left, right)]
    d_left, d_right = rep(left), rep(right)
    r_left, r_right = rep(raw[0]), rep(raw[1])
    raw_desc = A.image_desc(fmt)
    Q = rig_Q(w, h, True)
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    maps = [R.cone_rig(cv2, sw, sh, w, h, cv2.CV_16SC2, s) for s in (1, -1)]
    eng.set_rectification(maps[0], maps[1], (sw, sh))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    s2 = torch.cuda.Stream()
    disp = {k: [torch.empty((n, h, w), dtype=torch.float32, device=dev) for _ in range(2)]
            for k in ("plain", "cloud", "rect", "rect_cloud")}
    views = torch.empty((n, 2, h, w, 3), dtype=torch.uint8, device=dev)
    pts = torch.empty((n, N, 3), dtype=torch.float32, device=dev)
    cols = torch.empty((n, N, 3), dtype=torch.uint8, device=dev)
    pix = torch.empty((n, N), dtype=torch.int32, device=dev)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    wb = eng.point_cloud_workspace_bytes(n)
    work = torch.empty(wb // 8 + 1, dtype=torch.int64, device=dev)

    def cloud_of(d, bgr, stride, stream):
        eng.point_cloud_batch_device(n, d.data_ptr(), Q, pts.data_ptr(), counts.data_ptr(), N, work.data_ptr(), wb,
                                     d_bgr=bgr, bgr_stride=stride, d_colors=cols.data_ptr(), d_pixels=pix.data_ptr(),
                                     stream=stream.cuda_stream)

    def plain(i):
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), disp["plain"][i % 2].data_ptr(), st.cuda_stream)

    def cloud(i):
        d = disp["cloud"][i % 2]
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d.data_ptr(), st.cuda_stream)
        eng.join(s2.cuda_stream)
        cloud_of(d, d_left.data_ptr(), 0, s2)

    def rect(i):
        eng.match_rectified_batch_device(n, r_left.data_ptr(), r_right.data_ptr(), raw_desc,
                                         d_disp=disp["rect"][i % 2].data_ptr(), stream=st.cuda_stream)

    def rect_cloud(i):
        d = disp["rect_cloud"][i % 2]
        eng.match_rectified_batch_device(n, r_left.data_ptr(), r_right.data_ptr(), raw_desc, d_disp=d.data_ptr(),
                                         stream=st.cuda_stream)
        eng.join(s2.cuda_stream)
        eng.ingest_views_batch_device(n, r_left.data_ptr(), r_right.data_ptr(), views.data_ptr(), raw_desc, True,
                                      s2.cuda_stream)
        cloud_of(d, views.data_ptr(), 6 * N, s2)

    ms = B.windows(eng, st, (plain, cloud, rect, rect_cloud), args.steps, args.warmup, args.rounds, side=s2)
    eng.set_pipelined(False)

    # checks: the last cloud (camera path, coloured by the left views) and a plain one against the restatement
    def cloud_ok(m, img):
        wp, wc, wx = C.cloud(m, Q, img)
        k = len(wx)
        return bool(int(counts[0]) == k and np.array_equal(pts[0, :k].cpu().numpy().view(np.uint32), wp.view(np.uint32))
                    and np.array_equal(cols[0, :k].cpu().numpy(), wc) and np.array_equal(pix[0, :k].cpu().numpy(), wx)
                    and bool((counts == counts[0]).all()))

    cam = disp["rect_cloud"][(args.steps - 1) % 2][0].cpu().numpy()
    checks = {"camera_views_are_matched": bool(np.array_equal(
                  eng.ingest_views(raw[0], raw[1], fmt, rectified=True), views[0].cpu().numpy())),
              "camera_cloud_vs_restatement": cloud_ok(cam, views[0, 0].cpu().numpy())}
    m0 = disp["cloud"][0][0].cpu().numpy()
    reps = 20
    k_cloud = B.events_ms(lambda: cloud_of(disp["cloud"][0], d_left.data_ptr(), 0, st), reps, st)
    checks["cloud_vs_restatement"] = cloud_ok(m0, left)
    kept = int(counts.sum())
    rp = torch.empty((n, h, w, 3), dtype=torch.float32, device=dev)
    k_reproj = B.events_ms(lambda: eng.reproject_batch_device(n, disp["cloud"][0].data_ptr(), Q,
                                                              [(rp.data_ptr(), "points")], st.cuda_stream), reps, st)

    def torch_index():
        eng.reproject_batch_device(n, disp["cloud"][0].data_ptr(), Q, [(rp.data_ptr(), "points")], st.cuda_stream)
        d = disp["cloud"][0]
        keep = torch.isfinite(d) & torch.isfinite(rp).all(-1)
        return rp[keep], d_left[keep.view(n, h, w)].flip(-1)

    k_index = B.events_ms(torch_index, reps, st)
    p_idx, c_idx = torch_index()
    checks["torch_indexing_same_points"] = bool(p_idx.shape[0] == kept and torch.equal(
        p_idx.view(torch.int32), torch.cat([pts[i, :int(counts[i])] for i in range(n)]).view(torch.int32)))
    # bytes the cloud moves: maps read, colours read and written, points and pixel indices written
    cloud_bytes = n * N * 4 + kept * (3 + 12 + 3 + 4)
    cp = torch.empty(cloud_bytes // 2 + 1, dtype=torch.uint8, device=dev)
    cp_ms, cp_gbs = B.d2d_copy(cp, cloud_bytes // 2, reps)
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "plain": {"value": rate["plain"], "call": "adc_match_batch_device"},
            "cloud": {"value": rate["cloud"],
                      "call": "adc_match_batch_device + adc_point_cloud_batch_device (colours, pixels) on a second stream "
                              "after adc_join"},
            "cloud_vs_plain": round(rate["cloud"] / rate["plain"], 4),
            "rect": {"value": rate["rect"], "call": "adc_match_rectified_batch_device (640x480 BayerRG12p)"},
            "rect_cloud": {"value": rate["rect_cloud"],
                           "call": "adc_match_rectified_batch_device + adc_ingest_views_batch_device + "
                                   "adc_point_cloud_batch_device coloured by the left views"},
            "rect_cloud_vs_rect": round(rate["rect_cloud"] / rate["rect"], 4),
            "kernel": {"cloud_ms_per_256_maps": round(k_cloud, 4), "kept_points": kept, "bytes": cloud_bytes,
                       "achieved_gbs": round(cloud_bytes / (k_cloud * 1e-3) / 1e9, 1),
                       "d2d_copy_same_bytes_ms": round(cp_ms, 4), "d2d_copy_gbs": round(cp_gbs, 1),
                       "cloud_vs_copy": round(cp_ms / k_cloud, 4),
                       "reproject_points_ms": round(k_reproj, 4),
                       "reproject_then_torch_indexing_ms": round(k_index, 4)},
            "checks": checks,
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "card": B.card()}
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
