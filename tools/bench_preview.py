#!/usr/bin/env python
"""Previews on bench.py's workload (Cone 450x375x64, batch 256, device-resident, pipelined), in one process so that
every figure comes from the same run:

  python tools/bench_preview.py [--steps 5 --warmup 3 --rounds 3]

* plain    : adc_match_batch_device on packed BGR Cone (what bench.py's "value" times)
* preview  : the same batch, then, on a second stream that waits with adc_join, adc_preview_batch_device of its 256
             maps as 1920x1080 NV12 TURBO MINMAX frames (an encoder's input), into one buffer laid out as NV12 surfaces
  Each path is timed in `rounds` alternating windows of `steps` steps (CUDA events on the first stream, which waits for
  the second at the end of a window); medians reported, with the spread (min, max) of the windows.
* kernel   : adc_preview_batch_device alone over the 256 maps (NV12 1080p TURBO, MINMAX and FIXED), next to a
             device-to-device copy of the bytes it writes plus the maps it reads (read + write counted).
* host     : the OpenCV path for one map (cv2.normalize + applyColorMap + resize + cvtColor to I420, then the chroma
             interleaved to NV12 with numpy) on 16 threads, each thread rendering its share of the 256 maps.
Every timed output is checked against the numpy restatement (tests/preview_testlib.py).  The card's name and power
limit are recorded beside the numbers.  Prints one JSON line; writes nothing.
"""
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import preview_testlib as PV


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    D = 64
    FW, FH = 1920, 1080
    d_left, d_right = rep(left), rep(right)
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    s2 = torch.cuda.Stream()
    disp = {k: [torch.empty((n, h, w), dtype=torch.float32, device=dev) for _ in range(2)] for k in ("plain", "preview")}
    frame = FW * FH * 3 // 2
    frames = torch.empty(n * frame, dtype=torch.uint8, device=dev)
    nv12 = A.image_desc("nv12")
    wb = eng.preview_workspace_bytes(n)
    work = torch.empty(wb, dtype=torch.uint8, device=dev)

    def preview_of(d, stream, value_range=None):
        eng.preview_batch_device(n, d.data_ptr(), frames.data_ptr(), nv12, "turbo", value_range, (FW, FH),
                                 d_work=work.data_ptr(), work_bytes=wb, stream=stream.cuda_stream)

    def plain(i):
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), disp["plain"][i % 2].data_ptr(), st.cuda_stream)

    def preview(i):
        d = disp["preview"][i % 2]
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d.data_ptr(), st.cuda_stream)
        eng.join(s2.cuda_stream)
        preview_of(d, s2)

    ms = B.windows(eng, st, (plain, preview), args.steps, args.warmup, args.rounds, side=s2)
    eng.set_pipelined(False)
    m_last = disp["preview"][(args.steps - 1) % 2]
    want = PV.preview(m_last[0].cpu().numpy(), 20, None, (FW, FH), "nv12").reshape(-1)
    got = frames.view(n, frame)
    checks = {"pipelined_preview_vs_restatement": bool(torch.equal(
        got, torch.from_numpy(want).to(dev).expand_as(got)))}

    reps = 20
    k_minmax = B.events_ms(lambda: preview_of(m_last, st), reps, st)
    k_fixed = B.events_ms(lambda: preview_of(m_last, st, (4.0, 0.0)), reps, st)
    want_fixed = PV.preview(m_last[0].cpu().numpy(), 20, (4.0, 0.0), (FW, FH), "nv12").reshape(-1)
    checks["fixed_vs_restatement"] = bool(torch.equal(frames[:frame].cpu(), torch.from_numpy(want_fixed)))
    moved = n * frame + n * w * h * 4              # frames written, maps read (the MINMAX pass reads them once more)
    cp = torch.empty(moved // 2 + 1, dtype=torch.uint8, device=dev)
    cp_ms, cp_gbs = B.d2d_copy(cp, moved // 2, reps)

    # the host path: OpenCV on 16 threads, one map per task
    import cv2
    maps = m_last.cpu().numpy()

    def host_one(m):
        valid = np.isfinite(m)
        g = np.zeros(m.shape, np.uint8)
        cv2.normalize(m, g, 0, 255, cv2.NORM_MINMAX, cv2.CV_8U, valid.astype(np.uint8))
        bgr = cv2.applyColorMap(g, cv2.COLORMAP_TURBO)
        bgr[~valid] = 0
        i420 = cv2.cvtColor(cv2.resize(bgr, (FW, FH), interpolation=cv2.INTER_NEAREST), cv2.COLOR_BGR2YUV_I420)
        flat, q = i420.reshape(-1), FW * FH // 4
        return np.concatenate([flat[:FW * FH], np.stack([flat[FW * FH:FW * FH + q], flat[FW * FH + q:]], -1).reshape(-1)])

    before = cv2.getNumThreads()
    cv2.setNumThreads(1)
    with ThreadPoolExecutor(16) as pool:
        list(pool.map(host_one, maps[:16]))
        host_s = []
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            out = list(pool.map(host_one, maps))
            host_s.append(time.perf_counter() - t0)
    cv2.setNumThreads(before)
    checks["host_path_vs_restatement"] = bool(np.array_equal(out[0], want))

    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    spread = {k: [round(n * args.steps / (x * 1e-3), 2) for x in (max(v), min(v))] for k, v in ms.items()}
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "plain": {"value": rate["plain"], "min_max": spread["plain"], "call": "adc_match_batch_device"},
            "preview": {"value": rate["preview"], "min_max": spread["preview"],
                        "call": "adc_match_batch_device + adc_preview_batch_device (1920x1080 NV12, TURBO, MINMAX) "
                                "on a second stream after adc_join"},
            "preview_cost_pct": round(100.0 * (1.0 - rate["preview"] / rate["plain"]), 2),
            "kernel": {"minmax_ms_per_256_maps": round(k_minmax, 4), "fixed_ms_per_256_maps": round(k_fixed, 4),
                       "bytes": moved, "achieved_gbs_minmax": round(moved / (k_minmax * 1e-3) / 1e9, 1),
                       "d2d_copy_same_bytes_ms": round(cp_ms, 4), "d2d_copy_gbs": round(cp_gbs, 1),
                       "preview_vs_copy": round(cp_ms / k_minmax, 4)},
            "host_opencv_16_threads": {"s_per_256_maps": round(statistics.median(host_s), 4),
                                       "maps_per_s": round(n / statistics.median(host_s), 2)},
            "checks": checks,
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "card": B.card()}
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
