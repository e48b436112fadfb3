#!/usr/bin/env python
"""Speckle removal on bench.py's workload (Cone 450x375x64, batch 256, device-resident, pipelined), in one process so
that every figure comes from the same run:

  python tools/bench_speckles.py [--steps 5 --warmup 3 --rounds 3]

* plain   : adc_match_batch_device on packed BGR Cone (what bench.py's "value" times)
* f32     : the same batch, then, on a second stream that waits with adc_join, adc_filter_speckles_batch_device of its
            256 f32 maps (+inf = missing, max_size 200, max_diff 2)
* s16     : the same batch, then on the second stream the DISP_S16 reprojection and the S16 filter
            ((min_disparity - 1) * 16 missing, max_size 200, max_diff 2 * 16: INTEGRATION.md's call)
  Each path is timed in `rounds` alternating windows of `steps` steps (CUDA events on the first stream, which waits for
  the second at the end of a window); the medians are reported.  Consecutive steps alternate between two map buffers.
* kernel  : the filter alone over the 256 Cone maps, F32 and S16, CUDA events around each call (a fresh copy of the
            maps is made before each, outside the events), next to a device-to-device copy of the map bytes.
* adversarial : one 1920x1080 S16 map each: a one-pixel serpentine that makes one component, a constant map, a
            checkerboard of singletons and white noise; CUDA events as for the kernel.
* opencv  : cv2.filterSpeckles on the host over the same 256 S16 maps, one map per task on a pool of as many threads as
            there are cores (OpenCV releases the GIL), for context.
Every filtered map is checked against the numpy restatement (tests/speckle_testlib.py), and the matched maps against
the reference's Cone MEDIAN/DISP_L hash.  The card's name, power limit and clocks are recorded beside the numbers.
Prints one JSON line; writes nothing.
"""
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import adc_testlib as T
import speckle_testlib as S

MAX_SIZE, MAX_DIFF = 200, 2


def filter_ms(eng, n, src, dst, t, nv, md, work, wb, reps, st):
    """Median ms of adc_filter_speckles_batch_device over n maps (dst refreshed from src before each call, outside
    the events)."""
    out = []
    for _ in range(reps + 2):
        dst.copy_(src)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        eng.filter_speckles_batch_device(n, dst.data_ptr(), t, MAX_SIZE if n > 1 else dst.numel(), md, nv,
                                         work.data_ptr(), wb, st.cuda_stream)
        e1.record(st)
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return statistics.median(out[2:])


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    N, D = w * h, 64
    d_left, d_right = rep(left), rep(right)
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    s2 = torch.cuda.Stream()
    disp = {k: [torch.empty((n, h, w), dtype=torch.float32, device=dev) for _ in range(2)] for k in ("plain", "f32", "s16")}
    s16 = torch.empty((n, h, w), dtype=torch.int16, device=dev)
    wb = eng.speckle_workspace_bytes(n)
    work = torch.empty(wb, dtype=torch.uint8, device=dev)
    s16_invalid = -16.0

    def plain(i):
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), disp["plain"][i % 2].data_ptr(), st.cuda_stream)

    def f32(i):
        d = disp["f32"][i % 2]
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d.data_ptr(), st.cuda_stream)
        eng.join(s2.cuda_stream)
        eng.filter_speckles_batch_device(n, d.data_ptr(), "f32", MAX_SIZE, MAX_DIFF, None, work.data_ptr(), wb,
                                         s2.cuda_stream)

    def s16_path(i):
        d = disp["s16"][i % 2]
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d.data_ptr(), st.cuda_stream)
        eng.join(s2.cuda_stream)
        eng.reproject_batch_device(n, d.data_ptr(), np.eye(4), [(s16.data_ptr(), "disp_s16")], s2.cuda_stream)
        eng.filter_speckles_batch_device(n, s16.data_ptr(), "s16", MAX_SIZE, MAX_DIFF * 16, s16_invalid,
                                         work.data_ptr(), wb, s2.cuda_stream)
    s16_path.__name__ = "s16"

    ms = B.windows(eng, st, (plain, f32, s16_path), args.steps, args.warmup, args.rounds, side=s2)
    eng.set_pipelined(False)

    # checks: the matched maps are the reference's, the filtered ones the restatement's
    golden = B.golden()
    m0 = disp["plain"][0][0].cpu().numpy()
    raw16 = eng.reproject(m0, np.eye(4), ["disp_s16"])["disp_s16"]
    want_f = S.filter_f32(m0, np.inf, MAX_SIZE, MAX_DIFF)
    want_s = S.filter_s16(raw16, s16_invalid, MAX_SIZE, MAX_DIFF * 16)
    same_all = lambda t: bool((t.view(torch.int32 if t.element_size() == 4 else torch.int16) ==
                               t[:1].view(torch.int32 if t.element_size() == 4 else torch.int16)).all())
    checks = {"maps_are_reference_cone": all(T.sha(m) == golden for b in disp["plain"] for m in b.cpu().numpy()),
              "f32_vs_restatement": all(S.same_bits(b[0].cpu().numpy(), want_f) for b in disp["f32"]),
              "s16_vs_restatement": bool(np.array_equal(s16[0].cpu().numpy(), want_s)),
              "every_map_the_same": all(same_all(t) for t in disp["f32"] + [s16]),
              "filter_removes_something": bool((want_f != m0).any() and (want_s != raw16).any())}

    reps = 10
    src_f = disp["plain"][0].clone()
    src_s = torch.from_numpy(np.repeat(raw16[None], n, 0)).to(dev)
    dst_f, dst_s = torch.empty_like(src_f), torch.empty_like(src_s)
    k_f32 = filter_ms(eng, n, src_f, dst_f, "f32", None, MAX_DIFF, work, wb, reps, st)
    k_s16 = filter_ms(eng, n, src_s, dst_s, "s16", s16_invalid, MAX_DIFF * 16, work, wb, reps, st)
    checks["kernel_f32_vs_restatement"] = S.same_bits(dst_f[-1].cpu().numpy(), want_f)
    checks["kernel_s16_vs_restatement"] = bool(np.array_equal(dst_s[-1].cpu().numpy(), want_s))
    cp = torch.empty(n * N * 4, dtype=torch.uint8, device=dev)
    cp_f_ms, cp_f_gbs = B.d2d_copy(cp, n * N * 4, 20)
    cp_s_ms, cp_s_gbs = B.d2d_copy(cp, n * N * 2, 20)
    eng.close()

    # adversarial 1920x1080 maps (S16; new_val 0 marks the serpentine's background as missing)
    H2, W2 = 1080, 1920
    eng2 = A.Engine(W2, H2, A.ADCensusOption(max_disparity=D))
    rng = np.random.default_rng(1)
    serp = np.zeros((H2, W2), np.int16)
    serp[0::2] = 1
    for y in range(1, H2, 2):
        serp[y, W2 - 1 if (y // 2) % 2 == 0 else 0] = 1
    adv = {"serpentine": (serp, 0.0, 0), "constant": (np.full((H2, W2), 7, np.int16), 0.0, 0),
           "checkerboard": (np.where((np.arange(H2)[:, None] + np.arange(W2)[None]) % 2 == 0, 100, -100).astype(np.int16),
                            0.0, 1),
           "noise": (rng.integers(-40, 40, (H2, W2)).astype(np.int16), -41.0, 3)}
    wb2 = eng2.speckle_workspace_bytes(1)
    work2 = torch.empty(wb2, dtype=torch.uint8, device=dev)
    adversarial = {}
    for name, (m, nv, md) in adv.items():
        src = torch.from_numpy(m).to(dev)
        dst = torch.empty_like(src)
        t = filter_ms(eng2, 1, src, dst, "s16", nv, md, work2, wb2, reps, st)
        ok = bool(np.array_equal(dst.cpu().numpy(), S.filter_s16(m, nv, m.size, md)))
        adversarial[name] = {"ms": round(t, 4), "vs_restatement": ok}
        checks[f"adversarial_{name}_vs_restatement"] = ok
    eng2.close()

    # OpenCV on the host, all cores
    host = [raw16.copy() for _ in range(n)]
    cores = os.cpu_count()
    with ThreadPoolExecutor(cores) as pool:
        list(pool.map(lambda a: cv2.filterSpeckles(a, s16_invalid, MAX_SIZE, MAX_DIFF * 16), [raw16.copy()] * cores))
        t0 = time.perf_counter()
        list(pool.map(lambda a: cv2.filterSpeckles(a, s16_invalid, MAX_SIZE, MAX_DIFF * 16), host))
        cv_ms = (time.perf_counter() - t0) * 1e3
    checks["opencv_vs_restatement"] = all(np.array_equal(a, want_s) for a in host)

    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "plain": {"value": rate["plain"], "call": "adc_match_batch_device"},
            "f32": {"value": rate["f32"],
                    "call": "adc_match_batch_device + adc_filter_speckles_batch_device (F32) on a second stream after "
                            "adc_join"},
            "f32_vs_plain": round(rate["f32"] / rate["plain"], 4),
            "s16": {"value": rate["s16"],
                    "call": "adc_match_batch_device + adc_reproject_batch_device (disp_s16) + "
                            "adc_filter_speckles_batch_device (S16) on a second stream after adc_join"},
            "s16_vs_plain": round(rate["s16"] / rate["plain"], 4),
            "kernel_f32": {"ms_per_256_maps": round(k_f32, 4), "d2d_copy_of_map_bytes_ms": round(cp_f_ms, 4),
                           "d2d_copy_gbs": round(cp_f_gbs, 1)},
            "kernel_s16": {"ms_per_256_maps": round(k_s16, 4), "d2d_copy_of_map_bytes_ms": round(cp_s_ms, 4),
                           "d2d_copy_gbs": round(cp_s_gbs, 1)},
            "adversarial_1920x1080_s16": adversarial,
            "opencv_host_256_s16_maps": {"ms": round(cv_ms, 2), "threads": cores, "opencv": cv2.__version__,
                                         "ipp": bool(cv2.ipp.useIPP())},
            "checks": checks,
            "rounds": args.rounds, "steps_per_round": args.steps, "card": {**B.card(), **B.clocks()}}
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
