#!/usr/bin/env python
"""Resizing on the way in, on bench.py's workload (Cone 450x375x64, batch 256, device-resident, pipelined), in one
process so that every figure comes from the same run:

  python tools/bench_resize.py [--steps 5 --warmup 3 --rounds 3]

Source frames are Cone scaled up with cv2.resize(INTER_LINEAR) and encoded; each direct path is timed against the
packed-BGR call on the same frames converted and resized beforehand (its yardstick; the image content differs from
Cone's, and from path to path):
* bgr_area            : adc_match_rectified_batch_device on tight 900 x 750 BGR frames, ADC_RESIZE_AREA (2 x 2)
* bayer_rg12p_area    : the same on 900 x 750 BayerRG12p frames, ADC_RESIZE_AREA (2 x 2)
* nv12_bt709_linear   : the same on 1920 x 1080 NV12 | ADC_IMG_YUV_BT709 frames, ADC_RESIZE_LINEAR_EXACT
* <path>_pre          : adc_match_batch_device (packed BGR) on the frames of <path> converted and resized beforehand
  The AREA paths share one engine and the LINEAR_EXACT paths another (a geometry is per engine); each engine's paths
  are timed in alternating windows (`--rounds`); the medians are reported.
* host                : the 1920 x 1080 NV12 frames (BT.601, which OpenCV converts) through cv2.cvtColor + cv2.resize
                        (INTER_LINEAR_EXACT) on the host (both views of every pair, all OpenCV threads) followed by
                        adc_match_batch: wall clock over one batch, after a warm-up batch.
* kernels             : the resize ingestion (adc_profile_kernel id 14) of each direct path over one wave (CUDA events),
                        next to a device-to-device cudaMemcpyAsync that moves as many bytes (read + write) as the
                        kernel's algorithmic bytes (both raw frames read, 2*3*N written, per pair).
Every direct map is checked bit for bit against its yardstick's, and the host path's against a direct NV12 call.  The
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
import rawdepth_testlib as RD
import resize_testlib as RS
import yuv_video_testlib as V


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    rep16 = B.cone(n, raw=True)[2]
    h, w, _ = left.shape
    D = 64
    rng = np.random.default_rng(7)
    BT709 = A.IMG_YUV_BT709

    def up(img, size):
        return cv2.resize(img, size, interpolation=cv2.INTER_LINEAR)

    # direct frames (per view) and the packed BGR they stand for, resized beforehand
    bgr = [up(img, (2 * w, 2 * h)) for img in (left, right)]
    bayer = [RD.encode(up(img, (2 * w, 2 * h)), "bayer_rg12p", rng) for img in (left, right)]
    nv = [V.encode(up(img, (1920, 1080)), "nv12") for img in (left, right)]
    frames = {"bgr_area": (bgr, A.image_desc("bgr")), "bayer_rg12p_area": (bayer, A.image_desc("bayer_rg12p")),
              "nv12_bt709_linear": (nv, A.image_desc(A.IMG_NV12 | BT709))}
    pre = {"bgr_area": [RS.area(x, 2, 2) for x in bgr],
           "bayer_rg12p_area": [RS.area(RD.decode(x, "bayer_rg12p", 2 * w, 2 * h), 2, 2) for x in bayer],
           "nv12_bt709_linear": [RS.linear_exact(V.decode(x, "nv12", 1920, 1080, BT709), w, h) for x in nv]}
    direct_d = {k: [rep16(x) for x in f] for k, (f, _) in frames.items()}
    pre_d = {k: [rep(x) for x in f] for k, f in pre.items()}
    out = {k: torch.empty((n, h, w), dtype=torch.float32, device=dev) for k in list(frames) + [k + "_pre" for k in frames]}

    engines = {"area": A.Engine(w, h, A.ADCensusOption(max_disparity=D)),
               "linear_exact": A.Engine(w, h, A.ADCensusOption(max_disparity=D))}
    engines["area"].set_resize((2 * w, 2 * h), "area")
    engines["linear_exact"].set_resize((1920, 1080), "linear_exact")
    groups = {"area": ("bgr_area", "bayer_rg12p_area"), "linear_exact": ("nv12_bt709_linear",)}
    st = torch.cuda.current_stream()

    def path(eng, name):
        if name.endswith("_pre"):
            bufs, desc, entry = pre_d[name[:-4]], None, eng.match_batch_device
        else:
            bufs, desc, entry = direct_d[name], frames[name][1], eng.match_rectified_batch_device

        def run(_):
            if desc is None:
                entry(n, bufs[0].data_ptr(), bufs[1].data_ptr(), out[name].data_ptr(), stream=st.cuda_stream)
            else:
                entry(n, bufs[0].data_ptr(), bufs[1].data_ptr(), image=desc, d_disp=out[name].data_ptr(),
                      stream=st.cuda_stream)
        run.__name__ = name
        return run

    ms = {}
    for kind, names in groups.items():
        eng = engines[kind]
        eng.set_pipelined(True)
        ms.update(B.windows(eng, st, tuple(path(eng, k) for name in names for k in (name, name + "_pre")), args.steps,
                            args.warmup, args.rounds))
        eng.set_pipelined(False)

    # host path: cv2.cvtColor(NV12, BT.601) + cv2.resize(INTER_LINEAR_EXACT) of every view on all cores, then
    # adc_match_batch (pointer-array form); checked against the direct call on the same NV12 frames without a flag
    lin = engines["linear_exact"]
    lefts, rights = [nv[0]] * n, [nv[1]] * n

    def host_view(x):
        return cv2.resize(cv2.cvtColor(x, cv2.COLOR_YUV2BGR_NV12), (w, h), interpolation=cv2.INTER_LINEAR_EXACT)

    def host():
        return lin.match_batch_ptrs([host_view(x) for x in lefts], [host_view(x) for x in rights])

    threads = os.cpu_count()
    host_s, host_maps = B.host_seconds(host, args.rounds, threads=threads)
    d_nv = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    lin.match_rectified_batch_device(n, direct_d["nv12_bt709_linear"][0].data_ptr(),
                                     direct_d["nv12_bt709_linear"][1].data_ptr(), image=A.image_desc("nv12"),
                                     d_disp=d_nv.data_ptr(), stream=st.cuda_stream)
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    checks = {f"{k}_vs_{k}_pre": got[k].tobytes() == got[k + "_pre"].tobytes() for k in frames}
    d_nv = d_nv.cpu().numpy()
    checks["nv12_vs_host"] = all(d_nv[i].tobytes() == host_maps[i].tobytes() for i in range(n))
    checks["pre_is_cv2"] = np.array_equal(pre["bgr_area"][0], cv2.resize(bgr[0], (w, h), interpolation=cv2.INTER_AREA))

    kernels = {}
    for kind, names in groups.items():
        eng = engines[kind]
        kernels.update(B.kernels_vs_copy(eng, tuple(
            (f"resize_{k}", "rectify", (lambda k=k: eng.match_rectified(frames[k][0][0], frames[k][0][1],
                                                                        format=frames[k][1].format)))
            for k in names), reps=50, dev=dev))
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    host_rate = round(n / statistics.median(host_s), 2)
    calls = {"bgr_area": "adc_match_rectified_batch_device (900x750 BGR, ADC_RESIZE_AREA)",
             "bayer_rg12p_area": "adc_match_rectified_batch_device (900x750 BayerRG12p, ADC_RESIZE_AREA)",
             "nv12_bt709_linear": "adc_match_rectified_batch_device (1920x1080 NV12 | BT709, ADC_RESIZE_LINEAR_EXACT)"}
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s"}
    for k in frames:
        line[k] = {"value": rate[k], "call": calls[k]}
        line[k + "_pre"] = {"value": rate[k + "_pre"],
                            "call": "adc_match_batch_device (the same frames converted and resized beforehand)"}
        line[f"{k}_vs_pre"] = round(rate[k] / rate[k + "_pre"], 4)
    line.update({
        "host_cvtcolor_resize": {"value": host_rate, "threads": threads, "opencv": cv2.__version__,
                                 "call": "cv2.cvtColor(COLOR_YUV2BGR_NV12) + cv2.resize(INTER_LINEAR_EXACT) on the "
                                         "host (both views, 1920x1080) + adc_match_batch"},
        "nv12_bt709_linear_vs_host": round(rate["nv12_bt709_linear"] / host_rate, 2),
        "windows_ms": {k: [round(x, 2) for x in v] for k, v in ms.items()},
        "checks": checks,
        "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": lin.wave_pairs, "lanes": lin.lanes,
        "kernels": kernels,
        "card": B.card()})
    for eng in engines.values():
        eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
