#!/usr/bin/env python
"""Image input formats against the packed-BGR batch call on bench.py's workload (Cone 450x375x64, batch 256,
device-resident, pipelined), in one process so that every figure comes from the same run:

  python tools/bench_image_formats.py [--steps 5 --warmup 3 --rounds 3]

* bgr        : adc_match_batch_device on packed BGR [N, H, W, 3] (what bench.py's "value" times)
* rgb_planar : adc_match_images_batch_device on a torchvision-style RGB batch [N, 3, H, W]
* gray       : adc_match_images_batch_device on a gray batch [N, H, W] (Cone's green channel)
* gray_bgr   : adc_match_batch_device on the same gray images replicated to packed BGR: the yardstick for `gray`, whose
               image content (and so the data-dependent refinement work) differs from Cone's colour images
* sbs_bgra   : adc_match_images_batch_device on side-by-side BGRA frames [N, H, 2W, 4], right view at +4W bytes
  The four are timed in alternating windows (`--rounds`); the medians are reported.
* kernel     : the ingestion kernel alone over one wave (adc_profile_kernel id 13, CUDA events) in each format, next to
               a device-to-device cudaMemcpyAsync (torch copy_) of the bytes the two cudaMemcpy2DAsync calls of the
               packed-BGR path move for one wave (both views: 2*3*N per pair), timed in the same process.
Every timed colour map is checked against the unmodified reference's sha256 (tests/golden); the gray maps against the
single-pair adc_match_images result of the same gray images.  The card's name and power limit are recorded beside the
numbers.  Prints one JSON line; writes nothing.
"""
import sys

import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import adc_testlib as T
import images_testlib as IT


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    D = 64
    golden = B.golden()
    d_left, d_right = rep(left), rep(right)
    p_left, p_right = rep(IT.from_bgr(left, "rgb_planar")), rep(IT.from_bgr(right, "rgb_planar"))
    g_left, g_right = rep(left[:, :, 1].copy()), rep(right[:, :, 1].copy())
    gb_left, gb_right = rep(IT.gray_to_bgr(left[:, :, 1])), rep(IT.gray_to_bgr(right[:, :, 1]))
    sbs = rep(np.concatenate([IT.from_bgr(left, "bgra"), IT.from_bgr(right, "bgra")], axis=1))
    out = {k: torch.empty((n, h, w), dtype=torch.float32, device=dev) for k in ("bgr", "rgb_planar", "gray", "gray_bgr",
                                                                                    "sbs_bgra")}
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    desc_p = A.image_desc("rgb_planar")
    desc_g = A.image_desc("gray")
    desc_s = A.image_desc("bgra", 8 * w, 0, 8 * w * h)

    def bgr(_):
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), out["bgr"].data_ptr(), st.cuda_stream)

    def rgb_planar(_):
        eng.match_images_batch_device(n, p_left.data_ptr(), p_right.data_ptr(), image=desc_p,
                                      d_disp=out["rgb_planar"].data_ptr(), stream=st.cuda_stream)

    def gray(_):
        eng.match_images_batch_device(n, g_left.data_ptr(), g_right.data_ptr(), image=desc_g,
                                      d_disp=out["gray"].data_ptr(), stream=st.cuda_stream)

    def gray_bgr(_):
        eng.match_batch_device(n, gb_left.data_ptr(), gb_right.data_ptr(), out["gray_bgr"].data_ptr(), st.cuda_stream)

    def sbs_bgra(_):
        eng.match_images_batch_device(n, sbs.data_ptr(), sbs.data_ptr() + 4 * w, image=desc_s,
                                      d_disp=out["sbs_bgra"].data_ptr(), stream=st.cuda_stream)

    ms = B.windows(eng, st, (bgr, rgb_planar, gray, gray_bgr, sbs_bgra), args.steps, args.warmup, args.rounds)
    eng.set_pipelined(False)
    gray_single, _ = eng.match_images(left[:, :, 1].copy(), right[:, :, 1].copy(), format="gray")

    def all_equal(t, want_sha):
        a = t.cpu().numpy()
        return all(T.sha(a[i]) == want_sha for i in range(n))

    checks = {"bgr": all_equal(out["bgr"], golden), "rgb_planar": all_equal(out["rgb_planar"], golden),
              "sbs_bgra": all_equal(out["sbs_bgra"], golden), "gray": all_equal(out["gray"], T.sha(gray_single)),
              "gray_bgr": all_equal(out["gray_bgr"], T.sha(gray_single))}

    reps = 50
    N, S = h * w, eng.wave_pairs
    kernels = {}
    for fmt in ("rgb_planar", "gray", "bgra", "rgb"):
        # the kernel timing takes the format of the engine's last images call: make one single-pair call of that format
        one = {"rgb_planar": IT.from_bgr(left, "rgb_planar"), "gray": left[:, :, 1].copy(),
               "bgra": IT.from_bgr(left, "bgra"), "rgb": IT.from_bgr(left, "rgb")}[fmt]
        eng.match_images(one, one, format=fmt)
        k_ms, k_bytes = eng.profile_kernel("image_ingest", reps=reps)
        kernels[fmt] = {"ms_per_wave": round(k_ms, 4), "algorithmic_bytes": k_bytes,
                        "achieved_gbs": round(k_bytes / (k_ms * 1e-3) / 1e9, 1)}
    cp_bytes = S * 2 * 3 * N
    cp_ms, cp_gbs = B.d2d_copy(torch.zeros(cp_bytes, dtype=torch.uint8, device=dev), cp_bytes, reps)
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "bgr": {"value": rate["bgr"], "call": "adc_match_batch_device (packed BGR)"},
            "rgb_planar": {"value": rate["rgb_planar"], "call": "adc_match_images_batch_device ([N, 3, H, W] RGB)"},
            "gray": {"value": rate["gray"], "call": "adc_match_images_batch_device ([N, H, W] gray)"},
            "gray_bgr": {"value": rate["gray_bgr"], "call": "adc_match_batch_device (the gray images as packed BGR)"},
            "sbs_bgra": {"value": rate["sbs_bgra"],
                         "call": "adc_match_images_batch_device ([N, H, 2W, 4] side-by-side BGRA)"},
            "vs_bgr": {k: round(rate[k] / rate["bgr"], 4) for k in ("rgb_planar", "sbs_bgra")},
            "gray_vs_gray_bgr": round(rate["gray"] / rate["gray_bgr"], 4),
            "checks": checks,
            "checked_against": "colour: sha256 of the unmodified reference's MEDIAN/DISP_L; gray: the single-pair "
                               "adc_match_images map of the same gray images (also for gray_bgr)",
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": S, "lanes": eng.lanes,
            "ingest_kernel": {**kernels, "note": f"one wave, source bytes of both views + 2*3*N written per pair; CUDA "
                                                 f"events over {reps} launches"},
            "bgr_copies": {"bytes": cp_bytes, "ms": round(cp_ms, 4), "achieved_gbs": round(cp_gbs, 1),
                           "note": "one device-to-device cudaMemcpyAsync of the bytes the packed-BGR path's two "
                                   "cudaMemcpy2DAsync calls move per wave; read + write counted"},
            "card": B.card()}
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
