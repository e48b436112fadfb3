#!/usr/bin/env python
"""Per-pixel side maps against the plain batch call on bench.py's workload (Cone 450x375x64, batch 256, device-resident,
pipelined), in one process so that every figure comes from the same run:

  python tools/bench_output_maps.py [--steps 5 --warmup 3 --rounds 3]

* plain     : adc_match_batch_device (what bench.py's "value" times)
* side_maps : adc_match_outputs_batch_device with the final map + MIN_COST + PEAK_RATIO + OUTLIERS
* map_only  : adc_match_outputs_batch_device with WTA_LEFT + PEAK_RATIO and no final map: the pipeline stops after the WTA
  The three are timed in alternating windows (`--rounds`); the medians are reported.
* kernels   : k_confidence alone over one wave (adc_profile_kernel id 12, both confidence maps) next to k_wta (id 5) and a
              device-to-device cudaMemcpyAsync (torch copy_) that reads and writes k_confidence's bytes, in the same call.
Every timed map is checked against the unmodified reference's sha256 (tests/golden): the final maps against
MEDIAN/DISP_L, WTA_LEFT against WTA/DISP_L, OUTLIERS as lists against OUTLIER/MISMATCHES and OUTLIER/OCCLUSIONS, the
confidence maps against the numpy helper (tests/maps_testlib.py) on the engine's f32 optimised volume of the pair, whose
sha256 must be the reference's SO4/VOL_AGGR.  The card's name and power limit are recorded beside the numbers.  Prints
one JSON line; writes nothing.
"""
import sys

import torch

import benchlib as B
import adcensus_b200 as A
import adc_testlib as T
import maps_testlib as MT


def main():
    args = B.args(__file__)
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    D = 64
    hashes = B.cone_hashes()
    f32 = lambda: torch.empty((n, h, w), dtype=torch.float32, device=dev)
    d_left, d_right = rep(left), rep(right)
    d_disp, d_disp_s = f32(), f32()
    side = {"min_cost": f32(), "peak_ratio": f32(), "outliers": torch.empty((n, h, w), dtype=torch.uint8, device=dev)}
    only = {"wta_left": f32(), "peak_ratio": f32()}
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    _, single = eng.match_outputs(left, right, volumes=["opt"], layout="hwd", dtype="f32")
    vol_ok = T.sha(single["opt"]) == hashes["SO4/VOL_AGGR"]
    c1, ratio = MT.confidence(single["opt"])
    del single

    def plain(_):
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d_disp.data_ptr(), st.cuda_stream)

    def side_maps(_):
        eng.match_outputs_batch_device(n, d_left.data_ptr(), d_right.data_ptr(),
                                       maps=[(b.data_ptr(), m) for m, b in side.items()], d_disp=d_disp_s.data_ptr(),
                                       stream=st.cuda_stream)

    def map_only(_):
        eng.match_outputs_batch_device(n, d_left.data_ptr(), d_right.data_ptr(),
                                       maps=[(b.data_ptr(), m) for m, b in only.items()], stream=st.cuda_stream)

    ms = B.windows(eng, st, (plain, side_maps, map_only), args.steps, args.warmup, args.rounds)

    def all_equal(t, want_sha):
        a = t.cpu().numpy()
        return all(T.sha(a[i]) == want_sha for i in range(n))

    def lists_ok(t):
        a = t.cpu().numpy()
        for i in range(n):
            mis, occ = MT.outlier_lists(a[i])
            if T.sha(mis) != hashes["OUTLIER/MISMATCHES"] or T.sha(occ) != hashes["OUTLIER/OCCLUSIONS"]:
                return False
        return True

    checks = {
        "plain_maps": all_equal(d_disp, hashes["MEDIAN/DISP_L"]),
        "side_maps_final_maps": all_equal(d_disp_s, hashes["MEDIAN/DISP_L"]),
        "side_maps_min_cost": vol_ok and all_equal(side["min_cost"], T.sha(c1)),
        "side_maps_peak_ratio": vol_ok and all_equal(side["peak_ratio"], T.sha(ratio)),
        "side_maps_outliers": lists_ok(side["outliers"]),
        "map_only_wta_left": all_equal(only["wta_left"], hashes["WTA/DISP_L"]),
        "map_only_peak_ratio": vol_ok and all_equal(only["peak_ratio"], T.sha(ratio)),
    }

    reps = 50
    k_ms, k_bytes, cp_ms, cp_gbs = B.kernel_vs_copy(eng, "confidence", reps, dev)
    w_ms, w_bytes = eng.profile_kernel("wta", reps=reps)
    k_gbs = k_bytes / (k_ms * 1e-3) / 1e9
    w_gbs = w_bytes / (w_ms * 1e-3) / 1e9
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    line = {"workload": "cone_450x375_d64_batch256", "unit": "maps/s",
            "plain": {"value": rate["plain"], "call": "adc_match_batch_device"},
            "side_maps": {"value": rate["side_maps"],
                          "call": "adc_match_outputs_batch_device (final map + MIN_COST + PEAK_RATIO + OUTLIERS)"},
            "map_only": {"value": rate["map_only"],
                         "call": "adc_match_outputs_batch_device (WTA_LEFT + PEAK_RATIO, no final map)"},
            "side_maps_vs_plain": round(rate["side_maps"] / rate["plain"], 4),
            "checks": checks,
            "checked_against": "sha256 of the unmodified reference's MEDIAN/DISP_L, WTA/DISP_L, OUTLIER/MISMATCHES, "
                               "OUTLIER/OCCLUSIONS; confidence: numpy helper on the pair's optimised volume "
                               "(= reference SO4/VOL_AGGR sha256)",
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "confidence_kernel": {"ms_per_wave": round(k_ms, 4), "algorithmic_bytes": k_bytes, "achieved_gbs": round(k_gbs, 1),
                                  "note": f"N*Dp*4 read + 2*4*N written per pair; CUDA events over {reps} launches"},
            "wta_kernel": {"ms_per_wave": round(w_ms, 4), "algorithmic_bytes": w_bytes, "achieved_gbs": round(w_gbs, 1),
                           "note": "N*D*4 read + 8*N written per pair (both views)"},
            "d2d_copy": {"bytes": int(k_bytes // 2), "ms": round(cp_ms, 4), "achieved_gbs": round(cp_gbs, 1),
                         "note": "cudaMemcpyAsync device to device of half of k_confidence's bytes; read + write counted"},
            "confidence_vs_copy": round(k_gbs / cp_gbs, 3), "confidence_vs_wta_time": round(k_ms / w_ms, 3),
            "card": B.card()}
    eng.close()
    return B.emit(line, all(checks.values()))


if __name__ == "__main__":
    sys.exit(main())
