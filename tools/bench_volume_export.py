#!/usr/bin/env python
"""Volume export against the plain batch call on bench.py's workload (Cone 450x375x64, batch 256, device-resident,
pipelined), in one process so that every figure comes from the same run:

  python tools/bench_volume_export.py --export opt-dhw-bf16 [--steps 5 --warmup 3 --rounds 3]

* regular      : adc_match_batch_device (what bench.py's "value" times)
* export       : adc_match_volumes_batch_device with the map and one exported volume (stage-layout-dtype)
* volumes_only : the same without a map: the pipeline stops after the exported stage
  The exported volumes go to device rings of a few waves' volumes, allocated before the engine so that the engine's
  memory sizing sees them; a batch is cut into calls of one ring each.  Every pair of the workload is the Cone pair, so
  calls in flight that share a ring write the same values.  The three are timed in alternating windows (`--rounds`);
  the medians are reported.
* export kernel: the export kernel alone over one wave (adc_profile_kernel id 11, CUDA events) against a device-to-device
               cudaMemcpyAsync (torch copy_) that reads and writes the same number of bytes, timed in the same call.
Every timed map is checked against the unmodified reference's sha256 (tests/golden); the last call's exported volumes
against the single-pair adc_match_volumes export and, for f32, against the reference's Cone volumes (COST/VOL_INIT,
AGG4/VOL_AGGR, SO4/VOL_AGGR).  The card's name and power limit are recorded beside the numbers.  Prints one JSON line;
writes nothing.
"""
import sys

import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import adc_testlib as T

GOLDEN_TAP = {"cost": "COST/VOL_INIT", "aggr": "AGG4/VOL_AGGR", "opt": "SO4/VOL_AGGR"}


def main():
    args = B.args(__file__, export=dict(required=True, choices=[f"{s}-{l}-{d}" for s in ("cost", "aggr", "opt")
                                                                  for l in ("hwd", "dhw")
                                                                  for d in ("f32", "f16", "bf16")]))
    stage, layout, dtype = args.export.split("-")
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    D, N = 64, w * h
    tdt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[dtype]
    ring_pairs = min(n, 4 * B.default_wave_pairs(w, h))
    ring_x = torch.empty((ring_pairs, N * D), dtype=tdt, device=dev)        # export with map
    ring_v = torch.empty((ring_pairs, N * D), dtype=tdt, device=dev)        # volumes only
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    d_left, d_right = rep(left), rep(right)
    d_disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    d_disp_x = torch.empty_like(d_disp)
    hashes = B.cone_hashes()
    golden = hashes["MEDIAN/DISP_L"]
    _, single = eng.match_volumes(left, right, stage, layout, dtype)
    single = single[stage]

    def regular(_):
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d_disp.data_ptr(), st.cuda_stream)

    def export(_):
        for j in range(0, n, ring_pairs):
            eng.match_volumes_batch_device(min(ring_pairs, n - j), d_left[j:].data_ptr(), d_right[j:].data_ptr(),
                                           [(ring_x.data_ptr(), stage, layout, dtype)], d_disp=d_disp_x[j:].data_ptr(),
                                           stream=st.cuda_stream)

    def volumes_only(_):
        for j in range(0, n, ring_pairs):
            eng.match_volumes_batch_device(min(ring_pairs, n - j), d_left[j:].data_ptr(), d_right[j:].data_ptr(),
                                           [(ring_v.data_ptr(), stage, layout, dtype)], stream=st.cuda_stream)

    ms = B.windows(eng, st, (regular, export, volumes_only), args.steps, args.warmup, args.rounds)
    reg, exp = d_disp.cpu().numpy(), d_disp_x.cpu().numpy()
    reg_ok = all(T.sha(reg[i]) == golden for i in range(n))
    exp_maps_ok = all(T.sha(exp[i]) == golden for i in range(n))

    def volumes_ok(ring):
        raw = ring.view(torch.int32 if dtype == "f32" else torch.int16).cpu().numpy()
        want = single.view(np.int32 if dtype == "f32" else np.int16).reshape(-1)
        ok = all(np.array_equal(raw[i], want) for i in range(ring_pairs))
        if dtype == "f32":
            v = single if layout == "hwd" else np.ascontiguousarray(single.transpose(1, 2, 0))
            ok = ok and T.sha(v) == hashes[GOLDEN_TAP[stage]]
        return ok

    exp_vol_ok, vo_vol_ok = volumes_ok(ring_x), volumes_ok(ring_v)

    reps = 50
    k_ms, k_bytes, cp_ms, cp_gbs = B.kernel_vs_copy(eng, "cost_export", reps, dev)
    k_gbs = k_bytes / (k_ms * 1e-3) / 1e9
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    checked = "every timed map: sha256 of the unmodified reference's map"
    vol_checked = "every ring volume of the last call: the single-pair adc_match_volumes export" + \
        (", = sha256 of the unmodified reference's volume" if dtype == "f32" else "")
    line = {"workload": "cone_450x375_d64_batch256", "export": args.export, "unit": "maps/s",
            "regular": {"value": rate["regular"], "call": "adc_match_batch_device", "outputs_bit_identical": reg_ok,
                        "outputs_checked_against": checked},
            "export": {"value": rate["export"], "call": "adc_match_volumes_batch_device (map + volume)",
                       "maps_bit_identical": exp_maps_ok, "volumes_bit_identical": exp_vol_ok,
                       "maps_checked_against": checked, "volumes_checked_against": vol_checked},
            "volumes_only": {"value": rate["volumes_only"], "unit": "volumes/s",
                             "call": "adc_match_volumes_batch_device (volume, no map)", "volumes_bit_identical": vo_vol_ok,
                             "volumes_checked_against": vol_checked},
            "ring_pairs": ring_pairs, "rounds": args.rounds, "steps_per_round": args.steps,
            "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "export_kernel": {"ms_per_wave": round(k_ms, 4), "algorithmic_bytes": k_bytes, "achieved_gbs": round(k_gbs, 1),
                              "note": f"N*Dp*4 read + N*D*sizeof(element) written per pair; CUDA events over {reps} launches"},
            "d2d_copy": {"bytes": int(k_bytes // 2), "ms": round(cp_ms, 4), "achieved_gbs": round(cp_gbs, 1),
                         "note": "cudaMemcpyAsync device to device of half the export's bytes; read + write counted"},
            "export_vs_copy": round(k_gbs / cp_gbs, 3), "card": B.card()}
    eng.close()
    return B.emit(line, reg_ok and exp_maps_ok and exp_vol_ok and vo_vol_ok)


if __name__ == "__main__":
    sys.exit(main())
