#!/usr/bin/env python
"""Cost-input mode against the AD-census path on bench.py's workload (Cone 450x375x64, batch 256, device-resident,
pipelined), in one process so that both figures come from the same run:

  python tools/bench_cost_input.py --cost-input dhw-f32 [--steps 5 --warmup 3 --rounds 3]

* regular    : adc_match_batch_device (what bench.py's "value" times)
* cost_input : adc_match_cost_batch_device with the workload's own AD-census volume (debug tap VOL_INIT), converted once
               to the requested layout / element type, as the caller's cost.  A device ring of a few waves' volumes,
               allocated before the engine so that the engine's memory sizing sees it, is cycled through (the volumes
               are only read, so calls in flight may share them).
  The two are timed in alternating windows (`--rounds`); the medians are reported.
* ingest     : the ingestion kernel alone over one wave (adc_profile_kernel id 10, CUDA events) against a device-to-device
               cudaMemcpyAsync (torch copy_) that reads and writes the same number of bytes, timed in the same call.
Every timed map is checked: against the single-pair adc_match_cost map of the same (rounded) volume, which for f32 must
also be the unmodified reference's map (tests/golden).  The card's name and power limit are recorded beside the numbers.
Prints one JSON line; writes nothing.
"""
import sys

import numpy as np
import torch

import benchlib as B
import adcensus_b200 as A
import adc_testlib as T


def main():
    args = B.args(__file__, cost_input=dict(required=True, choices=[f"{l}-{d}" for l in ("hwd", "dhw")
                                                                       for d in ("f32", "f16", "bf16")]))
    layout, dtype = args.cost_input.split("-")
    dev = torch.device("cuda", 0)
    n = args.pairs
    left, right, rep = B.cone(n)
    h, w, _ = left.shape
    D, N = 64, w * h
    tdt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[dtype]
    ring = torch.empty((min(n, 4 * B.default_wave_pairs(w, h)), N * D), dtype=tdt, device=dev)
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    d_left, d_right = rep(left), rep(right)
    d_disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    d_disp_c = torch.empty_like(d_disp)

    eng.debug_run(left, right, "COST")
    vol = torch.from_numpy(eng.tap("VOL_INIT").copy()).to(dev)             # [H][W][D] f32
    if layout == "dhw":
        vol = vol.permute(2, 0, 1).contiguous()
    ring.copy_(vol.reshape(1, -1).to(tdt).expand(ring.shape[0], -1))
    one = ring[0].cpu()
    host = (one.view(torch.int16).numpy().view(np.uint16) if dtype == "bf16" else one.numpy()).reshape(tuple(vol.shape))
    want = T.sha(eng.match_cost(left, right, host, layout, dtype=dtype))
    golden = B.golden()

    def regular(_):
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d_disp.data_ptr(), st.cuda_stream)

    def cost(_):
        for j in range(0, n, ring.shape[0]):
            eng.match_cost_batch_device(min(ring.shape[0], n - j), d_left[j:].data_ptr(), d_right[j:].data_ptr(),
                                        ring.data_ptr(), d_disp_c[j:].data_ptr(), layout, dtype, st.cuda_stream)

    ms = B.windows(eng, st, (regular, cost), args.steps, args.warmup, args.rounds)
    reg, cst = d_disp.cpu().numpy(), d_disp_c.cpu().numpy()
    reg_ok = all(T.sha(reg[i]) == golden for i in range(n))
    cost_ok = all(T.sha(cst[i]) == want for i in range(n)) and (dtype != "f32" or want == golden)

    reps = 50
    ing_ms, ing_bytes, cp_ms, cp_gbs = B.kernel_vs_copy(eng, "cost_ingest", reps, dev)
    ing_gbs = ing_bytes / (ing_ms * 1e-3) / 1e9
    rate = {k: B.maps_per_s(v, n, args.steps) for k, v in ms.items()}
    line = {"workload": "cone_450x375_d64_batch256", "input": args.cost_input, "unit": "maps/s",
            "regular": {"value": rate["regular"], "call": "adc_match_batch_device", "outputs_bit_identical": reg_ok},
            "cost_input": {"value": rate["cost"], "call": "adc_match_cost_batch_device", "ring_pairs": ring.shape[0],
                           "outputs_bit_identical": cost_ok,
                           "outputs_checked_against": "every timed map: the single-pair adc_match_cost map of the same volume"
                                                      + (", = sha256 of the unmodified reference's map" if dtype == "f32" else "")},
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "ingest": {"ms_per_wave": round(ing_ms, 4), "algorithmic_bytes": ing_bytes, "achieved_gbs": round(ing_gbs, 1),
                       "note": f"N*D*sizeof(element) read + N*Dp*4 written per pair; CUDA events over {reps} launches"},
            "d2d_copy": {"bytes": int(ing_bytes // 2), "ms": round(cp_ms, 4), "achieved_gbs": round(cp_gbs, 1),
                         "note": "cudaMemcpyAsync device to device of half the ingestion's bytes; read + write counted"},
            "ingest_vs_copy": round(ing_gbs / cp_gbs, 3), "card": B.card()}
    eng.close()
    return B.emit(line, reg_ok and cost_ok)


if __name__ == "__main__":
    sys.exit(main())
