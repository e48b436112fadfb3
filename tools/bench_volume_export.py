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
import argparse
import json
import statistics
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import adcensus_b200 as A  # noqa: E402
import adc_testlib as T  # noqa: E402
from bench_cost_input import card  # noqa: E402

GOLDEN_TAP = {"cost": "COST/VOL_INIT", "aggr": "AGG4/VOL_AGGR", "opt": "SO4/VOL_AGGR"}


def alternating_windows(eng, st, paths, steps, warmup, rounds):
    """{path name: [ms per window]}: each path (a function that enqueues one step on `st`) is warmed up, then the paths
    are timed in `rounds` alternating windows of `steps` steps each, CUDA events around a window joined on `st`."""
    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(steps):
            fn()
        eng.join(st.cuda_stream)
        e1.record(st)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for fn in paths:
        for _ in range(max(2, warmup)):
            fn()
        eng.join(st.cuda_stream)
    ms = {fn.__name__: [] for fn in paths}
    for _ in range(rounds):
        for fn in paths:
            ms[fn.__name__].append(timed(fn))
    torch.cuda.synchronize()
    return ms


def d2d_copy(src, nbytes, reps):
    """(ms, GB/s with read + write counted) of a device-to-device copy (torch copy_, cudaMemcpyAsync) of the first
    `nbytes` bytes of the uint8 device tensor `src`, CUDA events over `reps` copies."""
    src = src[:nbytes]
    dst = torch.empty(nbytes, dtype=torch.uint8, device=src.device)
    dst.copy_(src)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dst.copy_(src)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return ms, 2 * nbytes / (ms * 1e-3) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--export", required=True,
                    choices=[f"{s}-{l}-{d}" for s in ("cost", "aggr", "opt") for l in ("hwd", "dhw") for d in ("f32", "f16", "bf16")])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timed windows of each path")
    ap.add_argument("--pairs", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_volume_export.py: no CUDA device (there is no CPU fallback)")
    stage, layout, dtype = args.export.split("-")
    dev = torch.device("cuda", 0)
    left, right = T.load_cone()
    h, w, _ = left.shape
    D, N, n = 64, w * h, args.pairs
    s_auto = min(32, max(2, (12288 + min(w, h) - 1) // min(w, h)))         # adc_create's default wave size
    tdt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[dtype]
    ring_pairs = min(n, 4 * s_auto)
    ring_x = torch.empty((ring_pairs, N * D), dtype=tdt, device=dev)        # export with map
    ring_v = torch.empty((ring_pairs, N * D), dtype=tdt, device=dev)        # volumes only
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    d_left = torch.from_numpy(np.repeat(left[None], n, 0)).to(dev)
    d_right = torch.from_numpy(np.repeat(right[None], n, 0)).to(dev)
    d_disp = torch.empty((n, h, w), dtype=torch.float32, device=dev)
    d_disp_x = torch.empty_like(d_disp)
    hashes = json.loads(str(np.load(T.GOLDEN_DIR / "golden_cone_full.npz")["hashes"]))
    golden = hashes["MEDIAN/DISP_L"]
    _, single = eng.match_volumes(left, right, stage, layout, dtype)
    single = single[stage]

    def regular():
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d_disp.data_ptr(), st.cuda_stream)

    def export():
        for j in range(0, n, ring_pairs):
            eng.match_volumes_batch_device(min(ring_pairs, n - j), d_left[j:].data_ptr(), d_right[j:].data_ptr(),
                                           [(ring_x.data_ptr(), stage, layout, dtype)], d_disp=d_disp_x[j:].data_ptr(),
                                           stream=st.cuda_stream)

    def volumes_only():
        for j in range(0, n, ring_pairs):
            eng.match_volumes_batch_device(min(ring_pairs, n - j), d_left[j:].data_ptr(), d_right[j:].data_ptr(),
                                           [(ring_v.data_ptr(), stage, layout, dtype)], stream=st.cuda_stream)

    ms = alternating_windows(eng, st, (regular, export, volumes_only), args.steps, args.warmup, args.rounds)
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
    k_ms, k_bytes = eng.profile_kernel("cost_export", reps=reps)
    cp_bytes = int(k_bytes // 2)                         # a copy of B bytes reads B and writes B
    cp_ms, cp_gbs = d2d_copy(ring_x.view(torch.uint8).reshape(-1), cp_bytes, reps)
    k_gbs = k_bytes / (k_ms * 1e-3) / 1e9
    rate = lambda v: round(n * args.steps / (statistics.median(v) * 1e-3), 2)
    checked = "every timed map: sha256 of the unmodified reference's map"
    vol_checked = "every ring volume of the last call: the single-pair adc_match_volumes export" + \
        (", = sha256 of the unmodified reference's volume" if dtype == "f32" else "")
    line = {"workload": "cone_450x375_d64_batch256", "export": args.export, "unit": "maps/s",
            "regular": {"value": rate(ms["regular"]), "call": "adc_match_batch_device", "outputs_bit_identical": reg_ok,
                        "outputs_checked_against": checked},
            "export": {"value": rate(ms["export"]), "call": "adc_match_volumes_batch_device (map + volume)",
                       "maps_bit_identical": exp_maps_ok, "volumes_bit_identical": exp_vol_ok,
                       "maps_checked_against": checked, "volumes_checked_against": vol_checked},
            "volumes_only": {"value": rate(ms["volumes_only"]), "unit": "volumes/s",
                             "call": "adc_match_volumes_batch_device (volume, no map)", "volumes_bit_identical": vo_vol_ok,
                             "volumes_checked_against": vol_checked},
            "ring_pairs": ring_pairs, "rounds": args.rounds, "steps_per_round": args.steps,
            "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "export_kernel": {"ms_per_wave": round(k_ms, 4), "algorithmic_bytes": k_bytes, "achieved_gbs": round(k_gbs, 1),
                              "note": f"N*Dp*4 read + N*D*sizeof(element) written per pair; CUDA events over {reps} launches"},
            "d2d_copy": {"bytes": cp_bytes, "ms": round(cp_ms, 4), "achieved_gbs": round(cp_gbs, 1),
                         "note": "cudaMemcpyAsync device to device of half the export's bytes; read + write counted"},
            "export_vs_copy": round(k_gbs / cp_gbs, 3), "card": card()}
    eng.close()
    print(json.dumps(line), flush=True)
    return 0 if (reg_ok and exp_maps_ok and exp_vol_ok and vo_vol_ok) else 1


if __name__ == "__main__":
    sys.exit(main())
