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
import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import adcensus_b200 as A  # noqa: E402
import adc_testlib as T  # noqa: E402


def card():
    """Name and power limit of the card (read-only nvidia-smi query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout
        name, limit = [c.strip() for c in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as ex:
        return {"name": torch.cuda.get_device_name(), "power_limit": None, "error": str(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cost-input", required=True, choices=[f"{l}-{d}" for l in ("hwd", "dhw") for d in ("f32", "f16", "bf16")])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timed windows of each path")
    ap.add_argument("--pairs", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cost_input.py: no CUDA device (there is no CPU fallback)")
    layout, dtype = args.cost_input.split("-")
    dev = torch.device("cuda", 0)
    left, right = T.load_cone()
    h, w, _ = left.shape
    D, N, n = 64, w * h, args.pairs
    s_auto = min(32, max(2, (12288 + min(w, h) - 1) // min(w, h)))         # adc_create's default wave size
    tdt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[dtype]
    ring = torch.empty((min(n, 4 * s_auto), N * D), dtype=tdt, device=dev)
    eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D))
    eng.set_pipelined(True)
    st = torch.cuda.current_stream()
    d_left = torch.from_numpy(np.repeat(left[None], n, 0)).to(dev)
    d_right = torch.from_numpy(np.repeat(right[None], n, 0)).to(dev)
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
    golden = json.loads(str(np.load(T.GOLDEN_DIR / "golden_cone_full.npz")["hashes"]))["MEDIAN/DISP_L"]

    def regular():
        eng.match_batch_device(n, d_left.data_ptr(), d_right.data_ptr(), d_disp.data_ptr(), st.cuda_stream)

    def cost():
        for j in range(0, n, ring.shape[0]):
            eng.match_cost_batch_device(min(ring.shape[0], n - j), d_left[j:].data_ptr(), d_right[j:].data_ptr(),
                                        ring.data_ptr(), d_disp_c[j:].data_ptr(), layout, dtype, st.cuda_stream)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(args.steps):
            fn()
        eng.join(st.cuda_stream)
        e1.record(st)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for fn in (regular, cost):
        for _ in range(max(2, args.warmup)):
            fn()
        eng.join(st.cuda_stream)
    ms_reg, ms_cost = [], []
    for _ in range(args.rounds):
        ms_reg.append(timed(regular))
        ms_cost.append(timed(cost))
    reg, cst = d_disp.cpu().numpy(), d_disp_c.cpu().numpy()
    reg_ok = all(T.sha(reg[i]) == golden for i in range(n))
    cost_ok = all(T.sha(cst[i]) == want for i in range(n)) and (dtype != "f32" or want == golden)

    reps = 50
    ing_ms, ing_bytes = eng.profile_kernel("cost_ingest", reps=reps)
    cp_bytes = int(ing_bytes // 2)                       # a copy of B bytes reads B and writes B
    src = ring.view(torch.uint8).reshape(-1)[:cp_bytes]
    dst = torch.empty(cp_bytes, dtype=torch.uint8, device=dev)
    dst.copy_(src)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dst.copy_(src)
    e1.record()
    torch.cuda.synchronize()
    cp_ms = e0.elapsed_time(e1) / reps
    ing_gbs = ing_bytes / (ing_ms * 1e-3) / 1e9
    cp_gbs = 2 * cp_bytes / (cp_ms * 1e-3) / 1e9
    rate = lambda ms: round(n * args.steps / (statistics.median(ms) * 1e-3), 2)
    line = {"workload": "cone_450x375_d64_batch256", "input": args.cost_input, "unit": "maps/s",
            "regular": {"value": rate(ms_reg), "call": "adc_match_batch_device", "outputs_bit_identical": reg_ok},
            "cost_input": {"value": rate(ms_cost), "call": "adc_match_cost_batch_device", "ring_pairs": ring.shape[0],
                           "outputs_bit_identical": cost_ok,
                           "outputs_checked_against": "every timed map: the single-pair adc_match_cost map of the same volume"
                                                      + (", = sha256 of the unmodified reference's map" if dtype == "f32" else "")},
            "rounds": args.rounds, "steps_per_round": args.steps, "wave_pairs": eng.wave_pairs, "lanes": eng.lanes,
            "ingest": {"ms_per_wave": round(ing_ms, 4), "algorithmic_bytes": ing_bytes, "achieved_gbs": round(ing_gbs, 1),
                       "note": f"N*D*sizeof(element) read + N*Dp*4 written per pair; CUDA events over {reps} launches"},
            "d2d_copy": {"bytes": cp_bytes, "ms": round(cp_ms, 4), "achieved_gbs": round(cp_gbs, 1),
                         "note": "cudaMemcpyAsync device to device of half the ingestion's bytes; read + write counted"},
            "ingest_vs_copy": round(ing_gbs / cp_gbs, 3), "card": card()}
    eng.close()
    print(json.dumps(line), flush=True)
    return 0 if (reg_ok and cost_ok) else 1


if __name__ == "__main__":
    sys.exit(main())
