"""What every tools/bench_*.py measures with: its command line, bench.py's Cone workload, the windowed and per-launch
CUDA-event timers, the kernel-against-copy comparison, the host-path timer, the card and the JSON line.  The scripts
import this module and no other bench script, so that changing one benchmark's helper cannot change what another
one measures.

Importing it puts the repository root and tests/ on sys.path (once), for adcensus_b200 and the test libraries.
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import adc_testlib as T  # noqa: E402


def args(script, **extra):
    """The parsed command line of `script` (its __file__): its own options `extra` (name: add_argument keywords,
    `cost_input` for --cost-input), then --steps, --warmup, --rounds and --pairs.  Exits when there is no CUDA
    device."""
    ap = argparse.ArgumentParser()
    for name, kw in extra.items():
        ap.add_argument("--" + name.replace("_", "-"), **kw)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternating timed windows of each path")
    ap.add_argument("--pairs", type=int, default=256)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit(f"{Path(script).name}: no CUDA device (there is no CPU fallback)")
    return a


def cone(n, raw=False):
    """bench.py's workload: the Cone pair (BGR [375][450][3]) and rep(a), which puts n replicas of the numpy array a
    on cuda:0 (raw: of a's bytes, for frames of 16-bit words)."""
    left, right = T.load_cone()
    dev = torch.device("cuda", 0)

    def rep(a):
        if raw:
            a = np.ascontiguousarray(a).view(np.uint8)
        return torch.from_numpy(np.repeat(a[None], n, 0)).to(dev)
    return left, right, rep


def cone_hashes():
    """{stage/tap: sha256} of the unmodified reference on Cone (tests/golden)."""
    return json.loads(str(np.load(T.GOLDEN_DIR / "golden_cone_full.npz")["hashes"]))


def golden():
    """sha256 of the unmodified reference's final Cone map."""
    return cone_hashes()["MEDIAN/DISP_L"]


def default_wave_pairs(w, h):
    """adc_create's default wave size for w x h images."""
    return min(32, max(2, (12288 + min(w, h) - 1) // min(w, h)))


def windows(eng, st, paths, steps, warmup, rounds, side=None):
    """{path name: [ms per window]}: each path (a function of the step index that enqueues one step on `st`, and
    perhaps on the stream `side`) is warmed up, then the paths are timed in `rounds` alternating windows of `steps`
    steps each, CUDA events on `st` around a window that ends when the engine (adc_join) and `side` are done."""
    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for i in range(steps):
            fn(i)
        eng.join(st.cuda_stream)
        if side is not None:
            st.wait_stream(side)
        e1.record(st)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for fn in paths:
        for i in range(max(2, warmup)):
            fn(i)
        eng.join(st.cuda_stream)
        torch.cuda.synchronize()
    ms = {fn.__name__: [] for fn in paths}
    for _ in range(rounds):
        for fn in paths:
            ms[fn.__name__].append(timed(fn))
    return ms


def events_ms(fn, reps, st):
    """Mean ms of fn() over `reps` calls, CUDA events on `st`, after one warm call."""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(reps):
        fn()
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


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


def kernel_vs_copy(eng, profile_name, reps, dev):
    """(kernel ms, algorithmic bytes, copy ms, copy GB/s): one pipeline kernel over one wave (adc_profile_kernel,
    `reps` launches) and a device-to-device copy that moves as many bytes, read + write."""
    k_ms, k_bytes = eng.profile_kernel(profile_name, reps=reps)
    cp_bytes = int(k_bytes // 2)                         # a copy of B bytes reads B and writes B
    cp_ms, cp_gbs = d2d_copy(torch.zeros(cp_bytes, dtype=torch.uint8, device=dev), cp_bytes, reps)
    return k_ms, k_bytes, cp_ms, cp_gbs


def kernels_vs_copy(eng, calls, reps, dev):
    """{name: row} of kernel_vs_copy for each (name, profile name, call) of `calls`, plus a note.  The profile ids
    replay the format of the engine's last images / rectified call, so `call` makes one call of that format first."""
    rows = {}
    for name, pid, call in calls:
        call()
        k_ms, k_bytes, cp_ms, cp_gbs = kernel_vs_copy(eng, pid, reps, dev)
        rows[name] = {"ms_per_wave": round(k_ms, 4), "algorithmic_bytes": k_bytes,
                      "achieved_gbs": round(k_bytes / (k_ms * 1e-3) / 1e9, 1),
                      "d2d_copy_same_bytes_ms": round(cp_ms, 4), "d2d_copy_gbs": round(cp_gbs, 1),
                      "kernel_vs_copy": round(cp_ms / k_ms, 4)}
    return {**rows, "note": f"one wave; CUDA events over {reps} launches; the copy is one cudaMemcpyAsync "
                            f"of algorithmic_bytes / 2, read + write counted"}


def remap(img, maps):
    """cv2.remap of img through (map1, map2) as the rectified entries resample: INTER_LINEAR, BORDER_CONSTANT 0."""
    import cv2
    return cv2.remap(img, *maps, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def host_seconds(fn, rounds, threads=None):
    """([s per call] of `rounds` calls after one warm call, the last call's result), on `threads` OpenCV threads if
    given (the setting is restored afterwards)."""
    import cv2
    if threads is not None:
        before = cv2.getNumThreads()
        cv2.setNumThreads(threads)
    fn()
    s = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        out = fn()
        s.append(time.perf_counter() - t0)
    if threads is not None:
        cv2.setNumThreads(before)
    return s, out


def maps_per_s(ms, n, steps):
    """Rate of windows of `steps` steps of n maps each, from the median window in ms."""
    return round(n * steps / (statistics.median(ms) * 1e-3), 2)


def card():
    """Name and power limit of the card (read-only nvidia-smi query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout
        name, limit = [c.strip() for c in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as ex:
        return {"name": torch.cuda.get_device_name(), "power_limit": None, "error": str(ex)}


def clocks():
    """SM clock now and its maximum (read-only nvidia-smi query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout
        sm, mx = [c.strip() for c in out.strip().splitlines()[0].split(",")]
        return {"sm_clock": sm, "max_sm_clock": mx}
    except Exception as ex:
        return {"error": str(ex)}


def emit(line, ok):
    """Prints the one JSON line; the exit code."""
    print(json.dumps(line), flush=True)
    return 0 if ok else 1
