"""Shared harness of the GPU test modules: engines from an adc_testlib.Option, bit-exact comparison, sentinel-guarded
device buffers, batched calls split for pipelined mode, every output of one batched call, one oracle run mapped to the
outputs the engine exports, the ptxas resource report, the golden fixtures and the C / C++ helper programs.

Importing this module also puts tools/ on sys.path, for the case definitions the tests share with the fixture
generators there.
"""
from __future__ import annotations

import functools
import json
import os
import re
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest

import adc_testlib as T

sys.path.insert(0, str(T.REPO / "tools"))

# (W, H, D, option overrides, seed): the stage-parity cases, also run by the export, map, speckle and reprojection tests
PARITY_CASES = [
    (64, 48, 16, {}, 1),
    (97, 61, 24, {}, 2),            # odd sizes
    (130, 70, 37, {}, 3),           # D not a multiple of 4 (padded stride)
    (50, 40, 64, {}, 4),            # D > W: out-of-image matches everywhere
    (9, 12, 8, {}, 5),              # W <= 9: census early return (adcensus_util.cpp:12)
    (40, 7, 8, {}, 6),              # H <= 7
    (80, 60, 32, {"cross_L1": 10, "cross_L2": 4, "cross_t1": 30, "cross_t2": 12, "so_tso": 25}, 7),
    (80, 60, 32, {"do_lr_check": 0}, 8),
    (80, 60, 32, {"do_filling": 0}, 9),
    (80, 60, 32, {"do_discontinuity_adjustment": 1}, 10),
    (120, 90, 48, {"lambda_ad": 7, "lambda_census": 20, "so_p1": 0.7, "so_p2": 2.5, "irv_ts": 10,
                   "irv_th": 0.3, "lrcheck_thres": 0.5}, 11),
    (150, 100, 130, {}, 12),        # 16 lanes per line, 9 values -> padded stride
    (80, 60, 32, {"min_disparity": 2, "max_disparity": 34}, 31),     # dmin > 0
    (80, 60, 32, {"min_disparity": -4, "max_disparity": 28}, 32),    # negative dmin
    (200, 40, 200, {}, 13),         # a whole warp per line
    (300, 24, 256, {}, 14),         # the largest range: 8 WTA chunks, WIDE voting (16-bit votes, one count per word)
    (64, 40, 255, {}, 15),          # D = 255 (padded to 256), WIDE voting
    (90, 200, 16, {"cross_L1": 70, "cross_L2": 30, "cross_t1": 300, "cross_t2": 300}, 16),   # arms never stop on colour: cross
    #                                 regions of up to 141 rows (the voting scan works in 96-row chunks), 141-tap windows
    (60, 300, 16, {"cross_L1": 130, "cross_L2": 17, "cross_t1": 300, "cross_t2": 300}, 17),  # L1 > 127: WIDE voting that
    #                                 enumerates (regions of more than 65535 pixels), fused aggregation with a larger
    #                                 shared-memory budget
    (700, 20, 12, {}, 18),          # a long row: the horizontal double pass of the aggregation cut into segments
    (33, 21, 5, {}, 19),            # D < 8: a single padded quad pair per pixel
]


# ---- engines and comparison ------------------------------------------------------------------------------------------
def engine(w, h, opt=None, **cfg):
    """An Engine of w x h with the fields of `opt` (an adc_testlib.Option; None = the defaults) and the engine
    configuration `cfg` (wave_pairs, lanes, debug_flags, ...)."""
    import adcensus_b200 as A
    o = A.ADCensusOption()
    if opt is not None:
        for name, _ in T.Option._fields_:
            if not name.startswith("_"):
                setattr(o, name, getattr(opt, name))
    return A.Engine(w, h, o, **cfg)


def bits(a):
    """The array's bit patterns: floating-point elements as unsigned integers of their own width (-0.0 and NaN payloads
    stay distinct), any other array as it is."""
    a = np.ascontiguousarray(a)
    return a.view(f"u{a.dtype.itemsize}") if a.dtype.kind == "f" else a


def same(name, got, want):
    """got and want have the same shape and the same bits, element for element.  A failure reports how many values
    differ, the largest absolute difference over the values finite in both, and how many are finite in one only."""
    assert got.shape == want.shape, f"{name}: shape {got.shape} vs {want.shape}"
    eq = bits(got) == bits(want)
    if eq.all():
        return
    fin = np.isfinite(got) & np.isfinite(want)
    md = float(np.abs(got[fin].astype(np.float64) - want[fin]).max()) if fin.any() else 0.0
    inf_mismatch = int((np.isfinite(got) != np.isfinite(want)).sum())
    raise AssertionError(f"{name}: {int((~eq).sum())} of {eq.size} values differ, max abs diff {md:.3e}, "
                         f"{inf_mismatch} finite/inf mismatches")


def cuda():
    """(torch, the device the GPU tests run on)."""
    import torch
    return torch, torch.device("cuda", 0)


def guarded(count, dtype, lead, tail, sentinel):
    """A device buffer of `count` elements of `dtype` with `lead` elements before them and `tail` after, every element
    set to `sentinel`: (the view of the count elements, a function that is true while every guard element still holds
    the sentinel, bit for bit)."""
    torch, dev = cuda()
    buf = torch.full((lead + count + tail,), sentinel, dtype=dtype, device=dev)
    as_int = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[buf.element_size()]

    def intact():
        guard = torch.cat([buf[:lead], buf[lead + count:]]).view(as_int)
        return bool((guard == torch.full((1,), sentinel, dtype=dtype, device=dev).view(as_int)).all())

    return buf[lead:lead + count], intact


# ---- batched calls ---------------------------------------------------------------------------------------------------
def split_calls(eng, n, pipelined, issue):
    """A batch of n pairs as one call, or in pipelined mode as two calls of half the batch each that flow into each
    other; then one join, a device synchronisation and pipelined mode off.  issue(first, count) makes one call."""
    torch, _ = cuda()
    st = torch.cuda.current_stream()
    eng.set_pipelined(pipelined)
    half = n // 2 if pipelined else n
    for first, count in ((0, half), (half, n - half)):
        if count:
            issue(first, count)
    eng.join(st.cuda_stream)
    torch.cuda.synchronize()
    eng.set_pipelined(False)


def batch_outputs(eng, entry, n, d_left, d_right, stride, *, image=None, volumes=(), maps=(), d_cost=None,
                  pipelined=False, **cost):
    """Every output of the batched entry point `entry` (a bound Engine method) over n pairs: pair i's views at
    d_left / d_right + i * stride bytes, the volume requests `volumes` [(stage, layout, dtype)], the side maps `maps`,
    the final map ("disp"), optionally a cost volume per pair (the tensor d_cost with the cost arguments `cost`).  Every
    destination starts as a sentinel (NaN volumes, -7 maps, 0xee outlier labels), so an element no call writes shows.
    Returns every output on the host; bf16 volumes as their int16 bit patterns."""
    torch, dev = cuda()
    h, w, D = eng.height, eng.width, eng.D
    tdt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
    out = {"disp": torch.full((n, h, w), -7.0, dtype=torch.float32, device=dev)}
    for stage, layout, dtype in volumes:
        out[stage] = torch.full((n, h, w, D) if layout == "hwd" else (n, D, h, w), float("nan"), dtype=tdt[dtype],
                                device=dev)
    for m in maps:
        out[m] = torch.full((n, h, w), 0xee, dtype=torch.uint8, device=dev) if m == "outliers" else \
            torch.full((n, h, w), -7.0, dtype=torch.float32, device=dev)
    if image is not None:
        cost["image"] = image

    def issue(first, count):
        if d_cost is not None:
            cost["d_cost"] = d_cost[first:].data_ptr()
        entry(count, d_left + first * stride, d_right + first * stride,
              maps=[(out[m][first:].data_ptr(), m) for m in maps],
              volumes=[(out[s][first:].data_ptr(), s, layout, dtype) for s, layout, dtype in volumes],
              d_disp=out["disp"][first:].data_ptr(), stream=torch.cuda.current_stream().cuda_stream, **cost)

    split_calls(eng, n, pipelined, issue)
    return {k: (v.view(torch.int16) if v.dtype == torch.bfloat16 else v).cpu().numpy() for k, v in out.items()}


# ---- the oracle ------------------------------------------------------------------------------------------------------
ORACLE_OUTPUTS = {("COST", "VOL_INIT"): "cost", ("AGG4", "VOL_AGGR"): "aggr", ("SO4", "VOL_AGGR"): "opt",
                  ("WTA", "DISP_L"): "wta_left", ("WTA", "DISP_R"): "wta_right",
                  ("OUTLIER", "MISMATCHES"): "mismatches", ("OUTLIER", "OCCLUSIONS"): "occlusions",
                  ("MEDIAN", "DISP_L"): "final"}


def oracle_outputs(W, H, opt, left, right):
    """One oracle run of one pair: the taps the engine's outputs are compared with, by output name (the three volumes
    [H][W][D], the WTA maps, the outlier lists, the final map)."""
    orc = T.Oracle(W, H, opt)
    orc.begin(left, right)
    out = {}
    for st in T.STAGES:
        orc.step()
        for tap in T.STAGE_TAPS[st]:
            if (st, tap) in ORACLE_OUTPUTS:
                out[ORACLE_OUTPUTS[(st, tap)]] = orc.tap(tap).copy()
    orc.close()
    return out


# ---- compiled code ---------------------------------------------------------------------------------------------------
def ptxas_report(src, extra_flags=()):
    """Compiles one .cu file for sm_90a with -Xptxas -v: {function: dict(regs, stack, spill_stores, spill_loads, lmem)}
    for every function ptxas reports (regs None for a function that is not a kernel entry).  Skips without nvcc."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not Path(nvcc).exists():
        pytest.skip(f"nvcc not found at {nvcc}")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                            *extra_flags, str(src), "-o", str(Path(d) / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    out, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'|Function properties for (\w+)", line)
        if m:
            cur = out.setdefault(m.group(1) or m.group(2), dict(regs=None, stack=None, spill_stores=None,
                                                                 spill_loads=None, lmem=0))
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            cur["stack"], cur["spill_stores"], cur["spill_loads"] = map(int, m.groups())
        m = re.search(r"Used (\d+) registers", line)
        if m:
            cur["regs"] = int(m.group(1))
        m = re.search(r"(\d+) bytes lmem", line)
        if m:
            cur["lmem"] = int(m.group(1))
    return out


_TOOLS_DIR = None


@functools.cache
def c_tool(name):
    """The helper program tests/c/<name>.cpp or tests/cpp/<name>.cpp, built once per session into a temporary
    directory (dropin_main against include/ and the shared library)."""
    global _TOOLS_DIR
    if _TOOLS_DIR is None:
        _TOOLS_DIR = tempfile.TemporaryDirectory(prefix="adc_tools_")
    exe = Path(_TOOLS_DIR.name) / name
    if name == "dropin_main":
        import adcensus_b200 as A
        lib = A.lib_path().parent
        cmd = ["g++", "-std=c++17", str(T.REPO / "tests" / "cpp" / f"{name}.cpp"), f"-I{T.REPO / 'include'}", f"-L{lib}",
               "-ladcensus_b200", f"-Wl,-rpath,{lib}", "-o", str(exe)]
    else:
        cmd = ["g++", "-O2", "-std=c++17", "-o", str(exe), str(T.REPO / "tests" / "c" / f"{name}.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return exe


# ---- golden fixtures -------------------------------------------------------------------------------------------------
def golden(name):
    """A JSON fixture under tests/golden, e.g. golden("golden_big.json")."""
    return json.loads((T.GOLDEN_DIR / name).read_text())


def golden_hashes(name):
    """The reference's sha256 per tap of tests/golden/golden_<name>.npz."""
    return json.loads(str(np.load(T.GOLDEN_DIR / f"golden_{name}.npz")["hashes"]))
