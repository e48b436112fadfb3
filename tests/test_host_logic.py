"""CPU tests of the host side: the C ABI library loads and exports everything the header declares,
the argument/err truth table that needs no GPU, the option block layout, and the multi-rank
sharding plumbing (world_size 2 over gloo)."""
import ctypes
import os
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import engine_testlib as E

ROOT = Path(__file__).resolve().parent.parent


def _lib():
    import adcensus_b200 as A
    from adcensus_b200.build import build_library
    build_library()
    return A, A.load_library()


def test_library_exports_every_declared_symbol():
    A, L = _lib()
    hdr = (ROOT / "include" / "adcensus_b200.h").read_text()
    names = sorted(set(re.findall(r"\b(adc_[a-z_0-9]+)\s*\(", hdr)))
    assert len(names) >= 18
    for n in names:
        assert hasattr(L, n), f"{n} is declared in include/adcensus_b200.h but not exported"
    # the C++ drop-in class is in the same library
    out = subprocess.run(["nm", "-DC", str(A.lib_path())], capture_output=True, text=True).stdout
    for m in ("ADCensusStereo::Initialize", "ADCensusStereo::Match", "ADCensusStereo::Reset", "ADCensusStereo::ADCensusStereo()"):
        assert m in out, m


def test_option_layout_matches_reference_struct():
    A, L = _lib()
    o = A.ADCensusOption()
    assert ctypes.sizeof(o) == 60
    offs = {n: getattr(A.ADCensusOption, n).offset for n, _ in A.ADCensusOption._fields_}
    assert offs["min_disparity"] == 0 and offs["max_disparity"] == 4 and offs["cross_L1"] == 16
    assert offs["so_p1"] == 32 and offs["so_tso"] == 40 and offs["irv_th"] == 48 and offs["lrcheck_thres"] == 52
    assert offs["do_lr_check"] == 56 and offs["do_filling"] == 57 and offs["do_discontinuity_adjustment"] == 58
    c = A.ADCensusOption(min_disparity=7)
    L.adc_default_option(ctypes.byref(c))        # the library's defaults == the reference constructor's
    for n, _ in A.ADCensusOption._fields_:
        if not n.startswith("_"):
            assert getattr(c, n) == pytest.approx(getattr(o, n)), n
    assert (o.max_disparity, o.lambda_ad, o.lambda_census, o.cross_L1, o.cross_L2, o.cross_t1, o.cross_t2) == (64, 10, 30, 34, 17, 20, 6)
    assert (o.so_tso, o.irv_ts, o.do_lr_check, o.do_filling, o.do_discontinuity_adjustment) == (15, 20, True, True, False)


def test_argument_errors_need_no_gpu():
    """ADCensusStereo.cpp:31,38: bad sizes and an empty disparity range fail before any device work."""
    A, L = _lib()
    h = ctypes.c_void_p()
    o = A.ADCensusOption()
    assert L.adc_create(0, 10, ctypes.byref(o), None, ctypes.byref(h)) == 1 and not h.value
    assert L.adc_create(10, -3, ctypes.byref(o), None, ctypes.byref(h)) == 1
    bad = A.ADCensusOption(min_disparity=10, max_disparity=10)
    assert L.adc_create(10, 10, ctypes.byref(bad), None, ctypes.byref(h)) == 1
    assert b"disparity" in L.adc_last_error()
    assert L.adc_create(10, 10, None, None, ctypes.byref(h)) == 1
    assert L.adc_match(None, None, None, None) == 1                      # Match before Initialize
    s = A.ADCensusStereo()
    assert s.Match(np.zeros((2, 2, 3), np.uint8), np.zeros((2, 2, 3), np.uint8)) is False
    assert s.Initialize(-1, 5, o) is False


def test_no_cpu_fallback_without_device():
    """On a box without a GPU, engine creation must fail loudly instead of computing on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    A, L = _lib()
    with pytest.raises(A.AdcError, match="no CUDA device|CUDA"):
        A.Engine(64, 48)


def test_product_never_touches_the_oracle():
    for f in list((ROOT / "adcensus_b200").rglob("*.py")) + list((ROOT / "adcensus_b200" / "csrc").glob("*")) + \
            list((ROOT / "include").glob("*")):
        if f.is_file() and f.suffix in (".py", ".cu", ".cuh", ".cpp", ".h"):
            txt = f.read_text()
            assert "adc_oracle" not in txt and "adc_testlib" not in txt and "libadcensus_ref" not in txt, f


def test_reference_style_cpp_caller_compiles_and_links():
    """A C++ program written against the reference's class interface builds against include/ and
    the shared library, and sees the reference's error truth table."""
    _lib()
    exe = E.c_tool("dropin_main")
    run = subprocess.run([str(exe)], capture_output=True, text=True, env=dict(os.environ, ADC_B200_QUIET="1"))
    assert run.returncode == 0, (run.returncode, run.stdout, run.stderr)
    assert "DROPIN_OK" in run.stdout or "DROPIN_NO_GPU" in run.stdout


def test_shard_bounds():
    from adcensus_b200.parallel import shard_bounds
    assert shard_bounds(4096, 8) == [(i * 512, (i + 1) * 512) for i in range(8)]
    b = shard_bounds(10, 4)
    assert b == [(0, 3), (3, 6), (6, 8), (8, 10)]
    assert shard_bounds(1, 3) == [(0, 1), (1, 1), (1, 1)]


_WORKER = r'''
import os
import numpy as np
import torch.distributed as dist
from adcensus_b200.parallel import run_sharded
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % os.environ["ADC_PORT"],
                        rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
H, W, n = 6, 8, 7
rng = np.random.default_rng(5)
lefts = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
rights = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
def fake_match(l, r):      # stands in for Engine.match_batch: any deterministic per-pair function
    return (l.astype(np.float32).sum(-1) - r.astype(np.float32).sum(-1)) * 0.25
rank = dist.get_rank()
out = run_sharded(fake_match, lefts if rank == 0 else None, rights if rank == 0 else None, H, W)
if rank == 0:
    want = fake_match(lefts, rights)
    assert out.shape == want.shape and np.array_equal(out, want), "gathered order or content wrong"
    print("SHARD_OK")
dist.destroy_process_group()
'''


def test_two_rank_scatter_gather_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    import socket
    with socket.socket() as sk:          # a port the kernel says is free right now (a fixed one can be in TIME_WAIT)
        sk.bind(("127.0.0.1", 0))
        port = str(sk.getsockname()[1])
    procs = []
    for r in range(2):
        path = os.pathsep.join(p for p in (str(ROOT), os.environ.get("PYTHONPATH")) if p)
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", ADC_PORT=port, PYTHONPATH=path)
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    outs = [p.communicate(timeout=180) for p in procs]
    for p, (so, se) in zip(procs, outs):
        assert p.returncode == 0, se[-2000:]
    assert "SHARD_OK" in outs[0][0]


def test_division_sequence_is_exact(tmp_path):
    """The aggregation's x / n (cross_aggregator.cpp:389) runs on the device as the compiler's IEEE fast-path sequence with the
    reciprocal hoisted (adc_div4, k_aggregate.cu).  tests/c/div_sequence.c replays that sequence on the CPU for every divisor
    1..65535, a dense sample of numerators and every approximate reciprocal within 3 ulp of 1/n: all quotients must be the
    IEEE ones."""
    import subprocess
    exe = tmp_path / "div_sequence"
    subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-o", str(exe), str(ROOT / "tests" / "c" / "div_sequence.c"), "-lm"], check=True)
    r = subprocess.run([str(exe), "300", "3"], capture_output=True, text=True)
    assert r.returncode == 0 and "total 0" in r.stdout, r.stdout
