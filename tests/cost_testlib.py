"""Test infrastructure of cost-input mode (adc_match_cost*): the CPU checkers with an injected cost volume and a
deterministic cost-volume generator.

``CostOracle`` is the C restatement (oracle/adc_oracle.c, wrapped unchanged by tests/c/orc_cost.c); ``CostReference``
is the unmodified reference behind tests/c/ref_cost_harness.cpp, which only tools/make_golden_cost.py builds (from the
checkout ADC_REFERENCE_DIR names) to record tests/golden/golden_cost_cases.json.
"""
from __future__ import annotations

import ctypes
import subprocess
from pathlib import Path

import numpy as np

import adc_testlib as T

C_DIR = T.REPO / "tests" / "c"
ORACLE_COST_LIB = T.ORACLE_DIR / "_build" / "libadc_oracle_cost.so"


def build_cost_oracle() -> Path:
    """Compiles the restatement with cost injection (same flags as oracle/Makefile's restatement)."""
    srcs = [C_DIR / "orc_cost.c"] + [T.ORACLE_DIR / f for f in ("adc_oracle.c", "adc_oracle.h", "adc_taps.h")]
    if not ORACLE_COST_LIB.exists() or any(s.stat().st_mtime > ORACLE_COST_LIB.stat().st_mtime for s in srcs):
        ORACLE_COST_LIB.parent.mkdir(parents=True, exist_ok=True)
        subprocess.run(["gcc", "-std=gnu11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Wextra",
                        f"-I{T.ORACLE_DIR}", "-o", str(ORACLE_COST_LIB), str(C_DIR / "orc_cost.c"), "-lm"], check=True)
    return ORACLE_COST_LIB


class _CostChecker(T._Checker):
    def begin_cost(self, left: np.ndarray, right: np.ndarray, cost_hwd: np.ndarray):
        """Stages as begin(), but the COST step installs `cost_hwd` (f32 [H][W][D]) instead of computing the cost."""
        left = np.ascontiguousarray(left, np.uint8)
        right = np.ascontiguousarray(right, np.uint8)
        cost = np.ascontiguousarray(cost_hwd, np.float32)
        assert cost.shape == (self.h, self.w, self.D), cost.shape
        self._keep = (left, right, cost)
        f = self._f("begin_cost")
        f.argtypes = [ctypes.c_void_p] * 4
        assert f(self.ctx, left.ctypes.data, right.ctypes.data, cost.ctypes.data) == 1

    def match_cost(self, left, right, cost_hwd) -> np.ndarray:
        self.begin_cost(left, right, cost_hwd)
        while self.step() >= 0:
            pass
        return self.tap("DISP_L").copy()


class CostOracle(_CostChecker):
    def __init__(self, width, height, opt=None):
        super().__init__(build_cost_oracle(), "occ", width, height, opt or T.default_option())


class CostReference(_CostChecker):
    def __init__(self, libpath: Path, width, height, opt=None):
        super().__init__(libpath, "refc", width, height, opt or T.default_option())


# ------------------------------------------------------------------------------------------------
def synthetic_cost(width: int, height: int, disp_range: int, seed: int, dmin: int = 0) -> np.ndarray:
    """Deterministic cost volume f32 [H][W][D] for T.synthetic_pair(width, height, disp_range, seed).

    Every value is a multiple of 1/32 in [0, 4): exactly representable in f16 and bf16, so one volume describes all three
    precisions.  Background costs lie in [1, 4); each pixel has one planted minimum in [0, 0.5) -- at the band disparity
    of synthetic_pair for seven pixels in eight, at a hashed disparity for the rest, so that the LR check finds
    mismatches and region voting / interpolation have real work.  Index d stands for disparity dmin + d."""
    D = int(disp_range)
    M = np.uint64(0xFFFFFFFFFFFFFFFF)
    ys = np.arange(height, dtype=np.uint64)[:, None, None]
    xs = np.arange(width, dtype=np.uint64)[None, :, None]
    ds = np.arange(D, dtype=np.uint64)[None, None, :]
    with np.errstate(over="ignore"):
        base = np.uint64(seed) * np.uint64(0xA24BAED4963EE407) & M
        r = T._splitmix64(base ^ (ys * np.uint64(0x9FB21C651E98DF25)) ^ (xs * np.uint64(0xC2B2AE3D27D4EB4F))
                          ^ (ds * np.uint64(0x165667B19E3779F9)))
        vol = (np.uint64(32) + r % np.uint64(96)).astype(np.int32)
        # band disparity of synthetic_pair (the right view is the left view shifted by it)
        lo = D // 8
        span = max(1, (3 * D) // 4 - lo)
        bands = T._splitmix64(np.uint64(seed) * np.uint64(1000003) + (np.arange(height) // 25).astype(np.uint64))
        band_d = (lo + (bands % np.uint64(span)).astype(np.int64)) - dmin
        p = T._splitmix64(base ^ np.uint64(0x5851F42D4C957F2D) ^ (ys[:, :, 0] * np.uint64(0x2545F4914F6CDD1D))
                          ^ (xs[:, :, 0] * np.uint64(0x9E3779B97F4A7C15)))
    planted = np.where((p & np.uint64(7)) == np.uint64(0), ((p >> np.uint64(8)) % np.uint64(D)).astype(np.int64),
                       np.broadcast_to(band_d[:, None], (height, width)))
    planted = np.clip(planted, 0, D - 1)
    low = ((p >> np.uint64(32)) % np.uint64(16)).astype(np.int32)
    np.put_along_axis(vol, planted[:, :, None], low[:, :, None], axis=2)
    return (vol.astype(np.float32) / np.float32(32.0))


def to_bf16_bits(a: np.ndarray) -> np.ndarray:
    """bfloat16 bit patterns (uint16) of an f32 array whose values are exactly representable in bfloat16."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    assert not (u & np.uint32(0xFFFF)).any(), "value not exactly representable in bfloat16"
    return (u >> np.uint32(16)).astype(np.uint16)


def cost_domain(a: np.ndarray) -> np.ndarray:
    """The value domain the engine applies to a caller's volume (include/adcensus_b200.h): NaN, +inf and values >=
    65536 -> 65536; negatives, -0.0 and -inf -> +0.0."""
    a = np.asarray(a, np.float32)
    with np.errstate(invalid="ignore"):
        out = np.where(a < np.float32(65536.0), a, np.float32(65536.0))
        out = np.where(out > 0, out, np.float32(0.0))
    return out.astype(np.float32)
