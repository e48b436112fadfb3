"""Test infrastructure of volume export (adc_match_volumes*): the expected contents of an exported volume."""
from __future__ import annotations

import numpy as np


def to_bf16_rn_bits(a: np.ndarray) -> np.ndarray:
    """bfloat16 bit patterns (uint16) of f32 values rounded to nearest, ties to even (__float2bfloat16_rn) -- what the
    volume export writes for ADC_COST_BF16.  Finite inputs (the engine's volumes hold no NaN)."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = (u + np.uint64(0x7FFF) + ((u >> np.uint64(16)) & np.uint64(1))) >> np.uint64(16)
    return (r & np.uint64(0xFFFF)).astype(np.uint16)


def export_of(vol_hwd: np.ndarray, layout: str, dtype: str) -> np.ndarray:
    """What the export must produce from an f32 [H][W][D] volume: [H][W][D] ("hwd") or [D][H][W] ("dhw"), as float32,
    float16 (IEEE round-to-nearest-even, 65520 and above -> +inf) or bfloat16 bit patterns."""
    v = vol_hwd if layout == "hwd" else np.ascontiguousarray(vol_hwd.transpose(2, 0, 1))
    if dtype == "f32":
        return np.ascontiguousarray(v, np.float32)
    if dtype == "f16":
        with np.errstate(over="ignore"):
            return v.astype(np.float16)
    return to_bf16_rn_bits(v)
