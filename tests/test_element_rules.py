"""Element-rule parity: every bit pattern through each per-element value rule of the engine on the device, against an
exact restatement of the rule.

The parity files compare maps and volumes with the oracle, so each per-element rule below is checked there only on the
values that images and a few specials produce.  Each rule is a small function with a finite domain, and a subtly wrong
kernel (a `<` for a `<=` in a clamp, `_rz` for `_rn`, NaN converted to 0 instead of INT_MIN) changes only a few bit
patterns of it.  This file enumerates the domains:

* cost input (`k_ingest.cu`): all 2^32 f32 patterns as a caller's cost volume, ingested in [H][W][D] and [D][H][W],
  exported as f32 (a bit copy: the value domain of include/adcensus_b200.h exactly), f16 and bf16 (round to nearest
  even); all 2^16 f16 and bf16 patterns in both layouts, exported as f32.  The restatements are integer numpy on the
  bit patterns; CPU tests pin them to numpy's float16 and torch's CPU bfloat16 conversions over all 2^32 patterns.
* reprojection (`k_reproject.cu`): all 2^32 f32 patterns as disparity maps of 4096 x 4096 (256 maps), `DISP_S16` and
  `DEPTH` against reproject_testlib; `POINTS` against live cv2.reprojectImageTo3D on 2^24 patterns (every sign,
  exponent and top 15 mantissa bits, random low bits, plus the specials); point clouds of two of the maps.
* gray (`k_cost.cu`): all 2^24 BGR colours in one 4096 x 4096 image (and permuted in the right view), against the
  oracle and a float64 restatement of cost_computor.cpp:69.
* division (`adc_div.cuh`): tests/cu/div_exhaustive.cu measures the hardware reciprocal over every divisor and runs the
  real adc_div4 over every divisor x every mantissa of three binades (see its header); a sample of its quotients is
  checked here against exact rational arithmetic.

Device memory stays under about 6 GB at every step: the enumerations run in chunks of 2^28 elements.
"""
from __future__ import annotations

import os
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor
from fractions import Fraction

import numpy as np
import pytest

import adc_testlib as T
import cloud_testlib as CL
import engine_testlib as E
import reproject_testlib as RP

ROOT = T.REPO
DIV_SRC = ROOT / "tests" / "cu" / "div_exhaustive.cu"
COST_MAX_BITS = 0x47800000          # ADC_COST_MAX = 65536.0f
CHUNK = 1 << 28                     # elements per enumeration step (1 GB of f32)
BLOCK = 1 << 20                     # elements per CPU work item: the restatements' temporaries stay in cache
_POOL = ThreadPoolExecutor(max_workers=os.cpu_count() or 4)


def _blocks(n, fn):
    """fn(lo, hi) over [0, n) in blocks of BLOCK elements on all cores (numpy releases the GIL); the list of results."""
    return list(_POOL.map(lambda lo: fn(lo, min(lo + BLOCK, n)), range(0, n, BLOCK)))


# ---- restatements, integer numpy on bit patterns -----------------------------------------------------------------------
def cost_domain(u):
    """uint32 f32 bits -> uint32: the value domain of cost input (include/adcensus_b200.h, "Value domain"): NaN (either
    sign), +inf and values >= ADC_COST_MAX become ADC_COST_MAX; negative values, -0.0 and -inf become +0.0; every other
    value (+0.0, positive subnormals included) stays as it is."""
    u = np.asarray(u, np.uint32)
    nan = (u & np.uint32(0x7FFFFFFF)) > np.uint32(0x7F800000)
    out = np.where(u >> np.uint32(31) != 0, np.uint32(0), np.minimum(u, np.uint32(COST_MAX_BITS)))
    out[nan] = COST_MAX_BITS
    return out


def f16_to_f32(h):
    """uint16 IEEE half bits -> uint32 f32 bits, exact (subnormals normalised; NaN keeps its payload, quiet)."""
    h = np.asarray(h, np.uint16).astype(np.uint32)
    s, e, m = (h & 0x8000) << 16, (h >> 10) & 0x1F, h & 0x3FF
    out = np.where(e == 0x1F, np.uint32(0x7F800000) | (m << 13), ((e + 112) << 23) | (m << 13))
    sub = (e == 0) & (m != 0)
    p = np.zeros_like(m)                        # floor(log2(m)) of the subnormals
    for k in range(1, 10):
        p[m >= (1 << k)] = k
    out = np.where(sub, ((p + 103) << 23) | ((m << (23 - p)) & 0x7FFFFF), out)
    out[(e == 0) & (m == 0)] = 0
    return out | s


def bf16_to_f32(b):
    """uint16 bfloat16 bits -> uint32 f32 bits: the upper half."""
    return np.asarray(b, np.uint16).astype(np.uint32) << 16


def f32_to_f16(u):
    """uint32 f32 bits -> uint16 IEEE half bits, round to nearest even: results below 2^-14 are half subnormals
    (2^-25 itself rounds to 0), values from 65520 up become inf, NaN becomes a quiet NaN with the top payload bits."""
    u = np.asarray(u, np.uint32)
    s = (u >> 16) & 0x8000
    a = u & 0x7FFFFFFF
    e = a >> 23
    # normal results: rebias the exponent (127 -> 15), round away 13 bits; a carry moves into the exponent, past the
    # largest finite half into 0x7c00 (inf)
    b = a - np.uint32(0x38000000)
    nrm = np.minimum((b + 0xFFF + ((b >> 13) & 1)) >> 13, 0x7C00)
    # subnormal results: the significand with its hidden bit, in units of 2^-24 (the smallest half subnormal), rounded
    sig = (a & 0x7FFFFF) | 0x800000
    sh = np.clip(126 - np.minimum(e, 126), 1, 25)       # 14 .. 25 where a subnormal result is taken
    sub = (sig + (np.uint32(1) << (sh - 1)) - 1 + ((sig >> sh) & 1)) >> sh
    out = np.where(a >= 0x38800000, nrm, sub)
    out = np.where(a > 0x7F800000, 0x7E00 | ((a >> 13) & 0x3FF), out)
    out = np.where(a == 0x7F800000, 0x7C00, out)
    return (out | s).astype(np.uint16)


def f32_to_bf16(u):
    """uint32 f32 bits -> uint16 bfloat16 bits, round to nearest even (overflow to inf); NaN becomes a quiet NaN."""
    u = np.asarray(u, np.uint32)
    r = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    return np.where((u & 0x7FFFFFFF) > 0x7F800000, (u >> 16) | 0x40, r).astype(np.uint16)


def _f16_nan(h):
    return (h & 0x7C00 == 0x7C00) & (h & 0x3FF != 0)


def _bf16_nan(b):
    return (b & 0x7F80 == 0x7F80) & (b & 0x7F != 0)


def _same_or_both_nan(got, want, is_nan):
    gn, wn = is_nan(got), is_nan(want)
    return bool(np.array_equal(gn, wn) and np.array_equal(got[~gn], want[~wn]))


def gray(bgr):
    """uint8 [..][3] BGR -> uint8: (r*0.299 + g*0.587) + b*0.114 in float64, one rounding per operation, truncated
    (cost_computor.cpp:69)."""
    b, g, r = (bgr[..., i].astype(np.float64) for i in range(3))
    return ((r * 0.299 + g * 0.587) + b * 0.114).astype(np.uint8)


def depth_bases(W, H, Q):
    """The d-independent part of rows 2 and 3 of reproject_testlib.points, flattened: ((+0.0 + Q[i][0]*x) + Q[i][1]*y)."""
    Q = np.asarray(Q, np.float64)
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    return [((np.zeros_like(xs) + Q[i, 0] * xs) + Q[i, 1] * ys).reshape(-1) for i in (2, 3)]


def depth_of(d, Q, base2, base3):
    """reproject_testlib.depth with the two d-independent partial sums given: the same operations in the same order, and
    OpenCV's Z = 10000 for d = FLT_MAX."""
    Q = np.asarray(Q, np.float64)
    with np.errstate(all="ignore"):
        dd = d.astype(np.float64)
        h2 = (base2 + Q[2, 2] * dd) + Q[2, 3] * 1.0
        h3 = (base3 + Q[3, 2] * dd) + Q[3, 3] * 1.0
        z = (h2.astype(np.float32).astype(np.float64) * (1.0 / h3)).astype(np.float32)
    return np.where(d == np.finfo(np.float32).max, np.float32(10000.0), z)


def _rational_f32(q: Fraction) -> int:
    """Bits of the f32 nearest to the positive rational q (ties to even); q must lie in the normal range."""
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    m = q / Fraction(2) ** (e - 23)                 # in [2^23, 2^24)
    f = m.numerator // m.denominator
    rem = m - f
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and f & 1):
        f += 1
    if f == 1 << 24:
        f, e = 1 << 23, e + 1
    assert -126 <= e <= 127
    return ((e + 127) << 23) | (f & 0x7FFFFF)


def _f32(bits):
    return Fraction(float(np.uint32(bits).view(np.float32)))


# ---- CPU: the restatements pinned --------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["f16", "bf16"])
def test_rounding_restatement_every_pattern(which):
    """f32_to_f16 equals numpy's astype(float16) and f32_to_bf16 torch's CPU .to(bfloat16) on all 2^32 f32 patterns
    (NaN compared as NaN: the payloads are the converters' own choice, and the engine's exports hold no NaN)."""
    import torch

    def part(lo, hi):
        u = np.arange(lo, hi, dtype=np.uint64).astype(np.uint32)
        if which == "f16":
            with np.errstate(all="ignore"):
                want = u.view(np.float32).astype(np.float16).view(np.uint16)
            return _same_or_both_nan(f32_to_f16(u), want, _f16_nan)
        want = torch.from_numpy(u.view(np.float32)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
        return _same_or_both_nan(f32_to_bf16(u), want, _bf16_nan)

    bad = [lo for lo in range(0, 1 << 32, 1 << 26) if not all(_blocks(1 << 26, lambda a, b: part(lo + a, lo + b)))]
    assert not bad, f"{which}: the restatement differs in the chunks starting at {[hex(b) for b in bad[:8]]}"


def test_widening_and_domain_restatements():
    """f16_to_f32 equals numpy's float16 -> float32 and bf16_to_f32 torch's CPU bfloat16 -> float32 on all 2^16 patterns
    (NaN as NaN), and cost_domain gives the header's value domain on the specials it names."""
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    want = h.view(np.float16).astype(np.float32).view(np.uint32)
    f32_nan = lambda a: (a & 0x7FFFFFFF) > 0x7F800000
    assert _same_or_both_nan(f16_to_f32(h), want, f32_nan)
    import torch
    want = torch.from_numpy(h.view(np.int16)).view(torch.bfloat16).float().numpy().view(np.uint32)
    assert _same_or_both_nan(bf16_to_f32(h), want, f32_nan)
    specials = np.array([np.nan, -np.nan, np.inf, -np.inf, -0.0, 0.0, -1.0, 1e-45, -1e-45, 65535.996, 65536.0, 65536.01,
                         3e38, 1.5], np.float32)
    want = np.array([65536, 65536, 65536, 0, 0, 0, 0, 1e-45, 0, 65535.996, 65536, 65536, 65536, 1.5], np.float32)
    assert np.array_equal(cost_domain(specials.view(np.uint32)), want.view(np.uint32))


def test_depth_restatement_matches_reproject_testlib():
    """depth_of with depth_bases is reproject_testlib.depth, bit for bit apart from NaN payloads, on the reprojection
    fixture's maps and on random patterns of every exponent under a stereoRectify Q."""
    z = np.load(T.GOLDEN_DIR / "golden_reproject_cases.npz")
    rng = np.random.default_rng(5)
    cases = [(z[f"{n}/disp"], z[f"{n}/Q"]) for n in sorted({k.split("/")[0] for k in z.files})]
    cases.append((rng.integers(0, 1 << 32, (64, 96), dtype=np.uint64).astype(np.uint32).view(np.float32), z["rig_free_1/Q"]))
    for disp, Q in cases:
        H, W = disp.shape
        got = depth_of(disp.reshape(-1), Q, *depth_bases(W, H, Q)).reshape(H, W)
        assert RP.same_nan(got, RP.depth(disp, Q))


def test_rational_rounding_helper():
    """_rational_f32 equals the f64 quotient rounded to f32 for integers below 2^24 (exact: 53 >= 2 * 24 + 2 bits, so
    the double rounding is innocuous), and rounds ties to even."""
    rng = np.random.default_rng(1)
    for a, b in rng.integers(1, 1 << 24, (4000, 2)):
        assert _rational_f32(Fraction(int(a), int(b))) == int(np.float32(float(a) / float(b)).view(np.uint32)), (a, b)
    assert _rational_f32(1 + Fraction(1, 2 ** 24)) == 0x3F800000        # tie, even below
    assert _rational_f32(1 + Fraction(3, 2 ** 24)) == 0x3F800002        # tie, even above
    assert _rational_f32(2 - Fraction(1, 2 ** 25)) == 0x40000000        # carry into the exponent


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip(f"nvcc not found at {nvcc}")
    return nvcc


def _library_nvflags():
    """The library's nvcc flags, from adcensus_b200/csrc/Makefile (ARCH and NVFLAGS, -Xptxas -v dropped)."""
    mk = (ROOT / "adcensus_b200" / "csrc" / "Makefile").read_text()
    arch = re.search(r"^ARCH = (.*)$", mk, re.M).group(1).split()
    flags = re.search(r"^NVFLAGS = \$\(ARCH\) (.*)$", mk, re.M).group(1).replace("-Xptxas -v", "").split()
    return arch + flags


def _build_div(out_dir):
    exe = out_dir / "div_exhaustive"
    r = subprocess.run([_nvcc(), *_library_nvflags(), "-o", str(exe), str(DIV_SRC)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def test_div_program_builds(tmp_path):
    """tests/cu/div_exhaustive.cu compiles with the library's flags and includes the library's header."""
    assert '#include "../../adcensus_b200/csrc/adc_div.cuh"' in DIV_SRC.read_text()
    assert "adc_div.cuh" in (ROOT / "adcensus_b200" / "csrc" / "k_aggregate.cu").read_text()
    _build_div(tmp_path)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return E.cuda()


def _arange_bits(torch, dev, first, count):
    """A device tensor of the f32 patterns first .. first + count - 1 (first a multiple of count, count <= 2^28)."""
    base = first - (1 << 32) if first >= 1 << 31 else first
    return (torch.arange(count, dtype=torch.int32, device=dev) + base).view(torch.float32)


@pytest.fixture(scope="module")
def cost_engine(torch_cuda):
    """4096 x 256 x 256: one pair's volume is 2^28 elements, one lane, one pair per wave."""
    eng = E.engine(4096, 256, T.default_option(max_disparity=256), wave_pairs=1, lanes=1)
    yield eng
    eng.close()


def _export(eng, cost, layout, cost_dtype, out_dtype):
    """The cost volume of one pair, ingested from `cost` (device tensor) and exported as `out_dtype`, on the host."""
    torch, dev = E.cuda()
    h, w = eng.height, eng.width
    img = torch.zeros((h, w, 3), dtype=torch.uint8, device=dev)
    tdt = {"f32": torch.int32, "f16": torch.int16, "bf16": torch.int16}[out_dtype]
    out = torch.full((cost.numel(),), -1, dtype=tdt, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    eng.match_volumes_batch_device(1, img.data_ptr(), img.data_ptr(), [(out.data_ptr(), "cost", layout, out_dtype)],
                                   d_cost=cost.data_ptr(), cost_layout=layout, cost_dtype=cost_dtype, stream=st)
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint32 if out_dtype == "f32" else np.uint16)


@pytest.mark.gpu
def test_cost_f32_every_pattern(torch_cuda, cost_engine):
    """All 2^32 f32 patterns as a caller's cost volume, 16 volumes of 2^28, [H][W][D] and [D][H][W] alternately (each
    exported in its own layout, so element i of the export is element i of the input): the f32 export is the value
    domain exactly, the f16 and bf16 exports its round-to-nearest-even, and no export holds a NaN."""
    torch, dev = torch_cuda
    for c in range(1 << 4):
        first = c * CHUNK
        layout = ("hwd", "dhw")[c & 1]
        cost = _arange_bits(torch, dev, first, CHUNK)
        got = {dt: _export(cost_engine, cost, layout, "f32", dt) for dt in ("f32", "f16", "bf16")}
        del cost

        def check(lo, hi):
            u = np.arange(first + lo, first + hi, dtype=np.uint64).astype(np.uint32)
            v = cost_domain(u)
            return (np.array_equal(got["f32"][lo:hi], v), np.array_equal(got["f16"][lo:hi], f32_to_f16(v)),
                    np.array_equal(got["bf16"][lo:hi], f32_to_bf16(v)), bool(_f16_nan(got["f16"][lo:hi]).any()),
                    bool(_bf16_nan(got["bf16"][lo:hi]).any()))

        res = np.array(_blocks(CHUNK, check))
        for j, what in enumerate(("f32 export", "f16 export", "bf16 export")):
            bad = np.flatnonzero(~res[:, j])
            assert not bad.size, f"{what}, {layout}: patterns {first + bad[0] * BLOCK:#x} .. differ ({bad.size} blocks)"
        assert not res[:, 3:].any(), f"a NaN in an export of patterns {first:#x} .."
        f32_nan = (got["f32"] & 0x7FFFFFFF) > 0x7F800000
        assert not f32_nan.any()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_cost_half_every_pattern(torch_cuda, cost_engine, dtype):
    """All 2^16 f16 (bf16) patterns, repeated over one volume, in both layouts, exported as f32: the exact widening
    followed by the value domain."""
    torch, dev = torch_cuda
    pat = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    widen = f16_to_f32 if dtype == "f16" else bf16_to_f32
    want = np.tile(cost_domain(widen(pat)), CHUNK >> 16)
    for layout in ("hwd", "dhw"):
        cost = (torch.arange(CHUNK, dtype=torch.int32, device=dev) & 0xFFFF).to(torch.int16)
        got = _export(cost_engine, cost, layout, dtype, "f32")
        del cost
        bad = np.flatnonzero(got != want)
        assert not bad.size, f"{dtype} {layout}: {bad.size} elements differ, first pattern {bad[0] & 0xFFFF:#06x}: " \
                             f"{got[bad[0]]:#010x} vs {want[bad[0]]:#010x}"


RP_W = RP_H = 4096
RP_DMIN = 5     # the +inf value of DISP_S16 is (5 - 1) * 16 = 64, not 0


@pytest.fixture(scope="module")
def map_engine(torch_cuda):
    """4096 x 4096, D = 1, min_disparity 5: 2^24 pixels per map, 256 maps for every f32 pattern."""
    eng = E.engine(RP_W, RP_H, T.default_option(min_disparity=RP_DMIN, max_disparity=RP_DMIN + 1), wave_pairs=1, lanes=1)
    yield eng
    eng.close()


def _rig_Q():
    """The Q of cv2.stereoRectify for a made-up rig without CALIB_ZERO_DISPARITY (tools/make_golden_reproject.py)."""
    return np.load(T.GOLDEN_DIR / "golden_reproject_cases.npz")["rig_free_1/Q"]


@pytest.mark.gpu
def test_reproject_every_pattern(torch_cuda, map_engine):
    """All 2^32 f32 patterns as 256 maps of 4096 x 4096, 16 maps per call: DISP_S16 equals reproject_testlib.disp_s16
    (saturate_cast<short>(d * 16) as x86 computes it, +inf as (min_disparity - 1) * 16) and DEPTH the restatement of
    cv::reprojectImageTo3D's Z, NaN compared as NaN."""
    torch, dev = torch_cuda
    Q = _rig_Q()
    N = RP_W * RP_H
    base2, base3 = depth_bases(RP_W, RP_H, Q)
    st = torch.cuda.current_stream().cuda_stream
    for c in range(1 << 4):
        first = c * CHUNK
        d = _arange_bits(torch, dev, first, CHUNK)
        dep = torch.full((CHUNK,), -7, dtype=torch.int32, device=dev)
        s16 = torch.full((CHUNK,), -7, dtype=torch.int16, device=dev)
        map_engine.reproject_batch_device(CHUNK // N, d.data_ptr(), Q, [(dep.data_ptr(), "depth"), (s16.data_ptr(), "disp_s16")], st)
        torch.cuda.synchronize()
        del d
        got_dep, got_s16 = dep.view(torch.float32).cpu().numpy(), s16.cpu().numpy()
        del dep, s16

        def check(lo, hi):
            u = np.arange(first + lo, first + hi, dtype=np.uint64).astype(np.uint32).view(np.float32)
            p = lo % N
            return (np.array_equal(got_s16[lo:hi], RP.disp_s16(u, RP_DMIN)),
                    RP.same_nan(got_dep[lo:hi], depth_of(u, Q, base2[p:p + hi - lo], base3[p:p + hi - lo])))

        res = np.array(_blocks(CHUNK, check))
        for j, what in enumerate(("DISP_S16", "DEPTH")):
            bad = np.flatnonzero(~res[:, j])
            assert not bad.size, f"{what}: patterns {first + bad[0] * BLOCK:#x} .. differ ({bad.size} blocks)"


def _points_map():
    """One 4096 x 4096 map of 2^24 patterns: every sign x exponent x top 15 mantissa bits, with random low 8 bits; the
    first pixels replaced by +-0, the subnormal edges, the smallest normals, FLT_MAX, +-inf and NaN."""
    rng = np.random.default_rng(24)
    u = (np.arange(1 << 24, dtype=np.uint32) << 8) | rng.integers(0, 256, 1 << 24, dtype=np.uint32)
    specials = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000, 0x80800000,
                0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001]
    u[:len(specials)] = specials
    return u.view(np.float32).reshape(RP_H, RP_W)


@pytest.mark.gpu
def test_reproject_points_budgeted(torch_cuda, map_engine):
    """POINTS of 2^24 patterns that take every exponent of both signs through the double arithmetic, against live
    cv2.reprojectImageTo3D (NaN compared as NaN)."""
    cv2 = pytest.importorskip("cv2")
    torch, dev = torch_cuda
    Q = _rig_Q()
    disp = _points_map()
    d = torch.from_numpy(disp).to(dev)
    pts = torch.full((3 * disp.size,), -7, dtype=torch.int32, device=dev)
    map_engine.reproject_batch_device(1, d.data_ptr(), Q, [(pts.data_ptr(), "points")],
                                      torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = pts.view(torch.float32).cpu().numpy().reshape(RP_H, RP_W, 3)
    want = cv2.reprojectImageTo3D(disp, Q)
    assert RP.same_nan(got, want)
    assert RP.same_nan(got, RP.points(disp, Q))


@pytest.mark.gpu
def test_point_cloud_every_pattern_maps(torch_cuda, map_engine):
    """adc_point_cloud_batch_device on two of the 256 pattern maps (d in [2, 8) and its negatives): counts, kept pixels
    and points equal the restatement of the keep rule (finite d, finite point, z_min <= Z <= z_max) with z bounds at the
    quartiles of the finite depths, so the bounds cut through finite values."""
    torch, dev = torch_cuda
    Q = _rig_Q()
    N = RP_W * RP_H
    maps = np.stack([(np.arange(N, dtype=np.uint32) | np.uint32(m << 24)).view(np.float32).reshape(RP_H, RP_W)
                     for m in (0x40, 0xC0)])
    base2, base3 = depth_bases(RP_W, RP_H, Q)
    z = np.concatenate([depth_of(m.reshape(-1), Q, base2, base3) for m in maps])
    z = z[np.isfinite(z)]
    z_range = (float(np.quantile(z, 0.25)), float(np.quantile(z, 0.75)))
    d = torch.from_numpy(maps).to(dev)
    work = torch.empty(map_engine.point_cloud_workspace_bytes(2), dtype=torch.uint8, device=dev)
    pts = torch.full((2 * N * 3,), -7, dtype=torch.int32, device=dev)
    pix = torch.full((2 * N,), -7, dtype=torch.int32, device=dev)
    counts = torch.full((2,), -7, dtype=torch.int32, device=dev)
    map_engine.point_cloud_batch_device(2, d.data_ptr(), Q, pts.data_ptr(), counts.data_ptr(), N, work.data_ptr(),
                                        work.numel(), d_pixels=pix.data_ptr(), z_range=z_range,
                                        stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    counts = counts.cpu().numpy()
    pts = pts.view(torch.float32).cpu().numpy().reshape(2, N, 3)
    pix = pix.cpu().numpy().reshape(2, N)
    for i in range(2):
        want_pts, _, want_pix = CL.cloud(maps[i], Q, None, *z_range)
        k = len(want_pix)
        assert 0 < k < N, (i, k)
        assert counts[i] == k, (i, counts[i], k)
        assert np.array_equal(pix[i, :k], want_pix), i
        assert np.array_equal(pts[i, :k].view(np.uint32), want_pts.view(np.uint32)), i


@pytest.mark.gpu
def test_gray_every_colour(torch_cuda, map_engine):
    """One 4096 x 4096 image holds each of the 2^24 BGR triples once, the right view the same triples in a permuted
    order; the GRAY_L / GRAY_R taps after the cost stage equal the oracle's gray of the same images and the float64
    restatement of cost_computor.cpp:69."""
    i = np.arange(1 << 24, dtype=np.uint32)
    left = np.stack([i & 255, (i >> 8) & 255, i >> 16], -1).astype(np.uint8).reshape(RP_H, RP_W, 3)
    right = left.reshape(-1, 3)[np.random.default_rng(9).permutation(1 << 24)].reshape(RP_H, RP_W, 3)
    map_engine.debug_run(left, right, "COST")
    got = {"GRAY_L": map_engine.tap("GRAY_L"), "GRAY_R": map_engine.tap("GRAY_R")}
    orc = T.Oracle(RP_W, RP_H, T.default_option(min_disparity=RP_DMIN, max_disparity=RP_DMIN + 1))
    orc.begin(left, right)
    orc.run_to("COST")
    for tap, img in (("GRAY_L", left), ("GRAY_R", right)):
        want = gray(img)
        assert np.array_equal(orc.tap(tap), want), f"oracle {tap}"
        bad = np.flatnonzero(got[tap] != want)
        assert not bad.size, f"{tap}: {bad.size} colours differ, first BGR {img.reshape(-1, 3)[bad[0]]}"
    orc.close()


@pytest.fixture(scope="module")
def div_run(torch_cuda, tmp_path_factory):
    """The output of tests/cu/div_exhaustive.cu, built with the library's flags: {name: value} and the sample rows."""
    exe = _build_div(tmp_path_factory.mktemp("div"))
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.rstrip().endswith("done"), r.stderr[-2000:] + r.stdout[-2000:]
    vals, sample, first = {}, [], []
    for line in r.stdout.splitlines():
        f = line.split()
        if f[0] == "sample":
            sample.append([int(v, 16) for v in f[1:]])
        elif f[0].endswith("_first"):
            first.append(line)
        elif f[0] != "done":
            vals.setdefault(f[0], []).append([float(v) for v in f[1:]])
    print("\n".join(line for line in r.stdout.splitlines() if not line.startswith("sample")))
    return vals, np.array(sample, np.uint64), first


@pytest.mark.gpu
def test_hardware_reciprocal_within_assumed_spread(div_run):
    """rcp.approx.ftz.f32 of every n in 1..65535 lies within 3 ulp of RN(1/n), the spread tests/c/div_sequence.c proves
    the refined sequence exact for."""
    vals = div_run[0]
    lo, hi = vals["rcp_ulp_min"][0][0], vals["rcp_ulp_max"][0][0]
    assert -3 <= lo <= hi <= 3, (lo, hi)
    assert sum(c for _, c in vals["rcp_ulp_hist"]) == 65535


@pytest.mark.gpu
@pytest.mark.parametrize("check", ["binade_1", "binade_lo", "binade_hi", "n_edge", "guard_x", "guard_n", "edge"])
def test_division_on_the_device(div_run, check):
    """adc_div4 over every divisor x every mantissa of [1, 2) and of the guards' binades equals __fdiv_rn, which equals
    the f64 quotient rounded to f32; the guard routes exactly {+0} U [1e-30f, 1e30f) x [1, 65535] to the fast branch;
    the fast sequence is exact at the guards' edges and at n = 65535, 65536."""
    vals, _, first = div_run
    checked = vals[f"{check}_checked"][0][0]
    want_checked = {"binade_1": 65535 << 23, "binade_lo": 65535 << 23, "binade_hi": 65535 << 23, "n_edge": 6 << 23,
                    "edge": 6 * 65535}
    if check in want_checked:
        assert checked == want_checked[check]
    assert vals[f"{check}_bad"][0][0] == 0, [f for f in first if f.startswith(check)]
    assert vals[f"{check}_bad_ref"][0][0] == 0


@pytest.mark.gpu
def test_division_sample_is_the_rational_quotient(div_run):
    """4096 (x, n) of the device run: __fdiv_rn and adc_div4 both give RN(x / n), computed with exact rationals."""
    sample = div_run[1]
    assert sample.shape == (4096, 4)
    for x, n, q, q4 in sample:
        want = _rational_f32(_f32(x) / _f32(n))
        assert int(q) == want and int(q4) == want, (hex(x), hex(n), hex(q), hex(q4), hex(want))
