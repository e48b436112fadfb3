#!/usr/bin/env python
"""Generates tests/golden/golden_ties_ref.json from the UNMODIFIED reference: sha256 of every tap after every stage for
the first pair of every tie case of tests/test_tie_parity.py.  Image cases run the reference behind oracle/_ref (built by
oracle/Makefile from the checkout ADC_REFERENCE_DIR names); cost-input cases run tests/c/ref_cost_harness.cpp, built
into a temporary directory as tools/make_golden_cost.py does.

The cases are defined here, so that the tests and this generator build the same inputs.  Each is a family of inputs
built so that the pipeline's first-minimum, strict-comparison and threshold rules meet exact equalities, under one
option set.  Every family has five distinct pairs (seeds), so that a batched call never holds two equal neighbours.
"""
import json
import os
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import adc_testlib as T  # noqa: E402
import make_golden_cost as GC  # noqa: E402
import make_golden_sweep as GS  # noqa: E402

W, H = 100, 64
N_PAIRS = 5
ADC_DBG_NO_RAY_TABLE, ADC_DBG_VOTE_ENUM = 1, 2
DEFAULT_RUNS = ("vote_enum", "no_ray_table")     # option sets that differ from "default" in engine debug flags only

# name -> (option overrides, engine debug flags).  "vote_enum" runs the defaults with region voting forced to enumerate
# its regions on the GPU, "no_ray_table" with the interpolation's generic ray walk; the oracle's run of either is the
# same as the defaults' (DEFAULT_RUNS), so neither is pinned separately.
OPTION_SETS = {
    "default": (dict(max_disparity=32), 0),
    "dneg_d27": (dict(min_disparity=-5, max_disparity=22), 0),          # D % 4 != 0, dmin < 0
    "wide_l1": (dict(max_disparity=32, cross_L1=130, cross_L2=40), 0),  # L1 > 127: WIDE voting
    "disc": (dict(max_disparity=32, do_discontinuity_adjustment=1), 0),
    "no_lr": (dict(max_disparity=32, do_lr_check=0), 0),
    "vote_enum": (dict(max_disparity=32), ADC_DBG_VOTE_ENUM),
    # the same, with interpolation walking its rays in double per step instead of the verified integer ray table
    "no_ray_table": (dict(max_disparity=32), ADC_DBG_NO_RAY_TABLE),
    # thresholds that exact counts and exact disparities reach: peak / total == 1/2, and |dl - dr| == 0 (exact non-zero
    # differences need both maps integer at once, which no input here produces on enough pixels to count on)
    "thresholds": (dict(max_disparity=32, irv_th=0.5, irv_ts=12, lrcheck_thres=0.0), 0),
    # no scanline penalties: each pass adds one value to a pixel's whole curve, so the curve's shape -- and the WTA map
    # a cost-input volume is built for -- survives exactly; with the LR check and filling as in the defaults
    "flat_so": (dict(max_disparity=32, so_p1=0.0, so_p2=0.0), 0),
    # the same without the LR check, and the discontinuity adjustment then runs on that map.  With
    # dmin != 0 it reads each curve at index round(d), not d - dmin (as the reference does), so it can move a pixel.
    "flat_so_disc": (dict(min_disparity=2, max_disparity=34, so_p1=0.0, so_p2=0.0, do_lr_check=0,
                          do_discontinuity_adjustment=1), 0),
}


# ---- image families ---------------------------------------------------------------------------------------------------
def _shift_pair(tex, pad, s):
    """(left, right) of a scene texture [H][W + 2 pad]: the right view is the left one at disparity s (left[x] =
    right[x - s])."""
    left = np.ascontiguousarray(tex[:, pad:pad + W])
    right = np.ascontiguousarray(tex[:, pad + s:pad + s + W])
    return left, right


def _noise(rng, h, w, run=1):
    """Random colours in runs of `run` equal pixels along x."""
    a = rng.integers(0, 256, (h, -(-w // run), 3), dtype=np.uint8)
    return np.ascontiguousarray(np.repeat(a, run, axis=1)[:, :w])


def _inner_shift(opt, i):
    """A disparity strictly inside the range, a few pixels from dmin."""
    return opt.min_disparity + 3 + i % 4


def fam_periodic_cols(opt, seed, i):
    """Columns periodic with period 8 or 13 (below D), right view shifted inside the range: the minimum repeats every
    period along d."""
    rng = np.random.default_rng(seed)
    p = (8, 13)[i % 2]
    pad = 64
    row = rng.integers(0, 256, (H, p, 3), dtype=np.uint8)
    tex = np.tile(row, (1, (W + 2 * pad) // p + 1, 1))[:, :W + 2 * pad]
    return _shift_pair(tex, pad, _inner_shift(opt, i))


def fam_periodic_tiles(opt, seed, i):
    """2-D periodic tiles (8 or 13 columns x 8 rows)."""
    rng = np.random.default_rng(seed)
    p = (8, 13)[i % 2]
    pad = 64
    tile = rng.integers(0, 256, (8, p, 3), dtype=np.uint8)
    tex = np.tile(tile, (H // 8 + 1, (W + 2 * pad) // p + 1, 1))[:H, :W + 2 * pad]
    return _shift_pair(tex, pad, _inner_shift(opt, i))


def fam_dot_lattice(opt, seed, i):
    """White isolated dots on black in the left view, the inverse (black dots on white) in the right one, shifted:
    every dot meets its inverse, so the AD sum reaches 765 and the census Hamming distance its maximum, 62."""
    rng = np.random.default_rng(seed)
    pad = 64
    tex = np.zeros((H, W + 2 * pad, 3), np.uint8)
    oy, ox = rng.integers(0, 10), rng.integers(0, 8)
    tex[oy::10, ox::8] = 255
    s = _inner_shift(opt, i)
    left, _ = _shift_pair(tex, pad, s)
    _, right = _shift_pair(255 - tex, pad, s)
    return left, right


def fam_saturated_steps(opt, seed, i):
    """Flat blocks whose colours step by exactly cross_t1 or cross_t2 (so the arm rules meet equality), 0 / 255 blocks,
    and a textured strip."""
    rng = np.random.default_rng(seed)
    pad = 64
    Wt = W + 2 * pad
    t1, t2 = opt.cross_t1, opt.cross_t2
    xs, ys = np.arange(Wt)[None, :], np.arange(H)[:, None]
    bx, by = (xs + seed) // 19, (ys + seed) // 21           # blocks longer than cross_L2 = 17
    base = 90 + int(rng.integers(0, 20))
    g = base + (bx % 2) * t2 + ((bx // 2) % 2) * t1 + (by % 2) * t1 + ((by // 2) % 2) * t2
    tex = np.repeat(g[:, :, None], 3, axis=2).clip(0, 255).astype(np.uint8)
    tex[:, :, 1] = (tex[:, :, 1].astype(int) + (by % 3) * t2).clip(0, 255).astype(np.uint8)
    # saturated blocks beside a textured strip
    c0 = pad + 30 + 4 * i
    tex[10:30, c0:c0 + 12] = 255
    tex[34:54, c0 + 12:c0 + 24] = 0
    tex[:, c0 + 24:c0 + 34] = _noise(rng, H, 10)
    return _shift_pair(tex, pad, _inner_shift(opt, i))


def fam_range_ends(opt, seed, i):
    """A textured right view shifted by exactly dmin (even pairs) or dmax - 1 (odd pairs): d1 at the range ends, so the
    left map is Invalid and the right map integer there."""
    rng = np.random.default_rng(seed)
    pad = max(abs(opt.min_disparity), abs(opt.max_disparity)) + 2
    tex = _noise(rng, H, W + 2 * pad, run=2)
    s = opt.min_disparity if i % 2 == 0 else opt.max_disparity - 1
    return _shift_pair(tex, pad, s)


def fam_identical(opt, seed, i):
    """Identical views: with dmin = 0 every pixel matches at the range end, so the LR check has nothing valid, voting
    finds no votes and interpolation no candidate."""
    rng = np.random.default_rng(seed)
    tex = _noise(rng, H, W, run=1 + i % 3)
    return tex, tex.copy()


def fam_occlusion_bars(opt, seed, i):
    """Foreground bars in front of a background of a few flat colours: long occlusion lists, and regions whose
    histograms have equal peaks."""
    rng = np.random.default_rng(seed)
    pad = 64
    Wt = W + 2 * pad
    s_bg = _inner_shift(opt, i)
    s_fg = s_bg + 12 + i % 3
    pal = rng.integers(0, 256, (4, 3), dtype=np.uint8)
    bg = pal[((np.arange(Wt)[None, :] // 6) + (np.arange(H)[:, None] // 9)) % 4]
    left = np.ascontiguousarray(bg[:, pad:pad + W])
    right = np.ascontiguousarray(bg[:, pad + s_bg:pad + s_bg + W])
    fg = rng.integers(0, 256, (3,), dtype=np.uint8)
    for x0 in range(8 + i, W, 24):
        for x in range(x0, min(x0 + 9, W)):
            left[:, x] = fg if (x - x0) % 4 else 255 - fg
            if 0 <= x - s_fg < W:
                right[:, x - s_fg] = left[:, x]
    return left, right


def fam_piecewise_regions(opt, seed, i):
    """Rectangles of a few constant colours: the interpolation's rays meet equal colour distances."""
    rng = np.random.default_rng(seed)
    pad = 64
    Wt = W + 2 * pad
    pal = rng.integers(0, 256, (3, 3), dtype=np.uint8)
    cx = rng.integers(5, 14, size=Wt // 5 + 1).cumsum()
    cy = rng.integers(4, 12, size=H // 4 + 1).cumsum()
    ix = np.searchsorted(cx, np.arange(Wt), side="right")
    iy = np.searchsorted(cy, np.arange(H), side="right")
    tex = pal[(ix[None, :] + 2 * iy[:, None]) % 3]
    return _shift_pair(np.ascontiguousarray(tex), pad, _inner_shift(opt, i) + 4)


IMAGE_FAMILIES = {
    "periodic_cols": fam_periodic_cols, "periodic_tiles": fam_periodic_tiles, "dot_lattice": fam_dot_lattice,
    "saturated_steps": fam_saturated_steps, "range_ends": fam_range_ends, "identical": fam_identical,
    "occlusion_bars": fam_occlusion_bars, "piecewise_regions": fam_piecewise_regions,
}


# ---- cost-input families: volumes of multiples of 1/32 in [0, 4), exact in f16 and bf16 ------------------------------
def _blocks(seed):
    """(column-block index [W], row-block index [H]) of the cost-input views' colour blocks."""
    bw, bh = 10 + seed % 3, 8 + seed % 2
    return np.arange(W) // bw, np.arange(H) // bh


def _cost_images(seed, i):
    """Views for a cost-input case: flat gray blocks, each 50 or more from its neighbours, so that every cross arm stops
    at its block's edge and aggregation averages equal curves only (the scanline penalties stay at P1 / P2 inside a
    block)."""
    bx, by = _blocks(seed)
    g = (40 + 50 * ((bx[None, :] + 2 * by[:, None] + i) % 4)).astype(np.uint8)
    left = np.ascontiguousarray(np.repeat(g[:, :, None], 3, axis=2))
    return left, np.ascontiguousarray(np.roll(left, -(3 + i), axis=1))


def cost_periodic_d(opt, seed, i):
    """C(d) periodic in d (period 3 to 7) with adjacent steps of 1/32, below the smallest scanline penalty P1 / 10:
    the minima repeat along d and stay tied through aggregation and all four passes."""
    D = opt.max_disparity - opt.min_disparity
    rng = np.random.default_rng(seed)
    P = 3 + (seed + i) % 5
    ph = rng.integers(0, P, (H // 8 + 1, W // 10 + 1))
    ph = np.repeat(np.repeat(ph, 8, 0), 10, 1)[:H, :W]
    k = 32 + (np.arange(D)[None, None, :] + ph[:, :, None]) % P
    return k.astype(np.float32) / np.float32(32)


def cost_plateau(opt, seed, i):
    """Blocks of pixels whose curve has a plateau of equal minima, or two equal minima at least 2 apart."""
    D = opt.max_disparity - opt.min_disparity
    rng = np.random.default_rng(seed)
    k = np.full((H, W, D), 96, np.int32)
    blk = rng.integers(0, 1 << 30, (H // 6 + 1, W // 7 + 1))
    blk = np.repeat(np.repeat(blk, 6, 0), 7, 1)[:H, :W]
    a = 2 + blk % (D - 8)
    kind = (blk >> 8) % 2
    for y in range(H):
        for x in range(W):
            d = int(a[y, x])
            if kind[y, x]:
                k[y, x, d:d + 4] = 8                            # plateau of four
            else:
                k[y, x, d] = k[y, x, d + 2 + int(blk[y, x] >> 12) % 5] = 8   # two minima 2..6 apart
    k += ((np.arange(D) * 7 + i) % 3)[None, None, :] * (k > 8)
    return k.astype(np.float32) / np.float32(32)


def cost_range_ends(opt, seed, i):
    """Minima at d = 0 or D - 1 (alternating blocks), and all-equal pixels."""
    D = opt.max_disparity - opt.min_disparity
    rng = np.random.default_rng(seed)
    k = 40 + rng.integers(0, 60, (H, W, D))
    blk = (np.arange(H)[:, None] // 5 + np.arange(W)[None, :] // 9 + i) % 4
    k[blk == 0, 0] = 4
    k[blk == 1, D - 1] = 4
    k[blk == 2, :] = 64
    k[blk == 3, D // 2] = 4
    return k.astype(np.float32) / np.float32(32)


def cost_blocks(opt, seed, i):
    """Column blocks (the views' blocks) alternating between two curves, in [2, 4):
      A: three equal minima at a..a+2 (d1 = a, parabola a + 0.5);
      B: one minimum at a + 2 with neighbours cmin + 1/32 and cmin + 3/32 (parabola a + 1.75).
    The other values fall by 1/32 per index.  Where the scanline passes keep the curves' shapes (no penalties), the map
    steps by 1.25 between blocks, so the edge test sees |gx| + |gy| == 5 exactly on both sides of each block edge; were
    those pixels edges, the discontinuity adjustment (which reads index round(d), off the minimum when dmin != 0) would
    move them to the lower cost at their neighbour's rounded disparity."""
    D = opt.max_disparity - opt.min_disparity
    bx, _ = _blocks(seed)
    a = 6 + (seed + i) % 7
    k = np.broadcast_to(120 - np.arange(D, dtype=np.int32).clip(0, 56), (H, W, D)).copy()
    A = (bx % 2 == 0)[None, :].repeat(H, 0)
    k[A, a - 1] = 66
    k[A, a:a + 3] = 64
    k[A, a + 3] = 66
    k[~A, a + 1] = 65
    k[~A, a + 2] = 64
    k[~A, a + 3] = 67
    return k.astype(np.float32) / np.float32(32)


def _teeth_images(seed, i):
    """Views of cost_vote_pairs: rows of 'teeth' -- 17 pixels of colour L, one spine pixel S, 17 pixels of colour R --
    between walls, every other row a wall row.  |L - S| = |R - S| = 15 < cross_t1 and |L - R| = 30, so a tooth pixel's
    arms cover its tooth and the spine, the spine's arms both teeth, and no vertical arm leaves its row."""
    S, L, R, Wc = 100, 85, 115, (200, 40, 200)
    left = np.empty((H, W, 3), np.uint8)
    left[:] = Wc
    x0 = 3 + (seed + i) % 5
    for y in range(1 + i % 2, H, 2):
        for s in (x0, x0 + 48):
            left[y, s:s + 17] = L
            left[y, s + 17] = S
            left[y, s + 18:s + 35] = R
    return left, np.ascontiguousarray(np.roll(left, -(3 + i), axis=1))


def cost_vote_pairs(opt, seed, i):
    """Teeth whose left half prefers disparity 2k and right half 2k + 1 in equal counts around a spine pixel whose
    curve dips at d = 0 (so it is Invalid and a mismatch): region voting then finds bins 2k and 2k + 1 tied at its peak,
    the two bins of one word of the narrow histogram.  Walls are flat."""
    D = opt.max_disparity - opt.min_disparity
    left, _ = _teeth_images(seed, i)
    k2 = 10 + 2 * ((seed + i) % 3)
    curve = {}
    for name, m in (("L", k2), ("R", k2 + 1)):
        c = np.full(D, 96, np.int32)
        c[0] = 74
        c[m - 1] = c[m + 1] = 80
        c[m] = 64
        curve[name] = c
    curve["S"] = np.full(D, 127, np.int32)
    curve["S"][0] = 0
    k = np.full((H, W, D), 96, np.int32)
    g = left[:, :, 0]
    for name, v in (("L", 85), ("S", 100), ("R", 115)):
        k[g == v] = curve[name]
    return k.astype(np.float32) / np.float32(32)


COST_FAMILIES = {"cost_periodic_d": cost_periodic_d, "cost_plateau": cost_plateau, "cost_range_ends": cost_range_ends,
                 "cost_blocks": cost_blocks, "cost_vote_pairs": cost_vote_pairs}
# cost families whose views are not _cost_images'
COST_IMAGES = {"cost_vote_pairs": _teeth_images}


# ---- cases ------------------------------------------------------------------------------------------------------------
def cases():
    """name -> (family, option set), every family x option set."""
    return {f"{fam}/{os_}": (fam, os_) for fam in (*IMAGE_FAMILIES, *COST_FAMILIES) for os_ in OPTION_SETS}


def option(case_name):
    return T.default_option(**OPTION_SETS[cases()[case_name][1]][0])


def debug_flags(case_name):
    return OPTION_SETS[cases()[case_name][1]][1]


def is_cost(case_name):
    return cases()[case_name][0] in COST_FAMILIES


def seed_of(case_name):
    """The case's first seed.  The DEFAULT_RUNS sets run the default set's pairs, so that their final maps meet the same
    hashes."""
    fam, os_ = cases()[case_name]
    os_ = "default" if os_ in DEFAULT_RUNS else os_
    return 7000 + 100 * list((*IMAGE_FAMILIES, *COST_FAMILIES)).index(fam) + list(OPTION_SETS).index(os_) * 10


def pairs(case_name):
    """The case's N_PAIRS inputs: [(left, right, cost volume f32 [H][W][D] or None)]."""
    fam, _ = cases()[case_name]
    opt = option(case_name)
    seed = seed_of(case_name)
    out = []
    for i in range(N_PAIRS):
        if fam in IMAGE_FAMILIES:
            left, right = IMAGE_FAMILIES[fam](opt, seed + i, i)
            out.append((left, right, None))
        else:
            left, right = COST_IMAGES.get(fam, _cost_images)(seed + i, i)
            out.append((left, right, COST_FAMILIES[fam](opt, seed + i, i)))
    return out


# A reference corner that is guarded, not emulated (DESIGN.md §8, SURVEY §8a A15): the discontinuity adjustment indexes
# a curve by round(d) without subtracting dmin, so an index outside [0, D) reads past the pixel's own curve; the oracle
# and the kernel skip such a pixel.  The dot lattice and the identical views with dmin = 2 reach that corner, so those
# two cases are not pinned.
REF_DIVERGES = ("dot_lattice/flat_so_disc", "identical/flat_so_disc")
# the cases pinned to the reference: every family x option set but the DEFAULT_RUNS (the same oracle run as default)
PINNED = sorted(n for n, (_, os_) in cases().items() if os_ not in DEFAULT_RUNS and n not in REF_DIVERGES)


def staged_hashes(checker, opt, left, right, cost=None):
    """sha256 of every tap after every stage of one pair, as make_golden_sweep.staged_hashes; with a cost volume the
    GRAY and CENSUS taps are left out (cost-input mode does not compute them)."""
    if cost is None:
        return GS.staged_hashes(checker, opt, left, right)
    import make_golden as G
    checker.begin_cost(left, right, cost)
    hashes = {}
    for st in T.STAGES:
        checker.step()
        for tap in GC.COST_STAGE_TAPS[st]:
            hashes[f"{st}/{tap}"] = T.sha(G.ref_case_tap(opt, tap, checker.tap(tap)))
    return hashes


def main():
    assert os.environ.get("ADC_REFERENCE_DIR"), "set ADC_REFERENCE_DIR to a checkout of the reference"
    T.build_oracle()
    assert T.have_ref(), "oracle/_ref could not be built from ADC_REFERENCE_DIR"
    import cost_testlib as CT
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cost_lib = GC.build_ref_cost_harness(Path(tmp))
        for name in PINNED:
            opt = option(name)
            left, right, cost = pairs(name)[0]
            ref = T.Reference(W, H, opt) if cost is None else CT.CostReference(cost_lib, W, H, opt)
            out[name] = staged_hashes(ref, opt, left, right, cost)
            ref.close()
            print(f"{name} final sha {out[name]['MEDIAN/DISP_L'][:16]}", flush=True)
    (T.GOLDEN_DIR / "golden_ties_ref.json").write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
