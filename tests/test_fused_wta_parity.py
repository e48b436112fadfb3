"""Fused scanline-WTA parity: the last scanline pass with both WTA views as its epilogue (k_scanline_wta writes disp_l and
per-band partial records of the right view, k_wta_merge folds them into disp_r; DESIGN.md 5.5) against the oracle, on
every instantiation the rule can pick, at the band edges, on inputs built to tie, on poisoned arenas and past 2^31 bytes.

The other parity files export volumes or run stage by stage, and either keeps the unfused pass 4 + k_wta; every case
here is a map-only call (sweep_testlib.check_case(volumes=False)), which fuses where so_wta_fused (so_plan.h) allows it.

CPU: the instantiations whose records fit a pair's volume anywhere in adc_create's domain (so_wta_main domain) against
the library's k_scanline_wta kernels; every one reached by a GPU case here; each edge case taking the path it is there
for; the tie cases' optimised volumes (oracle, SO4) reaching every merge rule at least once.
GPU: every case through one batched call, both WTA maps, the outlier lists and the final map bit for bit against each
pair's oracle run, on an engine with ADC_DBG_FUSED_SO_WTA; after each call the VOL_AGGR tap is refused, which shows the
fused form ran.  Three 4000 x 2100 x 64 pairs run under the AUTO rule against committed hashes.
"""
import functools
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import adc_testlib as T
import cost_testlib as CT
import engine_testlib as E  # puts tools/ on sys.path
import make_golden_sweep as GS
import make_golden_ties as GT
from adcensus_b200.engine import DBG_FUSED_SO_WTA, DBG_UNFUSED_SO_WTA, poison_flags
from sweep_testlib import Case, check_case, library_instantiations, plans, reached, so_lanes_per_line  # noqa: F401

AUTO, NEVER, ALWAYS = 0, 1, 2   # SoWtaForce
WTA_SYMBOLS = {"k_scanline_wta": re.compile(r"_Z14k_scanline_wtaILi(\d+)ELi(\d+)ELb([01])EE")}
FIELDS = 6                      # SO_WTA_FIELDS


def _rule(W, H, D, dmin=0, force=ALWAYS, opt_export=0, confidence=0, discontinuity=0, debug_run=0):
    r = subprocess.run([str(E.c_tool("so_wta_main"))] + [str(v) for v in (W, H, D, dmin, opt_export, confidence,
                                                                          discontinuity, debug_run, force)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return dict(zip(("fused", "band", "row_records", "plane", "vol"), map(int, r.stdout.split())))


@functools.cache
def domain():
    """{D: (K, LPS, FULL, widths the forced rule fuses, the first of them)} over adc_create's whole domain."""
    r = subprocess.run([str(E.c_tool("so_wta_main")), "domain"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    rows = [list(map(int, line.split())) for line in r.stdout.strip().split("\n")]
    return {D: (K, L, bool(F), n, w) for D, K, L, F, n, w in rows}


def fit_instantiations():
    return {("k_scanline_wta", K, L, F) for K, L, F, n, _ in domain().values() if n}


# ---- cases ----------------------------------------------------------------------------------------------------------
def _opt(D, dmin=0, **kw):
    return T.default_option(min_disparity=dmin, max_disparity=dmin + D, **kw)


def sweep_case(D):
    """The kernel sweep's case of range D (H, dmin, seed and pairs), at its width where the records fit, else at the
    nearest wider width where they do."""
    W, H, opt, seed = GS.sweep_case(D)
    while not _rule(W, H, D)["fused"]:
        W += 1
    return Case(f"sweep_D{D}", W, H, opt, seed)


FIT_DS = [D for D, (_, _, _, n, _) in sorted(domain().items()) if n]

# name -> (case, what it is there for).  Checked on the CPU by test_edge_cases_take_their_path.
EDGE_CASES = {
    # the records fill a pair's slice exactly: an overrun lands in the next pair of the wave
    "fill_d5_w15": (Case("fill_d5_w15", 15, 11, _opt(5), 501, wave_pairs=4, lanes=1), dict(exact_fill=True)),
    "fill_d5_w30": (Case("fill_d5_w30", 30, 9, _opt(5), 502, wave_pairs=4, lanes=1), dict(exact_fill=True)),
    "fill_d6_w63": (Case("fill_d6_w63", 63, 7, _opt(6), 503, wave_pairs=4, lanes=1), dict(exact_fill=True)),
    "fill_d9_w12": (Case("fill_d9_w12", 12, 13, _opt(9), 504, wave_pairs=4, lanes=1), dict(exact_fill=True, one_band=True)),
    "fill_d9_w24": (Case("fill_d9_w24", 24, 9, _opt(9), 505, wave_pairs=4, lanes=1), dict(exact_fill=True)),
    "fill_d9_w36": (Case("fill_d9_w36", 36, 7, _opt(9), 506, wave_pairs=4, lanes=1), dict(exact_fill=True)),
    # the last band's live warps (the CTA barrier count wta_threads) and a partly dead last warp, 8 and 16 lanes per line
    "lps8_r1": (Case("lps8_r1", 49, 11, _opt(40), 511), dict(lps=8, live_warps=1, dead_lines=True)),
    "lps8_r2": (Case("lps8_r2", 53, 11, _opt(40), 512), dict(lps=8, live_warps=2, dead_lines=True)),
    "lps8_r3": (Case("lps8_r3", 57, 11, _opt(40), 513), dict(lps=8, live_warps=3, dead_lines=True)),
    "lps8_r4": (Case("lps8_r4", 63, 11, _opt(40), 514), dict(lps=8, live_warps=4, dead_lines=True)),
    "lps16_r1": (Case("lps16_r1", 113, 9, _opt(100), 515), dict(lps=16, live_warps=1, dead_lines=True)),
    "lps16_r2": (Case("lps16_r2", 115, 9, _opt(100), 516), dict(lps=16, live_warps=2, dead_lines=True)),
    "lps16_r3": (Case("lps16_r3", 117, 9, _opt(100), 517), dict(lps=16, live_warps=3, dead_lines=True)),
    "lps16_r4": (Case("lps16_r4", 119, 9, _opt(100), 518), dict(lps=16, live_warps=4, dead_lines=True)),
    # one band; W < D
    "one_band_d20": (Case("one_band_d20", 14, 9, _opt(20), 521), dict(one_band=True)),
    "one_band_d64": (Case("one_band_d64", 16, 9, _opt(64), 522), dict(one_band=True, narrow=True)),
    "narrow_d64": (Case("narrow_d64", 60, 9, _opt(64), 523), dict(narrow=True)),
    "narrow_d128": (Case("narrow_d128", 120, 7, _opt(128), 524), dict(narrow=True)),
    # head-only and short passes, and a last ring slot of one step
    "h1": (Case("h1", 70, 1, _opt(48), 531), dict(H=1)),
    "h2": (Case("h2", 70, 2, _opt(48), 532), dict(H=2)),
    "h3": (Case("h3", 70, 3, _opt(48), 533), dict(H=3)),
    "h_slot_plus1": (Case("h_slot_plus1", 70, 17, _opt(48), 534), dict(one_past_slot=True)),
    "h_slot_plus1_lps16": (Case("h_slot_plus1_lps16", 91, 13, _opt(72), 535), dict(one_past_slot=True, lps=16)),
    # right pixels whose diagonal meets no column: dmin > 0, and dmin <= -D
    "dmin_pos": (Case("dmin_pos", 50, 11, _opt(40, 20), 541), dict(no_column=True)),
    "dmin_neg_d": (Case("dmin_neg_d", 45, 11, _opt(24, -24), 542), dict(no_column=True)),
    "dmin_below_neg_d": (Case("dmin_below_neg_d", 70, 9, _opt(40, -50), 543), dict(no_column=True)),
    # the y pass at Cone's width in more CTAs than stay resident (20 pairs per wave, one more in a second wave)
    "resident_overflow": (Case("resident_overflow", 450, 9, _opt(128), 551, wave_pairs=20, lanes=1, n=21),
                          dict(y_waves=2)),
}
POISON_CASES = [n for n in EDGE_CASES if n.startswith("fill_")] + ["lps8_r3"]


def edge_facts(c, plans):
    """What case c's fused pass meets, from so_plan.h (the plan executables)."""
    rule = _rule(c.W, c.H, c.D, c.opt.min_disparity)
    lps = so_lanes_per_line(c.Dp)
    band, lpw = rule["band"], 32 // lps
    rem = (c.W - 1) % band + 1                       # columns of the last band
    y = plans.so(c, 1)
    xr = np.arange(c.W)
    lo, hi = np.maximum(0, xr + c.opt.min_disparity), np.minimum(c.W - 1, xr + c.opt.min_disparity + c.D - 1)
    return dict(fused=bool(rule["fused"]), exact_fill=FIELDS * rule["plane"] == rule["vol"], lps=lps,
                live_warps=-(-rem // lpw), dead_lines=rem % lpw != 0, one_band=c.W <= band, narrow=c.W < c.D, H=c.H,
                one_past_slot=c.H > y["T"] and c.H % y["T"] == 1, no_column=bool((lo > hi).any()),
                y_waves=y["waves"])


# ---- tie families ---------------------------------------------------------------------------------------------------
# GT's cases whose options leave the fusion on (the discontinuity adjustment reads the optimised volume)
TIE_CASES = [n for n, (_, os_) in GT.cases().items() if not GT.OPTION_SETS[os_][0].get("do_discontinuity_adjustment")]
COST_INPUTS = [(layout, dtype) for layout in ("hwd", "dhw") for dtype in ("f32", "f16", "bf16")]

# Cost-input families built for the merge's rules.  Without scanline penalties each pass adds one value to a pixel's
# whole curve, and where a pixel's cross region holds only equal curves aggregation keeps the curve too, so the WTA
# meets the shapes built here.  Values are multiples of 1/32 below 4: exact in every element type.
ZERO_PEN = dict(so_p1=0.0, so_p2=0.0)
FT_OPTION_SETS = {"flat": _opt(32, **ZERO_PEN), "flat_dpos": _opt(32, 3, **ZERO_PEN), "flat_dneg": _opt(27, -6, **ZERO_PEN)}
BAND = 16   # so_wta_band at these ranges (8 lanes per line)


def _band_images(edge, i):
    """Views of flat 16-column blocks aligned with the bands, alternating in colour; with `edge` in {0, 15} that column
    of every band is a block of its own.  Neighbouring blocks differ by more than cross_t1, so no cross arm leaves its
    block."""
    x = np.arange(GT.W)
    cls = (x // BAND + i) % 2
    if edge is not None:
        cls = np.where(x % BAND == edge, 2, cls)
    g = np.broadcast_to((30 + 100 * cls).astype(np.uint8)[None, :], (GT.H, GT.W))
    left = np.ascontiguousarray(np.repeat(g[:, :, None], 3, axis=2))
    return left, np.ascontiguousarray(np.roll(left, -(3 + i), axis=1))


def ft_two_band_tie(D, seed, i):
    """One curve everywhere with two equal minima 16 + s apart: every right pixel's first minimum is tied in a later
    band."""
    a, s = 1 + (seed + i) % 6, (seed + i) % 5
    k = 96 + (np.arange(D) * 5 + i) % 7
    k[a] = k[min(a + BAND + s, D - 1)] = 64
    return GT._cost_images(seed, i), np.broadcast_to(k, (GT.H, GT.W, D))


def ft_band_edges(D, seed, i):
    """A low curve on the first (even i) or last (odd i) column of every band: the minimum of a right pixel sits at a
    record's first or last d, and its parabola takes a neighbour from the record before or after."""
    edge = 0 if i % 2 == 0 else BAND - 1
    x = np.arange(GT.W)[:, None]
    d = np.arange(D)[None, :]
    k = np.where(x % BAND == edge, 64 + (d * 3 + x // BAND + seed) % 5, 96 + (d + x // BAND) % 3)
    return _band_images(edge, i), np.broadcast_to(k, (GT.H, GT.W, D))


def ft_range_ends(D, seed, i):
    """Per band: the minimum at d = 0, at d = D - 1, or a flat curve; equal minima across bands."""
    x = np.arange(GT.W)[:, None]
    d = np.arange(D)[None, :]
    kind = (x // BAND + i + seed) % 3
    k = 96 + (d * 7 + x // BAND) % 4
    k = np.where((kind == 0) & (d == 0) | (kind == 1) & (d == D - 1), 64, k)
    k = np.where(kind == 2, 64, k)
    return _band_images(None, i), np.broadcast_to(k, (GT.H, GT.W, D))


def ft_flat_parabola(D, seed, i):
    """One V-shaped curve everywhere, c(a - 1) == c(a + 1): a flat parabola, whose neighbours cross a band boundary
    where the minimum sits on a band's first or last column."""
    a = 2 + (seed + 3 * i) % (D - 4)
    k = 64 + 2 * np.abs(np.arange(D) - a)
    return GT._cost_images(seed, i), np.broadcast_to(k, (GT.H, GT.W, D))


FT_FAMILIES = {"two_band_tie": ft_two_band_tie, "band_edges": ft_band_edges, "range_ends": ft_range_ends,
               "flat_parabola": ft_flat_parabola}
FT_CASES = [f"ft/{fam}/{os_}" for fam in FT_FAMILIES for os_ in FT_OPTION_SETS]


def tie_option(name):
    if name.startswith("ft/"):
        return FT_OPTION_SETS[name.split("/")[2]]
    return GT.option(name)


@functools.cache
def tie_pairs(name):
    if not name.startswith("ft/"):
        return GT.pairs(name)
    _, fam, os_ = name.split("/")
    opt = tie_option(name)
    seed = 9000 + 100 * list(FT_FAMILIES).index(fam) + 10 * list(FT_OPTION_SETS).index(os_)
    out = []
    for i in range(GT.N_PAIRS):
        (left, right), k = FT_FAMILIES[fam](opt.max_disparity - opt.min_disparity, seed + i, i)
        out.append((left, right, (np.asarray(k, np.float32) / np.float32(32)).copy()))
    return out


def tie_cost_input(name):
    """(layout, element type): the tie file's cycle through the option sets, and through the families here."""
    if name.startswith("ft/"):
        return COST_INPUTS[FT_CASES.index(name) % len(COST_INPUTS)]
    return COST_INPUTS[list(GT.OPTION_SETS).index(GT.cases()[name][1]) % len(COST_INPUTS)]


def tie_case(name):
    opt = tie_option(name)
    return Case(name, GT.W, GT.H, opt, 0)


def merge_rule_counts(vol, dmin, band):
    """On an optimised volume [H][W][D]: right pixels whose first minimum a later band ties, whose minimum sits at a
    record's first d with d > 0, at a record's last d with d < D - 1, and that see no column at all."""
    H, W, D = vol.shape
    xr, d = np.arange(W)[:, None], np.arange(D)[None, :]
    x = xr + dmin + d
    ok = (x >= 0) & (x < W)
    cr = np.where(ok[None], vol[:, np.clip(x, 0, W - 1), np.broadcast_to(d, x.shape)], np.inf)
    has = ok.any(axis=1)
    ds = cr.argmin(axis=2)
    m = np.take_along_axis(cr, ds[..., None], 2)
    xs = xr[None, :, 0] + dmin + ds
    later = ((cr == m) & (x[None] // band > xs[..., None] // band) & ok[None]).any(axis=2)
    first = (xs % band == 0) & (ds > 0)
    last = (((xs + 1) % band == 0) | (xs == W - 1)) & (ds < D - 1)
    return dict(later_band_tie=int((later & has).sum()), record_first=int((first & has).sum()),
                record_last=int((last & has).sum()), no_column=int(H * (~has).sum()))


@functools.cache
def tie_case_counts(name):
    """(merge_rule_counts summed over the case's pairs, the oracle's tie counters up to the WTA, summed)."""
    opt = tie_option(name)

    def one(p):
        left, right, cost = p
        orc = T.Oracle(GT.W, GT.H, opt) if cost is None else CT.CostOracle(GT.W, GT.H, opt)
        orc.begin(left, right) if cost is None else orc.begin_cost(left, right, cost)
        orc.run_to("SO4")
        r = merge_rule_counts(orc.tap("VOL_AGGR"), opt.min_disparity, BAND)
        orc.run_to("WTA")
        t = orc.tie_counts()
        orc.close()
        return r, t

    with ThreadPoolExecutor(GT.N_PAIRS) as ex:
        per = list(ex.map(one, tie_pairs(name)))
    return ({k: sum(r[k] for r, _ in per) for k in per[0][0]}, {k: sum(t[k] for _, t in per) for k in T.TIES})


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_reachable_instantiations_are_the_built_ones():
    """The k_scanline_wta instantiations whose records fit a pair's volume for some W, H, dmin adc_create accepts are
    exactly 23 (D in {5, 6} and 9..128), and exactly the ones in the library."""
    dom = domain()
    assert [D for D in dom if dom[D][3]] == [5, 6, *range(9, 129)]
    fit = fit_instantiations()
    assert len(fit) == 23, sorted(fit)
    assert not {(K, L) for _, K, L, _ in fit if L == 32} and ("k_scanline_wta", 1, 8, True) not in fit
    assert library_instantiations(WTA_SYMBOLS) == fit, sorted(library_instantiations(WTA_SYMBOLS) ^ fit)


def test_sweep_cases():
    """The fused sweep covers every range of the fit domain, at the sweep's shape or the nearest wider one that fits."""
    assert FIT_DS == [5, 6, *range(9, 129)]
    moved = 0
    for D in FIT_DS:
        c = sweep_case(D)
        W0, H0, opt0, _ = GS.sweep_case(D)
        assert (c.H, c.opt.min_disparity) == (H0, opt0.min_disparity) and c.W >= W0
        moved += c.W != W0
    print(f"{moved} of {len(FIT_DS)} sweep ranges moved to a wider width")


def _gpu_cases():
    return ([(sweep_case(D), DBG_FUSED_SO_WTA) for D in FIT_DS] + [(c, DBG_FUSED_SO_WTA) for c, _ in EDGE_CASES.values()]
            + [(tie_case(n), DBG_FUSED_SO_WTA | GT.debug_flags(n) if not n.startswith("ft/") else DBG_FUSED_SO_WTA)
               for n in TIE_CASES + FT_CASES])


def test_every_instantiation_is_covered(plans):
    """Every instantiation in the fit domain is launched fused by at least one GPU case of this file."""
    union = set()
    for c, flags in _gpu_cases():
        rule = plans.so_wta(c, flags, volumes=False)
        assert rule["fused"], c.name
        union |= reached(c, plans, fused=True)
    wta = {i for i in union if i[0] == "k_scanline_wta"}
    assert wta == fit_instantiations(), sorted(fit_instantiations() - wta)


def test_edge_cases_take_their_path(plans):
    """Each band-edge case is fused and meets what it is there for."""
    for name, (c, want) in EDGE_CASES.items():
        got = edge_facts(c, plans)
        assert got["fused"], name
        for k, v in want.items():
            assert got[k] == v, f"{name}: {k} = {got[k]}, expected {v} ({got})"
        if want.get("exact_fill"):   # several pairs per wave: an overrun would land in the next pair's slice
            assert c.wave_pairs >= 4, name
    assert {(c.W % 16) for n, (c, _) in EDGE_CASES.items() if n.startswith("lps8_")} == {1, 5, 9, 15}
    assert {(c.W % 8) for n, (c, _) in EDGE_CASES.items() if n.startswith("lps16_")} == {1, 3, 5, 7}


def test_large_case_is_fused_by_default():
    """4000 x 2100 x 64 fuses under the AUTO rule, each volume is past 2^31 bytes, and in a wave of three the second
    pair's records start past 2^31 bytes and the third pair's past 2^32."""
    g = E.golden("golden_limits.json")
    W, H, D = (g["F1_s1"][k] for k in ("width", "height", "max_disparity"))
    r = _rule(W, H, D, force=AUTO)
    assert r["fused"] and 2 ** 31 < 4 * r["vol"] < 2 ** 32 < 2 * 4 * r["vol"]
    assert g["F1_s1"]["checker"] == g["F1_s2"]["checker"] == "reference"
    assert not _rule(W, H, D, force=AUTO, confidence=1)["fused"]


def test_tie_cases_reach_the_merge_rules():
    """Across the tie cases, the oracle's optimised volumes have right pixels whose first minimum a later band ties,
    minima at a record's first d (d > 0) and last d (d < D - 1), and right pixels with no column; and the new families
    decide WTA_L, WTA_R and SUBPIX_FLAT."""
    tot = dict(later_band_tie=0, record_first=0, record_last=0, no_column=0)
    ties = dict.fromkeys(T.TIES, 0)
    for n in TIE_CASES + FT_CASES:
        r, t = tie_case_counts(n)
        for k in tot:
            tot[k] += r[k]
        if n.startswith("ft/"):
            for k in ties:
                ties[k] += t[k]
    print("merge rules over the tie cases:", tot, "oracle ties over the new families:", ties)
    assert all(v > 0 for v in tot.values()), tot
    assert ties["WTA_L"] > 0 and ties["WTA_R"] > 0 and ties["SUBPIX_FLAT"] > 0, ties
    for fam in FT_FAMILIES:   # each new family reaches the rule it is built for
        r = [tie_case_counts(f"ft/{fam}/{o}")[0] for o in FT_OPTION_SETS]
        need = {"two_band_tie": "later_band_tie", "band_edges": "record_first", "range_ends": "later_band_tie",
                "flat_parabola": "record_last"}[fam]
        assert sum(x[need] for x in r) > 0, (fam, r)


def test_cost_inputs_cover_every_type():
    assert {tie_cost_input(n) for n in FT_CASES} == set(COST_INPUTS)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _refused(eng):
    import adcensus_b200 as A
    with pytest.raises(A.AdcError, match="epilogue"):
        eng.tap("VOL_AGGR")


def _check_fused(c, flags=DBG_FUSED_SO_WTA, **kw):
    return check_case(c, debug_flags=flags, volumes=False, after=_refused, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("D", FIT_DS)
def test_fused_sweep(D):
    _check_fused(sweep_case(D))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EDGE_CASES))
def test_band_edge(name):
    c = EDGE_CASES[name][0]
    pairs = [T.synthetic_pair(c.W, c.H, c.D, c.seed + 7919 * k) for k in range(c.n)] if c.n > 5 else None
    _check_fused(c, pairs=pairs)


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True], ids=["plain", "pipelined"])
@pytest.mark.parametrize("name", TIE_CASES + FT_CASES)
def test_tie_case_fused(name, pipelined):
    flags = DBG_FUSED_SO_WTA | (0 if name.startswith("ft/") else GT.debug_flags(name))
    layout, dtype = tie_cost_input(name)
    _check_fused(tie_case(name), flags, pairs=tie_pairs(name), pipelined=pipelined, cost_layout=layout,
                 cost_dtype=dtype)


def _cone_case():
    left, right = T.load_cone()
    H, W = left.shape[:2]
    pairs = [(left, right)] + [T.synthetic_pair(W, H, 64, 561 + k) for k in range(3)]
    return Case("cone", W, H, T.default_option(), 561, wave_pairs=4, lanes=1, n=4), pairs


@pytest.mark.gpu
@pytest.mark.parametrize("byte", [0xFF, 0x7F, 0x01], ids=["ff", "7f", "01"])
@pytest.mark.parametrize("name", POISON_CASES + ["cone"])
def test_poisoned_arena(name, byte):
    """Batches of four on arenas filled with `byte` before every wave: a merge that reads a record slot the pass did not
    write meets the pattern."""
    if name == "cone":
        c, pairs = _cone_case()
    else:
        c0 = EDGE_CASES[name][0]
        c, pairs = Case(name, c0.W, c0.H, c0.opt, c0.seed, wave_pairs=4, lanes=1, n=4), None
    _check_fused(c, DBG_FUSED_SO_WTA | poison_flags(byte), pairs=pairs)


@pytest.mark.gpu
def test_vol_aggr_tap_shows_the_form():
    """A map-only call that stops after the WTA: fused, VOL_AGGR is refused; unfused, it is the oracle's SO4 volume.
    VOL_INIT is the SO3 volume either way.  Cone through adc_match under the defaults leaves VOL_AGGR refused."""
    W, H, D = 100, 37, 64
    opt = _opt(D)
    left, right = T.synthetic_pair(W, H, D, 571)
    orc = T.Oracle(W, H, opt)
    orc.begin(left, right)
    orc.run_to("SO3")
    so3 = orc.tap("VOL_INIT").copy()
    orc.run_to("SO4")
    so4 = orc.tap("VOL_AGGR").copy()
    orc.run_to("WTA")
    wta = orc.tap("DISP_L").copy(), orc.tap("DISP_R").copy()
    orc.close()
    for flags in (DBG_FUSED_SO_WTA, DBG_UNFUSED_SO_WTA):
        eng = E.engine(W, H, opt, debug_flags=flags)
        try:
            _, maps = eng.match_outputs(left, right, maps=("wta_left", "wta_right"), disparity=False)
            E.same(f"{flags} wta_left", maps["wta_left"], wta[0])
            E.same(f"{flags} wta_right", maps["wta_right"], wta[1])
            E.same(f"{flags} VOL_INIT", eng.tap("VOL_INIT"), so3)
            if flags == DBG_FUSED_SO_WTA:
                _refused(eng)
            else:
                E.same("unfused VOL_AGGR", eng.tap("VOL_AGGR"), so4)
        finally:
            eng.close()
    left, right = T.load_cone()
    eng = E.engine(left.shape[1], left.shape[0], T.default_option())
    try:
        want = T.Oracle(left.shape[1], left.shape[0], T.default_option()).match(left, right)
        E.same("cone match", eng.match(left, right), want)
        _refused(eng)
    finally:
        eng.close()


@pytest.mark.gpu
def test_large_volume_fused():
    """Three 4000 x 2100 x 64 pairs (seeds 1, 2, 1) in one wave under the AUTO rule (fused), through
    adc_match_outputs_batch_device with the WTA maps and the final map: each against the reference's hashes."""
    torch, dev = E.cuda()
    g = E.golden("golden_limits.json")
    cases = [g[n] for n in ("F1_s1", "F1_s2", "F1_s1")]
    W, H, D = cases[0]["width"], cases[0]["height"], cases[0]["max_disparity"]
    views = []
    for c in cases:
        left, right = T.synthetic_pair(W, H, D, c["seed"])
        assert [T.sha(left), T.sha(right)] == c["input_sha"]
        views.append((left, right))
    d_l = torch.from_numpy(np.stack([v[0] for v in views])).to(dev)
    d_r = torch.from_numpy(np.stack([v[1] for v in views])).to(dev)
    del views
    eng = E.engine(W, H, T.default_option(max_disparity=D), wave_pairs=3, lanes=1)
    try:
        assert eng.wave_pairs == 3
        got = E.batch_outputs(eng, eng.match_outputs_batch_device, 3, d_l.data_ptr(), d_r.data_ptr(), 3 * W * H,
                              maps=["wta_left", "wta_right"])
        _refused(eng)
    finally:
        eng.close()
    for i, c in enumerate(cases):
        for k, tap in (("wta_left", "WTA/DISP_L"), ("wta_right", "WTA/DISP_R"), ("disp", "MEDIAN/DISP_L")):
            assert T.sha(got[k][i]) == c["hashes"][tap], f"pair {i}: {k}"
