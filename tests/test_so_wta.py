"""The last scanline pass with the winner-takes-all as its epilogue (k_scanline_wta + k_wta_merge) against
the unfused pass 4 + k_wta: the selection rule on the CPU (adcensus_b200/csrc/so_plan.h), and both forms forced through
adc_config.debug_flags on the same inputs, compared bit for bit."""
import subprocess

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E

AUTO, NEVER, ALWAYS = 0, 1, 2   # SoWtaForce


def _rule(W, H, D, dmin=0, opt_export=0, confidence=0, discontinuity=0, debug_run=0, force=AUTO):
    r = subprocess.run([str(E.c_tool("so_wta_main"))] + [str(v) for v in (W, H, D, dmin, opt_export, confidence,
                                                                          discontinuity, debug_run, force)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    fused, band, row_records, plane, vol = map(int, r.stdout.split())
    return dict(fused=bool(fused), band=band, row_records=row_records, plane=plane, vol=vol)


def _row_records(W, D, dmin, band):
    """Records of one row, counted right pixel by right pixel: the bands its diagonal's in-image columns touch."""
    n = 0
    for xr in range(W):
        lo, hi = max(0, xr + dmin), min(W - 1, xr + dmin + D - 1)
        if lo <= hi:
            n += hi // band - lo // band + 1
    return n


def test_rule_bytes_at_the_benchmark_shapes():
    cone = _rule(450, 375, 64)
    assert cone["band"] == 16 and cone["fused"]
    assert 2 * 24 * cone["row_records"] <= 0.5 * 2 * 4 * 450 * 64          # records written + read: 44 % of 2V
    kitti = _rule(1242, 375, 128)
    assert kitti["band"] == 8 and not kitti["fused"]
    p1080 = _rule(1920, 1080, 192)
    assert p1080["band"] == 4 and not p1080["fused"]
    for W, D, dmin in ((450, 64, 0), (1242, 128, 0), (1920, 192, 0), (100, 64, 0), (133, 128, 0), (97, 50, -9),
                       (64, 64, 30), (41, 20, -50)):
        r = _rule(W, 7, D, dmin)
        assert r["row_records"] == _row_records(W, D, dmin, r["band"]), (W, D, dmin)


def test_rule_keeps_the_volume_where_it_is_read():
    for what in ("opt_export", "confidence", "discontinuity", "debug_run"):
        assert not _rule(450, 375, 64, **{what: 1})["fused"], what
        assert not _rule(450, 375, 64, force=ALWAYS, **{what: 1})["fused"], what
    assert not _rule(450, 375, 64, force=NEVER)["fused"]


def test_rule_forced_only_where_the_records_fit():
    kitti = _rule(1242, 375, 128, force=ALWAYS)
    assert kitti["fused"] and 6 * kitti["plane"] <= kitti["vol"]
    p1080 = _rule(1920, 1080, 192, force=ALWAYS)
    assert not p1080["fused"] and 6 * p1080["plane"] > p1080["vol"]


# name -> (W, H, min_disparity, max_disparity, seed).  Band widths 16 / 8 columns; most widths leave a partial last band.
CASES = {
    "cone_crop_d64": (450, 375, 0, 64, None),      # the benchmark's shape and pair: the rule fuses it
    "d64_partial": (100, 37, 0, 64, 11),          # 6 bands + 4 columns, FULL K = 8
    "d48_partial": (77, 29, 0, 48, 12),           # K = 6
    "d50_padded": (97, 31, -9, 41, 13),           # D not a multiple of 4, negative dmin
    "d20_padded": (41, 23, 0, 20, 14),            # K = 3, band wider than D
    "dmin_pos": (83, 19, 7, 71, 15),              # positive dmin: right pixels at the left edge see no column
    "d128_band8": (133, 21, 0, 128, 16),          # 16 lanes per line: band of 8 columns, 16 bands + 5 columns
}


def _pairs(W, H, D, seed, n):
    if seed is None:
        left, right = T.load_cone()
        return np.stack([left] * n), np.stack([right] * n)
    ps = [T.synthetic_pair(W, H, D, seed + k) for k in range(n)]
    return np.stack([p[0] for p in ps]), np.stack([p[1] for p in ps])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_fused_and_unfused_forms_agree(name):
    import adcensus_b200 as A
    W, H, dmin, dmax, seed = CASES[name]
    D = dmax - dmin
    opt = T.default_option(min_disparity=dmin, max_disparity=dmax)
    rule = _rule(W, H, D, dmin, force=ALWAYS)
    lefts, rights = _pairs(W, H, D, seed, 3)
    out = {}
    for form, flag in (("unfused", A.engine.DBG_UNFUSED_SO_WTA), ("fused", A.engine.DBG_FUSED_SO_WTA)):
        eng = E.engine(W, H, opt, wave_pairs=2, lanes=2, debug_flags=flag)
        try:
            disp, maps = eng.match_outputs(lefts[1], rights[1], maps=("wta_left", "wta_right"))
            out[form] = dict(disp=disp, batch=eng.match_batch(lefts, rights), **maps)
        finally:
            eng.close()
    for k in ("wta_left", "wta_right", "disp", "batch"):
        E.same(f"{name} {k} (records fit: {rule['fused']})", out["fused"][k], out["unfused"][k])
