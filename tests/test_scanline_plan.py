"""CPU test of the scanline passes' launch plan (adcensus_b200/csrc/so_plan.h): slot length T, ring depth NS and the
residency that follows from them, for the three benchmark shapes on an H100 SXM (132 SMs, 228 KB shared memory per SM)."""
import subprocess

import pytest

import engine_testlib as E


def _plan(W, H, Dp, S, axis):
    r = subprocess.run([str(E.c_tool("so_plan_main")), str(W), str(H), str(Dp), str(S), str(axis)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    T, NS, smem, ctas, per_sm, waves = map(int, r.stdout.split())
    return dict(T=T, NS=NS, smem=smem, ctas=ctas, per_sm=per_sm, waves=waves)


# (W, H, Dp, wave pairs as adc_create picks them, axis) -> (T, NS, CTAs, CTAs per SM, waves)
CASES = {
    "cone_x": ((450, 375, 64, 32, 0), (2, 4, 768, 6, 1)),
    "cone_y": ((450, 375, 64, 32, 1), (2, 3, 928, 8, 1)),      # 6 CTAs per SM would leave 136 CTAs for a second wave
    "kitti_x": ((1242, 375, 128, 32, 0), (2, 4, 1504, 6, 2)),
    "kitti_y": ((1242, 375, 128, 32, 1), (2, 3, 4992, 8, 5)),
    "1080p_x": ((1920, 1080, 192, 12, 0), (2, 4, 3240, 8, 4)),
    "1080p_y": ((1920, 1080, 192, 12, 1), (2, 4, 5760, 8, 6)),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_scanline_plan_choices(name):
    args, (T, NS, ctas, per_sm, waves) = CASES[name]
    p = _plan(*args)
    assert (p["T"], p["NS"], p["ctas"], p["per_sm"], p["waves"]) == (T, NS, ctas, per_sm, waves), p
    assert p["T"] * p["NS"] >= 4                              # every warp keeps at least four steps in flight
    assert (p["smem"] + 1024) * p["per_sm"] <= 228 * 1024


def test_scanline_plan_serves_every_disparity_range():
    for Dp in range(4, 257, 4):
        for axis in (0, 1):
            p = _plan(450, 375, Dp, 32, axis)
            assert p["T"] >= 2 and p["per_sm"] >= 1, (Dp, axis, p)
