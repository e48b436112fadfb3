"""The AD-census cost computed inside the first horizontal aggregation pass (k_cost_arm_sum_h, k_aggregate.cu): its
launch plan (adcensus_b200/csrc/ca_plan.h) on the CPU, its compiled resources, and on the GPU the volumes it produces
against the separate cost kernel and the unfused aggregation."""
import subprocess

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E

CSRC = T.REPO / "adcensus_b200" / "csrc"

# H100: 228 KB of shared memory per SM, 1 KB reserved per CTA; the kernel is planned for two CTAs per SM
SMEM_PER_SM, SMEM_RESERVED = 228 * 1024, 1024


def _plan(W, D, L1):
    Dp = (D + 3) // 4 * 4
    r = subprocess.run([str(E.c_tool("ca_plan_main")), str(W), str(Dp), str(L1)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.split("\n")
    qc, Ls, nseg, nchunks, gm, lpc, threads, smem, ok, budget = map(int, lines[0].split())
    segs = [tuple(map(int, ln.split())) for ln in lines[1:] if ln.strip()]
    return dict(qc=qc, Ls=Ls, nseg=nseg, nchunks=nchunks, gm=gm, lpc=lpc, threads=threads, smem=smem, ok=ok,
                budget=budget, Dp=Dp), segs


# (W, D, cross_L1)
PLAN_SHAPES = {
    "cone": (450, 64, 34), "kitti": (1242, 128, 34), "1080p": (1920, 192, 34), "d256": (450, 256, 34),
    "l1_130": (450, 64, 130), "odd_w": (97, 24, 34), "d37": (131, 37, 34), "odd_long": (1001, 61, 34),
    "d5": (33, 5, 34), "wide_l1_130": (1920, 192, 130),
}


@pytest.mark.parametrize("name", sorted(PLAN_SHAPES))
def test_cost_fused_plan(name):
    W, D, L1 = PLAN_SHAPES[name]
    p, segs = _plan(W, D, L1)
    assert p["ok"], p
    L1c = min(max(L1, 0), 255)
    # shared memory within the budget, and two CTAs per SM
    assert p["smem"] <= p["budget"] and 2 * (p["smem"] + SMEM_RESERVED) <= SMEM_PER_SM, p
    assert p["qc"] in (4, 8) and p["nchunks"] * p["qc"] * 4 >= p["Dp"], p
    assert p["threads"] % 32 == 0 and 32 <= p["threads"] <= 256, p
    # the segments tile the row: consecutive, no gaps, the last one ends at W
    assert p["Ls"] % 4 == 0 and len(segs) == p["nseg"], (p, segs)
    assert segs[0][0] == 0 and segs[-1][1] == W, segs
    for (a0, a1, _, _), (b0, _, _, _) in zip(segs, segs[1:]):
        assert a1 == b0 and a1 - a0 == p["Ls"], segs
    for s0, s1, m0, m1 in segs:
        # the cost range covers every tap of the segment's windows, [s0 - L1c, s1 + L1c) within the row ...
        assert m0 <= max(0, s0 - L1c) and m1 >= min(W, s1 + L1c), (s0, s1, m0, m1)
        assert 0 <= m0 and m0 % 4 == 0 and m1 <= W, (s0, s1, m0, m1)
        # ... and fits the cost rows the shared memory is sized for
        assert (m1 - m0 + 3) // 4 <= p["gm"], (p, s0, s1, m0, m1)
        assert (s1 - s0 + 3) // 4 <= p["Ls"] // 4
    if W <= 450 and L1 <= 34:
        assert p["nseg"] == 1, p                      # Cone and smaller rows are one segment


def test_cost_fused_plan_cone_choice():
    p, _ = _plan(450, 64, 34)
    assert (p["qc"], p["nseg"], p["nchunks"], p["threads"]) == (8, 1, 2, 256), p


def test_cost_fused_kernel_resources():
    """ptxas -v: no stack frame, no spills in any instantiation of k_cost_arm_sum_h, and at most 128 registers, which
    two CTAs of 256 threads per SM need; k_cost_volume keeps its 64 registers."""
    flags = ("-Xcompiler", "-ffp-contract=off")
    fused = {k: v for k, v in E.ptxas_report(CSRC / "k_aggregate.cu", flags).items()
             if "k_cost_arm_sum_h" in k and v["regs"] is not None}
    assert len(fused) == 4, sorted(fused)
    for name, f in fused.items():
        assert (f["stack"], f["spill_stores"], f["spill_loads"]) == (0, 0, 0), (name, f)
        assert f["regs"] <= 128, (name, f)
    cost = {k: v for k, v in E.ptxas_report(CSRC / "k_cost.cu", flags).items()
            if "k_cost_volume" in k and v["regs"] is not None}
    assert len(cost) == 2, sorted(cost)
    for name, f in cost.items():
        assert f["spill_stores"] == 0 and f["regs"] == 64, (name, f)


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_fused_cost_launch_count():
    """The fused path replaces k_cost_volume + the first horizontal pass by one launch: AGG4 takes 4 launches more than
    ARMS (the fused kernel, three double passes, the last divided pass); it took 5 with the separate cost kernel."""
    w, h, D = 97, 61, 24
    opt = T.default_option(max_disparity=D)
    left, right = T.synthetic_pair(w, h, D, 2)
    eng = E.engine(w, h, opt)
    c0 = eng.launch_count
    eng.debug_run(left, right, "ARMS")
    arms = eng.launch_count - c0
    c0 = eng.launch_count
    eng.debug_run(left, right, "AGG4")
    agg4 = eng.launch_count - c0
    eng.close()
    assert agg4 - arms == 4, (arms, agg4)


def _fused_cases():
    cases = [(w, h, D, over, seed) for (w, h, D, over, seed) in E.PARITY_CASES]
    cases.append(("cone", None, 64, {}, None))
    cases.append((1920, 1080, 192, {}, 41))          # rows cut into segments
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("case", _fused_cases(), ids=lambda c: f"{c[0]}x{c[1]}x{c[2]}")
def test_fused_cost_export_and_aggregation(case, cone):
    """The COST export written by the fused kernel equals the separate cost kernel's volume (debug_run("COST") /
    VOL_INIT); the same call's AGGR export and final map equal those of an engine that runs the unfused aggregation."""
    import adcensus_b200 as A
    w, h, D, over, seed = case
    if w == "cone":
        left, right = cone
        h, w, _ = left.shape
        opt = T.default_option()
    else:
        opt = T.default_option(**{"max_disparity": D, **over})
        left, right = T.synthetic_pair(w, h, D, seed)
    kw = dict(wave_pairs=1, lanes=1)
    eng = E.engine(w, h, opt, **kw)
    eng.debug_run(left, right, "COST")
    want_cost = eng.tap("VOL_INIT").copy()
    disp, vols = eng.match_volumes(left, right, ["cost", "aggr"])
    eng.close()
    assert np.array_equal(E.bits(vols["cost"]), E.bits(want_cost)), f"{w}x{h}x{D}: COST export differs from k_cost_volume"
    ref = E.engine(w, h, opt, debug_flags=A.engine.DBG_UNFUSED_AGG, **kw)
    rdisp, rvols = ref.match_volumes(left, right, ["aggr"])
    ref.close()
    assert np.array_equal(E.bits(vols["aggr"]), E.bits(rvols["aggr"])), f"{w}x{h}x{D}: AGGR differs from the unfused passes"
    assert np.array_equal(E.bits(disp), E.bits(rdisp)), f"{w}x{h}x{D}: final map differs from the unfused pipeline"
