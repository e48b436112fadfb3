"""The batched parity check of the kernel sweep and the option-space cases: a case, the launch plans the kernels take
for it (printed by tests/c/ca_plan_main.cpp and so_plan_main.cpp from the headers the kernels are launched with), the
template instantiations one run of it launches, and the run itself against the oracle."""
from __future__ import annotations

import os
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E  # puts tools/ on sys.path
import maps_testlib as MT
import make_golden_sweep as GS

SMEM_RESERVED_PER_CTA = 1024     # shared memory the driver reserves per CTA on sm_90


class Case:
    """One batched GPU run: W x H x D with `opt`, n pairs in waves of `wave_pairs` over `lanes` lanes."""

    def __init__(self, name, W, H, opt, seed, wave_pairs=2, lanes=2, n=5):
        self.name, self.W, self.H, self.opt, self.seed = name, W, H, opt, seed
        self.D = opt.max_disparity - opt.min_disparity
        self.Dp = (self.D + 3) // 4 * 4
        self.L1 = opt.cross_L1
        self.wave_pairs, self.lanes, self.n = wave_pairs, lanes, n


# ---- cases ----------------------------------------------------------------------------------------------------------
def sweep_case(D):
    W, H, opt, seed = GS.sweep_case(D)
    return Case(f"D{D}", W, H, opt, seed)


def _opt(D, **kw):
    return T.default_option(max_disparity=D, **kw)


LONG_ARMS = dict(cross_L1=255, cross_L2=120, cross_t1=50, cross_t2=25)
# name -> (case, what its plans must be).  Shapes found with the plan executables; test_plan_branch_cases checks them.
PLAN_CASES = {
    # fused cost + first horizontal pass (ca_plan): rows in 2 and 3 segments at L1 = 34, qc = 8, exact and not
    "cost_rows_2seg": (Case("cost_rows_2seg", 501, 23, _opt(45), 61), dict(ca_nseg=2, ca_qc=8)),
    "cost_rows_3seg": (Case("cost_rows_3seg", 861, 19, _opt(64), 62), dict(ca_nseg=3, ca_qc=8)),
    # L1 = 130: 3 segments of 164 outputs, shorter than 2 L1, so a segment's halos span a whole neighbouring segment
    "cost_rows_l1_130": (Case("cost_rows_l1_130", 486, 17, _opt(61, cross_L1=130, cross_L2=40, cross_t1=60, cross_t2=30), 63),
                         dict(ca_nseg=3, ca_qc=8, ca_short=True)),
    # D < 32: four quads per CTA, D not a multiple of 4, rows in 2 segments
    "cost_rows_qc4": (Case("cost_rows_qc4", 825, 13, _opt(23), 64), dict(ca_nseg=2, ca_qc=4)),
    # arms too long for the fused cost plan: the separate cost kernel, exact and padded D; at W = 701 the row does not
    # fit k_arm_sum2t's plan either, so both axes take the LDG double pass with eight quads
    "cost_volume_exact": (Case("cost_volume_exact", 509, 13, _opt(32, **LONG_ARMS), 65), dict(ca_ok=False)),
    "cost_volume_padded_ldg": (Case("cost_volume_padded_ldg", 701, 13, _opt(37, **LONG_ARMS), 66),
                               dict(ca_ok=False, tmaps=False)),
    # k_arm_sum2t down columns cut into segments, one line per CTA, eight and four quads
    "cols_seg_qc8": (Case("cols_seg_qc8", 21, 709, _opt(64), 67), dict(t1_nseg=3, t1_qc=8, t1_lpc=1)),
    "cols_seg_qc4": (Case("cols_seg_qc4", 13, 809, _opt(23), 68), dict(t1_nseg=2, t1_qc=4, t1_lpc=1)),
    # the LDG double pass on rows in segments: Q = 4 (generic QC) and Q = 3 (no TMA plan at all, Q < 4)
    "ldg_rows_q4": (Case("ldg_rows_q4", 1001, 13, _opt(14), 69), dict(ldg0_nseg=2, ldg0_qc=0, t0_nseg=2)),
    "ldg_rows_q3": (Case("ldg_rows_q3", 1001, 13, _opt(11), 70), dict(ldg0_nseg=2, ldg0_qc=0, tmaps=False)),
    # scanline slots of T = 2 steps on the row passes, for 8, 16 and 32 lanes per line, K not FULL, an odd step count
    "so_t2_lps8": (Case("so_t2_lps8", 33, 1057, _opt(61), 71, wave_pairs=8, lanes=1), dict(so_T0=2, lps=8)),
    "so_t2_lps16": (Case("so_t2_lps16", 33, 659, _opt(93), 72, wave_pairs=8, lanes=1), dict(so_T0=2, lps=16)),
    "so_t2_lps32": (Case("so_t2_lps32", 33, 329, _opt(200), 73, wave_pairs=8, lanes=1), dict(so_T0=2, lps=32)),
}

SWEEP_DS = list(range(1, 257))


def all_cases():
    return [sweep_case(D) for D in SWEEP_DS] + [c for c, _ in PLAN_CASES.values()]


SYMBOLS = {
    "k_scanline": re.compile(r"_Z10k_scanlineILi(\d+)ELi(\d+)ELb([01])EE"),
    "k_cost_volume": re.compile(r"_Z13k_cost_volumeILb([01])EE"),
    "k_cost_arm_sum_h": re.compile(r"_Z16k_cost_arm_sum_hILb([01])ELi(\d+)EE"),
    "k_arm_sum2t": re.compile(r"_Z11k_arm_sum2tILb([01])ELi(\d+)EE"),
    "k_arm_sum2": re.compile(r"_Z10k_arm_sum2ILb([01])ELi(\d+)EE"),
    "k_vote_scan": re.compile(r"_Z11k_vote_scanILb([01])EE"),
    "k_vote_push": re.compile(r"_Z11k_vote_pushILb([01])EE"),
}


def library_instantiations(symbols=SYMBOLS):
    """{(template, args...)} of the templates in `symbols` (by default the seven above), read from the built library's
    device symbols."""
    from adcensus_b200.build import build_library
    cuobjdump = Path(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")).parent / "cuobjdump"
    if not cuobjdump.exists():
        pytest.skip(f"cuobjdump not found at {cuobjdump}")
    r = subprocess.run([str(cuobjdump), "-symbols", str(build_library())], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    found = set()
    for name, rx in symbols.items():
        for m in rx.finditer(r.stdout):
            args = tuple(int(g) for g in m.groups())
            if name in ("k_scanline", "k_scanline_wta"):
                found.add((name, args[0], args[1], bool(args[2])))
            else:
                found.add((name, bool(args[0]), *args[1:]))
    return found


# ---- plans ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def plans():
    return Plans()


def _device_figures():
    """(SM count, shared memory per SM, reserved per CTA) of device 0, or an H100 SXM's where there is no GPU."""
    import torch
    if torch.cuda.is_available():
        p = torch.cuda.get_device_properties(0)
        return p.multi_processor_count, p.shared_memory_per_multiprocessor, SMEM_RESERVED_PER_CTA
    return 132, 228 * 1024, SMEM_RESERVED_PER_CTA


class Plans:
    def __init__(self):
        self.dev = _device_figures()

    def _run(self, exe, *args):
        r = subprocess.run([str(E.c_tool(exe)), *map(str, args)], capture_output=True, text=True)
        assert r.returncode == 0, (exe, args, r.stdout, r.stderr)
        return r.stdout

    def ca(self, c):
        v = list(map(int, self._run("ca_plan_main", c.W, c.Dp, c.L1).split("\n")[0].split()))
        return dict(zip(("qc", "Ls", "nseg", "nchunks", "gm", "lpc", "threads", "smem", "ok", "budget"), v))

    def arm(self, c):
        out = []
        for line in self._run("ca_plan_main", "arm", c.W, c.H, c.Dp, c.L1).strip().split("\n"):
            v = list(map(int, line.split()))
            out.append(dict(zip(("dir", "t_ok", "t_qc", "t_Ls", "t_nseg", "t_nchunks", "t_lpc", "t_threads", "t_smem",
                                 "ldg_qc_log2", "ldg_Ls", "ldg_nseg", "ldg_smem", "form", "smem_attr"), v)))
        return out

    def so(self, c, axis):
        v = list(map(int, self._run("so_plan_main", c.W, c.H, c.Dp, c.wave_pairs, axis, *self.dev).split()))
        return dict(zip(("T", "NS", "smem", "ctas", "ctas_per_sm", "waves"), v))

    def so_wta(self, c, debug_flags=0, volumes=True, confidence=False):
        """so_wta_fused for a batched run of case c (check_case's requests): dict(fused, band, row_records, plane, vol)."""
        import adcensus_b200 as A
        force = 1 if debug_flags & A.engine.DBG_UNFUSED_SO_WTA else 2 if debug_flags & A.engine.DBG_FUSED_SO_WTA else 0
        v = list(map(int, self._run("so_wta_main", c.W, c.H, c.D, c.opt.min_disparity, int(volumes), int(confidence),
                                    int(c.opt.do_discontinuity_adjustment != 0), 0, force).split()))
        return dict(zip(("fused", "band", "row_records", "plane", "vol"), v))


def so_lanes_per_line(Dp):
    return 8 if Dp <= 64 else (16 if Dp <= 128 else 32)


A2_TMA, A2_LDG = 1, 0     # the forms arm_sum2_form (ca_plan.h) picks


def reached(c, plans, fused=False):
    """The instantiations of the seven templates one batched run of case c launches, by the launch rules of
    k_aggregate.cu, k_cost.cu, k_scanline.cu and k_vote.cu (a run that matches, so every stage runs, with the fused
    aggregation):
      cost:      k_cost_arm_sum_h<D == Dp, ca_plan.qc> where ca_plan is ok, else k_cost_volume<D == Dp>;
      axis dir:  k_arm_sum2t<dir, qc> where the TMA plans of both axes are ok and, on rows, the row is one segment; else
                 k_arm_sum2<dir, 8 if Qc == 8 else 0> (generic QC).  This restates arm_sum2_form, and the form the plan
                 executable prints for the axis must agree with it;
      scanline:  k_scanline<ceil(Dp / LPS), LPS, D == K * LPS>, LPS = so_lanes_per_line(Dp), and with the same
                 arguments k_scanline_wta where the last pass runs `fused` with the WTA (Plans.so_wta);
      voting:    k_vote_scan<WIDE> and k_vote_push<WIDE>, WIDE iff D > 254 or L1 > 127."""
    out = set()
    exact = c.D == c.Dp
    ca = plans.ca(c)
    out.add(("k_cost_arm_sum_h", exact, ca["qc"]) if ca["ok"] else ("k_cost_volume", exact))
    arm = plans.arm(c)
    tmaps = bool(arm[0]["t_ok"] and arm[1]["t_ok"])
    for a in arm:
        # the fused aggregation runs on every shape: both plans fit the shared memory the passes are launched under
        assert a["t_smem"] <= a["smem_attr"] and a["ldg_smem"] <= a["smem_attr"], (c.name, a)
        tma = tmaps and not (a["dir"] == 0 and a["t_nseg"] > 1)
        assert a["form"] == (A2_TMA if tma else A2_LDG), (c.name, a)
        if tma:
            out.add(("k_arm_sum2t", a["dir"] == 1, a["t_qc"]))
        else:
            out.add(("k_arm_sum2", a["dir"] == 1, 8 if a["ldg_qc_log2"] == 3 else 0))
    lps = so_lanes_per_line(c.Dp)
    K = -(-c.Dp // lps)
    out.add(("k_scanline", K, lps, c.D == K * lps))
    if fused:
        out.add(("k_scanline_wta", K, lps, c.D == K * lps))
    wide = c.D > 254 or min(c.L1, 255) > 127
    out.add(("k_vote_scan", wide))
    out.add(("k_vote_push", wide))
    return out


# ---- the GPU run ----------------------------------------------------------------------------------------------------
def _oracle_outputs(c, left, right, cost):
    if cost is None:
        return E.oracle_outputs(c.W, c.H, c.opt, left, right)
    import cost_testlib as CT
    orc = CT.CostOracle(c.W, c.H, c.opt)
    orc.begin_cost(left, right, cost)
    out = {}
    for st in T.STAGES:
        orc.step()
        for tap in T.STAGE_TAPS[st]:
            if (st, tap) in E.ORACLE_OUTPUTS:
                out[E.ORACLE_OUTPUTS[(st, tap)]] = orc.tap(tap).copy()
    orc.close()
    return out


def check_case(c, debug_flags=0, pairs=None, confidence=False, pipelined=False, cost_layout="hwd", cost_dtype="f32",
               volumes=True, after=None):
    """One match_outputs_batch_device call over the case's pairs, exporting the three volumes (f32, [H][W][D]), the
    WTA maps, the outlier map and the final map, each pair compared bit for bit with its own oracle run, on an engine
    created with `debug_flags`; returns every output of the call on the host.
    volumes=False: no volume export (the call then reads the optimised volume only where the options do, so the last
    scanline pass may take the WTA as its epilogue); not with confidence.  after(eng): called with the engine after the
    call, before it is closed.
    pairs: [(left, right)] or [(left, right, cost volume f32 [H][W][D])] instead of the sweep's pairs; with cost volumes
    the call matches from them (given as `cost_layout` / `cost_dtype`; their values must be exact in that type).
    confidence: also export MIN_COST / PEAK_RATIO and compare them with maps_testlib.confidence of the oracle's SO4
    volume.  pipelined: the batch as two calls that flow into each other."""
    torch, dev = E.cuda()
    if pairs is None:
        pairs = GS.sweep_pairs(c.W, c.H, c.D, c.seed)[:c.n]
    pairs = [(p[0], p[1], p[2] if len(p) > 2 else None) for p in pairs]
    has_cost = pairs[0][2] is not None
    assert all((p[2] is not None) == has_cost for p in pairs)
    assert volumes or not confidence, "the confidence maps read the optimised volume"
    maps = ["wta_left", "wta_right", "outliers"] + (["min_cost", "peak_ratio"] if confidence else [])
    # the oracle runs overlap in threads (ctypes releases the GIL during the call) while the GPU runs the batch
    with ThreadPoolExecutor(len(pairs)) as ex:
        futs = [ex.submit(_oracle_outputs, c, l, r, v) for l, r, v in pairs]
        d_l = torch.from_numpy(np.stack([p[0] for p in pairs])).to(dev)
        d_r = torch.from_numpy(np.stack([p[1] for p in pairs])).to(dev)
        cost = {}
        if has_cost:
            import cost_testlib as CT
            vols = [v if cost_layout == "hwd" else np.ascontiguousarray(v.transpose(2, 0, 1)) for _, _, v in pairs]
            vols = [CT.to_bf16_bits(v) if cost_dtype == "bf16" else v.astype({"f32": np.float32, "f16": np.float16}[cost_dtype])
                    for v in vols]
            for v, (_, _, v32) in zip(vols, pairs):
                back = (v.astype(np.uint32) << 16).view(np.float32) if cost_dtype == "bf16" else v.astype(np.float32)
                assert np.array_equal(back, v32 if cost_layout == "hwd" else v32.transpose(2, 0, 1)), "volume not exact"
            cost = dict(d_cost=torch.from_numpy(np.stack(vols).view(np.int16) if cost_dtype == "bf16" else np.stack(vols)).to(dev), cost_layout=cost_layout, cost_dtype=cost_dtype)
        eng = E.engine(c.W, c.H, c.opt, wave_pairs=c.wave_pairs, lanes=c.lanes, debug_flags=debug_flags)
        assert (eng.wave_pairs, eng.lanes) == (c.wave_pairs, c.lanes), (eng.wave_pairs, eng.lanes)
        got = E.batch_outputs(eng, eng.match_outputs_batch_device, len(pairs), d_l.data_ptr(), d_r.data_ptr(),
                              3 * c.W * c.H, volumes=[(s, "hwd", "f32") for s in ("cost", "aggr", "opt") if volumes],
                              maps=maps, pipelined=pipelined, **cost)
        if after is not None:
            after(eng)
        eng.close()
        want = [f.result() for f in futs]
    for i, w in enumerate(want):
        tag = f"{c.name} ({c.W}x{c.H}x{c.D}, dmin {c.opt.min_disparity}) pair {i}"
        if volumes:
            E.same(f"{tag} COST/VOL_INIT", got["cost"][i], w["cost"])
            E.same(f"{tag} AGG4/VOL_AGGR", got["aggr"][i], w["aggr"])
            E.same(f"{tag} SO4/VOL_AGGR", got["opt"][i], w["opt"])
        E.same(f"{tag} WTA/DISP_L", got["wta_left"][i], w["wta_left"])
        E.same(f"{tag} WTA/DISP_R", got["wta_right"][i], w["wta_right"])
        assert set(np.unique(got["outliers"][i])) <= {0, 1, 2}, f"{tag} OUTLIER: labels other than 0, 1, 2"
        mis, occ = MT.outlier_lists(got["outliers"][i])
        E.same(f"{tag} OUTLIER/MISMATCHES", mis, w["mismatches"].reshape(-1, 2))
        E.same(f"{tag} OUTLIER/OCCLUSIONS", occ, w["occlusions"].reshape(-1, 2))
        if confidence:
            c1, ratio = MT.confidence(w["opt"])
            E.same(f"{tag} MIN_COST", got["min_cost"][i], c1)
            E.same(f"{tag} PEAK_RATIO", got["peak_ratio"][i], ratio)
        E.same(f"{tag} MEDIAN/DISP_L", got["disp"][i], w["final"])
    return got
