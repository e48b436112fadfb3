"""The batched parity check of the kernel sweep and the option-space cases: a case, the launch plans the kernels take
for it (printed by tests/c/ca_plan_main.cpp and so_plan_main.cpp from the headers the kernels are launched with), the
template instantiations one run of it launches, and the run itself against the oracle."""
from __future__ import annotations

import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

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


def so_lanes_per_line(Dp):
    return 8 if Dp <= 64 else (16 if Dp <= 128 else 32)


A2_TMA, A2_LDG = 1, 0     # the forms arm_sum2_form (ca_plan.h) picks


def reached(c, plans):
    """The instantiations of the seven templates one batched run of case c launches, by the launch rules of
    k_aggregate.cu, k_cost.cu, k_scanline.cu and k_vote.cu (a run that matches, so every stage runs, with the fused
    aggregation):
      cost:      k_cost_arm_sum_h<D == Dp, ca_plan.qc> where ca_plan is ok, else k_cost_volume<D == Dp>;
      axis dir:  k_arm_sum2t<dir, qc> where the TMA plans of both axes are ok and, on rows, the row is one segment; else
                 k_arm_sum2<dir, 8 if Qc == 8 else 0> (generic QC).  This restates arm_sum2_form, and the form the plan
                 executable prints for the axis must agree with it;
      scanline:  k_scanline<ceil(Dp / LPS), LPS, D == K * LPS>, LPS = so_lanes_per_line(Dp);
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
    wide = c.D > 254 or min(c.L1, 255) > 127
    out.add(("k_vote_scan", wide))
    out.add(("k_vote_push", wide))
    return out


# ---- the GPU run ----------------------------------------------------------------------------------------------------
def check_case(c):
    """One match_outputs_batch_device call over the case's pairs, exporting the three volumes (f32, [H][W][D]), the
    WTA maps, the outlier map and the final map, each pair compared bit for bit with its own oracle run; returns every
    output of the call on the host."""
    torch, dev = E.cuda()
    # the oracle runs overlap in threads (ctypes releases the GIL during the call) while the GPU runs the batch
    pairs = GS.sweep_pairs(c.W, c.H, c.D, c.seed)[:c.n]
    with ThreadPoolExecutor(len(pairs)) as ex:
        futs = [ex.submit(E.oracle_outputs, c.W, c.H, c.opt, l, r) for l, r in pairs]
        d_l = torch.from_numpy(np.stack([p[0] for p in pairs])).to(dev)
        d_r = torch.from_numpy(np.stack([p[1] for p in pairs])).to(dev)
        eng = E.engine(c.W, c.H, c.opt, wave_pairs=c.wave_pairs, lanes=c.lanes)
        assert (eng.wave_pairs, eng.lanes) == (c.wave_pairs, c.lanes), (eng.wave_pairs, eng.lanes)
        got = E.batch_outputs(eng, eng.match_outputs_batch_device, len(pairs), d_l.data_ptr(), d_r.data_ptr(),
                              3 * c.W * c.H, volumes=[(s, "hwd", "f32") for s in ("cost", "aggr", "opt")],
                              maps=["wta_left", "wta_right", "outliers"])
        eng.close()
        want = [f.result() for f in futs]
    for i, w in enumerate(want):
        tag = f"{c.name} ({c.W}x{c.H}x{c.D}, dmin {c.opt.min_disparity}) pair {i}"
        E.same(f"{tag} COST/VOL_INIT", got["cost"][i], w["cost"])
        E.same(f"{tag} AGG4/VOL_AGGR", got["aggr"][i], w["aggr"])
        E.same(f"{tag} SO4/VOL_AGGR", got["opt"][i], w["opt"])
        E.same(f"{tag} WTA/DISP_L", got["wta_left"][i], w["wta_left"])
        E.same(f"{tag} WTA/DISP_R", got["wta_right"][i], w["wta_right"])
        mis, occ = MT.outlier_lists(got["outliers"][i])
        E.same(f"{tag} OUTLIER/MISMATCHES", mis, w["mismatches"].reshape(-1, 2))
        E.same(f"{tag} OUTLIER/OCCLUSIONS", occ, w["occlusions"].reshape(-1, 2))
        E.same(f"{tag} MEDIAN/DISP_L", got["disp"][i], w["final"])
    return got
