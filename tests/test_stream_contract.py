"""Stream-order parity: every asynchronous entry point of include/adcensus_b200.h against the oracle or a restatement,
with its inputs produced late and its results consumed early, and engines driven from two threads.

The gate.  On the caller's stream a delay kernel (torch.cuda._sleep) runs first, then the copy of the real inputs into
buffers that held a decoy batch until then.  Right after the call, on the stream that may read the results (the
caller's stream; in pipelined mode a second stream joined with adc_join), every output is snapshot and then the inputs
(and the cost volume) are overwritten with the decoy again.  An entry point that reads its inputs before the gate opens
gives the decoy's results; one whose results are read before they are complete leaves sentinels in the snapshot; one
that still reads its inputs after the consumer overwrote them gives the decoy's results.  Two preconditions keep a pass
from being vacuous: the decoy's expected results differ from the real ones on every pair, and the consumer stream is
still busy right after the snapshot has been enqueued (the gate was still closed when the call returned).

CPU: every function of the header that takes a stream is in the matrix; the expected results and the preconditions;
the two engines of the threaded run share a template instantiation and each reaches one the other does not.
GPU: the matrix -- 11 entry points on the legacy default stream, a torch pool stream and the per-thread default stream,
each as one call joined per call and as two pipelined calls joined once onto another stream; the host entry points
between two un-joined pipelined batches; adc_get_right_disparity after a batch; adc_set_rectification between two
pipelined rectified calls; adc_destroy of one engine while another has un-joined work; two engines on two threads in a
fresh interpreter (tests/stream_contract_worker.py).
"""
import functools
import os
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import pytest

import adc_testlib as T
import cloud_testlib as CL
import cost_testlib as CT
import engine_testlib as E  # puts tools/ on sys.path
import export_testlib as X
import maps_testlib as MT
import rectify_testlib as R
import reproject_testlib as RP
import speckle_testlib as SP
import yuv_testlib as Y

W, H = 72, 48
N_PAIRS, WAVE, LANES = 7, 2, 2           # four waves: both lanes reused, the last wave partial
SRC_W, SRC_H = 80, 56                    # raw frames of the rectified entry
OPTS = {"d24": dict(max_disparity=24), "dneg": dict(min_disparity=-4, max_disparity=20)}
SPECKLE = (30, 0.25)                     # max_size, max_diff of the speckle entry (f32 maps, new_val = +inf)
GATE_MS, GATE_FACTOR = 20.0, 5.0         # the gate lasts at least this long, and this many times the longest call
HEADER = T.REPO / "include" / "adcensus_b200.h"
WORKER = Path(__file__).with_name("stream_contract_worker.py")
KINDS = ("real", "decoy")
STREAMS = ("legacy", "pool", "per_thread")


def option(case):
    return T.default_option(**OPTS[case])


def _q():
    return np.load(T.GOLDEN_DIR / "golden_reproject_cases.npz")["rig_zero_0/Q"]


def _maps(version):
    """Both views' float remap tables of rectification `version` (1 or 2), output W x H from SRC_W x SRC_H frames."""
    return tuple(R.warp_maps(W, H, SRC_W, SRC_H, 10 * version + v) for v in range(2))


# ---- inputs and what they must give (CPU) -----------------------------------------------------------------------------
@functools.cache
def inputs(case, kind):
    """The batch of one kind: packed BGR pairs, their NV12 frames, raw frames for the rectified entry and cost volumes
    (f32 [H][W][D], exact in bf16), each [n][...] per view."""
    o = option(case)
    D = o.max_disparity - o.min_disparity
    base = 100 if kind == "real" else 200
    bgr = [T.synthetic_pair(W, H, D, base + i) for i in range(N_PAIRS)]
    raw = [T.synthetic_pair(SRC_W, SRC_H, D, base + 50 + i) for i in range(N_PAIRS)]
    return {
        "bgr": tuple(np.stack([p[v] for p in bgr]) for v in range(2)),
        "nv12": tuple(np.stack([Y.encode(p[v], "nv12") for p in bgr]) for v in range(2)),
        "raw": tuple(np.stack([p[v] for p in raw]) for v in range(2)),
        "cost": np.stack([CT.synthetic_cost(W, H, D, base + i, o.min_disparity) for i in range(N_PAIRS)]),
    }


def _cost_final(case, l, r, c):
    return CT.CostOracle(W, H, option(case)).match_cost(l, r, c)


@functools.cache
def expected(case, kind):
    """Oracle runs of the batch of one kind: "bgr" (every output of oracle_outputs), "nv12" (the final maps of the
    decoded frames, and the decoded views), "rect1" / "rect2" (the final maps of the raw frames through rectification
    1 / 2), "cost" (the final maps of the cost volumes)."""
    x = inputs(case, kind)
    o = option(case)
    l, r = x["bgr"]
    dec = [tuple(Y.decode(x["nv12"][v][i], "nv12", W, H) for v in range(2)) for i in range(N_PAIRS)]
    rect = {k: [tuple(R.remap(x["raw"][v][i], *_maps(k)[v]) for v in range(2)) for i in range(N_PAIRS)] for k in (1, 2)}
    with ThreadPoolExecutor(8) as ex:
        bgr = [ex.submit(E.oracle_outputs, W, H, o, l[i], r[i]) for i in range(N_PAIRS)]
        nv12 = [ex.submit(E.oracle_outputs, W, H, o, *dec[i]) for i in range(N_PAIRS)]
        rc = {k: [ex.submit(E.oracle_outputs, W, H, o, *rect[k][i]) for i in range(N_PAIRS)] for k in (1, 2)}
        cost = [ex.submit(_cost_final, case, l[i], r[i], x["cost"][i]) for i in range(N_PAIRS)]
        out = {"bgr": [f.result() for f in bgr], "nv12": np.stack([f.result()["final"] for f in nv12]),
               "views": np.stack([np.stack(d) for d in dec]), "cost": np.stack([f.result() for f in cost])}
        for k in (1, 2):
            out[f"rect{k}"] = np.stack([f.result()["final"] for f in rc[k]])
    return out


def finals(case, kind):
    return np.stack([w["final"] for w in expected(case, kind)["bgr"]])


@functools.cache
def disparity_maps(case, kind):
    """The maps the reprojection, speckle and cloud entries read: the final maps with a few invalid (+inf) pixels and
    small blobs lifted by 7.5, which the speckle filter removes."""
    rng = np.random.default_rng(1 if kind == "real" else 2)
    out = finals(case, kind).copy()
    for m in out:
        m[rng.random(m.shape) < 0.03] = np.inf
        for y, x in zip(rng.integers(0, H - 2, 12), rng.integers(0, W - 2, 12)):
            m[y:y + 2, x:x + 2] += np.float32(7.5)
    return out


def _speckled(case, kind):
    return np.stack([SP.filter_f32(m, np.inf, *SPECKLE) for m in disparity_maps(case, kind)])


# ---- the entry points ---------------------------------------------------------------------------------------------------
def _same_nan(tag, got, want):
    assert RP.same_nan(got, want), f"{tag}: differs (NaN-insensitive)"


def _same_outliers(tag, got, want):
    mis, occ = MT.outlier_lists(got)
    E.same(f"{tag} mismatches", mis, want[0])
    E.same(f"{tag} occlusions", occ, want[1])


class Entry:
    """One asynchronous entry point set up over the batch: inputs behind the gate, outputs that start as sentinels
    (guarded by sentinel elements on both sides on the device), the call over pairs [first, first + count) and what
    every output must hold for the real and for the decoy batch."""

    def __init__(self, name, case, caller_stream=False, **cfg):
        self.name, self.case = name, case
        self.eng = E.engine(W, H, option(case), wave_pairs=WAVE, lanes=LANES, **cfg)
        self.caller_stream = caller_stream   # enqueued on the caller's stream, not on the engine's lanes
        self.gated = []     # (buffer, real, decoy)
        self.outs = {}      # name: (buffer, sentinel or None for an in-place buffer, guard check or None)
        self.cmp = {}       # name: comparison (default E.same)
        self.issue = None   # (first, count, stream handle) -> None
        self.want = None    # kind -> {name: per-pair expected values}

    def gate_in(self, real, decoy, pinned=False):
        torch, dev = E.cuda()
        r = torch.from_numpy(np.ascontiguousarray(real)).to(dev)
        d = torch.from_numpy(np.ascontiguousarray(decoy)).to(dev)
        buf = torch.empty(r.shape, dtype=r.dtype, pin_memory=True) if pinned else torch.empty_like(r)
        self.gated.append((buf, r, d))
        return buf

    def out(self, name, shape, dtype, sentinel, pinned=False):
        torch, _ = E.cuda()
        if pinned:
            buf, intact = torch.empty(shape, dtype=dtype, pin_memory=True), None
        else:
            flat, intact = E.guarded(int(np.prod(shape)), dtype, 64, 64, sentinel)
            buf = flat.view(shape)
        self.outs[name] = (buf, sentinel, intact)
        return buf

    def in_place(self, name, buf):
        self.outs[name] = (buf, None, None)

    def close(self):
        E.cuda()[0].cuda.synchronize()
        self.eng.close()


def _bgr_views(e, kind_key="bgr", pinned=False):
    (rl, rr), (dl, dr) = inputs(e.case, "real")[kind_key], inputs(e.case, "decoy")[kind_key]
    return e.gate_in(rl, dl, pinned), e.gate_in(rr, dr, pinned)


def _final_want(e, key="bgr"):
    if key == "bgr":
        return lambda kind: {"disp": finals(e.case, kind)}
    return lambda kind: {"disp": expected(e.case, kind)[key]}


def b_match(case):
    torch, _ = E.cuda()
    e = Entry("adc_match_batch_device", case)
    L, Rv = _bgr_views(e)
    d = e.out("disp", (N_PAIRS, H, W), torch.float32, -7.0)
    e.issue = lambda f, c, st: e.eng.match_batch_device(c, L[f:].data_ptr(), Rv[f:].data_ptr(), d[f:].data_ptr(), st)
    e.want = _final_want(e)
    return e


def b_pinned(case):
    torch, _ = E.cuda()
    e = Entry("adc_match_batch_pinned_async", case)
    L, Rv = _bgr_views(e, pinned=True)       # filled by a device-to-host copy behind the gate
    d = e.out("disp", (N_PAIRS, H, W), torch.float32, -7.0, pinned=True)
    e.issue = lambda f, c, st: e.eng.match_batch_pinned_async(c, L[f:].data_ptr(), Rv[f:].data_ptr(), d[f:].data_ptr(), st)
    e.want = _final_want(e)
    return e


def b_cost(case):
    torch, _ = E.cuda()
    e = Entry("adc_match_cost_batch_device", case)
    L, Rv = _bgr_views(e)
    bits = {k: CT.to_bf16_bits(inputs(case, k)["cost"].transpose(0, 3, 1, 2)).view(np.int16) for k in KINDS}
    C = e.gate_in(bits["real"], bits["decoy"])
    d = e.out("disp", (N_PAIRS, H, W), torch.float32, -7.0)
    e.issue = lambda f, c, st: e.eng.match_cost_batch_device(c, L[f:].data_ptr(), Rv[f:].data_ptr(), C[f:].data_ptr(),
                                                             d[f:].data_ptr(), "dhw", "bf16", st)
    e.want = _final_want(e, "cost")
    return e


def b_volumes(case):
    torch, _ = E.cuda()
    e = Entry("adc_match_volumes_batch_device", case)
    L, Rv = _bgr_views(e)
    D = e.eng.D
    d = e.out("disp", (N_PAIRS, H, W), torch.float32, -7.0)
    cost = e.out("cost", (N_PAIRS, D, H, W), torch.int16, -1)            # bf16 bits, sentinel NaN
    opt = e.out("opt", (N_PAIRS, H, W, D), torch.float32, float("nan"))
    e.issue = lambda f, c, st: e.eng.match_volumes_batch_device(
        c, L[f:].data_ptr(), Rv[f:].data_ptr(), [(cost[f:].data_ptr(), "cost", "dhw", "bf16"),
                                                 (opt[f:].data_ptr(), "opt", "hwd", "f32")], d[f:].data_ptr(), stream=st)
    e.want = lambda kind: {"disp": finals(case, kind),
                           "cost": [X.export_of(w["cost"], "dhw", "bf16").view(np.int16) for w in expected(case, kind)["bgr"]],
                           "opt": [w["opt"] for w in expected(case, kind)["bgr"]]}
    return e


def b_outputs(case):
    torch, _ = E.cuda()
    e = Entry("adc_match_outputs_batch_device", case)
    L, Rv = _bgr_views(e)
    D = e.eng.D
    d = e.out("disp", (N_PAIRS, H, W), torch.float32, -7.0)
    maps = {m: e.out(m, (N_PAIRS, H, W), torch.float32, -7.0) for m in ("wta_left", "wta_right")}
    maps["outliers"] = e.out("outliers", (N_PAIRS, H, W), torch.uint8, 0xee)
    aggr = e.out("aggr", (N_PAIRS, H, W, D), torch.float32, float("nan"))
    e.cmp["outliers"] = _same_outliers
    e.issue = lambda f, c, st: e.eng.match_outputs_batch_device(
        c, L[f:].data_ptr(), Rv[f:].data_ptr(), maps=[(t[f:].data_ptr(), m) for m, t in maps.items()],
        volumes=[(aggr[f:].data_ptr(), "aggr", "hwd", "f32")], d_disp=d[f:].data_ptr(), stream=st)
    e.want = lambda kind: {"disp": finals(case, kind),
                           "wta_left": [w["wta_left"] for w in expected(case, kind)["bgr"]],
                           "wta_right": [w["wta_right"] for w in expected(case, kind)["bgr"]],
                           "outliers": [(w["mismatches"].reshape(-1, 2), w["occlusions"].reshape(-1, 2))
                                        for w in expected(case, kind)["bgr"]],
                           "aggr": [w["aggr"] for w in expected(case, kind)["bgr"]]}
    return e


def b_images(case):
    import adcensus_b200 as A
    torch, _ = E.cuda()
    e = Entry("adc_match_images_batch_device", case)
    L, Rv = _bgr_views(e, "nv12")
    d = e.out("disp", (N_PAIRS, H, W), torch.float32, -7.0)
    desc = A.image_desc("nv12")
    e.issue = lambda f, c, st: e.eng.match_images_batch_device(c, L[f:].data_ptr(), Rv[f:].data_ptr(), image=desc,
                                                               d_disp=d[f:].data_ptr(), stream=st)
    e.want = _final_want(e, "nv12")
    return e


def b_rectified(case):
    torch, _ = E.cuda()
    e = Entry("adc_match_rectified_batch_device", case)
    e.eng.set_rectification(*_maps(1), src_size=(SRC_W, SRC_H))
    L, Rv = _bgr_views(e, "raw")
    d = e.out("disp", (N_PAIRS, H, W), torch.float32, -7.0)
    e.issue = lambda f, c, st: e.eng.match_rectified_batch_device(c, L[f:].data_ptr(), Rv[f:].data_ptr(),
                                                                  d_disp=d[f:].data_ptr(), stream=st)
    e.want = _final_want(e, "rect1")
    return e


def b_reproject(case):
    torch, _ = E.cuda()
    e = Entry("adc_reproject_batch_device", case, caller_stream=True)
    M = e.gate_in(disparity_maps(case, "real"), disparity_maps(case, "decoy"))
    pts = e.out("points", (N_PAIRS, H, W, 3), torch.float32, -7.0)
    dep = e.out("depth", (N_PAIRS, H, W), torch.float32, -7.0)
    s16 = e.out("disp_s16", (N_PAIRS, H, W), torch.int16, 0x5a5a)
    Q = _q()
    e.cmp.update(points=_same_nan, depth=_same_nan)
    e.issue = lambda f, c, st: e.eng.reproject_batch_device(
        c, M[f:].data_ptr(), Q, [(pts[f:].data_ptr(), "points"), (dep[f:].data_ptr(), "depth"),
                                 (s16[f:].data_ptr(), "disp_s16")], st)
    dmin = option(case).min_disparity
    e.want = lambda kind: {"points": [RP.points(m, Q) for m in disparity_maps(case, kind)],
                           "depth": [RP.depth(m, Q) for m in disparity_maps(case, kind)],
                           "disp_s16": [RP.disp_s16(m, dmin) for m in disparity_maps(case, kind)]}
    return e


def b_speckles(case):
    torch, dev = E.cuda()
    e = Entry("adc_filter_speckles_batch_device", case, caller_stream=True)
    M = e.gate_in(disparity_maps(case, "real"), disparity_maps(case, "decoy"))
    e.in_place("maps", M)
    wb = e.eng.speckle_workspace_bytes(N_PAIRS)
    work = torch.empty(wb, dtype=torch.uint8, device=dev)
    e.issue = lambda f, c, st: e.eng.filter_speckles_batch_device(c, M[f:].data_ptr(), "f32", *SPECKLE, None,
                                                                  work.data_ptr(), wb, st)
    e.want = lambda kind: {"maps": _speckled(case, kind)}
    return e


def b_ingest(case):
    import adcensus_b200 as A
    torch, _ = E.cuda()
    e = Entry("adc_ingest_views_batch_device", case, caller_stream=True)
    L, Rv = _bgr_views(e, "nv12")
    v = e.out("views", (N_PAIRS, 2, H, W, 3), torch.uint8, 0x5a)
    desc = A.image_desc("nv12")
    e.issue = lambda f, c, st: e.eng.ingest_views_batch_device(c, L[f:].data_ptr(), Rv[f:].data_ptr(), v[f:].data_ptr(),
                                                               image=desc, stream=st)
    e.want = lambda kind: {"views": expected(case, kind)["views"]}
    return e


def b_cloud(case):
    torch, dev = E.cuda()
    e = Entry("adc_point_cloud_batch_device", case, caller_stream=True)
    M = e.gate_in(disparity_maps(case, "real"), disparity_maps(case, "decoy"))
    B = e.gate_in(inputs(case, "real")["bgr"][0], inputs(case, "decoy")["bgr"][0])
    cap = H * W
    pts = e.out("points", (N_PAIRS, cap, 3), torch.float32, -7.0)
    col = e.out("colors", (N_PAIRS, cap, 3), torch.uint8, 0x5a)
    pix = e.out("pixels", (N_PAIRS, cap), torch.int32, -7)
    cnt = e.out("counts", (N_PAIRS,), torch.int32, -7)
    wb = e.eng.point_cloud_workspace_bytes(N_PAIRS)
    work = torch.empty((wb + 7) // 8, dtype=torch.int64, device=dev)
    Q = _q()
    e.issue = lambda f, c, st: e.eng.point_cloud_batch_device(
        c, M[f:].data_ptr(), Q, pts[f:].data_ptr(), cnt[f:].data_ptr(), cap, work.data_ptr(), wb, d_bgr=B[f:].data_ptr(),
        d_colors=col[f:].data_ptr(), d_pixels=pix[f:].data_ptr(), stream=st)

    def want(kind):
        clouds = [CL.cloud(m, Q, b) for m, b in zip(disparity_maps(case, kind), inputs(case, kind)["bgr"][0])]
        return {"counts": np.array([len(c[2]) for c in clouds], np.int32),
                "points": [c[0] for c in clouds], "colors": [c[1] for c in clouds], "pixels": [c[2] for c in clouds]}

    def prefix(tag, got, want):   # the first count entries; nothing past them is specified
        E.same(tag, got[:len(want)], want)

    e.cmp.update(points=prefix, colors=prefix, pixels=prefix)
    e.want = want
    return e


BUILDERS = {"adc_match_batch_device": b_match, "adc_match_batch_pinned_async": b_pinned,
            "adc_match_cost_batch_device": b_cost, "adc_match_volumes_batch_device": b_volumes,
            "adc_match_outputs_batch_device": b_outputs, "adc_match_images_batch_device": b_images,
            "adc_match_rectified_batch_device": b_rectified, "adc_reproject_batch_device": b_reproject,
            "adc_filter_speckles_batch_device": b_speckles, "adc_ingest_views_batch_device": b_ingest,
            "adc_point_cloud_batch_device": b_cloud}
# functions that take a stream but only make it wait (no input to read, no output to write)
JOIN_ONLY = {"adc_join"}
MATRIX = [(name, "d24") for name in BUILDERS] + [("adc_match_batch_device", "dneg"),
                                                 ("adc_match_outputs_batch_device", "dneg")]


def _differs(a, b):
    if isinstance(a, tuple):
        return any(_differs(x, y) for x, y in zip(a, b))
    a, b = np.asarray(a), np.asarray(b)
    return a.shape != b.shape or not np.array_equal(E.bits(a), E.bits(b))


def check_outputs(e, got, kind="real"):
    """Every output of every pair against the expected values of the batch of one kind."""
    want = e.want(kind)
    for name, w in want.items():
        cmp = e.cmp.get(name, E.same)
        if name == "counts":
            E.same(f"{e.name} counts", got[name], w)
            continue
        for i in range(N_PAIRS):
            cmp(f"{e.name} {name} pair {i}", got[name][i], w[i])


# ---- CPU --------------------------------------------------------------------------------------------------------------
def stream_functions():
    """The functions of the header with a `void* stream` parameter."""
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    return {m.group(1) for m in re.finditer(r"\bint\s+(adc_\w+)\s*\(([^;{]*?)\)\s*;", text)
            if re.search(r"\bvoid\s*\*\s*stream\b", m.group(2))}


def test_every_stream_entry_point_is_in_the_matrix():
    """A function of the header that takes a stream and is not in the matrix (nor adc_join, which the pipelined legs
    use) would be an asynchronous entry point whose ordering nothing checks."""
    fns = stream_functions()
    assert len(fns) >= 12 and "adc_match_batch_device" in fns and "adc_join" in fns, sorted(fns)
    assert fns - JOIN_ONLY == set(BUILDERS), (sorted(fns - JOIN_ONLY - set(BUILDERS)), sorted(set(BUILDERS) - fns))
    assert {name for name, _ in MATRIX} == set(BUILDERS)


@pytest.mark.parametrize("case", sorted(OPTS))
def test_decoy_differs_on_every_pair(case):
    """The preconditions the matrix relies on, on the CPU: for every entry point, the decoy batch's expected primary
    output differs from the real batch's on every pair; the speckle filter changes every real map (so that filtering
    the decoy, or not filtering at all, shows); and the maps the reprojection and the cloud read hold invalid pixels."""
    for key in ("nv12", "rect1", "rect2", "cost"):
        a, b = expected(case, "real")[key], expected(case, "decoy")[key]
        assert all(_differs(a[i], b[i]) for i in range(N_PAIRS)), key
    fr, fd = finals(case, "real"), finals(case, "decoy")
    assert all(_differs(fr[i], fd[i]) for i in range(N_PAIRS))
    fr, fd = disparity_maps(case, "real"), disparity_maps(case, "decoy")
    assert all(_differs(expected(case, "real")["rect1"][i], expected(case, "real")["rect2"][i]) for i in range(N_PAIRS))
    sr, sd = _speckled(case, "real"), _speckled(case, "decoy")
    assert all(_differs(sr[i], sd[i]) and _differs(sr[i], fr[i]) for i in range(N_PAIRS))
    assert np.isinf(fr).any()
    q = _q()
    for i in range(N_PAIRS):
        cr, cd = CL.cloud(fr[i], q), CL.cloud(fd[i], q)
        assert _differs(cr[0], cd[0]) and _differs(cr[2], cd[2]), i


def test_worker_engines_share_and_differ_in_instantiations():
    """The two engines of the threaded run launch at least one template instantiation in common (whose first launch
    the two threads race for) and each at least one the other does not."""
    import sweep_testlib as ST
    import stream_contract_worker as WK
    plans = ST.Plans()
    got = [ST.reached(ST.Case(f"thread {k}", w, h, T.default_option(**o), 0), plans)
           for k, (w, h, o) in enumerate(WK.SHAPES)]
    assert got[0] & got[1] and got[0] - got[1] and got[1] - got[0], got


# ---- GPU: the harness ----------------------------------------------------------------------------------------------------
def stream_of(kind):
    """A torch stream of the kind: the legacy default stream (handle 0), a pool stream (non-blocking), or the
    per-thread default stream (handle 2, cudaStreamPerThread) as an external stream."""
    torch, _ = E.cuda()
    if kind == "legacy":
        s = torch.cuda.default_stream()
        if s.cuda_stream != 0:
            pytest.skip(f"torch's default stream is not the legacy default stream (handle {s.cuda_stream})")
        return s
    if kind == "pool":
        return torch.cuda.Stream()
    try:
        return torch.cuda.ExternalStream(2)
    except Exception as ex:   # noqa: BLE001 -- torch decides whether it takes the handle
        pytest.skip(f"torch does not accept the per-thread default stream as an external stream: {ex}")


def _elapsed_ms(stream, fn):
    torch, _ = E.cuda()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        a.record()
        fn()
        b.record()
    b.synchronize()
    return a.elapsed_time(b)


@pytest.fixture(scope="module")
def gate():
    """Cycles of the delay kernel, calibrated once: the gate lasts at least GATE_FACTOR times the longest ungated call
    of the matrix (one call over the whole batch, per-call join, measured with CUDA events after one warm-up call) and
    at least GATE_MS."""
    torch, _ = E.cuda()
    s = torch.cuda.Stream()
    calls = {}
    for name in BUILDERS:
        e = BUILDERS[name]("d24")
        for buf, real, _ in e.gated:
            buf.copy_(real)
        torch.cuda.synchronize()
        for _ in range(2):
            calls[name] = _elapsed_ms(s, lambda: e.issue(0, N_PAIRS, s.cuda_stream))
        e.close()
    probe = 1 << 24
    _elapsed_ms(s, lambda: torch.cuda._sleep(probe))
    per_ms = probe / _elapsed_ms(s, lambda: torch.cuda._sleep(probe))
    target = max(GATE_MS, GATE_FACTOR * max(calls.values()))
    cycles = int(per_ms * target * 1.25)
    gate_ms = _elapsed_ms(s, lambda: torch.cuda._sleep(cycles))
    print(f"\nstream contract: ungated calls (ms) " + ", ".join(f"{k} {v:.2f}" for k, v in calls.items()) +
          f"; gate {cycles} cycles = {gate_ms:.1f} ms")
    assert gate_ms >= target, (gate_ms, target)
    return cycles


def run_gated(e, stream, pipelined, cycles, between=None, expect_busy=True):
    """One gated run of entry e on `stream`: inputs reset to the decoy and outputs to their sentinels; then on the
    stream the gate and the real inputs, the batch as one call (plain) or two pipelined calls joined with adc_join onto
    a second stream; on the consumer stream the snapshots and the decoy written back over the inputs.  `between`
    (optional) runs on the host after the calls, before the join; expect_busy=False when it synchronises with the
    gate, so that the consumer may find the work done.  Returns every output as the consumer saw it
    (pinned outputs read on the host after the consumer stream's synchronisation)."""
    torch, _ = E.cuda()
    torch.cuda.synchronize()
    for buf, _, decoy in e.gated:
        buf.copy_(decoy)
    for buf, sentinel, _ in e.outs.values():
        if sentinel is not None:
            buf.fill_(sentinel)
    snaps = {name: torch.empty(buf.shape, dtype=buf.dtype, device="cuda") for name, (buf, _, _) in e.outs.items()}
    consumer = torch.cuda.Stream() if pipelined else stream
    torch.cuda.synchronize()
    e.eng.set_pipelined(pipelined)
    half = N_PAIRS // 2 if pipelined else N_PAIRS
    with torch.cuda.stream(stream):
        torch.cuda._sleep(cycles)
        for buf, real, _ in e.gated:
            buf.copy_(real, non_blocking=True)
        for first, count in ((0, half), (half, N_PAIRS - half)):
            if count:
                e.issue(first, count, stream.cuda_stream)
    if between is not None:
        between()
    if pipelined:
        e.eng.join(consumer.cuda_stream)
        if e.caller_stream:   # the entry's work is on the caller's stream: a consumer elsewhere waits for that
            consumer.wait_stream(stream)
    with torch.cuda.stream(consumer):
        for name, (buf, _, _) in e.outs.items():
            snaps[name].copy_(buf, non_blocking=True)
        busy = not consumer.query()
        for buf, _, decoy in e.gated:
            buf.copy_(decoy, non_blocking=True)
    consumer.synchronize()
    pinned = {name: buf.numpy().copy() for name, (buf, _, _) in e.outs.items() if not buf.is_cuda}
    e.eng.set_pipelined(False)
    got = {name: (t.view(torch.int16) if t.dtype == torch.bfloat16 else t).cpu().numpy() for name, t in snaps.items()}
    torch.cuda.synchronize()
    assert busy or not expect_busy, "the consumer stream had finished right after the snapshot was enqueued: the gate did not hold"
    for name, (_, _, intact) in e.outs.items():
        assert intact is None or intact(), f"{e.name}: a guard element of {name} was overwritten"
    return got, pinned


# ---- GPU: the matrix ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "pipelined"])
@pytest.mark.parametrize("stream_kind", STREAMS)
@pytest.mark.parametrize("entry,case", MATRIX)
def test_stream_order(entry, case, stream_kind, mode, gate):
    """Inputs written behind the gate on the caller's stream, outputs snapshot right after the call (plain: on the
    caller's stream after the per-call join; pipelined: two calls, adc_join onto a second stream, snapshot there), the
    inputs overwritten with the decoy right after: every output of every pair equals the expected result of the real
    inputs, bit for bit, and the host reads the same from pinned outputs after the consumer stream's synchronisation."""
    s = stream_of(stream_kind)
    e = BUILDERS[entry](case)
    try:
        got, pinned = run_gated(e, s, mode == "pipelined", gate)
        check_outputs(e, got)
        if pinned:
            check_outputs(e, pinned)
    finally:
        e.close()


# ---- GPU: host calls and asynchronous calls on one engine ------------------------------------------------------------
@pytest.mark.gpu
def test_right_map_is_the_last_host_match(gate):
    """adc_match(A), then an un-joined pipelined batch of other pairs, then adc_get_right_disparity: the right-view map
    of A (the oracle's WTA/DISP_R), not that of the batch's first pair, which the batch's first wave computes into the
    same lane."""
    torch, _ = E.cuda()
    e = b_match("d24")
    try:
        dl, dr = inputs("d24", "decoy")["bgr"]
        want = expected("d24", "decoy")["bgr"][0]
        E.same("adc_match", e.eng.match(dl[0], dr[0]), want["final"])
        right = {}
        got, _ = run_gated(e, torch.cuda.Stream(), True, gate, between=lambda: right.setdefault("r", e.eng.right_disparity()), expect_busy=False)
        E.same("right map after a pipelined batch", right["r"], want["wta_right"])
        check_outputs(e, got)
        E.same("right map after the join", e.eng.right_disparity(), want["wta_right"])
    finally:
        e.close()


def _host_calls(eng, case):
    """name -> (call, check) of the host entry points: each call takes pair 0 of the decoy batch (or its final map)."""
    l, r = (v[0] for v in inputs(case, "decoy")["bgr"])
    w = expected(case, "decoy")["bgr"][0]
    m = disparity_maps(case, "decoy")[0]
    Q = _q()
    nl, nr = (v[0] for v in inputs(case, "decoy")["nv12"])

    def volumes():
        disp, vols = eng.match_volumes(l, r, ["cost", "aggr", "opt"])
        E.same("match_volumes disp", disp, w["final"])
        for s in ("cost", "aggr", "opt"):
            E.same(f"match_volumes {s}", vols[s], w[s])

    def outputs():
        disp, out = eng.match_outputs(l, r, maps=["wta_left", "wta_right", "outliers"], volumes=["opt"])
        E.same("match_outputs disp", disp, w["final"])
        E.same("match_outputs wta_left", out["wta_left"], w["wta_left"])
        E.same("match_outputs wta_right", out["wta_right"], w["wta_right"])
        _same_outliers("match_outputs outliers", out["outliers"], (w["mismatches"].reshape(-1, 2),
                                                                   w["occlusions"].reshape(-1, 2)))
        E.same("match_outputs opt", out["opt"], w["opt"])

    def reproject():
        out = eng.reproject(m, Q, ("points", "depth", "disp_s16"))
        _same_nan("reproject points", out["points"], RP.points(m, Q))
        _same_nan("reproject depth", out["depth"], RP.depth(m, Q))
        E.same("reproject disp_s16", out["disp_s16"], RP.disp_s16(m, option(case).min_disparity))

    def cloud():
        pts, cols, pix = eng.point_cloud(m, Q, l, pixels=True)
        want = CL.cloud(m, Q, l)
        E.same("point_cloud points", pts, want[0])
        E.same("point_cloud colors", cols, want[1])
        E.same("point_cloud pixels", pix, want[2])

    return {
        "match": lambda: (E.same("adc_match", eng.match(l, r), w["final"]),
                          E.same("adc_match right map", eng.right_disparity(), w["wta_right"])),
        "match_volumes": volumes,
        "match_outputs": outputs,
        "reproject": reproject,
        "filter_speckles": lambda: E.same("filter_speckles", eng.filter_speckles(m, *SPECKLE),
                                          SP.filter_f32(m, np.inf, *SPECKLE)),
        "point_cloud": cloud,
        "ingest_views": lambda: E.same("ingest_views", eng.ingest_views(nl, nr, "nv12"),
                                       expected(case, "decoy")["views"][0]),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("host", ["match", "match_volumes", "match_outputs", "reproject", "filter_speckles",
                                  "point_cloud", "ingest_views"])
def test_host_call_between_pipelined_batches(host, gate):
    """A host entry point between the two un-joined calls of a gated pipelined batch, after a smaller host call, so
    that the device staging grows (is freed and allocated again) while the batch is in flight: the host call matches
    its reference, and both calls of the batch match the oracle after the join."""
    torch, _ = E.cuda()
    e = b_outputs("d24")
    try:
        m = disparity_maps("d24", "decoy")[0]
        e.eng.reproject(m, _q(), "disp_s16")          # the smallest staging of the host entries
        calls = _host_calls(e.eng, "d24")
        issue = e.issue
        state = {"calls": 0}

        def issue_then_host(first, count, st):
            issue(first, count, st)
            state["calls"] += 1
            if state["calls"] == 1:
                calls[host]()

        e.issue = issue_then_host
        got, _ = run_gated(e, torch.cuda.Stream(), True, gate, expect_busy=False)
        assert state["calls"] == 2
        check_outputs(e, got)
    finally:
        e.close()


@pytest.mark.gpu
def test_rectification_changes_between_pipelined_calls(gate):
    """adc_set_rectification between two un-joined pipelined rectified calls of a gated batch: the first call's pairs
    match the oracle under the old maps, the second call's under the new ones."""
    torch, _ = E.cuda()
    e = b_rectified("d24")
    try:
        issue = e.issue
        state = {"calls": 0}

        def issue_then_swap(first, count, st):
            issue(first, count, st)
            state["calls"] += 1
            if state["calls"] == 1:
                e.eng.set_rectification(*_maps(2), src_size=(SRC_W, SRC_H))

        e.issue = issue_then_swap
        got, _ = run_gated(e, torch.cuda.Stream(), True, gate, expect_busy=False)
        half = N_PAIRS // 2
        for i in range(N_PAIRS):
            E.same(f"pair {i}", got["disp"][i], expected("d24", "real")["rect1" if i < half else "rect2"][i])
    finally:
        e.close()


@pytest.mark.gpu
def test_destroy_other_engine_during_pipelined_work(gate):
    """adc_destroy of engine A while engine B has un-joined pipelined work behind the gate: B's results are intact."""
    torch, _ = E.cuda()
    e = b_outputs("d24")
    other = E.engine(W, H, option("d24"), wave_pairs=WAVE, lanes=LANES)
    try:
        l, r = (v[0] for v in inputs("d24", "decoy")["bgr"])
        other.match(l, r)
        got, _ = run_gated(e, torch.cuda.Stream(), True, gate, between=other.close, expect_busy=False)
        check_outputs(e, got)
    finally:
        other.close()
        e.close()


# ---- GPU: two engines on two threads --------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_engines_on_two_threads(gate):
    """Two engines on two threads of a fresh interpreter (no kernel launched before, so the first launches of the
    instantiations both shapes reach really race), each on its own stream with three gated batch calls, plain and
    pipelined alternating, against the oracle; one thread makes an argument error while the other has a call in
    flight and has made its own, and each reads its own adc_last_error."""
    path = os.pathsep.join(p for p in (str(T.REPO), str(T.REPO / "tests"), os.environ.get("PYTHONPATH")) if p)
    r = subprocess.run([sys.executable, str(WORKER), str(gate)], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, PYTHONPATH=path))
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    assert "STREAM_WORKER_OK" in r.stdout, r.stdout[-3000:]
