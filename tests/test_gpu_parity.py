"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle, stage by stage.

Bar (BASELINE.json north_star): bit-exact census / arms / support counts / WTA integer indices;
<= 1e-4 on float costs; <= 0.01 px on sub-pixel disparity.  The kernels are built to be bit-exact
on the float stages too, and these tests assert exact equality there as well (a failure prints the
max abs difference so a tolerance-level deviation can be told from a real bug).
"""
import numpy as np
import pytest

import adc_testlib as T
import engine_testlib as E  # puts tools/ on sys.path

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", E.PARITY_CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}-{i}" for i, c in enumerate(E.PARITY_CASES)])
def test_stage_parity_synthetic(case):
    w, h, D, over, seed = case
    opt = T.default_option(**{"max_disparity": D, **over})
    left, right = T.synthetic_pair(w, h, D, seed)
    orc = T.Oracle(w, h, opt)
    eng = E.engine(w, h, opt)
    orc.begin(left, right)
    for st in T.STAGES:
        orc.step()
        eng.debug_run(left, right, st)
        for tap in T.STAGE_TAPS[st]:
            E.same(f"{st}/{tap}", eng.tap(tap), orc.tap(tap))
    # the public entry point gives the same map as the staged run
    E.same("match", eng.match(left, right), orc.tap("DISP_L"))
    eng.close()


def test_cone_all_stages(cone):
    left, right = cone
    h, w, _ = left.shape
    orc = T.Oracle(w, h)
    eng = E.engine(w, h, T.default_option())
    orc.begin(left, right)
    for st in T.STAGES:
        orc.step()
        eng.debug_run(left, right, st)
        for tap in T.STAGE_TAPS[st]:
            E.same(f"cone {st}/{tap}", eng.tap(tap), orc.tap(tap))
    final = eng.match(left, right)
    E.same("cone match", final, orc.tap("DISP_L"))
    eng.close()


def test_batch_equals_single():
    w, h, D = 96, 64, 32
    opt = T.default_option(max_disparity=D)
    pairs = [T.synthetic_pair(w, h, D, 100 + i) for i in range(11)]
    lefts = np.stack([p[0] for p in pairs])
    rights = np.stack([p[1] for p in pairs])
    eng = E.engine(w, h, opt, wave_pairs=4, lanes=2)
    singles = [eng.match(l, r) for l, r in pairs]
    batch = eng.match_batch(lefts, rights)
    for i in range(len(pairs)):
        E.same(f"batch[{i}]", batch[i], singles[i])
    ptrs = eng.match_batch_ptrs([p[0] for p in pairs], [p[1] for p in pairs])
    for i in range(len(pairs)):
        E.same(f"ptrs[{i}]", ptrs[i], singles[i])
    orc = T.Oracle(w, h, opt)
    E.same("vs oracle", singles[3], orc.match(*pairs[3]))
    eng.close()


def test_error_truth_table():
    """Mirrors ADCensusStereo.cpp:31,38,71,74: bad sizes / empty range / null pointers -> false."""
    import adcensus_b200 as A
    s = A.ADCensusStereo()
    assert s.Match(np.zeros((4, 4, 3), np.uint8), np.zeros((4, 4, 3), np.uint8)) is False  # before Initialize
    assert s.Initialize(0, 10, A.ADCensusOption()) is False
    assert s.Initialize(10, -1, A.ADCensusOption()) is False
    assert s.Initialize(10, 10, A.ADCensusOption(min_disparity=5, max_disparity=5)) is False
    assert s.Initialize(32, 24, A.ADCensusOption(max_disparity=8)) is True
    assert s.Match(None, np.zeros((24, 32, 3), np.uint8)) is False
    out = s.Match(np.zeros((24, 32, 3), np.uint8), np.zeros((24, 32, 3), np.uint8))
    assert out.shape == (24, 32)
    assert s.Reset(40, 30, A.ADCensusOption(max_disparity=16)) is True
    assert s.Match(np.zeros((30, 40, 3), np.uint8), np.zeros((30, 40, 3), np.uint8)).shape == (30, 40)
    s.Release()


def test_golden_cases_on_gpu():
    """The committed golden vectors (produced by the unmodified reference, tools/make_golden.py):
    every tap after every stage must hash to the reference's sha256."""
    import make_golden as G
    for name in ("cone_crop", "synth_a", "synth_b", "synth_opts", "synth_disc"):
        left, right, opt = G.case_inputs(name)
        hashes = E.golden_hashes(name)
        h, w, _ = left.shape
        eng = E.engine(w, h, opt)
        for st in T.STAGES:
            eng.debug_run(left, right, st)
            for tap in T.STAGE_TAPS[st]:
                assert T.sha(eng.tap(tap)) == hashes[f"{st}/{tap}"], f"{name}: {st}/{tap}"
        eng.close()


def test_cone_final_equals_reference_golden(cone):
    left, right = cone
    hashes = E.golden_hashes("cone_full")
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option())
    out = eng.match(left, right)
    assert T.sha(out) == hashes["MEDIAN/DISP_L"] and hashes["MEDIAN/DISP_L"].startswith("77d70a58d1aa5c71")
    # batched + pinned-async entry points give the same bits
    import torch
    n = 20
    hl = torch.from_numpy(np.repeat(left[None], n, 0)).pin_memory()
    hr = torch.from_numpy(np.repeat(right[None], n, 0)).pin_memory()
    hd = torch.empty((n, h, w), dtype=torch.float32).pin_memory()
    eng.match_batch_pinned_async(n, hl.data_ptr(), hr.data_ptr(), hd.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert (hd.numpy().view(np.uint32) == out.view(np.uint32)[None]).all()
    eng.close()


def test_cpp_dropin_program_on_gpu(tmp_path, cone):
    """The reference-style C++ caller (tests/cpp/dropin_main.cpp, written against ADCensusStereo.h as main.cpp uses it)
    runs Match on the Cone pair on the device; the map it writes must hash to the unmodified reference's."""
    import subprocess
    exe = E.c_tool("dropin_main")
    left, right = cone
    h, w, _ = left.shape
    left.tofile(tmp_path / "left.bgr"); right.tofile(tmp_path / "right.bgr")
    run = subprocess.run([str(exe), str(tmp_path / "left.bgr"), str(tmp_path / "right.bgr"), str(w), str(h), "0", "64",
                          str(tmp_path / "disp.f32")], capture_output=True, text=True)
    assert run.returncode == 0 and "DROPIN_OK" in run.stdout, (run.returncode, run.stdout[-500:], run.stderr[-500:])
    assert "cost aggregating! timing" in run.stdout     # the reference's six timing lines are kept
    got = np.fromfile(tmp_path / "disp.f32", np.float32).reshape(h, w)
    hashes = E.golden_hashes("cone_full")
    assert T.sha(got) == hashes["MEDIAN/DISP_L"], "C++ drop-in class produced a different Cone map than the reference"


@pytest.mark.parametrize("flag", ["DBG_VOTE_ENUM", "DBG_VOTE_GLOBAL_STATE", "DBG_NO_RAY_TABLE", "DBG_UNFUSED_AGG"])
def test_alternate_code_paths(flag, cone):
    """Kernels that only unusual parameters reach, forced through adc_config.debug_flags, against the oracle:
    DBG_VOTE_ENUM          the voting kernel finds the histograms a filled pixel belongs to by enumerating the inverse cross
                           region instead of walking precomputed adjacency lists (taken when the lists do not fit);
    DBG_VOTE_GLOBAL_STATE  its per-slot state in global instead of shared memory (more than 32768 pending pixels);
    DBG_NO_RAY_TABLE       interpolation rays evaluated in double per step (image sizes for which the integer ray table is
                           not exact);
    DBG_UNFUSED_AGG        the eight single aggregation passes through the whole pipeline (arms too long for the fused plan).
    The 64x40 pair with D = 255 (2439 pending pixels) takes the voting kernel's WIDE instantiation."""
    import adcensus_b200 as A
    fl = getattr(A.engine, flag)
    cases = [cone + (64,)]
    for (w, h, D, seed) in ((120, 90, 48, 3), (97, 61, 24, 5), (64, 40, 255, 15)):
        l, r = T.synthetic_pair(w, h, D, seed)
        cases.append((l, r, D))
    for left, right, D in cases:
        h, w, _ = left.shape
        opt = T.default_option(max_disparity=D)
        orc = T.Oracle(w, h, opt)
        eng = E.engine(w, h, opt, debug_flags=fl)
        orc.begin(left, right); orc.run_to("VOTE")
        eng.debug_run(left, right, "VOTE")
        c = eng.counters()   # [13] = 1 when the adjacency lists were used (they need room in the idle cost volume,
        #                      which small images with long lists do not have -- Cone does)
        if flag == "DBG_VOTE_ENUM":
            assert c[13] == 0, f"adjacency lists used although enumeration was forced: counters {c}"
        elif (w, h) == (450, 375):
            assert c[13] == 1, f"Cone fell back to enumeration: counters {c}"
        for tap in ("DISP_L", "MISMATCHES", "OCCLUSIONS"):
            E.same(f"{flag} VOTE/{tap}", eng.tap(tap), orc.tap(tap))
        E.same(f"{flag} final", eng.match(left, right), orc.match(left, right))
        eng.close()


def test_pipelined_batches(cone):
    """adc_set_pipelined: three async batch calls in a row without a join in between (different inputs, different output
    buffers, more pairs than one wave), one adc_join at the end; every map must equal the single-pair result."""
    import torch
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option(), wave_pairs=4, lanes=3)
    single = [eng.match(left, right), eng.match(right, left), eng.match(left[:, ::-1].copy(), right[:, ::-1].copy())]
    ins = [(left, right), (right, left), (left[:, ::-1].copy(), right[:, ::-1].copy())]
    n = 10
    st = torch.cuda.current_stream()
    eng.set_pipelined(True)
    outs, keep = [], []
    for l, r in ins:
        dl = torch.from_numpy(np.repeat(l[None], n, 0)).cuda()
        dr = torch.from_numpy(np.repeat(r[None], n, 0)).cuda()
        dd = torch.zeros((n, h, w), dtype=torch.float32, device="cuda")
        keep.append((dl, dr))
        eng.match_batch_device(n, dl.data_ptr(), dr.data_ptr(), dd.data_ptr(), st.cuda_stream)
        outs.append(dd)
    eng.join(st.cuda_stream)
    torch.cuda.synchronize()
    for want, got in zip(single, outs):
        assert (got.cpu().numpy().view(np.uint32) == want.view(np.uint32)[None]).all()
    eng.set_pipelined(False)
    eng.close()


def test_limits_fail_at_create_not_at_match():
    """The reference has no size limits (ADCensusStereo.cpp:31-41 only rejects non-positive sizes); this engine has
    three (include/adcensus_b200.h: ADC_MAX_*).  A size beyond them must make Initialize fail -- never pass Initialize
    and then fail Match -- and the largest accepted height must really run."""
    import adcensus_b200 as A
    s = A.ADCensusStereo()
    assert s.Initialize(64, 4097, A.ADCensusOption(max_disparity=8)) is False and "height" in s.last_error
    assert s.Initialize(64, 48, A.ADCensusOption(max_disparity=257)) is False and "disparity range" in s.last_error
    assert s.Initialize(10001, 8, A.ADCensusOption(max_disparity=8)) is False and "width" in s.last_error
    # a tall image above the old 2048-row limit of the median kernel, against the oracle
    w, h, D = 24, 2100, 8
    opt = T.default_option(max_disparity=D)
    left, right = T.synthetic_pair(w, h, D, 21)
    eng = E.engine(w, h, opt)
    E.same("tall image", eng.match(left, right), T.Oracle(w, h, opt).match(left, right))
    eng.close()


def test_sync_entry_points_join_in_pipelined_mode(cone):
    """adc_set_pipelined only changes the asynchronous entry points: a synchronous batch call on pinned buffers must
    return with its maps complete (round-1 defect: the join was skipped for pinned buffers)."""
    import ctypes
    import adcensus_b200 as A
    left, right = cone
    h, w, _ = left.shape
    eng = E.engine(w, h, T.default_option(), wave_pairs=4, lanes=3)
    want = eng.match(left, right)
    L = A.load_library()
    n = 9
    nb_img, nb_map = n * h * w * 3, n * h * w * 4
    pl, pr, pd = L.adc_host_alloc(nb_img), L.adc_host_alloc(nb_img), L.adc_host_alloc(nb_map)
    assert pl and pr and pd
    al = np.ctypeslib.as_array(ctypes.cast(pl, ctypes.POINTER(ctypes.c_uint8)), (n, h, w, 3))
    ar = np.ctypeslib.as_array(ctypes.cast(pr, ctypes.POINTER(ctypes.c_uint8)), (n, h, w, 3))
    ad = np.ctypeslib.as_array(ctypes.cast(pd, ctypes.POINTER(ctypes.c_float)), (n, h, w))
    al[:], ar[:] = left[None], right[None]
    eng.set_pipelined(True)
    for _ in range(2):
        ad[:] = -1.0
        assert L.adc_match_batch_strided(eng._h, n, pl, pr, pd) == 0
        assert (ad.view(np.uint32) == want.view(np.uint32)[None]).all(), "maps incomplete on return"
    eng.set_pipelined(False)
    eng.close()
    for q in (pl, pr, pd):
        L.adc_host_free(q)


@pytest.mark.parametrize("name", ["cloth3", "wood2", "piano"])
def test_real_pairs_vs_reference_goldens(name):
    """The reference's other bundled Middlebury pairs (Cloth3 view1/view5 at D = 128 is its own usage example,
    main.cpp:30) through every stage, against sha256 hashes produced by the unmodified reference
    (tools/make_golden_big.py): real data at D = 128, 626x555 / 653x555 / 707x481."""
    g = E.golden("golden_big.json")[name]
    z = np.load(T.GOLDEN_DIR / "real_pairs.npz")
    left, right = z[f"{name}_left"], z[f"{name}_right"]
    assert [T.sha(left), T.sha(right)] == g["input_sha"]
    h, w, _ = left.shape
    opt = T.default_option(max_disparity=g["max_disparity"])
    eng = E.engine(w, h, opt)
    for st in T.STAGES:
        eng.debug_run(left, right, st)
        for tap in T.STAGE_TAPS[st]:
            assert T.sha(eng.tap(tap)) == g["hashes"][f"{st}/{tap}"], f"{name}: {st}/{tap}"
    out = eng.match(left, right)
    assert T.sha(out) == g["hashes"]["MEDIAN/DISP_L"]
    E.same(f"{name} final", out, z[f"{name}_final"])
    # the right-view map the reference keeps private (ADCensusStereo.cpp:245-310) through the public entry point
    assert T.sha(eng.right_disparity()) == g["hashes"]["WTA/DISP_R"]
    eng.close()


@pytest.mark.parametrize("name", ["kitti_s1", "kitti_s2", "p1080_s1"])
def test_baseline_configs_vs_reference_goldens(name):
    """BASELINE.json configs 3 and 4 (synthetic 1242x375x128, 1920x1080x192): the aggregated volume, the optimised
    volume, both WTA maps, the outlier lists and the final map against the unmodified reference's hashes
    (one long reference run per 1080p pair, done once by tools/make_golden_big.py)."""
    g = E.golden("golden_big.json")[name]
    w, h, D = g["width"], g["height"], g["max_disparity"]
    seed = int(name.rsplit("_s", 1)[1])
    left, right = T.synthetic_pair(w, h, D, seed)
    assert [T.sha(left), T.sha(right)] == g["input_sha"]
    eng = E.engine(w, h, T.default_option(max_disparity=D))
    out = eng.match(left, right)
    assert T.sha(out) == g["hashes"]["MEDIAN/DISP_L"], f"{name}: final map"
    for st, taps in (("COST", ["CENSUS_L", "VOL_INIT"]), ("ARMS", ["ARMS", "SUPCNT_H", "SUPCNT_V"]), ("AGG2", ["VOL_AGGR"]),
                     ("AGG4", ["VOL_AGGR"]), ("SO4", ["VOL_AGGR"]), ("WTA", ["DISP_L", "DISP_R"]),
                     ("OUTLIER", ["MISMATCHES", "OCCLUSIONS"]), ("VOTE", ["DISP_L"])):
        eng.debug_run(left, right, st)
        for tap in taps:
            assert T.sha(eng.tap(tap)) == g["hashes"][f"{st}/{tap}"], f"{name}: {st}/{tap}"
    batch = eng.match_batch(np.stack([left, left, left]), np.stack([right, right, right]))
    assert (batch.view(np.uint32) == out.view(np.uint32)[None]).all()
    eng.close()


_SHARD_WORKER = r'''
import os
import numpy as np
import torch
import torch.distributed as dist
import adc_testlib as T
import adcensus_b200 as A
from adcensus_b200.parallel import run_sharded_device
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
if world > 1:
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%s" % os.environ["ADC_PORT"], rank=rank, world_size=world, device_id=dev)
w, h, D, n = 96, 64, 32, 11
eng = A.Engine(w, h, A.ADCensusOption(max_disparity=D), device=rank, wave_pairs=2, lanes=2)
d_l = d_r = d_out = None
if rank == 0:
    pairs = [T.synthetic_pair(w, h, D, 200 + i) for i in range(n)]
    d_l = torch.from_numpy(np.stack([p[0] for p in pairs])).to(dev)
    d_r = torch.from_numpy(np.stack([p[1] for p in pairs])).to(dev)
    d_out = torch.zeros((n, h, w), dtype=torch.float32, device=dev)
for _ in range(2):          # twice: buffers and streams are reused
    run_sharded_device(eng, d_l, d_r, d_out, n, h, w, dev)
torch.cuda.synchronize()
if rank == 0:
    out = d_out.cpu().numpy()
    orc = T.Oracle(w, h, T.default_option(max_disparity=D))
    for i in (0, 5, 6, 10):   # both sides of the rank boundary, first and last
        want = orc.match(*pairs[i])
        assert out[i].tobytes() == want.tobytes(), "pair %d differs from the oracle (order or content)" % i
    single = [eng.match(*p) for p in pairs]
    assert all(out[i].tobytes() == single[i].tobytes() for i in range(n))
    print("SHARD_OK")
eng.close()
if world > 1:
    dist.destroy_process_group()
'''


@pytest.mark.parametrize("world", [1, 2])
def test_sharded_batch_real_engine(tmp_path, world):
    """adcensus_b200.parallel.run_sharded_device (BASELINE configs[4] form) with the REAL engine: rank 0 owns the batch,
    NCCL scatter -> Match -> NCCL gather, order and bits against the oracle.  world = 2 needs two GPUs."""
    import os, socket, subprocess, sys
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    script = tmp_path / "worker.py"
    script.write_text(_SHARD_WORKER)
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = str(sk.getsockname()[1])
    procs = []
    for r in range(world):
        path = os.pathsep.join(p for p in (str(T.REPO), str(T.REPO / "tests"), os.environ.get("PYTHONPATH")) if p)
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), ADC_PORT=port, PYTHONPATH=path)
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    outs = [p.communicate(timeout=600) for p in procs]
    for p, (so, se) in zip(procs, outs):
        assert p.returncode == 0, se[-3000:]
    assert "SHARD_OK" in outs[0][0]


def test_loaded_gpu_batch_equals_reference(cone):
    """Every map of a batch that really loads the GPU (default wave size and lane count, several waves in flight, two
    calls back to back) against the reference's sha256.  Single-pair runs leave most SMs idle and hid a shared-memory
    proxy-ordering bug of the scanline ring that corrupted about one pair in four of a full wave."""
    import torch
    left, right = cone
    h, w, _ = left.shape
    want = E.golden_hashes("cone_full")["MEDIAN/DISP_L"]
    eng = E.engine(w, h, T.default_option())
    n = 4 * eng.wave_pairs + 3
    dl = torch.from_numpy(np.repeat(left[None], n, 0)).cuda()
    dr = torch.from_numpy(np.repeat(right[None], n, 0)).cuda()
    dd = torch.zeros((n, h, w), dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream()
    for _ in range(2):
        eng.match_batch_device(n, dl.data_ptr(), dr.data_ptr(), dd.data_ptr(), st.cuda_stream)
    torch.cuda.synchronize()
    out = dd.cpu().numpy()
    bad = [i for i in range(n) if T.sha(out[i]) != want]
    assert not bad, f"{len(bad)} of {n} maps differ from the reference: pairs {bad[:8]}"
    eng.close()
