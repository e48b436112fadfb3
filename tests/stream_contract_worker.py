"""Two engines on two threads, in an interpreter of their own (run by tests/test_stream_contract.py with the gate's delay
in cycles as its argument): no kernel has been launched in the process before, so the two threads' first launches of the
template instantiations both shapes reach race for the one-time kernel set-up.

Each thread owns an engine, a stream and a second stream for pipelined joins, and makes CALLS gated batch calls
(plain and pipelined alternating): on its stream the decoy and sentinels, a delay kernel, the real inputs, the call;
then on the consumer stream a snapshot of the maps and the decoy written back over the inputs.  The maps must equal the
oracle's, computed before the threads start.  During the first pipelined call, with both threads' work in flight,
thread 1 makes an argument error (n = -1), thread 0 then makes another, and each must read its own adc_last_error.
Prints STREAM_WORKER_OK, or the failures and exits 1.
"""
import sys
import threading

import numpy as np

# (W, H, option overrides) of the two engines: both reach k_vote_scan<false>, only the first an exact scanline
# instantiation (D = 24 = 3 * 8) and only the second a padded one (D = 37)
SHAPES = [(72, 48, dict(max_disparity=24)), (64, 40, dict(max_disparity=37))]
N_PAIRS, WAVE, LANES, CALLS = 5, 2, 2, 3
WAIT_S = 120


def expected():
    """Per engine: (option, real pairs, decoy pairs, the oracle's final maps of the real pairs)."""
    import adc_testlib as T
    import engine_testlib as E
    out = []
    for k, (w, h, o) in enumerate(SHAPES):
        opt = T.default_option(**o)
        D = opt.max_disparity - opt.min_disparity
        real = [T.synthetic_pair(w, h, D, 300 + 10 * k + i) for i in range(N_PAIRS)]
        decoy = [T.synthetic_pair(w, h, D, 400 + 10 * k + i) for i in range(N_PAIRS)]
        want = np.stack([E.oracle_outputs(w, h, opt, l, r)["final"] for l, r in real])
        other = np.stack([E.oracle_outputs(w, h, opt, l, r)["final"] for l, r in decoy])
        assert all((E.bits(want[i]) != E.bits(other[i])).any() for i in range(N_PAIRS)), "decoy gives the real maps"
        out.append((opt, real, decoy, want))
    return out


def main(cycles):
    import torch
    import adcensus_b200 as A
    import engine_testlib as E

    cases = expected()
    L = A.load_library()
    failures = []
    start = threading.Barrier(2, timeout=WAIT_S)
    erred = [threading.Event(), threading.Event()]

    def own_error(k, eng):
        """Thread 1 makes its error first; thread 0 makes its own after that; thread 1 reads its text only after
        thread 0 has made its error.  Both threads have a pipelined call in flight meanwhile."""
        if k == 1:
            assert L.adc_match_batch_device(eng._h, -1, None, None, None, None) == 1   # ADC_ERR_ARG
            erred[1].set()
            assert erred[0].wait(WAIT_S), "thread 0 made no error"
            msg = L.adc_last_error().decode()
            assert "adc_match_batch_device: bad arguments" in msg, f"thread 1 reads {msg!r}"
        else:
            assert erred[1].wait(WAIT_S), "thread 1 made no error"
            assert L.adc_set_pipelined(None, 1) == 1
            erred[0].set()
            msg = L.adc_last_error().decode()
            assert "adc_set_pipelined: engine is NULL" in msg, f"thread 0 reads {msg!r}"

    def run(k):
        try:
            opt, real, decoy, want = cases[k]
            w, h, _ = SHAPES[k]
            dev = torch.device("cuda", 0)
            torch.cuda.set_device(dev)
            eng = E.engine(w, h, opt, wave_pairs=WAVE, lanes=LANES)
            st, st2 = torch.cuda.Stream(), torch.cuda.Stream()
            src = {kind: [torch.from_numpy(np.stack([p[v] for p in pairs])).to(dev) for v in range(2)]
                   for kind, pairs in (("real", real), ("decoy", decoy))}
            views = [torch.empty_like(t) for t in src["real"]]
            disp = torch.empty((N_PAIRS, h, w), dtype=torch.float32, device=dev)
            snap = torch.empty_like(disp)
            torch.cuda.current_stream().synchronize()
            start.wait()
            for call in range(CALLS):
                pipelined = call % 2 == 1
                eng.set_pipelined(pipelined)
                half = N_PAIRS // 2 if pipelined else N_PAIRS
                with torch.cuda.stream(st):
                    for v in range(2):
                        views[v].copy_(src["decoy"][v], non_blocking=True)
                    disp.fill_(-7.0)
                    torch.cuda._sleep(cycles)
                    for v in range(2):
                        views[v].copy_(src["real"][v], non_blocking=True)
                    for first, count in ((0, half), (half, N_PAIRS - half)):
                        if count:
                            eng.match_batch_device(count, views[0][first:].data_ptr(), views[1][first:].data_ptr(),
                                                   disp[first:].data_ptr(), st.cuda_stream)
                consumer = st2 if pipelined else st
                if pipelined:
                    eng.join(consumer.cuda_stream)
                with torch.cuda.stream(consumer):
                    snap.copy_(disp, non_blocking=True)
                    busy = not consumer.query()
                    for v in range(2):
                        views[v].copy_(src["decoy"][v], non_blocking=True)
                if call == 1:
                    own_error(k, eng)
                consumer.synchronize()
                eng.set_pipelined(False)
                assert busy, f"call {call}: the consumer stream had finished right after the snapshot: the gate did not hold"
                got = snap.cpu().numpy()
                for i in range(N_PAIRS):
                    E.same(f"thread {k} call {call} ({'pipelined' if pipelined else 'plain'}) pair {i}", got[i], want[i])
            st.synchronize()
            st2.synchronize()
            eng.close()
        except BaseException as ex:   # noqa: BLE001 -- reported to the parent, which asserts the exit code
            failures.append(f"thread {k}: {ex!r}")
            erred[k].set()
            start.abort()

    threads = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    if failures:
        print("\n".join(failures))
        return 1
    print("STREAM_WORKER_OK")
    return 0


if __name__ == "__main__":
    sys.exit(main(int(sys.argv[1])))
