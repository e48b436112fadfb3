// ca_plan.h -- window-record sizes and the launch plan of the fused cost + first horizontal arm sum (k_cost_arm_sum_h,
// k_aggregate.cu).  Plain C++ with no CUDA dependency, so that tests/test_cost_fused_agg.py can check the plan on the CPU.
#pragma once
#include <stddef.h>

#ifdef __CUDACC__
#define CA_HD __host__ __device__
#else
#define CA_HD
#endif

// arm length the window records and the fused kernels are sized for; words per window record (header + one nibble per
// tap of a group's union of at most 2 * L1c + 4 taps, padded to 16 bytes)
CA_HD inline int arm_L1c(int L1) { return L1 < 0 ? 0 : (L1 > 255 ? 255 : L1); }
CA_HD inline int arm_rec_words(int L1) { const int nw = (2 * arm_L1c(L1) + 4 + 7) / 8; return (1 + nw + 3) / 4 * 4; }

#define CA_AD_REP 8                 // replicas of the 766-entry AD table (k_cost_volume keeps 16: see ca_smem_bytes)
#define CA_SMEM_BUDGET (113 * 1024) // shared memory per CTA: two CTAs per SM on an H100 (228 KB per SM, 1 KB reserved per CTA)
#define CA_MAX_THREADS 256
#define CA_ROWS_PER_CTA 4           // the tables are staged once per CTA

// Shared memory of a CTA whose cost positions span at most gm groups of four and whose outputs span at most ngo groups:
//   costs [4 gm + 8 over-read rows][qc] float4 | census table [64][32] | AD table [766][CA_AD_REP]
//   | right-image entries [4 gm + 4 qc] x (packed BGR, census low, census high) | left-image entries [4 gm] x 3
//   | window records of the output groups [ngo][rw]
inline size_t ca_smem_bytes(int qc, int gm, int ngo, int rw) {
    return (size_t)(4 * gm + 8) * qc * 16 + (size_t)(64 * 32 + 766 * CA_AD_REP) * 4 + (size_t)3 * (4 * gm + 4 * qc) * 4 +
           (size_t)3 * 4 * gm * 4 + (size_t)ngo * rw * 4;
}

// Cost positions [m0, m1) of the segment whose outputs are [s0, s1): every tap a window of the segment can reach,
// m0 rounded down to a multiple of four (the cost blocks are groups of four positions).
CA_HD inline void ca_cost_range(int W, int L1c, int s0, int s1, int* m0, int* m1) {
    *m0 = (s0 - L1c > 0 ? s0 - L1c : 0) & ~3;
    *m1 = s1 + L1c < W ? s1 + L1c : W;
}

// qc disparity quads per CTA, rows cut into nseg segments of Ls outputs (a multiple of 4; one segment when the row fits),
// gm = the most cost groups of a segment, threads per CTA.  ok = false: not applicable (the arms are too long for the budget).
struct CaPlan { int qc, Ls, nseg, nchunks, gm, lpc, threads; size_t smem; bool ok; };

inline CaPlan ca_plan(int W, int Dp, int L1) {
    CaPlan p{};
    const int Q = Dp / 4, L1c = arm_L1c(L1), rw = arm_rec_words(L1);
    p.qc = Q >= 8 ? 8 : 4;
    const int gw = (W + 3) / 4;
    auto gm_of = [&](int ls) { const int g = (ls + 2 * L1c + 6) / 4; return g < gw ? g : gw; };   // m1 - m0 <= ls + 2 L1c + 3
    int ls = (W + 3) & ~3;
    while (ls > 64 && ca_smem_bytes(p.qc, gm_of(ls), ls / 4, rw) > CA_SMEM_BUDGET) ls -= 4;
    if (ca_smem_bytes(p.qc, gm_of(ls), ls / 4, rw) > CA_SMEM_BUDGET) { p.ok = false; return p; }
    p.nseg = (W + ls - 1) / ls;
    p.Ls = ((W + p.nseg - 1) / p.nseg + 3) & ~3;        // the segments evened out
    p.nseg = (W + p.Ls - 1) / p.Ls;
    p.gm = gm_of(p.Ls);
    p.smem = ca_smem_bytes(p.qc, p.gm, p.Ls / 4, rw);
    p.nchunks = (Q + p.qc - 1) / p.qc;
    p.lpc = CA_ROWS_PER_CTA;
    // threads: as few whole warps as give every thread the same number of groups
    const int slots = CA_MAX_THREADS / p.qc, iters = (p.gm + slots - 1) / slots;
    p.threads = (((p.gm + iters - 1) / iters) * p.qc + 31) / 32 * 32;
    if (p.threads > CA_MAX_THREADS) p.threads = CA_MAX_THREADS;
    p.ok = true;
    return p;
}
