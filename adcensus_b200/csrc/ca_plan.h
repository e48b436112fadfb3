// ca_plan.h -- window-record sizes and the launch plans of the fused aggregation kernels of k_aggregate.cu: the fused cost +
// first horizontal arm sum (k_cost_arm_sum_h) and the double passes (k_arm_sum2t, k_arm_sum2).  Plain C++ with no CUDA
// dependency, so that tests/test_cost_fused_agg.py and tests/test_kernel_sweep.py can check the plans on the CPU.
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

// Window records of one pair (k_aggregate.cu), RW words each: [H][GW] records of the horizontal axis (GW = ceil(W/4)
// groups per row), then [GH][W] records of the vertical axis (group index outermost, so that neighbouring columns are
// neighbouring records).  Counted in records: the pair holds arm_pair_recs(H, W) of them, and the record of group g of
// line `line` (a row for dir 0, a column for dir 1) is number arm_line_rec(W, H, dir, line) + g * arm_rec_gstride(W, dir).
CA_HD inline size_t arm_pair_recs(int H, int W) {
    const size_t GW = (size_t)((W + 3) >> 2), GH = (size_t)((H + 3) >> 2);
    return GW * H + GH * W;
}
CA_HD inline size_t arm_line_rec(int W, int H, int dir, int line) {
    return dir ? (size_t)((W + 3) >> 2) * H + line : (size_t)line * ((W + 3) >> 2);
}
CA_HD inline int arm_rec_gstride(int W, int dir) { return dir ? W : 1; }

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

// Segment length (a multiple of 4) of a line of L outputs cut into segments of at most ls outputs, evened out.
inline int ca_even_segments(int L, int ls) {
    const int nseg = (L + ls - 1) / ls;
    return ((L + nseg - 1) / nseg + 3) & ~3;
}

// Threads of a CTA whose groups of outputs are taken by qc threads each: as few whole warps as give every thread the same
// number of groups, at most CA_MAX_THREADS.
inline int ca_threads(int groups, int qc) {
    const int slots = CA_MAX_THREADS / qc, iters = (groups + slots - 1) / slots;
    const int t = (((groups + iters - 1) / iters) * qc + 31) / 32 * 32;
    return t > CA_MAX_THREADS ? CA_MAX_THREADS : t;
}

// Dynamic shared memory per CTA the double passes (k_arm_sum2t, k_arm_sum2) are launched under (the launch attribute):
// the most a plan's smem may be.
#define A2_SMEM_ATTR (200 * 1024)

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
    p.Ls = ca_even_segments(W, ls);
    p.nseg = (W + p.Ls - 1) / p.Ls;
    p.gm = gm_of(p.Ls);
    p.smem = ca_smem_bytes(p.qc, p.gm, p.Ls / 4, rw);
    p.nchunks = (Q + p.qc - 1) / p.qc;
    p.lpc = CA_ROWS_PER_CTA;
    p.threads = ca_threads(p.gm, p.qc);
    p.ok = true;
    return p;
}

// Plan of the TMA-staged double pass (k_arm_sum2t, k_aggregate.cu) for one axis (dir 0 = rows, 1 = columns): quads per
// CTA, box length, segment length, lines per CTA, shared-memory sizes.
struct ArmSum2tPlan { int qc, BR, Ls, nseg, nchunks, rows_s_cap, threads, lpc; size_t smem; bool ok; };
inline ArmSum2tPlan plan_arm_sum2t(int W, int H, int Dp, int L1, int dir) {
    const int budget_kb = 104;            // shared memory per CTA (two CTAs per SM); 72 and 130 KB measured slower or equal
    ArmSum2tPlan pl{};
    const int Q = Dp / 4, L = dir ? H : W, L1c = arm_L1c(L1);
    if (Q < 4) { pl.ok = false; return pl; }                      // (tiny disparity ranges take the LDG kernel)
    const int BR = 64;
    auto need = [&](int qc, int ls, bool whole, int* rows_s_cap) {
        const int rows_m = (whole ? L : ls + 2 * L1c + 3) + 13;   // + 8 over-read rows, + rounding, + the row that holds the mbarrier
        const int rows_s = whole ? L : ls + 4 * L1c + 3;
        *rows_s_cap = (rows_s + BR - 1) / BR * BR + 8;
        return (size_t)(*rows_s_cap + rows_m) * qc * 16 + 16 + (size_t)(rows_m / 4 + 1) * arm_rec_words(L1) * 4 + (size_t)rows_m * 4 + 64;   // tiles | mid | mbarrier | records | divisors
    };
    const size_t budget = (size_t)budget_kb * 1024;
    int qc = Q >= 8 ? 8 : 4, cap = 0;
    if (need(8, 0, true, &cap) > budget && need(4, 0, true, &cap) <= budget) qc = 4;   // a whole line with 4 quads beats segments with 8
    pl.qc = qc; pl.BR = BR;
    if (need(qc, 0, true, &cap) <= budget) { pl.Ls = (L + 3) & ~3; pl.nseg = 1; }
    else {
        int ls = (L + 3) & ~3;
        while (ls > 64 && need(qc, ls, false, &cap) > budget) ls -= 4;
        if (need(qc, ls, false, &cap) > budget) { pl.ok = false; return pl; }
        pl.Ls = ca_even_segments(L, ls);
        pl.nseg = (L + pl.Ls - 1) / pl.Ls;
    }
    pl.smem = need(qc, pl.Ls, pl.nseg == 1, &pl.rows_s_cap);
    pl.nchunks = (Q + qc - 1) / qc;
    pl.threads = ca_threads(((pl.nseg == 1 ? L : pl.Ls) + 3) / 4, qc);
    // lines per CTA: each line after the first loads while the previous one finishes.  A line cut into segments keeps one
    // per CTA (1920x1080x192's vertical pass measured 3 % slower with two or four).
    pl.lpc = pl.nseg > 1 ? 1 : 4;
    pl.ok = true;
    return pl;
}

// Segment length / chunk width of the LDG double pass (k_arm_sum2, k_aggregate.cu) for one axis: the largest segment whose
// `mid` rows fit the shared-memory budget; a whole line when it fits.  ok is a constant: the plan applies to every shape,
// because the budget grows to what a segment of 64 outputs needs.
struct ArmSum2Plan { int Ls, qc_log2, nseg, nchunks, rows_m_cap; size_t smem; static constexpr bool ok = true; };
inline ArmSum2Plan plan_arm_sum2(int W, int H, int Dp, int L1, int dir) {
    const int budget_kb = 60;    // shared memory per CTA the plan may use (40 KB: 8 % slower on Cone; 75 / 100 KB: no faster)
    ArmSum2Plan pl{};
    const int Q = Dp / 4, L = dir ? H : W, L1c = arm_L1c(L1);
    int ql = 0;
    while ((1 << ql) < Q && ql < 3) ql++;                 // Qc = min(8, Q rounded up to a power of two); 4 quads measured 4-25 % slower
    const int Qc = 1 << ql;
    size_t budget = (size_t)budget_kb * 1024;
    const size_t need_min = (size_t)(2 * L1c + 16 + 64) * Qc * 16;    // a segment of at least 64 outputs
    if (budget < need_min) budget = need_min;
    const int rows_max = (int)(budget / ((size_t)Qc * 16));
    int Ls;
    if (L + 12 <= rows_max) Ls = (L + 3) & ~3;             // the whole line
    else Ls = ca_even_segments(L, (rows_max - 2 * L1c - 16) & ~3);
    pl.Ls = Ls; pl.qc_log2 = ql;
    pl.nseg = (L + Ls - 1) / Ls;
    pl.nchunks = (Q + Qc - 1) / Qc;
    const int rows = (pl.nseg == 1 ? L : Ls + 2 * L1c + 3) + 4 + 8;   // + the rows the last trip of a walk may touch
    pl.rows_m_cap = (rows + 3) & ~3;
    pl.smem = (size_t)pl.rows_m_cap * Qc * 16 + (size_t)(pl.rows_m_cap / 4 + 1) * arm_rec_words(L1) * 4 + (size_t)pl.rows_m_cap * 4 + 16;   // mid | records | divisors
    return pl;
}

// Form of the double pass on axis dir (0 = rows, 1 = columns): the TMA-staged kernel when the TMA plans of both axes are
// ok and, on rows, the row is one segment (a row cut into segments would re-fetch 4 L1 source positions per segment);
// the LDG kernel otherwise.  The launcher, the tensor-map encoder and the tests read this one rule.
enum { A2_LDG = 0, A2_TMA = 1 };
inline int arm_sum2_form(int W, int H, int Dp, int L1, int dir) {
    const ArmSum2tPlan rows = plan_arm_sum2t(W, H, Dp, L1, 0), cols = plan_arm_sum2t(W, H, Dp, L1, 1);
    if (!rows.ok || !cols.ok) return A2_LDG;
    return dir == 0 && rows.nseg > 1 ? A2_LDG : A2_TMA;
}
