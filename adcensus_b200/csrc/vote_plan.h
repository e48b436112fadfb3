// vote_plan.h -- when region voting (k_vote.cu) may keep its forward and adjacency lists in the idle cost volume.  Plain
// C++ with no CUDA dependency, so that tests/test_size_limits.py can sweep the rule on the CPU over every shape
// adc_create accepts.
#pragma once

#ifdef __CUDACC__
#define VOTE_HD __host__ __device__
#else
#define VOTE_HD
#endif

// The histograms of the ns pending pixels come first in a pair's stretch of hist_stride 32-bit words (the idle cost
// volume, N * Dp words): HW words per pixel, two 16-bit counts per word, or one 32-bit count in the WIDE form.
VOTE_HD inline bool vote_wide(int D, int L1) { return D > 254 || L1 > 127; }
VOTE_HD inline int vote_hist_words(int D, bool wide) { return wide ? D : (D + 1) >> 1; }
// the forward lists follow them, 8-byte aligned (in 32-bit words)
VOTE_HD inline long long vote_fwd_offset(long long ns, int HW) { return (ns * HW + 1) & ~1ll; }

// room = the sum of the pending pixels' region sizes (sup_h, < 65536 each) = the number of forward-list entries
// k_vote_scan writes, two words each.  Each of k_vote_slots' VOTE_ROOM_CTAS CTAs of a pair folds its part with
// vote_room_add (per thread, then over the warps), which is exact up to VOTE_ROOM_MAX and VOTE_ROOM_SAT beyond; operands
// are at most VOTE_ROOM_SAT, so a + b never wraps.  The CTA then merges its part into the pair's counter with one atomic,
// vote_room_merge: a part of at most VOTE_ROOM_PART_MAX is added, a larger one sets VOTE_ROOM_OVER.  The exact parts sum
// to at most VOTE_ROOM_CTAS * VOTE_ROOM_PART_MAX = VOTE_ROOM_MAX, so they never carry into that bit, the order does not
// matter, and the counter holds the exact room when room <= VOTE_ROOM_MAX and no part was larger, and a value above
// VOTE_ROOM_MAX otherwise (a room above VOTE_ROOM_MAX always has such a part).
#define VOTE_ROOM_MAX (1u << 30)
#define VOTE_ROOM_SAT (VOTE_ROOM_MAX + 1u)
#define VOTE_ROOM_CTAS 64
#define VOTE_ROOM_PART_MAX (VOTE_ROOM_MAX / VOTE_ROOM_CTAS)
#define VOTE_ROOM_OVER (1u << 31)
VOTE_HD inline unsigned vote_room_add(unsigned a, unsigned b) { return a + b < VOTE_ROOM_SAT ? a + b : VOTE_ROOM_SAT; }
VOTE_HD inline unsigned vote_room_merge(unsigned counter, unsigned part) {
    return part <= VOTE_ROOM_PART_MAX ? counter + part : counter | VOTE_ROOM_OVER;
}

// Forward lists: room entries after the histograms.  Admitted only while the counter is exact and at most 2^30, so the
// int cursors of k_vote_scan and k_vote_push (which end at room, or run < 2^13 past it) stay below 2^31 and the entries
// k_vote_push streams are the entries k_vote_scan wrote.  A pair over the limit enumerates (the same fixed point).
VOTE_HD inline bool vote_use_fwd(long long ns, int HW, long long room, long long hist_stride) {
    return room <= VOTE_ROOM_MAX && vote_fwd_offset(ns, HW) + 2 * room <= hist_stride;
}
// Adjacency lists: the n_adj real entries of the forward lists (<= room), after them.
VOTE_HD inline bool vote_use_adj(bool use_fwd, long long ns, int HW, long long room, long long n_adj, long long hist_stride) {
    return use_fwd && n_adj <= room && vote_fwd_offset(ns, HW) + 2 * room + n_adj <= hist_stride;
}
