// Sweeps region voting's list admission rule (adcensus_b200/csrc/vote_plan.h) over the extremes of the shapes adc_create
// accepts: every D from 1 to 256 in both histogram forms, image sizes up to the largest the shape limits allow, pending
// counts from 0 to N, true forward-list sizes up to N * 65535 and every counter value k_vote_slots' saturating
// accumulation can leave.  Wherever the rule admits the forward lists it checks that the true entry count and every int
// cursor stay below 2^31, that k_vote_push streams exactly the entries k_vote_scan wrote, and that the lists fit the
// pair's stretch of the idle cost volume.
// Usage: vote_plan_main   ->   "ok <checks>" and exit 0, or the first violations, one per line, and exit 1
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <vector>

#include "../../adcensus_b200/csrc/vote_plan.h"

static const long long MAX_HEIGHT = 4096, MAX_WIDTH = 10000, MAX_PIXELS = 1ll << 28;   // adc_create's shape limits
static const long long SUP_MAX = 65535;                  // a region size as sup_h holds it
static const long long PUSH_OVERSHOOT = 8 * 1024;        // k_vote_push's streaming index runs past n by < 8 * VP_THREADS
static long long checks = 0, failures = 0;

// prints the first three violations of each check
#define CHECK(cond, ...)                                                                   \
    do {                                                                                   \
        static int shown = 0;                                                              \
        checks++;                                                                          \
        if (!(cond)) {                                                                     \
            failures++;                                                                    \
            if (shown++ < 3) { printf("FAIL " __VA_ARGS__); printf("  [%s]\n", #cond); } \
        }                                                                                  \
    } while (0)

static void add_clamped(std::vector<long long>& v, long long x, long long lo, long long hi) {
    if (x >= lo && x <= hi) v.push_back(x);
}

static std::vector<long long> uniq(std::vector<long long> v) {
    std::sort(v.begin(), v.end());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    return v;
}

// The accumulation.  Each of k_vote_slots' CTAs folds its part of the region sizes with vote_room_add (per thread, then
// over the warps, in an order nobody controls) and merges the part into the pair's counter with vote_room_merge, in an
// order nobody controls either.  Every operand is a value the fold can hold.
//  - The fold: if adding two such values is exact while the sum is at most VOTE_ROOM_MAX, stays above VOTE_ROOM_MAX once
//    the sum is, and never leaves [0, VOTE_ROOM_SAT], then by induction a CTA's part is its exact sum S when
//    S <= VOTE_ROOM_MAX and a value in (VOTE_ROOM_MAX, VOTE_ROOM_SAT] otherwise, whatever the grouping and the order.
//  - The merge: exact parts are at most VOTE_ROOM_PART_MAX, and VOTE_ROOM_CTAS of them sum to at most VOTE_ROOM_MAX below
//    VOTE_ROOM_OVER, so adding them never carries into the flag and the merges commute.  The counter is then the exact
//    room when every part is at most VOTE_ROOM_PART_MAX, and VOTE_ROOM_OVER plus the exact parts' sum otherwise; a room
//    above VOTE_ROOM_MAX always has a part above VOTE_ROOM_PART_MAX (pigeonhole).
static void check_accumulation() {
    const long long MX = VOTE_ROOM_MAX, SAT = VOTE_ROOM_SAT, PART = VOTE_ROOM_PART_MAX, OVER = VOTE_ROOM_OVER;
    std::vector<long long> v;
    for (long long x : {0ll, 1ll, 2ll, SUP_MAX - 1, SUP_MAX, SUP_MAX + 1, PART - 1, PART, PART + 1, MX / 2, MX / 2 + 1,
                        MX - SUP_MAX, MX - 1, MX, MX + 1, SAT - 1, SAT, 0x1fffffffll, 0x20000000ll, 0x3fffffffll,
                        0x40000000ll, 0x40000001ll, 0x5fffffffll, 0x7ffffffell, 0x7fffffffll})
        add_clamped(v, x, 0, SAT);
    v = uniq(v);
    for (long long a : v)
        for (long long b : v) {
            const long long r = vote_room_add((unsigned)a, (unsigned)b);
            CHECK(r >= 0 && r <= SAT, "fold %lld + %lld -> %lld: outside [0, VOTE_ROOM_SAT]\n", a, b, r);
            if (a + b <= MX) CHECK(r == a + b, "fold %lld + %lld -> %lld: not exact below VOTE_ROOM_MAX\n", a, b, r);
            else             CHECK(r > MX, "fold %lld + %lld -> %lld: a sum above VOTE_ROOM_MAX reads as admissible\n", a, b, r);
        }
    CHECK((long long)VOTE_ROOM_CTAS * PART <= MX, "the exact parts of %d CTAs can sum past VOTE_ROOM_MAX\n", VOTE_ROOM_CTAS);
    CHECK(OVER > MX && OVER + MX <= UINT32_MAX && (OVER & (2 * MX - 1)) == 0,
          "VOTE_ROOM_OVER %lld is not a flag above the exact parts' sums\n", OVER);
    // merging: counters the merges of exact parts and the flag can reach, and every part a CTA can hold
    std::vector<long long> cs;
    for (long long c : {0ll, 1ll, PART, MX - PART, MX - 1, MX, OVER, OVER + 1, OVER + MX - PART, OVER + MX}) cs.push_back(c);
    for (long long c : cs)
        for (long long p : v)
            for (long long q : v) {
                const long long r = vote_room_merge((unsigned)c, (unsigned)p);
                CHECK(vote_room_merge(vote_room_merge((unsigned)c, (unsigned)p), (unsigned)q) ==
                      vote_room_merge(vote_room_merge((unsigned)c, (unsigned)q), (unsigned)p),
                      "merge of parts %lld and %lld into %lld depends on their order\n", p, q, c);
                if (p <= PART) CHECK(r == c + p, "merge of part %lld into %lld -> %lld: not exact\n", p, c, r);
                else           CHECK(r > MX && (r & ~(unsigned long long)OVER) == (c & ~(unsigned long long)OVER),
                                     "merge of part %lld into %lld -> %lld: not flagged\n", p, c, r);
            }
    // a room above VOTE_ROOM_MAX, cut into VOTE_ROOM_CTAS parts as evenly or as unevenly as possible, has a flagged part
    for (long long T : {MX + 1, MX + 2, 2 * MX, 1ll << 33}) {
        unsigned c_even = 0, c_one = 0;
        for (int i = 0; i < VOTE_ROOM_CTAS; i++) {
            const long long even = T / VOTE_ROOM_CTAS + (i < T % VOTE_ROOM_CTAS ? 1 : 0);
            c_even = vote_room_merge(c_even, (unsigned)std::min(even, SAT));
            c_one = vote_room_merge(c_one, (unsigned)(i == 0 ? std::min(T, SAT) : 0));
        }
        CHECK(c_even > MX && c_one > MX, "room %lld leaves counters %u / %u\n", T, c_even, c_one);
    }
}

// The counter values a true room T can leave (see check_accumulation): T itself while T <= VOTE_ROOM_MAX, and whenever a
// part was flagged VOTE_ROOM_OVER plus any sum of exact parts.
static std::vector<long long> counter_values(long long T) {
    const long long MX = VOTE_ROOM_MAX, OVER = VOTE_ROOM_OVER;
    std::vector<long long> v{OVER, OVER + 1, OVER + MX - 1, OVER + MX};
    add_clamped(v, OVER + T, OVER, OVER + MX);
    if (T <= MX) v.push_back(T);
    return uniq(v);
}

static void check_shape(int D, bool wide, long long N) {
    const int Dp = (D + 3) / 4 * 4, HW = vote_hist_words(D, wide);
    const long long stride = N * Dp;   // dm.vol_stride: the pair's stretch of the idle cost volume, in 32-bit words
    std::vector<long long> nss{0, 1, 2, 3, N / 1024, N / 16, N / 4, N / 2, N - 1, N};
    for (long long c : {0ll, 1ll << 30, 1ll << 31, 1ll << 32, (long long)VOTE_ROOM_MAX, (long long)VOTE_ROOM_OVER})
        for (long long d = -2; d <= 2; d++) nss.push_back((stride - 2 * c) / HW + d);
    std::vector<long long> ns_v;
    for (long long ns : nss) add_clamped(ns_v, ns, 0, N);
    for (long long ns : uniq(ns_v)) {
        const long long fwd_off = vote_fwd_offset(ns, HW);
        CHECK(fwd_off <= stride, "D=%d wide=%d N=%lld ns=%lld: histograms end at %lld > %lld\n", D, wide, N, ns, fwd_off, stride);
        const long long tmax = ns * SUP_MAX;
        std::vector<long long> ts{0, 1, ns, tmax, tmax - 1, (stride - fwd_off) / 2, (stride - fwd_off) / 2 + 1};
        for (long long t : {(long long)VOTE_ROOM_MAX, (long long)VOTE_ROOM_SAT, (long long)VOTE_ROOM_OVER, 1ll << 32, 1ll << 33})
            for (long long d = -2; d <= 2; d++) ts.push_back(t + d);
        ts.push_back((1ll << 31) - PUSH_OVERSHOOT);
        std::vector<long long> t_v;
        for (long long t : ts) add_clamped(t_v, t, 0, tmax);
        for (long long T : uniq(t_v))
            for (long long c : counter_values(T)) {
                if (!vote_use_fwd(ns, HW, c, stride)) continue;
                // k_vote_scan: the cursor (int, counters[9]) ends at T; k_vote_push streams (int)room entries
                CHECK(T + PUSH_OVERSHOOT <= INT32_MAX, "D=%d wide=%d N=%lld ns=%lld T=%lld counter=%lld: forward lists admitted "
                      "with an entry count an int cursor cannot hold\n", D, wide, N, ns, T, c);
                CHECK(c == T, "D=%d wide=%d N=%lld ns=%lld T=%lld counter=%lld: k_vote_push would stream %lld entries of the %lld "
                      "written\n", D, wide, N, ns, T, c, c, T);
                CHECK(fwd_off + 2 * c <= stride, "D=%d wide=%d N=%lld ns=%lld counter=%lld: forward lists past the stride\n",
                      D, wide, N, ns, c);
                // k_vote_push: n_adj = the entries that are real edges (<= T); its prefix sum is capped at VOTE_ROOM_SAT
                std::vector<long long> a_v;
                for (long long a : {0ll, 1ll, T / 2, T - ns, T, T + 1, (long long)VOTE_ROOM_SAT, stride - fwd_off - 2 * c,
                                    stride - fwd_off - 2 * c + 1})
                    add_clamped(a_v, a, 0, std::max(T, (long long)VOTE_ROOM_SAT));
                for (long long n_adj : uniq(a_v)) {
                    if (!vote_use_adj(true, ns, HW, c, n_adj, stride)) continue;
                    CHECK(fwd_off + 2 * c + n_adj <= stride, "D=%d wide=%d N=%lld ns=%lld counter=%lld n_adj=%lld: adjacency "
                          "lists past the stride\n", D, wide, N, ns, c, n_adj);
                    CHECK(n_adj <= INT32_MAX, "D=%d wide=%d N=%lld ns=%lld n_adj=%lld: adjacency offsets overflow int\n",
                          D, wide, N, ns, n_adj);
                }
            }
    }
}

int main() {
    check_accumulation();
    for (int D = 1; D <= 256; D++) {
        const long long W = MAX_WIDTH - D, H = MAX_HEIGHT;   // width + range <= 10000, height <= 4096
        const long long nmax = std::min(W * H, MAX_PIXELS);
        for (long long N : {1ll, 2ll, 1ll << 20, nmax / 2, nmax - 1, nmax})
            for (bool wide : {false, true}) check_shape(D, wide, N);
    }
    if (failures) {
        printf("%lld of %lld checks failed\n", failures, checks);
        return 1;
    }
    printf("ok %lld\n", checks);
    return 0;
}
