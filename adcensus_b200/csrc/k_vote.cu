// k_vote.cu -- iterative region voting (reference: multistep_refiner.cpp:153-227), incremental form.
//
// The reference runs 5 iterations x {mismatch list, occlusion list}; inside a sweep the pixels are
// visited in raster order and a filled pixel is immediately visible to the later ones.  For a pending
// pixel p the vote is a histogram over its cross region R(p) (vertical arm of p, then the horizontal arm
// of every pixel on it) of the rounded disparities of the valid pixels, reading q's value "as of now" if
// q precedes p in raster order and "as of the start of the sweep" otherwise.
//
// Exact parallel form used here.  Every pending pixel owns a histogram in memory that is kept equal to
// what the reference's scan would count for it, and the sweep is the fixed point of
//     derive: value(p) = vote(hist(p))                     for every p whose histogram changed
//     push:   value(q) changed a -> b  =>  hist(p)[a]--, hist(p)[b]++   for every pending p of the swept
//             list with q in R(p) and p after q in raster order
// iterated until no value changes.  The sequential result is the unique fixed point of that map
// (induction over raster order: the first pending pixel depends on nothing that moves, pixel p only on
// earlier ones), so the iteration order is free; a round without changes certifies it.  When a sweep has
// converged its fills are committed: they become visible to the pixels BEFORE them and to the other list
// (one more push of "invalid -> b"), and the filled pixels leave the lists.  Histogram counts are
// integers, so the order of the pushes is irrelevant; derive and push never overlap (CTA barrier between
// them), so every derive sees a consistent histogram.
//
// Why: the pull form (re-scan R(p) whenever something near p changed) visits ~27 M pixels per Cone pair
// behind a tile-granular "dirty" filter; the sequential reference 7.7 M.  Here the regions are scanned
// twice (2.7 M visits each): the first scan builds the histograms and counts, for every pending pixel t,
// how many regions contain it; the second writes those regions' owners into t's adjacency list (CSR by
// target; 2.1 M entries on Cone -- pending pixels come in blobs).  Only pending pixels ever change, so a
// value change of t is then: walk t's list (coalesced) and touch those histograms.  All of it -- the two
// scans with their counters and cursors in shared memory, then 12.7 k value changes, 32 k 64-bin derives,
// ~50 rounds -- runs in ONE CTA per stereo pair with nothing but CTA barriers between the phases, beside
// the bandwidth-bound kernels of the other lanes.  (Batch-wide scan kernels were tried first: their two
// million global atomics per pair made them cost more whole-GPU time than the voting they prepared.)
// If the adjacency lists do not fit the idle cost volume they live in (pathological inputs: huge regions
// that are almost entirely invalid), the pair falls back to enumerating the inverse region of every change
// on the fly from transposed arm tables (push_enum below).
//
// Two instantiations of the scan and push kernels, WIDE = D > 254 || L1 > 127.  The narrow one keeps a slot's vote in
// one byte (255 = none) and the histogram counts in 16 bits, two per word (a region of L1 <= 127 holds < 65536 pixels).
// WIDE keeps the vote in 16 bits (0xffff = none) and one 32-bit count per word, which covers every D <= 256 and
// L1 <= 255.  For L1 > 127 the uint16 support counts the forward lists are reserved from may wrap, so those pairs
// always enumerate.
#include "adc_common.cuh"
#include <type_traits>

#define VP_THREADS 1024
#define VP_WARPS (VP_THREADS / 32)
#define VI_WARPS 8
#define VP_MAXD 256
#define VOTE_OUTSIDE 256   // vstate of a valid pixel whose rounded disparity lies outside [0,D): no histogram counts it
// counters (ADC_CNT ints per pair): 2 = fixed-point rounds, 3 = derives, 4..8 = microseconds spent in the phases of
// k_vote_push, 9 = forward-list cursor, 10/11 = active list sizes, 12 = changes, 13 = 1 when the adjacency lists are in
// use, 14 = total adjacency entries, 15 = forward-list room

// ---- state maps: vstate[p] = rounded disparity index of a valid pixel, VOTE_OUTSIDE, or -1 = invalid; alr = the
// horizontal arms alone (2 bytes per pixel), which is all the region scans read of a row ----
__global__ void k_vote_encode(AdcDims dm, const float* __restrict__ disp, const uchar4* __restrict__ arms,
                              uchar2* __restrict__ alr, int* __restrict__ vstate) {
    const int pair = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dm.N) return;
    const float d = disp[(size_t)pair * dm.N + i];
    int v = -1;
    if (d != ADC_INVALID_F) {
        const int di = (int)roundf(d) - dm.dmin;   // lround: half away from zero
        v = di >= 0 && di < dm.D ? di : VOTE_OUTSIDE;
    }
    vstate[(size_t)pair * dm.N + i] = v;
    const uchar4 a = arms[(size_t)pair * dm.N + i];
    alr[(size_t)pair * dm.N + i] = make_uchar2(a.x, a.y);
}

// ---- transposed per-pixel tables for the fallback: vertical arms (top,bottom) as [x][y] ----
__global__ void __launch_bounds__(256)
k_vote_transpose(AdcDims dm, const uchar4* __restrict__ arms, uchar2* __restrict__ atbT) {
    __shared__ uchar2 tile[32][33];
    const int pair = blockIdx.z;
    const int x0 = blockIdx.x * 32, y0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
    const uchar4* A = arms + (size_t)pair * dm.N;
    uchar2* T = atbT + (size_t)pair * dm.N;
    for (int j = ty; j < 32; j += 8) {
        const int x = x0 + tx, y = y0 + j;
        if (x < dm.W && y < dm.H) { const uchar4 a = __ldg(A + y * dm.W + x); tile[j][tx] = make_uchar2(a.z, a.w); }
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
        const int x = x0 + j, y = y0 + tx;
        if (x < dm.W && y < dm.H) T[(size_t)x * dm.H + y] = tile[tx][j];
    }
}

// ---- slots.  slot = position in the active list (+ n0 for the occlusion list).  vstate[p]: rounded disparity
// index of a valid pixel (VOTE_OUTSIDE = outside [0,D)), -1 = invalid, -(slot+2) = invalid and pending in slot. ----
__global__ void __launch_bounds__(256)
k_vote_slots(AdcDims dm, const int* __restrict__ vlist, int* __restrict__ counters, int* __restrict__ vstate,
             int* __restrict__ pslotT, const uint16_t* __restrict__ sup) {
    const int pair = blockIdx.y;
    const int n0 = counters[pair * ADC_CNT + 10], n1 = counters[pair * ADC_CNT + 11];
    unsigned room = 0;   // sum of the region sizes = upper bound of the forward lists (saturating)
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n0 + n1; s += gridDim.x * blockDim.x) {
        const int p = s < n0 ? vlist[((size_t)pair * 2 + 0) * dm.N + s] : vlist[((size_t)pair * 2 + 1) * dm.N + (s - n0)];
        const int y = p / dm.W, x = p - y * dm.W;
        vstate[(size_t)pair * dm.N + p] = -(s + 2);
        pslotT[(size_t)pair * dm.N + (size_t)x * dm.H + y] = s;
        room += sup[(size_t)pair * dm.N + p];
    }
    room = __reduce_add_sync(0xffffffffu, min(room, 0x00ffffffu));
    if ((threadIdx.x & 31) == 0 && room) {
        const unsigned old = atomicAdd(reinterpret_cast<unsigned*>(counters + pair * ADC_CNT + 15), min(room, 0x1fffffffu));
        if (old > 0x3fffffffu) atomicExch(reinterpret_cast<unsigned*>(counters + pair * ADC_CNT + 15), 0x7fffffffu);   // stays "too big"
    }
}

// ---- region scan of one slot by one warp.  A group of LPR lanes takes one region row, so a trip covers 4 x 32/LPR rows,
// the first 2*LPR columns of each fetched before any is consumed (8 independent loads in flight per lane); the horizontal
// arms of all rows are fetched up front (lane r holds rows r, r+32, r+64) and handed out by shuffle.  With LPR = 8 the
// typical Cone region (a dozen rows of a dozen-odd pixels) is one trip.  `visit` is called in warp-uniform control flow
// (it may use warp collectives); -1 (an invalid pixel that is nobody's slot) stands in for "no pixel here".
template <int LPR, typename F>
__device__ __forceinline__ void vote_scan_region(int p, int W, const uchar4* __restrict__ A, const uchar2* __restrict__ ALR,
                                                 const int* __restrict__ VS, int lane, F&& visit) {
    constexpr int RPT = 32 / LPR;          // rows per step of a trip
    const int y = p / W, x = p - y * W;
    const uchar4 a = __ldg(A + p);
    const int top = a.z, rows = top + (int)a.w + 1;
    const int rbase = (y - top) * W + x;
    const int grp = lane / LPR, sub = lane % LPR;
    // the horizontal arms are cached 96 rows at a time (lane r holds rows r, r+32, r+64 of the chunk); a region has
    // up to 2*L1+1 <= 511 rows, the default L1 = 34 gives at most 69: one chunk
    for (int rb = 0; rb < rows; rb += 96) {
        const int rows_c = min(rows - rb, 96);
        const int cbase = rbase + rb * W;
        unsigned ar[3];
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const int ri = lane + 32 * j;
            uchar2 v = make_uchar2(0, 0);
            if (ri < rows_c) v = __ldg(ALR + cbase + ri * W);
            ar[j] = (unsigned)v.x | ((unsigned)v.y << 8);
        }
        for (int r0 = 0; r0 < rows_c; r0 += 4 * RPT) {
            int v0[4], v1[4], cl[4], ch[4], ro[4];
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const int ri = r0 + RPT * t + grp;
                unsigned a2 = __shfl_sync(0xffffffffu, ar[0], ri & 31);
                if (rows_c > 32) {
                    const unsigned a2b = __shfl_sync(0xffffffffu, ar[1], ri & 31), a2c = __shfl_sync(0xffffffffu, ar[2], ri & 31);
                    a2 = ri < 32 ? a2 : (ri < 64 ? a2b : a2c);
                }
                ro[t] = cbase + ri * W;
                cl[t] = -(int)(a2 & 255u) + sub;
                ch[t] = ri < rows_c ? (int)(a2 >> 8) : -0x10000;     // rows past the chunk: empty segment
                v0[t] = cl[t] <= ch[t] ? __ldg(VS + ro[t] + cl[t]) : -1;
                v1[t] = cl[t] + LPR <= ch[t] ? __ldg(VS + ro[t] + cl[t] + LPR) : -1;
            }
            int more = 0;
#pragma unroll
            for (int t = 0; t < 4; t++) more = max(more, (ch[t] - cl[t]) / LPR);
            more = __reduce_max_sync(0xffffffffu, more);          // LPR-column chunks the widest row of the trip needs, minus one
#pragma unroll
            for (int t = 0; t < 4; t++) visit(v0[t]);
            if (more >= 1) {
#pragma unroll
                for (int t = 0; t < 4; t++) visit(v1[t]);
            }
            for (int k = 2; k <= more; k++) {                     // wider rows
#pragma unroll
                for (int t = 0; t < 4; t++) visit(cl[t] + LPR * k <= ch[t] ? __ldg(VS + ro[t] + cl[t] + LPR * k) : -1);
            }
        }
    }
}

// ---- batch-wide scan: histogram of every slot (D counters packed two per 32-bit word, a region holding < 65536 pixels;
// WIDE: one per word) and, when there is room, its forward list: an entry (t, s) for every pending pixel t of the region
// of slot s, written compacted at a base taken from the pair's cursor (counters[9]).  A slot reserves as many entries as
// its region has pixels and marks the ones it does not use (-1): the lists of a pair are ONE dense array of `room`
// entries that k_vote_push streams through.
__host__ __device__ inline long long vote_fwd_offset(long long ns, int HW) { return (ns * HW + 1) & ~1ll; }   // in 32-bit words, 8-byte aligned
template <bool WIDE>
__global__ void __launch_bounds__(VI_WARPS * 32)
k_vote_scan(AdcParams P, const uchar4* __restrict__ arms, const uchar2* __restrict__ alr_all, const int* __restrict__ vstate_all,
            const uint16_t* __restrict__ sup_all, const int* __restrict__ vlist, int* counters, unsigned* __restrict__ hist_all,
            long long hist_stride, int force_enum) {
    __shared__ int s_hist[VI_WARPS][VP_MAXD];
    const AdcDims& dm = P.dm;
    const int pair = blockIdx.y;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int W = dm.W, D = dm.D, HW = WIDE ? D : (D + 1) >> 1;
    int* cnt = counters + pair * ADC_CNT;
    const int n0 = cnt[10], n1 = cnt[11], ns = n0 + n1;
    const long long room = (unsigned)cnt[15];
    const bool use_fwd = !force_enum && vote_fwd_offset(ns, HW) + 2 * room <= hist_stride;
    const uchar4* A = arms + (size_t)pair * dm.N;
    const uchar2* ALR = alr_all + (size_t)pair * dm.N;
    const int* VS = vstate_all + (size_t)pair * dm.N;
    const uint16_t* sup = sup_all + (size_t)pair * dm.N;
    unsigned* hist = hist_all + (size_t)pair * hist_stride;
    int2* fwd = reinterpret_cast<int2*>(hist + vote_fwd_offset(ns, HW));
    int* hs = s_hist[wid];
    for (int s = blockIdx.x * VI_WARPS + wid; s < ns; s += gridDim.x * VI_WARPS) {
        const int p = s < n0 ? vlist[((size_t)pair * 2 + 0) * dm.N + s] : vlist[((size_t)pair * 2 + 1) * dm.N + (s - n0)];
        for (int b = lane; b < D; b += 32) hs[b] = 0;
        int fb = 0, fn = 0;
        const int reserved = (int)sup[p];
        if (use_fwd) {
            if (lane == 0) fb = atomicAdd(cnt + 9, reserved);
            fb = __shfl_sync(0xffffffffu, fb, 0);
        }
        __syncwarp();
        vote_scan_region<8>(p, W, A, ALR, VS, lane, [&](int v) {
            if (v >= 0 && v < D) atomicAdd(&hs[v], 1);
            if (use_fwd) {
                const bool edge = v < -1 && -v - 2 != s;
                const unsigned m = __ballot_sync(0xffffffffu, edge);
                if (edge) fwd[fb + fn + __popc(m & ((1u << lane) - 1u))] = make_int2(-v - 2, s);
                fn += __popc(m);
            }
        });
        __syncwarp();
        for (int w2 = lane; w2 < HW; w2 += 32) {
            if constexpr (WIDE) {
                hist[(size_t)s * HW + w2] = (unsigned)hs[w2];
            } else {
                const unsigned c0 = (unsigned)hs[2 * w2], c1 = (2 * w2 + 1 < D) ? (unsigned)hs[2 * w2 + 1] : 0u;
                hist[(size_t)s * HW + w2] = c0 | (c1 << 16);
            }
        }
        if (use_fwd)
            for (int k2 = fn + lane; k2 < reserved; k2 += 32) fwd[fb + k2] = make_int2(-1, -1);
        __syncwarp();
    }
}

// One CTA per stereo pair.  Per-slot state (current vote, dirty / dead flags) lives in shared memory when the
// lists fit (VP_SMEM_SLOTS slots; global memory otherwise -- one CTA = one SM, so plain accesses are coherent);
// the histograms live in global memory and are read at L2 (ld.cg) because the pushes are L2 atomics; the
// adjacency lists and the fallback's arm / slot tables are immutable here and go through the read-only path.
#define VP_SMEM_SLOTS 32768
#define VP_FLAG_DIRTY 1
#define VP_FLAG_DEAD 2

template <bool WIDE> using VoteVal = typename std::conditional<WIDE, uint16_t, uint8_t>::type;   // a slot's vote

template <bool WIDE>
__global__ void __launch_bounds__(VP_THREADS)
k_vote_push(AdcParams P, const uchar2* __restrict__ alr_all,
            const uchar2* __restrict__ atbT_all, const int* __restrict__ pslotT_all, unsigned* hist_all, long long hist_stride, int* cur_all, VoteVal<WIDE>* val_all, uint8_t* flag_all,
            const int* __restrict__ vlist, int* counters, int* work_all, int2* chg_all,
            float* disp_old, float* disp_new, uint8_t* label, int cols_cap, int slot_cap, int force_enum) {
    using VT = VoteVal<WIDE>;
    constexpr int NONE = WIDE ? 0xffff : 255;   // "no vote"; a change record packs old and new vote in VB-bit fields
    constexpr int VB = WIDE ? 16 : 8;
    constexpr int NHW = WIDE ? 8 : 4;           // histogram words per lane, at most
    extern __shared__ __align__(16) unsigned char vp_smem[];
    __shared__ int s_nwork, s_nchg, s_warp[32], s_base, s_fits;
    const AdcDims& dm = P.dm;
    const int pair = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int W = dm.W, H = dm.H, D = dm.D, HW = WIDE ? D : (D + 1) >> 1;
    const int L1 = max(P.L1, 0), R = 2 * L1 + 1;
    const uchar2* ALR = alr_all + (size_t)pair * dm.N;
    const uchar2* ATB = atbT_all + (size_t)pair * dm.N;
    const int* pslotT = pslotT_all + (size_t)pair * dm.N;
    unsigned* hist = hist_all + (size_t)pair * hist_stride;
    int* work = work_all + (size_t)pair * dm.N;
    int2* chg = chg_all + (size_t)pair * dm.N;
    float* d_old = disp_old + (size_t)pair * dm.N;
    float* d_new = disp_new + (size_t)pair * dm.N;
    uint8_t* lab = label + (size_t)pair * dm.N;
    int* cnt = counters + pair * ADC_CNT;
    const int n0 = __ldcg(cnt + 10), n1 = __ldcg(cnt + 11), ns = n0 + n1;
    const int* list0 = vlist + ((size_t)pair * 2 + 0) * dm.N;
    const int* list1 = vlist + ((size_t)pair * 2 + 1) * dm.N;
    auto pix = [&](int s) { return s < n0 ? __ldg(list0 + s) : __ldg(list1 + (s - n0)); };
    // shared memory: [fallback column lists][val][flg][cur]
    unsigned short* cols = reinterpret_cast<unsigned short*>(vp_smem) + (size_t)wid * cols_cap;
    unsigned char* after_hist = vp_smem + (size_t)VP_WARPS * cols_cap * 2;
    VT* val;         // [slot] current vote, NONE = none
    uint8_t* flg;    // [slot] VP_FLAG_*
    int* cur;        // [slot + 1] list lengths -> list starts -> fill cursors (= list ends once filled)
    const bool state_smem = ns <= slot_cap;
    if (state_smem) {
        val = reinterpret_cast<VT*>(after_hist);
        flg = reinterpret_cast<uint8_t*>(val + slot_cap);
        cur = reinterpret_cast<int*>(flg + slot_cap);
    } else {
        val = val_all + (size_t)pair * dm.N;
        flg = flag_all + (size_t)pair * dm.N;
        cur = cur_all + (size_t)pair * (dm.N + 1);
    }
    for (int i = tid; i < ns; i += VP_THREADS) { val[i] = NONE; flg[i] = VP_FLAG_DIRTY; }
    for (int i = tid; i <= ns; i += VP_THREADS) cur[i] = 0;
    __syncthreads();
    int rounds_total = 0, derives = 0, changes = 0;

    // ---- adjacency lists (CSR by target) from the forward lists of k_vote_scan: count, prefix, fill
    const long long room = (unsigned)__ldcg(cnt + 15);
    const long long fwd_off = vote_fwd_offset(ns, HW);
    const bool use_fwd = !force_enum && fwd_off + 2 * room <= hist_stride;
    const int2* fwd = reinterpret_cast<const int2*>(hist + fwd_off);
    // adjacency entry = the slot whose histogram counts the target.  (Whether that slot's pixel comes after the target in
    // raster order -- all a push needs to know about it -- is a comparison of slot numbers: the lists are in raster order.)
    int* adj = reinterpret_cast<int*>(hist) + fwd_off + (use_fwd ? 2 * room : 0);
    unsigned long long t_start = 0;
    if (tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));
    // Both passes stream through the pair's forward entries, eight independent 8-byte loads per thread in flight (the
    // first version walked list by list, two entries per lane in flight, and spent 1.9 of the kernel's 3.6 ms here).
    auto for_each_edge = [&](auto&& f) {
        const int n = (int)room;                       // (< 2^30: use_fwd)
        for (int i0 = tid; i0 < n; i0 += 8 * VP_THREADS) {
            int2 e[8];
#pragma unroll
            for (int j = 0; j < 8; j++) e[j] = i0 + j * VP_THREADS < n ? __ldg(fwd + i0 + j * VP_THREADS) : make_int2(-1, -1);
#pragma unroll
            for (int j = 0; j < 8; j++)
                if (e[j].x >= 0) f(e[j].x, e[j].y);
        }
    };
    if (use_fwd) for_each_edge([&](int t, int) { atomicAdd(&cur[t + 1], 1); });   // length of t's list, kept at index t + 1
    __syncthreads();
    // ---- inclusive prefix sum over cur[0..ns]: cur[t] = start of t's list, cur[ns] = number of entries
    if (tid == 0) { s_base = 0; s_fits = 1; }
    __syncthreads();
    for (int i0 = 0; i0 <= ns; i0 += VP_THREADS) {
        const int i = i0 + tid;
        const int v = i <= ns ? (state_smem ? cur[i] : __ldcg(cur + i)) : 0;
        int inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) s_warp[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            const int w = s_warp[lane];
            int wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
            s_warp[lane] = wi - w;
        }
        __syncthreads();
        const int base = s_base;
        if (i <= ns) cur[i] = base + s_warp[wid] + inc;
        __syncthreads();
        if (tid == VP_THREADS - 1) {
            const long long nb = (long long)base + s_warp[VP_WARPS - 1] + inc;
            if (nb > 0x3fffffff) s_fits = 0;
            s_base = (int)min(nb, (long long)0x3fffffff);
        }
        __syncthreads();
    }
    const int n_adj = s_base;
    const bool use_adj = use_fwd && s_fits && fwd_off + 2 * room + n_adj <= hist_stride;
    // ---- fill (afterwards cur[t] = end of t's list = start of t + 1's)
    if (use_adj) for_each_edge([&](int t, int s) { adj[atomicAdd(&cur[t], 1)] = s; });
    __syncthreads();
    if (tid == 0) {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        __stcg(cnt + 13, use_adj ? 1 : 0); __stcg(cnt + 14, n_adj); __stcg(cnt + 4, (int)((t1 - t_start) / 1000));   // us spent building the lists
    }

    // value change of the pixel in slot t (a -> b, NONE = invalid) -> histograms of the pending pixels whose region
    // holds it.
    //   phase 0 (inside the sweep of list k): pixels of list k that come after it in raster order
    //   phase 1 (commit, a == NONE):          pixels of list k before it, and every pixel of the other list
    auto touch = [&](int s, bool after, int a, int b, int k, int phase) {
        const int f = flg[s];
        if (f & VP_FLAG_DEAD) return;
        const int kk = s >= n0 ? 1 : 0;
        bool go;
        if (phase == 0) go = kk == k && after;
        else            go = (kk != k || !after) && val[s] == NONE;   // (pixels filled by this very sweep are leaving)
        if (!go) return;
        unsigned* h = hist + (size_t)s * HW;
        if constexpr (WIDE) {
            if (a < D) atomicSub(h + a, 1u);
            if (b < D) atomicAdd(h + b, 1u);
        } else {
            if (a < D) atomicSub(h + (a >> 1), 1u << ((a & 1) * 16));
            if (b < D) atomicAdd(h + (b >> 1), 1u << ((b & 1) * 16));
        }
        // (racecheck flags this byte: concurrent pushes may read and set the same slot's flag -- every writer stores the same
        //  value into its own byte and a reader that still sees 0 merely stores it again; the flags are consumed after a barrier)
        if (!(f & VP_FLAG_DIRTY)) flg[s] = (uint8_t)VP_FLAG_DIRTY;
    };
    auto push_adj = [&](int t, int a, int b, int k, int phase) {
        // (global-memory cursors were advanced by L2 atomics: read them at L2)
        const int e0 = t > 0 ? (state_smem ? cur[t - 1] : __ldcg(cur + t - 1)) : 0, e1 = state_smem ? cur[t] : __ldcg(cur + t);
        for (int e = e0 + lane; e < e1; e += 128) {          // four entries per lane per trip, loads first
            int v[4];
#pragma unroll
            for (int j = 0; j < 4; j++) v[j] = e + 32 * j < e1 ? adj[e + 32 * j] : -1;
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (v[j] >= 0) touch(v[j], v[j] > t, a, b, k, phase);
        }
    };
    // Fallback: inverse region by enumeration.  p' = (px,py) has q = (qx,qy) in R(p') iff the horizontal arm of
    // (px,qy) reaches qx and the vertical arm of (px,py) reaches qy.  Columns first, then four columns x three row
    // groups of candidates per trip (independent loads).
    auto push_enum = [&](int q, int a, int b, int k, int phase) {
        const int qy = q / W, qx = q - qy * W;
        int ncols = 0;
        for (int c0 = 0; c0 < R; c0 += 32) {
            const int px_l = qx - L1 + c0 + lane;
            bool cover = false;
            if (px_l >= 0 && px_l < W && c0 + lane < R) {
                const uchar2 ar = __ldg(ALR + qy * W + px_l);     // (left, right) of (px, qy)
                cover = px_l >= qx ? (px_l - qx <= (int)ar.x) : (qx - px_l <= (int)ar.y);
            }
            const unsigned m = __ballot_sync(0xffffffffu, cover);
            if (cover) cols[ncols + __popc(m & ((1u << lane) - 1u))] = (unsigned short)(c0 + lane);
            ncols += __popc(m);
        }
        __syncwarp();
        for (int c = 0; c < ncols; c += 4) {
            int px[4];
#pragma unroll
            for (int j = 0; j < 4; j++) px[j] = c + j < ncols ? qx - L1 + (int)cols[c + j] : -1;
            for (int r0 = 0; r0 < R; r0 += 96) {
                int slot[4][3];
#pragma unroll
                for (int t = 0; t < 3; t++) {
                    const int ro = r0 + 32 * t + lane, py = qy - L1 + ro;
                    const bool rok = ro < R && py >= 0 && py < H;
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        slot[j][t] = -1;
                        if (rok && px[j] >= 0) {
                            const uchar2 tb = __ldg(ATB + (size_t)px[j] * H + py);   // (top, bottom) of (px, py)
                            const bool cov = py >= qy ? (py - qy <= (int)tb.x) : (qy - py <= (int)tb.y);
                            if (cov) slot[j][t] = -2;
                        }
                    }
                }
#pragma unroll
                for (int t = 0; t < 3; t++) {
                    const int py = qy - L1 + r0 + 32 * t + lane;
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        if (slot[j][t] == -2) slot[j][t] = __ldg(pslotT + (size_t)px[j] * H + py);
                }
#pragma unroll
                for (int t = 0; t < 3; t++) {
                    const int py = qy - L1 + r0 + 32 * t + lane;
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        if (slot[j][t] >= 0) touch(slot[j][t], py > qy || (py == qy && px[j] > qx), a, b, k, phase);
                }
            }
        }
        __syncwarp();
    };

    auto vote = [&](const unsigned hv[], int nw) -> int {   // multistep_refiner.cpp:199-214 on the packed histogram words of this lane
        int peak = 0, best = 0x7fffffff, total = 0;
        for (int i = 0; i < nw; i++) {
            const int w2 = lane + 32 * i;
            if constexpr (WIDE) {
                const int c = (int)hv[i];
                if (peak < c) { peak = c; best = w2; }         // strict '<': the lowest disparity wins ties
                total += c;
            } else {
                const int c0 = (int)(hv[i] & 0xffffu), c1 = (int)(hv[i] >> 16);
                if (peak < c0) { peak = c0; best = 2 * w2; }       // strict '<': the lowest disparity wins ties
                if (peak < c1) { peak = c1; best = 2 * w2 + 1; }
                total += c0 + c1;
            }
        }
        const int gpeak = __reduce_max_sync(0xffffffffu, peak);
        const int gbest = __reduce_min_sync(0xffffffffu, peak == gpeak ? best : 0x7fffffff);
        total = __reduce_add_sync(0xffffffffu, total);
        if (gpeak > 0 && total > P.irv_ts && __fdiv_rn(__fmul_rn((float)gpeak, 1.0f), (float)total) > P.irv_th) return gbest;
        return NONE;
    };
    const int nhw = (HW + 31) / 32;   // histogram words per lane (<= NHW)
    // phase clock of thread 0 (diagnostics, adc_debug_counters): ns spent collecting / deriving / pushing
    // (kept in shared memory: only thread 0 touches them, and registers are short here)
    __shared__ unsigned long long s_clk[4];   // mark, collect, derive, push
    enum { ns_collect = 1, ns_derive = 2, ns_push = 3 };
    auto lap = [&](int acc) {
        if (tid == 0) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            s_clk[acc] += t - s_clk[0];
            s_clk[0] = t;
        }
    };
    if (tid == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        s_clk[0] = t; s_clk[1] = s_clk[2] = s_clk[3] = 0;
    }

    for (int it = 0; it < 5; it++) {
        for (int k = 0; k < 2; k++) {
            const int n = k == 0 ? n0 : n1, base = k == 0 ? 0 : n0;
            if (n == 0) continue;
            bool any_change = false;
            while (true) {
                __syncthreads();   // (everybody has read the previous round's counters)
                if (tid == 0) { s_nwork = 0; s_nchg = 0; }
                __syncthreads();
                // ---- collect the pixels of this list whose histogram changed since their last derive
                for (int i0 = 0; i0 < n; i0 += VP_THREADS) {
                    const int i = i0 + tid;
                    const bool d = i < n && (flg[base + i] & VP_FLAG_DIRTY);
                    if (d) flg[base + i] = 0;
                    const unsigned m = __ballot_sync(0xffffffffu, d);
                    int o = 0;
                    if (lane == 0 && m) o = atomicAdd(&s_nwork, __popc(m));
                    o = __shfl_sync(0xffffffffu, o, 0);
                    if (d) work[o + __popc(m & ((1u << lane) - 1u))] = base + i;
                }
                __syncthreads();
                lap(ns_collect);
                const int nwork = s_nwork;
                if (nwork == 0) break;
                rounds_total++;
                // ---- derive: vote of every such pixel from its histogram, four pixels per trip (their loads in flight together)
                for (int t = 4 * wid; t < nwork; t += 4 * VP_WARPS) {
                    int sl[4];
                    unsigned hv[4][NHW];
#pragma unroll
                    for (int u = 0; u < 4; u++) sl[u] = work[min(t + u, nwork - 1)];
#pragma unroll
                    for (int u = 0; u < 4; u++) {
#pragma unroll
                        for (int j = 0; j < NHW; j++) {
                            const int w2 = lane + 32 * j;
                            hv[u][j] = (j < nhw && w2 < HW) ? __ldcg(hist + (size_t)sl[u] * HW + w2) : 0u;
                        }
                    }
                    int r[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) r[u] = vote(hv[u], nhw);
                    if (lane == 0) {
#pragma unroll
                        for (int u = 0; u < 4; u++) {
                            if (t + u >= nwork) break;
                            derives++;
                            const int a = val[sl[u]];
                            if (r[u] != a) {
                                val[sl[u]] = (VT)r[u];
                                chg[atomicAdd(&s_nchg, 1)] = make_int2(sl[u], a | (r[u] << VB));
                            }
                        }
                    }
                }
                __syncthreads();
                lap(ns_derive);
                const int nchg = s_nchg;
                if (nchg == 0) break;
                any_change = true;
                changes += nchg;
                // ---- push the changes into the histograms of the later pixels of this list
                for (int t = wid; t < nchg; t += VP_WARPS) {
                    const int2 c = chg[t];
                    if (use_adj) push_adj(c.x, c.y & NONE, (c.y >> VB) & NONE, k, 0);
                    else         push_enum(pix(c.x), c.y & NONE, (c.y >> VB) & NONE, k, 0);
                }
                __syncthreads();
                lap(ns_push);
            }
            if (!any_change) continue;   // nothing moved in this sweep (uniform across the CTA)
            // ---- commit: the pixels filled by this sweep become visible to everybody and leave the list
            __syncthreads();
            if (tid == 0) s_nchg = 0;
            __syncthreads();
            for (int i0 = 0; i0 < n; i0 += VP_THREADS) {
                const int i = i0 + tid;
                bool f = false;
                int v = NONE;
                if (i < n && !(flg[base + i] & VP_FLAG_DEAD)) { v = val[base + i]; f = v != NONE; }
                const unsigned m = __ballot_sync(0xffffffffu, f);
                int o = 0;
                if (lane == 0 && m) o = atomicAdd(&s_nchg, __popc(m));
                o = __shfl_sync(0xffffffffu, o, 0);
                if (f) {
                    const int p = pix(base + i);
                    const float fv = (float)(v + dm.dmin);
                    d_old[p] = fv;
                    d_new[p] = fv;
                    lab[p] = 0;
                    chg[o + __popc(m & ((1u << lane) - 1u))] = make_int2(base + i, p);
                }
            }
            __syncthreads();
            const int ncommit = s_nchg;
            changes += ncommit;
            for (int t = wid; t < ncommit; t += VP_WARPS) {
                const int2 c = chg[t];
                if (use_adj) push_adj(c.x, NONE, (int)val[c.x], k, 1);
                else         push_enum(c.y, NONE, (int)val[c.x], k, 1);
            }
            __syncthreads();
            for (int t = tid; t < ncommit; t += VP_THREADS) flg[chg[t].x] = (uint8_t)VP_FLAG_DEAD;
            __syncthreads();
        }
    }
    derives = __reduce_add_sync(0xffffffffu, lane == 0 ? derives : 0);
    if (lane == 0) atomicAdd(cnt + 3, derives);
    if (tid == 0) {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        __stcg(cnt + 2, rounds_total); __stcg(cnt + 12, changes);
        __stcg(cnt + 5, (int)((t1 - t_start) / 1000)); __stcg(cnt + 6, (int)(s_clk[ns_derive] / 1000));      // us: whole kernel, derive phases,
        __stcg(cnt + 7, (int)(s_clk[ns_push] / 1000)); __stcg(cnt + 8, (int)(s_clk[ns_collect] / 1000));             // push phases, collect phases
    }
}

// The histograms (ns * HW <= N * D words), forward lists and adjacency lists live in w.vote_hist, the idle cost volume.
template <bool WIDE>
static void launch_scan_push(const AdcParams& P, const AdcWave& w, int L1, int force_enum, cudaStream_t st) {
    const AdcDims& dm = P.dm;
    unsigned* hist = w.vote_hist;
    int gx = (adc_sm_count() * 8 + w.S - 1) / w.S;
    if (gx < 1) gx = 1;
    dim3 igrid(gx, w.S);
    k_vote_scan<WIDE><<<igrid, VI_WARPS * 32, 0, st>>>(P, w.arms, w.vote_alr, w.vote_state, w.sup_h, w.vlist, w.counters,
                                                       hist, dm.vol_stride, force_enum);
    const int cols_cap = (2 * L1 + 1 + 7) / 8 * 8;
    // shared memory: column lists (fallback), then val / flg / cur for as many slots as fit
    const size_t fixed = (size_t)VP_WARPS * cols_cap * 2;
    const size_t slot_bytes = sizeof(VoteVal<WIDE>) + 1 + 4;
    int slot_cap = (int)((220 * 1024 - fixed - 16) / slot_bytes) & ~15;
    if (slot_cap > VP_SMEM_SLOTS) slot_cap = VP_SMEM_SLOTS;
    if ((P.dbg & 4) && slot_cap > 256) slot_cap = 256;   // ADC_DBG_VOTE_GLOBAL_STATE: global-memory copy of the per-slot state (tests)
    const size_t smem = fixed + (slot_bytes - 4) * (size_t)slot_cap + ((size_t)slot_cap + 1) * 4;
    static AdcOnce attr_once;
    if (adc_once_needed(attr_once)) {
        cudaFuncSetAttribute(k_vote_push<WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 222 * 1024);   // (+ static < 227 KB)
        adc_once_done(attr_once);
    }
    k_vote_push<WIDE><<<w.S, VP_THREADS, smem, st>>>(P, w.vote_alr, w.vote_atbT, w.vote_pslotT, hist, dm.vol_stride, w.vote_off,
                                                     reinterpret_cast<VoteVal<WIDE>*>(w.vote_val), w.vote_dirtyb, w.vlist,
                                                     w.counters, w.vote_work, w.vote_chg, w.disp_l, w.disp_t, w.label,
                                                     cols_cap, slot_cap, force_enum);
}

// Region voting for every D and L1: the active lists, the state maps, the incremental histograms, then the outlier lists
// rebuilt from the labels (every listed pixel that is still invalid).  disp_l = committed state, disp_t = working copy;
// both hold the post-outlier map here.
void adc_launch_voting(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches) {
    const AdcDims& dm = P.dm;
    const int L1 = P.L1 > 0 ? P.L1 : 0;
    adc_launch_active_lists(P, w, st, launches);
    dim3 egrid((dm.N + 255) / 256, w.S);
    k_vote_encode<<<egrid, 256, 0, st>>>(dm, w.disp_l, w.arms, w.vote_alr, w.vote_state);
    cudaMemsetAsync(w.vote_pslotT, 0xff, (size_t)w.S * dm.N * sizeof(int), st);
    dim3 tgrid((dm.W + 31) / 32, (dm.H + 31) / 32, w.S);
    k_vote_transpose<<<tgrid, 256, 0, st>>>(dm, w.arms, w.vote_atbT);
    dim3 sgrid(64, w.S);
    k_vote_slots<<<sgrid, 256, 0, st>>>(dm, w.vlist, w.counters, w.vote_state, w.vote_pslotT, w.sup_h);
    // ADC_DBG_VOTE_ENUM forces the enumeration fallback (tests); L1 > 127 takes it always (the support counts may wrap)
    const int force_enum = (P.dbg & 2) || L1 > 127 ? 1 : 0;
    if (dm.D > 254 || L1 > 127) launch_scan_push<true>(P, w, L1, force_enum, st);
    else                        launch_scan_push<false>(P, w, L1, force_enum, st);
    *launches += 5;
    adc_launch_build_lists(P, w, st, launches);
}
