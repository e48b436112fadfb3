// k_scanline.cu -- stage 3: the four chained scanline-optimisation passes
// (reference: scanline_optimizer.cpp:40-61 sequencing, :63-171 horizontal, :173-279 vertical).
//
// One warp owns one scanline (a row for the +-x passes, a column for the +-y passes) and walks it
// serially; the D disparities of a pixel are spread over the 32 lanes, K consecutive ones per
// lane, and live in registers from one step to the next.  Per step the recurrence is
//     L(d) = ( C(d) + min( Lp(d), Lp(d-1)+P1, Lp(d+1)+P1, minLp+P2 ) ) / 2
// (no "- minLp" term, and a "/2": scanline_optimizer.cpp:144-151), with Lp padded by Large_Float
// on both ends and the running minimum taken over the pads too (:96,:107-110).  Neighbour values
// cross lanes through two shuffles; the minimum over d is one REDUX on order-preserving integer
// keys.  Only add/min/exact scalings occur, so the result is bit-identical to the CPU path.
//
// Memory system: everything a step needs that does not depend on the recurrence -- the pixel's
// cost vector (Dp floats) and a small "penalty record" -- is streamed into a per-warp shared
// memory ring by the TMA engine: one tensor copy brings the costs of the warp's lines for T
// consecutive steps, a second one their records, so HBM/L2 latency never sits on the serial
// chain and the number of bytes in flight per SM is set by the ring depth, not by register
// scoreboards.
//
// Penalty record.  P1/P2 depend on d1 = Dc(left[p], left[p_prev]) and d2 = Dc(right[xr],
// right[xr_prev]) with xr = x - d - dmin, through (d1 < tso, d2 < tso).  The reference declares d2
// once per pixel (initialised to d1) and only overwrites it while 0 < xr < W-1, so for
// disparities past the valid interval it keeps the value of the last valid one ("sticky d2",
// :116-121).  Closed form: valid d form [lo,hi] = [max(0,x-dmin-(W-2)), min(D-1,x-dmin-1)];
// d<lo -> d1, d in [lo,hi] -> map(x-d-dmin), d>hi -> map(x-hi-dmin), empty interval -> d1.
// k_so_records folds all of that into, per pixel, one word (d1 < tso) and a D-bit string
// (bit d = d2(d) < tso); the bit string is a window of a per-row bit vector of the right image
// stored mirrored, so that increasing d walks increasing bit positions.
#include "adc_common.cuh"
#include "so_plan.h"
#include <cuda.h>     // CUtensorMap and its enums only: the encoder is fetched through the runtime
#include <string.h>

template <int K>
struct Piece { static constexpr int G = (K % 4 == 0) ? 4 : ((K % 2 == 0) ? 2 : 1); static constexpr int NP = K / G; };

template <int K>
__device__ __forceinline__ void ld_vec(const float* p, int lane, int Dp, float (&v)[K]) {   // generic/shared pointer
    constexpr int G = Piece<K>::G, NP = Piece<K>::NP;
#pragma unroll
    for (int j = 0; j < NP; j++) {
        const int d = lane * K + j * G;
        if (d < Dp) {
            if (G == 4) { const float4 t = *reinterpret_cast<const float4*>(p + d); v[j*G] = t.x; v[j*G+1] = t.y; v[j*G+2] = t.z; v[j*G+3] = t.w; }
            else if (G == 2) { const float2 t = *reinterpret_cast<const float2*>(p + d); v[j*G] = t.x; v[j*G+1] = t.y; }
            else v[j] = p[d];
        } else {
#pragma unroll
            for (int g = 0; g < G; g++) v[j * G + g] = 0.f;
        }
    }
}

template <int K>
__device__ __forceinline__ void st_vec(float* __restrict__ p, int lane, int Dp, const float (&v)[K]) {
    constexpr int G = Piece<K>::G, NP = Piece<K>::NP;
#pragma unroll
    for (int j = 0; j < NP; j++) {
        const int d = lane * K + j * G;
        if (d < Dp) {
            if (G == 4) *reinterpret_cast<float4*>(p + d) = make_float4(v[j*G], v[j*G+1], v[j*G+2], v[j*G+3]);
            else if (G == 2) *reinterpret_cast<float2*>(p + d) = make_float2(v[j*G], v[j*G+1]);
            else p[d] = v[j];
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Bit rows of the right image: for variant v in {h-fwd, h-bwd, v-fwd, v-bwd}, bit(xr) of row y says
// whether the colour distance between right(y,xr) and its predecessor along the path is < tso.
// Stored mirrored: bit j of the row holds xr = W-1-j.
// ---------------------------------------------------------------------------------------------
__host__ __device__ inline int so_row_words(int W) { return (W + 31) / 32 + 2; }

__global__ void __launch_bounds__(128)
k_so_bitrows(AdcDims dm, int tso, const uint8_t* __restrict__ dmap, unsigned* __restrict__ bitrows) {
    const int pair = blockIdx.y, y = blockIdx.x;
    const int W = dm.W, rw = so_row_words(W);
    const uint8_t* mh = dmap + ((size_t)pair * 4 + 2) * dm.N;   // right image, distance to (y, x-1)
    const uint8_t* mv = dmap + ((size_t)pair * 4 + 3) * dm.N;   // right image, distance to (y-1, x)
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;  // warp = variant
    unsigned* out = bitrows + (((size_t)pair * 4 + wid) * dm.H + y) * rw;
    for (int w0 = 0; w0 < rw; w0++) {
        const int j = w0 * 32 + lane;
        const int xr = W - 1 - j;
        bool bit = false;
        if (xr > 0 && xr < W - 1) {   // the only positions the reference ever looks at (scanline_optimizer.cpp:120)
            int v;
            if (wid == 0) v = mh[y * W + xr];                 // +x pass: right[xr] vs right[xr-1]
            else if (wid == 1) v = mh[y * W + xr + 1];        // -x pass: right[xr] vs right[xr+1]
            else if (wid == 2) v = y > 0 ? mv[y * W + xr] : 255;            // +y pass: row y vs y-1 (never a path head's successor at y=0)
            else v = y + 1 < dm.H ? mv[(y + 1) * W + xr] : 255;             // -y pass: row y vs y+1
            bit = v < tso;
        }
        const unsigned m = __ballot_sync(0xffffffffu, bit);
        if (lane == 0) out[w0] = m;
    }
}

// per-pixel record for one pass direction (so_rec_words, so_plan.h)
// (one launch writes the records of all four pass directions, blockIdx.z = direction)
__global__ void __launch_bounds__(256)
k_so_records(AdcDims dm, int tso, const uint8_t* __restrict__ dmap,
             const unsigned* __restrict__ bitrows, unsigned* __restrict__ rec) {
    const int pair = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dm.N) return;
    const int sx = blockIdx.z == 0 ? 1 : (blockIdx.z == 1 ? -1 : 0);
    const int sy = blockIdx.z == 2 ? 1 : (blockIdx.z == 3 ? -1 : 0);
    const int W = dm.W, D = dm.D, dmin = dm.dmin;
    const int y = i / W, x = i - y * W;
    const bool fwd = (sx + sy) > 0;
    const int pstep = sx + sy * W;
    const int variant = sx ? (fwd ? 0 : 1) : (fwd ? 2 : 3);
    const int rw = so_row_words(W), nrec = so_rec_words(dm.Dp);
    unsigned* out = rec + (((size_t)pair * 4 + variant) * dm.N + i) * nrec;
    // d1: this pixel vs the one the path came from (undefined for path heads, which never use it)
    const uint8_t* ml = dmap + ((size_t)pair * 4 + (sx ? 0 : 1)) * dm.N;
    const int pi_from = i - pstep;
    int d1 = 0;
    if (fwd) d1 = ml[i];
    else if (pi_from >= 0 && pi_from < dm.N) d1 = ml[pi_from];
    const unsigned a1 = d1 < tso ? 0xffffffffu : 0u;
    const int lo = max(0, x - dmin - (W - 2));
    const int hi = min(D - 1, x - dmin - 1);
    const unsigned* row = bitrows + (((size_t)pair * 4 + variant) * dm.H + y) * rw;
    const int j0 = W - 1 - x + dmin;           // bit position of d = 0  (xr = x - dmin)
    auto window = [&](int d0) -> unsigned {     // bits d0..d0+31 of the string, 0 where out of the row
        const int j = j0 + d0;                   // |j| < W + D + 64: plain int
        const int wlo = j >> 5;                  // arithmetic shift = floor division also for negative j
        const int sh = j & 31;
        const unsigned a = (wlo >= 0 && wlo < rw) ? row[wlo] : 0u;
        const unsigned b = (wlo + 1 >= 0 && wlo + 1 < rw) ? row[wlo + 1] : 0u;
        return __funnelshift_r(a, b, sh);
    };
    unsigned fill_hi = a1;
    if (lo <= hi) fill_hi = (window(hi) & 1u) ? 0xffffffffu : 0u;
    const int nw = (dm.Dp + 31) / 32 + 1;
    auto word = [&](int w0) -> unsigned {
        if (lo > hi) return a1;
        const int d0 = w0 * 32;
        const unsigned raw = window(d0);
        // masks of the bits with d < lo and d > hi inside this word
        const unsigned m_lo = lo <= d0 ? 0u : (lo >= d0 + 32 ? 0xffffffffu : ((1u << (lo - d0)) - 1u));
        const unsigned m_hi = hi >= d0 + 31 ? 0u : (hi < d0 ? 0xffffffffu : ~((2u << (hi - d0)) - 1u));
        return (raw & ~m_lo & ~m_hi) | (a1 & m_lo) | (fill_hi & m_hi);
    };
    if (nrec == 4) {   // D <= 64: the whole record is one 128-bit store
        *reinterpret_cast<uint4*>(out) = make_uint4(a1, word(0), nw > 1 ? word(1) : 0u, nw > 2 ? word(2) : 0u);
        return;
    }
    out[0] = a1;
    for (int w0 = 0; w0 < nw; w0++) out[1 + w0] = word(w0);
    for (int w0 = 1 + nw; w0 < nrec; w0++) out[w0] = 0u;
}

// ---------------------------------------------------------------------------------------------
// The serial kernel.  A group of LPS lanes (8, 16 or 32) owns one scanline and keeps K = Dp/LPS
// consecutive disparities per lane, so a warp advances 32/LPS neighbouring scanlines in lockstep.
// Fewer lanes per line = more disparities per lane = the per-step bookkeeping (barriers, copy
// issue, neighbour shuffles, the min butterfly) is amortised over more cost values; the kernel
// was issue-bound with 2 values per lane.
//
// Ring: NS slots per warp, slot k holding steps kT .. kT+T-1 of all the warp's lines.  The volume
// is described as a 4-D tensor [S][H][W][Dp] and the records as [4S][H][W][nrec], so a box
// {Dp, T steps, LPW rows} (+-x passes) or {Dp, LPW columns, T rows} (+-y passes) is one tensor copy;
// positions outside the pair's image (a partial last slot, a warp's dead lines) are zero-filled by
// the hardware, never read from the neighbouring pair.  A backward pass fetches the box that ends
// at its step and walks it in reverse.
__device__ __forceinline__ unsigned so_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
    unsigned ok, spins = 0;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (!ok && ++spins > (1u << 24)) __trap();   // a copy that never completes is a bug: fail the launch instead of hanging the device
    } while (!ok);
}
__device__ __forceinline__ void tma_load_4d(unsigned dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, unsigned bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                 ::"r"(dst), "l"(reinterpret_cast<unsigned long long>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
                 : "memory");
}

// WTA: the last pass (-y) with the winner-takes-all as its epilogue (DESIGN.md 5.5).  It stores no volume: each warp
// overwrites the costs of a step in its ring slot with the step's L, takes the left view's first minimum of each of its
// columns from the registers, and once all warps of the CTA have finished a slot, the CTA reads the slot's rows along the
// right view's diagonals and writes one partial record per (row, right pixel) to dst (so_plan.h).  The slot is refilled
// only after that.
template <int K, int LPS, bool FULL, bool WTA>   // FULL: D == LPS*K, every lane's K values are real disparities (no padding logic)
__device__ __forceinline__ void so_pass(const CUtensorMap& tm_cost, const CUtensorMap& tm_rec, const AdcParams& P,
                                        float* __restrict__ dst, float* __restrict__ disp_l, int sx, int sy, int T, int NS) {
    constexpr int LPW = 32 / LPS;               // lines per warp
    if constexpr (WTA) { sx = 0; sy = -1; }
    extern __shared__ __align__(128) unsigned char so_smem[];
    const AdcDims& dm = P.dm;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int sub = lane / LPS, gl = lane % LPS;   // line within the warp, lane within the line's group
    const int line0 = (blockIdx.x * SO_WARPS + wid) * LPW;   // first line of this warp
    const int line = line0 + sub;
    const int pair = blockIdx.y;
    const int n_lines = sx ? dm.H : dm.W, n_steps = sx ? dm.W : dm.H;
    if (line0 >= n_lines) return;                // a warp of the grid's last CTA without lines: no copies, no barriers
    const bool live = line < n_lines;            // dead groups run along (uniform control flow) but store nothing
    // FULL: D == Dp == K * LPS is known at compile time, and with it every size below
    const int W = dm.W, D = FULL ? K * LPS : dm.D, Dp = FULL ? K * LPS : dm.Dp;
    const int pstep = sx + sy * W;               // signed pixel stride along the path
    const int nrec = so_rec_words(Dp);
    const bool fwd = sx + sy > 0;
    const int variant = sx ? (sx > 0 ? 0 : 1) : (sy > 0 ? 2 : 3);
    const unsigned cost_region = so_cost_region(Dp, T), slot_bytes = so_slot_bytes(Dp, T);
    unsigned char* wring = so_smem + (size_t)wid * NS * slot_bytes;
    const unsigned bar0 = so_smem_u32(so_smem + (size_t)SO_WARPS * NS * slot_bytes) + (unsigned)(wid * NS) * 8u;
    const unsigned tx = (unsigned)(T * LPW * (Dp + nrec) * 4);   // a box's bytes count in full, zero-filled positions too
    const int nch = (n_steps + T - 1) / T;       // slots' worth of steps; the last one may be partial

    auto issue = [&](int c) {   // lane 0: steps cT .. cT+T-1 of the warp's lines into slot c % NS
        const int s = c % NS;
        const unsigned bar = bar0 + 8u * (unsigned)s, d0 = so_smem_u32(wring + (size_t)s * slot_bytes);
        const int p0 = fwd ? c * T : n_steps - (c + 1) * T;   // first box position along the path
        mbar_expect_tx(bar, tx);
        if (sx) {
            tma_load_4d(d0, &tm_cost, 0, p0, line0, pair, bar);
            tma_load_4d(d0 + cost_region, &tm_rec, 0, p0, line0, pair * 4 + variant, bar);
        } else {
            tma_load_4d(d0, &tm_cost, 0, line0, p0, pair, bar);
            tma_load_4d(d0 + cost_region, &tm_rec, 0, line0, p0, pair * 4 + variant, bar);
        }
    };
    if (lane == 0) {
        for (int j = 0; j < NS; j++) mbar_init(bar0 + 8u * j, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int c = 0; c < NS && c < nch; c++) issue(c);
    }
    __syncwarp();

    // The step being read is step t of chunk c, in ring slot `slot`, whose mbarrier completes phase `phase` for it.
    int c = 0, t = 0, slot = 0;
    unsigned phase = 0;
    const int bit0 = gl * K;   // first disparity of this lane inside the record's bit string
    auto fetch = [&](float (&C)[K], bool& a1, unsigned& bits) -> float* {   // returns the step's row of costs in the slot
        if (t == 0) mbar_wait(bar0 + 8u * (unsigned)slot, phase);
        const int pos = fwd ? t : T - 1 - t;
        const int row = sx ? sub * T + pos : pos * LPW + sub;   // box {Dp, T, LPW} or {Dp, LPW, T}
        unsigned char* sl = wring + (size_t)slot * slot_bytes;
        float* cs = reinterpret_cast<float*>(sl) + row * Dp;
        if constexpr (FULL && K == 8) {
            // a lane's eight costs are two 16-byte chunks 32 bytes apart: the lanes of a 128-bit load phase would hit four bank
            // groups twice, so lanes with (gl >> 2) & 1 read their second chunk first -- eight different bank groups per phase
            const int b = (gl >> 2) & 1;
            const float4 u = *reinterpret_cast<const float4*>(cs + 8 * gl + 4 * b);
            const float4 v = *reinterpret_cast<const float4*>(cs + 8 * gl + 4 - 4 * b);
            const float4 lo = b ? v : u, hi = b ? u : v;
            C[0] = lo.x; C[1] = lo.y; C[2] = lo.z; C[3] = lo.w;
            C[4] = hi.x; C[5] = hi.y; C[6] = hi.z; C[7] = hi.w;
        } else ld_vec<K>(cs, gl, Dp, C);
        const unsigned* rw = reinterpret_cast<const unsigned*>(sl + cost_region) + row * nrec;
        a1 = rw[0] != 0u;
        bits = __funnelshift_r(rw[1 + (bit0 >> 5)], rw[2 + (bit0 >> 5)], bit0 & 31);
        if (!WTA && ++t == T) {   // WTA: the slot is advanced by wta_advance, after the CTA has read it
            // Every lane has read the slot before it is refilled.  The refill is a write of the ASYNC proxy (the TMA engine),
            // the reads above went through the generic proxy: each lane orders its reads against that proxy before the
            // barrier (DESIGN.md 5.3: without the proxy fence pairs of a loaded GPU came out wrong).
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0 && c + NS < nch) issue(c + NS);
            t = 0;
            c++;
            if (++slot == NS) { slot = 0; phase ^= 1u; }
        }
        return cs;
    };

    bool valid[K];
#pragma unroll
    for (int k = 0; k < K; k++) valid[k] = FULL || (gl * K + k) < D;

    // ---- WTA epilogue (WTA only; step s of the pass is image row H - 1 - s)
    // the CTA's warps that own columns: they alone take part in its barriers
    const int wta_threads = 32 * min(SO_WARPS, (n_lines - (int)blockIdx.x * SO_WARPS * LPW + LPW - 1) / LPW);
    // Left view of this group's column: the first minimum over d is the lowest d holding the group's minimum m (the
    // reference's strict '>' scan from Large_Float, ADCensusStereo.cpp:209-222); its neighbours are read from the row.
    auto wta_left = [&](const float* row, const float (&V)[K], float m, int step) {
        int kk = K;
#pragma unroll
        for (int k = K - 1; k >= 0; k--)
            if (valid[k] && V[k] == m) kk = k;
        const unsigned bal = __ballot_sync(0xffffffffu, kk < K);
        const unsigned grp = LPS == 32 ? bal : (bal >> (sub * LPS)) & ((1u << LPS) - 1u);
        __syncwarp();   // the row's values stored by the other lanes
        if (live && gl == __ffs(grp) - 1) {
            const int bd = gl * K + kk;
            float out = ADC_INVALID_F;   // a minimum at either end of the range (or none) is Invalid (:224-227)
            if (m < ADC_LARGE_F && bd > 0 && bd < D - 1) out = adc_subpixel(row[bd - 1], row[bd + 1], m, dm.dmin + bd);
            disp_l[(size_t)pair * dm.N + (size_t)(dm.H - 1 - step) * W + line] = out;
        }
    };
    // Right view: cost_R(xr, d) = cost(xr + dmin + d, d).  For each step of the slot and each right pixel whose diagonal
    // crosses the band, the first minimum over the diagonal's d-range inside the band, its in-range neighbours and the
    // range's first and last cost (the fields of so_plan.h; k_wta_merge folds them).
    auto wta_records = [&](int nt, int s0) {
        constexpr int CB = SO_WARPS * LPW;   // band width
        const int x0 = blockIdx.x * CB, NJ = CB + D - 1, nb = (W + CB - 1) / CB, dmin = dm.dmin;
        const long long plane = (long long)dm.H * nb * NJ;
        float* R = dst + (size_t)pair * dm.vol_stride;
        const size_t wstride = (size_t)NS * slot_bytes / 4;   // floats between two warps' rings
        const int xcap = W - 1 - x0;                           // the band's last column inside the image
        for (int tt = 0; tt < nt; tt++) {
            const int y = dm.H - 1 - (s0 + tt);
            const float* rb = reinterpret_cast<const float*>(so_smem + (size_t)slot * slot_bytes) + (T - 1 - tt) * LPW * Dp;
            for (int j = threadIdx.x; j < NJ; j += wta_threads) {
                const int xr = x0 - dmin - (D - 1) + j;
                const int ilo = max(0, j - (D - 1)), ihi = min(min(CB - 1, j), xcap);   // band columns on the diagonal
                if (xr < 0 || xr >= W || ilo > ihi) continue;
                const int dd0 = D - 1 - j;                                              // d of band column i: i + dd0
                auto at = [&](int i) { return rb[(size_t)(i / LPW) * wstride + (i % LPW) * Dp + i + dd0]; };
                float m = ADC_LARGE_F;
                int a = -1;
                const float* pw = rb + dd0;   // band column i = w * LPW + s sits at pw + w * (wstride + LPW) + s * (Dp + 1)
#pragma unroll 1
                for (int w = 0; w < SO_WARPS; w++, pw += wstride + LPW) {
                    const float* p = pw;
#pragma unroll
                    for (int s = 0; s < LPW; s++, p += Dp + 1) {
                        const int i = w * LPW + s;
                        if (i >= ilo && i <= ihi) {
                            const float v = *p;
                            if (m > v) { m = v; a = i; }
                        }
                    }
                }
                const long long r = ((long long)y * nb + blockIdx.x) * NJ + j;
                R[r] = m;
                R[plane + r] = __int_as_float(a < 0 ? -1 : a + dd0);
                R[2 * plane + r] = a > ilo ? at(a - 1) : ADC_LARGE_F;
                R[3 * plane + r] = a >= 0 && a < ihi ? at(a + 1) : ADC_LARGE_F;
                R[4 * plane + r] = at(ilo);
                R[5 * plane + r] = at(ihi);
            }
        }
    };
    // after step `step`: at the end of a slot (or of the pass) the CTA takes the slot's records, then the slot is refilled
    auto wta_advance = [&](int step) {
        if (++t < T && step + 1 < n_steps) return;
        asm volatile("bar.sync 1, %0;" ::"r"(wta_threads) : "memory");   // every warp's rows of the slot are stored
        wta_records(t, step + 1 - t);
        // the refill is a write of the async proxy after generic reads and writes of the slot (see fetch)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("bar.sync 1, %0;" ::"r"(wta_threads) : "memory");   // nobody reads the slot any more
        if (lane == 0 && c + NS < nch) issue(c + NS);
        t = 0;
        c++;
        if (++slot == NS) { slot = 0; phase ^= 1u; }
    };

    // the path head: L = C  (scanline_optimizer.cpp:99-100)
    long long pi = (long long)(sy ? (sy > 0 ? 0 : dm.H - 1) : line) * W + (sx ? (sx > 0 ? 0 : W - 1) : line);
    float* O = dst + (size_t)pair * dm.vol_stride;
    float L[K];
    float* row;
    {
        bool a1;
        unsigned bits;
        row = fetch(L, a1, bits);
    }
    if (!WTA && live) st_vec<K>(O + (size_t)pi * Dp, gl, Dp, L);
    float minL = ADC_LARGE_F;
#pragma unroll
    for (int k = 0; k < K; k++) {
        if (!valid[k]) L[k] = ADC_LARGE_F;
        minL = fminf(minL, L[k]);
    }
#pragma unroll
    for (int o = LPS / 2; o >= 1; o >>= 1) minL = fminf(minL, __shfl_xor_sync(0xffffffffu, minL, o));
    if constexpr (WTA) {   // the head's row in the slot holds L already
        wta_left(row, L, minL, 0);
        wta_advance(0);
    }

    for (int step = 1; step < n_steps; step++) {
        float C[K];
        bool a1;
        unsigned bits;
        row = fetch(C, a1, bits);
        pi += pstep;

        const float up = __shfl_up_sync(0xffffffffu, L[K - 1], 1, LPS);
        const float down = __shfl_down_sync(0xffffffffu, L[0], 1, LPS);
        const float left_in = gl == 0 ? ADC_LARGE_F : up;
        const float right_in = gl == LPS - 1 ? ADC_LARGE_F : down;
        // the three penalty classes of this pixel's left-image term (scanline_optimizer.cpp:129-141)
        const float P1a = a1 ? P.p1 : P.p1_4, P1b = a1 ? P.p1_4 : P.p1_10;   // d2 < tso  /  d2 >= tso
        const float P2a = a1 ? P.p2 : P.p2_4, P2b = a1 ? P.p2_4 : P.p2_10;
        const float m4a = __fadd_rn(minL, P2a), m4b = __fadd_rn(minL, P2b);

        float Ln[K];
        float mn = ADC_LARGE_F;
#pragma unroll
        for (int k = 0; k < K; k++) {
            const bool a2 = (bits >> k) & 1u;
            const float P1 = a2 ? P1a : P1b;
            const float l1 = L[k];
            const float l2 = __fadd_rn(k > 0 ? L[k - 1] : left_in, P1);
            const float l3 = __fadd_rn(k < K - 1 ? L[k + 1] : right_in, P1);
            const float l4 = a2 ? m4a : m4b;
            float v = __fadd_rn(C[k], fminf(fminf(l1, l2), fminf(l3, l4)));
            v = __fmul_rn(v, 0.5f);
            Ln[k] = v;
            if (valid[k]) mn = fminf(mn, v);
        }
        if constexpr (WTA) {
            if constexpr (FULL && K == 8) {   // the bank-group order of fetch's loads
                const int b = (gl >> 2) & 1;
                const float4 lo = make_float4(Ln[0], Ln[1], Ln[2], Ln[3]), hi = make_float4(Ln[4], Ln[5], Ln[6], Ln[7]);
                *reinterpret_cast<float4*>(row + 8 * gl + 4 * b) = b ? hi : lo;
                *reinterpret_cast<float4*>(row + 8 * gl + 4 - 4 * b) = b ? lo : hi;
            } else st_vec<K>(row, gl, Dp, Ln);
        } else if (live) st_vec<K>(O + (size_t)pi * Dp, gl, Dp, Ln);
#pragma unroll
        for (int k = 0; k < K; k++) L[k] = valid[k] ? Ln[k] : ADC_LARGE_F;
#pragma unroll
        for (int o = LPS / 2; o >= 1; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        minL = mn;
        if constexpr (WTA) {
            wta_left(row, Ln, mn, step);
            wta_advance(step);
        }
    }
}

template <int K, int LPS, bool FULL>
__global__ void __launch_bounds__(SO_WARPS * 32, SO_MIN_CTAS)
k_scanline(const __grid_constant__ CUtensorMap tm_cost, const __grid_constant__ CUtensorMap tm_rec, AdcParams P,
           float* __restrict__ dst, int sx, int sy, int T, int NS) {
    so_pass<K, LPS, FULL, false>(tm_cost, tm_rec, P, dst, nullptr, sx, sy, T, NS);
}

template <int K, int LPS, bool FULL>   // the -y pass; rec = the right view's records
__global__ void __launch_bounds__(SO_WARPS * 32, SO_MIN_CTAS)
k_scanline_wta(const __grid_constant__ CUtensorMap tm_cost, const __grid_constant__ CUtensorMap tm_rec, AdcParams P,
               float* __restrict__ rec, float* __restrict__ disp_l, int T, int NS) {
    so_pass<K, LPS, FULL, true>(tm_cost, tm_rec, P, rec, disp_l, 0, -1, T, NS);
}

// The fused pass exists only where its records can fit a pair's volume for some shape adc_create accepts
// (so_wta_fused): never with 32 lanes per line (a band of 4 columns), nor at D = 8 (K = 1, FULL).
// tests/test_fused_wta_parity.py derives that set over the whole domain and compares it with the library's kernels.
template <int K, int LPS, bool FULL>
constexpr bool so_wta_built() { return LPS != 32 && !(K == 1 && FULL); }

template <int K, int LPS, bool FULL, bool WTA>
static int launch_scanline_kf(const AdcParams& P, const AdcWave& w, const CUtensorMap& tc, const CUtensorMap& tr,
                              int T, int NS, size_t smem, float* dst, int sx, int sy, cudaStream_t st) {
    if constexpr (WTA && !so_wta_built<K, LPS, FULL>()) {
        return 1;
    } else {
        constexpr int LPW = 32 / LPS;
        const int n_lines = sx ? P.dm.H : P.dm.W;
        const void* fn;
        if constexpr (WTA) fn = (const void*)k_scanline_wta<K, LPS, FULL>;
        else fn = (const void*)k_scanline<K, LPS, FULL>;
        static AdcOnce attr_once;
        if (adc_once_needed(attr_once)) {
            cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, SO_SMEM_MAX);
            cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            adc_once_done(attr_once);
        }
        const int lines_per_block = SO_WARPS * LPW;
        dim3 grid((n_lines + lines_per_block - 1) / lines_per_block, w.S);
        if constexpr (WTA) k_scanline_wta<K, LPS, FULL><<<grid, SO_WARPS * 32, smem, st>>>(tc, tr, P, dst, w.disp_l, T, NS);
        else k_scanline<K, LPS, FULL><<<grid, SO_WARPS * 32, smem, st>>>(tc, tr, P, dst, sx, sy, T, NS);
        return 0;
    }
}

void adc_launch_so_bitrows(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches) {
    dim3 grid(P.dm.H, w.S);
    k_so_bitrows<<<grid, 128, 0, st>>>(P.dm, P.tso, w.dmap, w.so_bitrows);
    dim3 rgrid((P.dm.N + 255) / 256, w.S, 4);
    k_so_records<<<rgrid, 256, 0, st>>>(P.dm, P.tso, w.dmap, w.so_bitrows, w.so_rec);
    *launches += 2;
}

// Tensor maps of a lane's two volumes and of its records, one per pass axis, with the boxes of that axis's plan
// (encoded once per lane at adc_create, for its capacity of S pairs).
bool adc_so_tmaps_encode(const AdcParams& P, int S, float* volA, float* volB, unsigned* so_rec, AdcSoTmaps* out) {
    memset(out, 0, sizeof(*out));
    const AdcTmapEncodeFn enc = adc_tmap_encoder();
    if (!enc) return false;
    int dev = 0, smem_sm = 0, smem_res = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&smem_res, cudaDevAttrReservedSharedMemoryPerBlock, dev) != cudaSuccess) { cudaGetLastError(); return false; }
    const AdcDims& dm = P.dm;
    const int Dp = dm.Dp, nrec = so_rec_words(Dp), LPW = 32 / so_lanes_per_line(Dp);
    for (int axis = 0; axis < 2; axis++) {
        const SoPlan pl = so_plan(dm.W, dm.H, Dp, S, axis, adc_sm_count(), (size_t)smem_sm, (size_t)smem_res);
        if (pl.T == 0) return false;
        out->T[axis] = pl.T; out->NS[axis] = pl.NS; out->smem[axis] = (unsigned)pl.smem;
        const cuuint32_t bx = axis ? (cuuint32_t)LPW : (cuuint32_t)pl.T, by = axis ? (cuuint32_t)pl.T : (cuuint32_t)LPW;
        const cuuint32_t estr[4] = {1, 1, 1, 1};
        for (int v = 0; v < 2; v++) {   // volumes [S][H][W][Dp]
            const cuuint64_t gdim[4] = {(cuuint64_t)Dp, (cuuint64_t)dm.W, (cuuint64_t)dm.H, (cuuint64_t)S};
            const cuuint64_t gstr[3] = {(cuuint64_t)Dp * 4, (cuuint64_t)dm.W * Dp * 4, (cuuint64_t)dm.vol_stride * 4};
            const cuuint32_t box[4] = {(cuuint32_t)Dp, bx, by, 1};
            CUtensorMap tm;
            if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, v ? volB : volA, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
                return false;
            memcpy(out->cost[v][axis], &tm, 128);
        }
        {   // records [S][4][H][W][nrec], seen as [4S][H][W][nrec]
            const cuuint64_t gdim[4] = {(cuuint64_t)nrec, (cuuint64_t)dm.W, (cuuint64_t)dm.H, (cuuint64_t)S * 4};
            const cuuint64_t gstr[3] = {(cuuint64_t)nrec * 4, (cuuint64_t)dm.W * nrec * 4, (cuuint64_t)dm.N * nrec * 4};
            const cuuint32_t box[4] = {(cuuint32_t)nrec, bx, by, 1};
            CUtensorMap tm;
            if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 4, so_rec, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
                return false;
            memcpy(out->rec[axis], &tm, 128);
        }
    }
    return true;
}

template <bool WTA>
static int launch_scanline(const AdcParams& P, const AdcWave& w, const float* src, float* dst, int sx, int sy,
                           cudaStream_t st, unsigned long long* launches) {
    const int Dp = P.dm.Dp;
    if (Dp > 256 || !w.so_tm || (src != w.volA && src != w.volB)) return 1;   // D > 256 not supported; a source without a map
    const int axis = sx ? 0 : 1;
    CUtensorMap tc, tr;
    memcpy(&tc, w.so_tm->cost[src == w.volB ? 1 : 0][axis], 128);
    memcpy(&tr, w.so_tm->rec[axis], 128);
    const int T = w.so_tm->T[axis], NS = w.so_tm->NS[axis];
    const size_t smem = w.so_tm->smem[axis];
    int rc = 1;
#define SO_GO(KK, LL) rc = (P.dm.D == KK * LL ? launch_scanline_kf<KK, LL, true, WTA>(P, w, tc, tr, T, NS, smem, dst, sx, sy, st) \
                                                  : launch_scanline_kf<KK, LL, false, WTA>(P, w, tc, tr, T, NS, smem, dst, sx, sy, st))
    switch (so_lanes_per_line(Dp)) {
        case 8:   // K = ceil(Dp / 8)
            switch ((Dp + 7) / 8) { case 1: SO_GO(1, 8); break; case 2: SO_GO(2, 8); break; case 3: SO_GO(3, 8); break; case 4: SO_GO(4, 8); break;
                                    case 5: SO_GO(5, 8); break; case 6: SO_GO(6, 8); break; case 7: SO_GO(7, 8); break; default: SO_GO(8, 8); }
            break;
        case 16:
            switch ((Dp + 15) / 16) { case 5: SO_GO(5, 16); break; case 6: SO_GO(6, 16); break; case 7: SO_GO(7, 16); break; default: SO_GO(8, 16); }
            break;
        default:
            switch ((Dp + 31) / 32) { case 5: SO_GO(5, 32); break; case 6: SO_GO(6, 32); break; case 7: SO_GO(7, 32); break; default: SO_GO(8, 32); }
    }
#undef SO_GO
    if (rc) return rc;
    ++*launches;
    return 0;
}

int adc_launch_scanline(const AdcParams& P, const AdcWave& w, const float* src, float* dst, int sx, int sy,
                        cudaStream_t st, unsigned long long* launches) {
    return launch_scanline<false>(P, w, src, dst, sx, sy, st, launches);
}

int adc_launch_scanline_wta(const AdcParams& P, const AdcWave& w, const float* src, float* rec, cudaStream_t st,
                            unsigned long long* launches) {
    return launch_scanline<true>(P, w, src, rec, 0, -1, st, launches);
}

size_t adc_so_rec_bytes(const AdcDims& dm) { return (size_t)4 * dm.N * so_rec_words(dm.Dp) * 4; }   // four pass directions
size_t adc_so_bitrow_bytes(const AdcDims& dm) { return (size_t)4 * dm.H * so_row_words(dm.W) * 4; }
