// so_plan.h -- sizes and launch plan of the scanline passes (k_scanline.cu).  Plain C++ with no CUDA dependency, so that
// tests/test_scanline_plan.py can check the plan's choices on the CPU.
#pragma once
#include <stddef.h>

#ifdef __CUDACC__
#define SO_HD __host__ __device__
#else
#define SO_HD
#endif

#define SO_WARPS 4          // warps per CTA
#define SO_MIN_CTAS 8       // __launch_bounds__ minimum of CTAs per SM: registers never hold residency below this
#define SO_SMEM_MAX (160 * 1024)   // dynamic shared memory a scanline CTA may be given

// per-pixel penalty record of one pass direction: word 0 = (d1 < tso), words 1.. = bit d -> (d2(d) < tso), padded to 16 bytes
SO_HD inline int so_rec_words(int Dp) { return ((1 + (Dp + 31) / 32 + 1) + 3) / 4 * 4; }
// lanes per line: as few as keep K = ceil(Dp / lanes) <= 8 (Dp is a multiple of 4, at most 256)
SO_HD inline int so_lanes_per_line(int Dp) { return Dp <= 64 ? 8 : (Dp <= 128 ? 16 : 32); }
// a region of a ring slot, rounded up to the 128-byte alignment of a tensor copy's shared-memory destination
SO_HD inline unsigned so_region(unsigned bytes) { return (bytes + 127u) / 128u * 128u; }
// one ring slot of a warp: the costs of its lines for T steps, then their records
SO_HD inline unsigned so_cost_region(int Dp, int T) { return so_region((unsigned)(T * (32 / so_lanes_per_line(Dp)) * Dp * 4)); }
SO_HD inline unsigned so_slot_bytes(int Dp, int T) {
    return so_cost_region(Dp, T) + so_region((unsigned)(T * (32 / so_lanes_per_line(Dp)) * so_rec_words(Dp) * 4));
}
// a CTA's rings plus one 8-byte mbarrier per (warp, slot)
inline size_t so_smem_bytes(int Dp, int T, int NS) { return (size_t)SO_WARPS * NS * (so_slot_bytes(Dp, T) + 8); }

// Plan of one pass: T steps per ring slot, NS slots per warp, and what follows from them.
struct SoPlan { int T, NS; size_t smem; int ctas, ctas_per_sm, waves; };

// The device enters as its SM count, its shared memory per SM and the shared memory it reserves per CTA.  The plan takes
// the candidate that runs the pass in the fewest waves of resident CTAs, and among those the one that keeps the most steps
// in flight when a slot is refilled, T * (NS - 1).  A pass whose grid just overflows one wave (Cone's y pass: 928 CTAs
// against 6 x 132 resident with 8 steps of 4 lines in flight) would run a second wave of a few CTAs through the whole
// scanline; a shallower ring lets more CTAs stay resident instead.
inline SoPlan so_plan(int W, int H, int Dp, int S, int axis_y, int sm_count, size_t smem_per_sm, size_t smem_reserved_per_cta) {
    static const int cand[][2] = {{4, 3}, {2, 4}, {4, 2}, {2, 3}, {3, 2}, {2, 2}};   // {T, NS}, most steps in flight at a refill first
    const int lines_per_cta = SO_WARPS * (32 / so_lanes_per_line(Dp));
    const int n_lines = axis_y ? W : H;
    SoPlan best{};
    for (const auto& c : cand) {
        SoPlan p{};
        p.T = c[0]; p.NS = c[1];
        p.smem = so_smem_bytes(Dp, p.T, p.NS);
        if (p.smem > SO_SMEM_MAX) continue;
        p.ctas_per_sm = (int)(smem_per_sm / (p.smem + smem_reserved_per_cta));
        if (p.ctas_per_sm > SO_MIN_CTAS) p.ctas_per_sm = SO_MIN_CTAS;
        if (p.ctas_per_sm < 1) continue;
        p.ctas = (n_lines + lines_per_cta - 1) / lines_per_cta * S;
        const int resident = p.ctas_per_sm * sm_count;
        p.waves = (p.ctas + resident - 1) / resident;
        if (best.T == 0 || p.waves < best.waves) best = p;
    }
    return best;
}

// ---- the last pass (-y) with the winner-takes-all as its epilogue (k_scanline_wta, k_wta_merge) ----------
// A CTA of the y pass owns a band of so_wta_band columns.  Per row it writes disp_l and, for every right pixel xr whose
// diagonal x = xr + dmin + d crosses the band, one partial record of the right view over that diagonal's d-range inside
// the band (SO_WTA_FIELDS floats, field-major); k_wta_merge folds a right pixel's records in band order.
#define SO_WTA_FIELDS 6     // minimum, first argmin (d, as int bits), cost at argmin-1 and argmin+1, at the range's first and last d
SO_HD inline int so_wta_band(int Dp) { return SO_WARPS * (32 / so_lanes_per_line(Dp)); }
// record slots of one band in one row: j = 0 .. band + D - 2 holds right pixel xr = x0 - dmin - (D - 1) + j
SO_HD inline int so_wta_slots(int Dp, int D) { return so_wta_band(Dp) + D - 1; }
// floats of one field plane of one pair: H rows x bands x slots
inline long long so_wta_plane(int W, int H, int D, int Dp) {
    const int c = so_wta_band(Dp);
    return (long long)H * ((W + c - 1) / c) * so_wta_slots(Dp, D);
}
// records one row actually carries: slots whose right pixel lies in the image and whose diagonal meets a band column < W
inline long long so_wta_row_records(int W, int D, int Dp, int dmin) {
    const int c = so_wta_band(Dp);
    long long n = 0;
    for (int x0 = 0; x0 < W; x0 += c) {
        const int lo = x0 - dmin - (D - 1) > 0 ? x0 - dmin - (D - 1) : 0;
        const int xe = x0 + c < W ? x0 + c : W;
        const int hi = xe - 1 - dmin < W - 1 ? xe - 1 - dmin : W - 1;
        if (hi >= lo) n += hi - lo + 1;
    }
    return n;
}

// What else a run does with the optimised volume of pass 4, besides the winner-takes-all.
struct SoVolumeUse {
    bool opt_export;      // an ADC_VOL_OPT export
    bool confidence;      // a MIN_COST or PEAK_RATIO map
    bool discontinuity;   // the discontinuity adjustment (reads the volume at the end of the refinement)
    bool debug_run;       // adc_debug_run*: it may stop at SO4, and adc_debug_get may tap the volume afterwards
};
enum SoWtaForce { SO_WTA_AUTO = 0, SO_WTA_NEVER = 1, SO_WTA_ALWAYS = 2 };   // ALWAYS: still only where the records fit

// Whether pass 4 runs fused with the winner-takes-all.  The fused form never stores the optimised volume, so it needs
// nobody to read it afterwards; its records take the volume's place in the pair's slice (vol_floats floats), so they must
// fit there.  It replaces a volume store and the WTA's volume read (2V per pair) by the records written and read again; it
// is taken where that traffic is at most half of 2V, i.e. where the band is wide against the disparity range (Cone,
// D = 64 on 16 columns: 44 %; 1242 x 375 x 128 on 8 columns: 80 %; 1920 x 1080 x 192 on 4 columns: 152 %).
inline bool so_wta_fused(const SoVolumeUse& use, int force, int W, int H, int D, int Dp, int dmin, long long vol_floats) {
    if (use.opt_export || use.confidence || use.discontinuity || use.debug_run || force == SO_WTA_NEVER) return false;
    if ((long long)SO_WTA_FIELDS * so_wta_plane(W, H, D, Dp) > vol_floats) return false;
    if (force == SO_WTA_ALWAYS) return true;
    const double traffic = 2.0 * SO_WTA_FIELDS * 4.0 * (double)so_wta_row_records(W, D, Dp, dmin);   // per row: written + read
    const double staged = 2.0 * 4.0 * W * Dp;                                                         // per row: volume store + WTA read
    return traffic <= 0.5 * staged;
}
