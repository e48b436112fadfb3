// k_refine.cu -- stage 5: multi-step disparity refinement (reference: multistep_refiner.cpp:60-87):
// LR-check outlier detection (:90-151), iterative region voting (:153-227), 16-ray proper
// interpolation (:229-305), optional depth-discontinuity adjustment (:307-371) and the in-place 3x3
// median (adcensus_util.cpp:55-81 called with in == out at multistep_refiner.cpp:86).
//
// The reference runs all of these sequentially *in place*, and the in-place order is part of the
// answer.  Each kernel below is a parallel schedule that provably reproduces the sequential
// result (argument given at each kernel); none of them approximates.
#include "adc_common.cuh"
#include <stdlib.h>
#include <algorithm>

// =============================================================================================
// 1. Outlier detection.  The raster scan reads disp_left[col_rl] of the same row while already
//    having invalidated pixels to the left of x.  Whether a pixel gets invalidated depends only on
//    the ORIGINAL maps (its own disparity and the right map), so: phase 1 computes that predicate
//    for every pixel; phase 2 classifies, seeing +inf for col_rl < x that phase 1 marked, and the
//    original value otherwise (col_rl == x reads the pixel itself before it is invalidated).
// =============================================================================================
__global__ void k_outlier_mark(AdcParams P, const float* __restrict__ disp_l, const float* __restrict__ disp_r,
                               uint8_t* __restrict__ flag) {
    const AdcDims& dm = P.dm;
    const int pair = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dm.N) return;
    const int y = i / dm.W, x = i - y * dm.W;
    const float d = disp_l[(size_t)pair * dm.N + i];
    uint8_t f = 0;
    if (d == ADC_INVALID_F) f = 1;
    else {
        const long col_r = lroundf(__fsub_rn((float)x, d));
        if (col_r < 0 || col_r >= dm.W) f = 1;
        else {
            const float dr = disp_r[(size_t)pair * dm.N + y * dm.W + col_r];
            if (fabsf(__fsub_rn(d, dr)) > P.lr_thres) f = 2;
        }
    }
    flag[(size_t)pair * dm.N + i] = f;
}

__global__ void k_outlier_classify(AdcParams P, const float* __restrict__ disp_l, const float* __restrict__ disp_r,
                                   const uint8_t* __restrict__ flag, float* __restrict__ disp_out,
                                   uint8_t* __restrict__ label) {
    const AdcDims& dm = P.dm;
    const int pair = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dm.N) return;
    const size_t o = (size_t)pair * dm.N;
    const int y = i / dm.W, x = i - y * dm.W;
    const uint8_t f = flag[o + i];
    const float d = disp_l[o + i];
    uint8_t lab = 0;
    if (f == 1) lab = 1;
    else if (f == 2) {
        const long col_r = lroundf(__fsub_rn((float)x, d));
        const float dr = disp_r[o + y * dm.W + col_r];
        const int col_rl = (int)lroundf(__fadd_rn((float)col_r, dr));
        lab = 1;
        if (col_rl > 0 && col_rl < dm.W) {
            const int j = y * dm.W + col_rl;
            const float dl = (col_rl < x && flag[o + j] != 0) ? ADC_INVALID_F : disp_l[o + j];
            if (dl > d) lab = 2;
        }
    }
    label[o + i] = lab;
    disp_out[o + i] = f ? ADC_INVALID_F : d;
}

void adc_launch_outlier(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches) {
    dim3 grid((P.dm.N + 255) / 256, w.S);
    k_outlier_mark<<<grid, 256, 0, st>>>(P, w.disp_l, w.disp_r, w.flag);
    k_outlier_classify<<<grid, 256, 0, st>>>(P, w.disp_l, w.disp_r, w.flag, w.disp_t, w.label);
    *launches += 2;
}

// =============================================================================================
// 2. Pixel lists.  Iterative region voting (:153-227) itself is in k_vote.cu; it works on the active lists built
//    here and leaves the outlier lists, rebuilt here, to the interpolation.
// =============================================================================================

// ---- ordered (raster) pixel lists of the two outlier classes: row counts -> scan -> scatter ----
__global__ void __launch_bounds__(128)
k_list_row_counts(AdcDims dm, const uint8_t* __restrict__ label, const uint16_t* __restrict__ region_size, int min_size,
                  int* __restrict__ rowcnt) {
    // region_size != NULL: only pixels whose cross region holds more than min_size pixels (see adc_launch_active_lists)
    const int pair = blockIdx.y, y = blockIdx.x;
    const uint8_t* lab = label + (size_t)pair * dm.N + (size_t)y * dm.W;
    const uint16_t* rs = region_size ? region_size + (size_t)pair * dm.N + (size_t)y * dm.W : nullptr;
    int c1 = 0, c2 = 0;
    for (int x = threadIdx.x; x < dm.W; x += 128) {
        uint8_t v = lab[x];
        if (rs && (int)rs[x] <= min_size) v = 0;
        c1 += v == 1; c2 += v == 2;
    }
    __shared__ int s1[4], s2[4];
    c1 = __reduce_add_sync(0xffffffffu, c1);
    c2 = __reduce_add_sync(0xffffffffu, c2);
    if ((threadIdx.x & 31) == 0) { s1[threadIdx.x >> 5] = c1; s2[threadIdx.x >> 5] = c2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        rowcnt[((size_t)pair * 2 + 0) * dm.H + y] = s1[0] + s1[1] + s1[2] + s1[3];
        rowcnt[((size_t)pair * 2 + 1) * dm.H + y] = s2[0] + s2[1] + s2[2] + s2[3];
    }
}

// exclusive scan of the row counts (in place), one warp per (pair, class)
__global__ void __launch_bounds__(64)
k_list_row_scan(AdcDims dm, int* __restrict__ rowcnt, int* __restrict__ counters, int slot) {
    const int pair = blockIdx.x, k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int* rc = rowcnt + ((size_t)pair * 2 + k) * dm.H;
    int base = 0;
    for (int y0 = 0; y0 < dm.H; y0 += 32) {
        const int y = y0 + lane;
        const int v = y < dm.H ? rc[y] : 0;
        int inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (y < dm.H) rc[y] = base + inc - v;
        base += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) counters[pair * ADC_CNT + slot + k] = base;
}

__global__ void __launch_bounds__(128)
k_list_row_scatter(AdcDims dm, const uint8_t* __restrict__ label, const uint16_t* __restrict__ region_size, int min_size,
                   const int* __restrict__ rowoff, int* __restrict__ pend) {
    const int pair = blockIdx.y, y = blockIdx.x;
    const uint8_t* lab = label + (size_t)pair * dm.N + (size_t)y * dm.W;
    const uint16_t* rs = region_size ? region_size + (size_t)pair * dm.N + (size_t)y * dm.W : nullptr;
    __shared__ int s_cnt[2][4];
    int base1 = rowoff[((size_t)pair * 2 + 0) * dm.H + y], base2 = rowoff[((size_t)pair * 2 + 1) * dm.H + y];
    int* l1 = pend + ((size_t)pair * 2 + 0) * dm.N;
    int* l2 = pend + ((size_t)pair * 2 + 1) * dm.N;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int x0 = 0; x0 < dm.W; x0 += 128) {
        const int x = x0 + threadIdx.x;
        uint8_t v = x < dm.W ? lab[x] : 0;
        if (rs && x < dm.W && (int)rs[x] <= min_size) v = 0;
        const unsigned b1 = __ballot_sync(0xffffffffu, v == 1), b2 = __ballot_sync(0xffffffffu, v == 2);
        if (lane == 0) { s_cnt[0][wid] = __popc(b1); s_cnt[1][wid] = __popc(b2); }
        __syncthreads();
        int o1 = base1, o2 = base2, t1 = 0, t2 = 0;
#pragma unroll
        for (int w2 = 0; w2 < 4; w2++) {
            if (w2 < wid) { o1 += s_cnt[0][w2]; o2 += s_cnt[1][w2]; }
            t1 += s_cnt[0][w2]; t2 += s_cnt[1][w2];
        }
        const unsigned lt = (1u << lane) - 1u;
        if (v == 1) l1[o1 + __popc(b1 & lt)] = y * dm.W + x;
        if (v == 2) l2[o2 + __popc(b2 & lt)] = y * dm.W + x;
        base1 += t1; base2 += t2;
        __syncthreads();
    }
}

void adc_launch_build_lists(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches) {
    dim3 grid(P.dm.H, w.S);
    k_list_row_counts<<<grid, 128, 0, st>>>(P.dm, w.label, nullptr, 0, w.rowcnt);
    k_list_row_scan<<<w.S, 64, 0, st>>>(P.dm, w.rowcnt, w.counters, 0);
    k_list_row_scatter<<<grid, 128, 0, st>>>(P.dm, w.label, nullptr, 0, w.rowcnt, w.pend);
    *launches += 3;
}

// Lists of the pixels that can still be filled by voting: a vote needs more than irv_ts valid pixels in
// the pixel's cross region (multistep_refiner.cpp:211), and that region -- the vertical arm of p, then the
// horizontal arm of every pixel on it -- is exactly the horizontal-first support region whose size
// cross_aggregator.cpp:271-325 already counted.  A pixel whose whole region is not larger than irv_ts can
// never pass, in any sweep, whatever its neighbours become: it is left out of the voting lists (about 40 %
// of the listed pixels on Cone) and simply stays in the outlier lists for the interpolation step.
void adc_launch_active_lists(const AdcParams& P, const AdcWave& w, cudaStream_t st, unsigned long long* launches) {
    const bool exact = P.L1 <= 127;   // beyond that the reference's uint16 counts may wrap
    dim3 grid(P.dm.H, w.S);
    k_list_row_counts<<<grid, 128, 0, st>>>(P.dm, w.label, exact ? w.sup_h : nullptr, P.irv_ts, w.rowcnt);
    k_list_row_scan<<<w.S, 64, 0, st>>>(P.dm, w.rowcnt, w.counters, 10);
    k_list_row_scatter<<<grid, 128, 0, st>>>(P.dm, w.label, exact ? w.sup_h : nullptr, P.irv_ts, w.rowcnt, w.vlist);
    *launches += 3;
}

// =============================================================================================
// 3. Proper interpolation.  For each pixel still in a list: 16 rays (angle accumulated in double
//    from the float quotient 3.1415926f/16), first valid disparity met along each; mismatches take
//    the candidate whose colour is closest (first wins), occlusions the smallest disparity; no
//    candidate -> 0.0 (the reference's value-initialised fill vector).  Results of one list are
//    written after the whole list has been evaluated (Jacobi), the occlusion list then sees the
//    filled mismatches -- hence one launch per list reading disp_old and writing disp_new.
//    The ray coordinates are evaluated exactly as the reference does, lround(y + m*sin) in double
//    without contraction, with sin/cos tables from the host's libm.
//    16 lanes = 16 rays of one pixel; two pixels per warp.
// =============================================================================================
__global__ void __launch_bounds__(256)
k_interpolate(AdcParams P, int k, const uint8_t* __restrict__ bgr, const float* __restrict__ disp_old,
              float* __restrict__ disp_new, const int* __restrict__ pend, const int* __restrict__ counters,
              const double* __restrict__ ray_sin, const double* __restrict__ ray_cos,
              const short2* __restrict__ ray_off) {
    const AdcDims& dm = P.dm;
    const int pair = blockIdx.y;
    const int n = counters[pair * ADC_CNT + k];
    const int* list = pend + ((size_t)pair * 2 + k) * dm.N;
    const uint8_t* left = bgr + (size_t)pair * 2 * dm.N * 3;
    const float* d_old = disp_old + (size_t)pair * dm.N;
    float* d_new = disp_new + (size_t)pair * dm.N;
    const int ray = threadIdx.x & 15;
    const int slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const int n_slots = (gridDim.x * blockDim.x) >> 4;
    const unsigned half_mask = 0xffffu << (threadIdx.x & 16);
    const double sa = ray_sin[ray], ca = ray_cos[ray];
    for (int base = 0; base < n; base += n_slots) {   // uniform trip count for the whole warp
        const int idx = base + slot;
        const bool active = idx < n;
        int p = 0, x = 0, y = 0;
        if (active) { p = list[idx]; y = p / dm.W; x = p - y * dm.W; }
        int dist = 0x7fffffff;
        float dval = ADC_LARGE_F;
        bool found = false;
        if (active) {
            const uchar3 c0 = adc_load_bgr(left, p);
            for (int m = 1; m < P.max_search; m++) {
                long yy, xx;
                if (ray_off) {   // integer offsets, verified on the host to equal the expression below for this image size
                    const short2 o = __ldg(ray_off + ray * P.max_search + m);
                    yy = y + o.y; xx = x + o.x;
                } else {
                    yy = lround(__dadd_rn((double)y, __dmul_rn((double)m, sa)));
                    xx = lround(__dadd_rn((double)x, __dmul_rn((double)m, ca)));
                }
                if (yy < 0 || yy >= dm.H || xx < 0 || xx >= dm.W) break;
                const int q = (int)yy * dm.W + (int)xx;
                const float d = d_old[q];
                if (d != ADC_INVALID_F) {
                    const uchar3 c = adc_load_bgr(left, q);
                    dist = abs((int)c0.x - (int)c.x) + abs((int)c0.y - (int)c.y) + abs((int)c0.z - (int)c.z);
                    dval = d;
                    found = true;
                    break;
                }
            }
        }
        // combine the 16 rays of this pixel (half-warp)
        const unsigned any = __ballot_sync(0xffffffffu, found) & half_mask;
        float result = 0.0f;
        if (k == 0) {
            // smallest colour distance, earliest ray on ties (strict '>' in the reference, min_dist starts at 9999)
            int key = (found && dist < 9999) ? ((dist << 4) | ray) : 0x7fffffff;
#pragma unroll
            for (int o = 8; o >= 1; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
            const int win = key & 15;
            const float dw = __shfl_sync(0xffffffffu, dval, (threadIdx.x & 16) | win);
            if (key != 0x7fffffff) result = dw;     // all candidates farther than 9999 keep d = 0.0f
        } else {
            float mv = found ? dval : ADC_LARGE_F;
#pragma unroll
            for (int o = 8; o >= 1; o >>= 1) mv = fminf(mv, __shfl_xor_sync(0xffffffffu, mv, o));
            result = mv;
        }
        if (any == 0) result = 0.0f;
        if (active && ray == 0) d_new[p] = result;
    }
}

// Fast path of the same step, used when the integer ray table is available (it is whenever it was verified exact
// for this image size, see engine.cu).  The generic kernel spends ~15 instructions per ray step on coordinates,
// four bounds tests and a float load; here the walk runs on a padded byte map (0 = invalid pixel: keep going,
// 1 = valid: candidate found, 2 = outside the image: the ray ends) with the ray table in shared memory as linear
// offsets into that map: one shared load, one add, one byte load and a test per step.
__global__ void __launch_bounds__(256)
k_interp_map(AdcDims dm, int B, const float* __restrict__ disp, uint8_t* __restrict__ imap) {
    const int Wp = dm.W + 2 * B, Hp = dm.H + 2 * B;
    const int pair = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Wp * Hp) return;
    const int yp = i / Wp, xp = i - yp * Wp;
    const int y = yp - B, x = xp - B;
    uint8_t v = 2;
    if (y >= 0 && y < dm.H && x >= 0 && x < dm.W) v = disp[(size_t)pair * dm.N + y * dm.W + x] != ADC_INVALID_F ? 1 : 0;
    imap[(size_t)pair * Wp * Hp + i] = v;
}

__global__ void __launch_bounds__(256)
k_interpolate_fast(AdcParams P, int k, const unsigned* __restrict__ bgrx, const float* __restrict__ disp_old,
                   float* __restrict__ disp_new, const int* __restrict__ pend, const int* __restrict__ counters,
                   const short2* __restrict__ ray_off, const uint8_t* __restrict__ imap_all) {
    extern __shared__ int ip_off[];   // [16][max_search]: dy * Wp + dx
    const AdcDims& dm = P.dm;
    const int L = P.max_search, B = L - 1, Wp = dm.W + 2 * B, Hp = dm.H + 2 * B;
    for (int i = threadIdx.x; i < 16 * L; i += blockDim.x) { const short2 o = ray_off[i]; ip_off[i] = (int)o.y * Wp + (int)o.x; }
    __syncthreads();
    const int pair = blockIdx.y;
    const int n = counters[pair * ADC_CNT + k];
    const int* list = pend + ((size_t)pair * 2 + k) * dm.N;
    const unsigned* left = bgrx + (size_t)pair * 2 * dm.N;   // packed B | G<<8 | R<<16
    const float* d_old = disp_old + (size_t)pair * dm.N;
    float* d_new = disp_new + (size_t)pair * dm.N;
    const uint8_t* imap = imap_all + (size_t)pair * Wp * Hp;
    const int ray = threadIdx.x & 15;
    const int slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const int n_slots = (gridDim.x * blockDim.x) >> 4;
    const unsigned half_mask = 0xffffu << (threadIdx.x & 16);
    const int* myoff = ip_off + ray * L;
    for (int base = 0; base < n; base += n_slots) {   // uniform trip count for the whole warp
        const int idx = base + slot;
        const bool active = idx < n;
        int p = 0;
        int dist = 0x7fffffff;
        float dval = ADC_LARGE_F;
        bool found = false;
        if (active) {
            p = list[idx];
            const int y = p / dm.W, x = p - y * dm.W;
            const uint8_t* c0p = imap + (y + B) * Wp + (x + B);
            int m = 1, hit = 2;
            for (; m < L; m++) {
                hit = c0p[myoff[m]];
                if (hit) break;
            }
            if (m < L && hit == 1) {
                const short2 o = __ldg(ray_off + ray * L + m);
                const int q = (y + o.y) * dm.W + (x + o.x);
                const unsigned a = __ldg(left + p), b = __ldg(left + q);
                const unsigned ad = __vabsdiffu4(a, b);
                dist = (int)(ad & 255u) + (int)((ad >> 8) & 255u) + (int)((ad >> 16) & 255u);
                dval = d_old[q];
                found = true;
            }
        }
        // combine the 16 rays of this pixel (half-warp) -- as in k_interpolate
        const unsigned any = __ballot_sync(0xffffffffu, found) & half_mask;
        float result = 0.0f;
        if (k == 0) {
            int key = (found && dist < 9999) ? ((dist << 4) | ray) : 0x7fffffff;
#pragma unroll
            for (int o = 8; o >= 1; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
            const int win = key & 15;
            const float dw = __shfl_sync(0xffffffffu, dval, (threadIdx.x & 16) | win);
            if (key != 0x7fffffff) result = dw;
        } else {
            float mv = found ? dval : ADC_LARGE_F;
#pragma unroll
            for (int o = 8; o >= 1; o >>= 1) mv = fminf(mv, __shfl_xor_sync(0xffffffffu, mv, o));
            result = mv;
        }
        if (any == 0) result = 0.0f;
        if (active && ray == 0) d_new[p] = result;
    }
}

void adc_launch_interp_list(const AdcParams& P, const AdcWave& w, int k, cudaStream_t st, unsigned long long* launches) {
    dim3 grid(592, w.S);
    const int L = P.max_search, B = L - 1;
    const size_t map_bytes = (size_t)(P.dm.W + 2 * B) * (P.dm.H + 2 * B);
    if (w.ray_off && L >= 2 && map_bytes <= (size_t)P.dm.N * 8 && (size_t)16 * L * sizeof(int) <= 48 * 1024) {
        uint8_t* imap = reinterpret_cast<uint8_t*>(w.vote_chg);   // voting's change list, 8 bytes per pixel, idle by now
        dim3 mgrid((unsigned)((map_bytes + 255) / 256), w.S);
        k_interp_map<<<mgrid, 256, 0, st>>>(P.dm, B, w.disp_l, imap);
        k_interpolate_fast<<<grid, 256, (size_t)16 * L * sizeof(int), st>>>(P, k, w.bgrx, w.disp_l, w.disp_t, w.pend, w.counters,
                                                                            w.ray_off, imap);
        *launches += 2;
        return;
    }
    k_interpolate<<<grid, 256, 0, st>>>(P, k, w.bgr, w.disp_l, w.disp_t, w.pend, w.counters, w.ray_sin, w.ray_cos, w.ray_off);
    ++*launches;
}

// =============================================================================================
// 4. Depth-discontinuity adjustment (default OFF in ADCensusOption).  Sobel edge mask on the
//    disparity map, then per row a strictly sequential left-to-right pass (pixel x may copy from
//    x-1, which may itself have just been changed) -> one thread per row.  The reference indexes
//    the cost volume with lround(d) without subtracting dmin (multistep_refiner.cpp:331); indices
//    outside [0,D) are undefined behaviour there and skipped here (the CPU checker does the same).
// =============================================================================================
__global__ void k_edge_mask(AdcDims dm, const float* __restrict__ disp, uint8_t* __restrict__ edge) {
    const int pair = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dm.N) return;
    const int y = i / dm.W, x = i - y * dm.W;
    uint8_t e = 0;
    if (y >= 1 && y < dm.H - 1 && x >= 1 && x < dm.W - 1) {
        const float* r1 = disp + (size_t)pair * dm.N + i;
        const float* r0 = r1 - dm.W;
        const float* r2 = r1 + dm.W;
        const float A = __fadd_rn(-r0[-1], r0[1]);
        const float B = __fadd_rn(__fmul_rn(-2.0f, r1[-1]), __fmul_rn(2.0f, r1[1]));
        const float C = __fadd_rn(-r2[-1], r2[1]);
        const float gx = __fadd_rn(__fadd_rn(A, B), C);
        const float T = __fsub_rn(__fsub_rn(-r0[-1], __fmul_rn(2.0f, r0[0])), r0[1]);
        const float U = __fadd_rn(__fadd_rn(r2[-1], __fmul_rn(2.0f, r2[0])), r2[1]);
        const float gy = __fadd_rn(T, U);
        if (__fadd_rn(fabsf(gx), fabsf(gy)) > 5.0f) e = 1;
    }
    edge[(size_t)pair * dm.N + i] = e;
}

__global__ void k_discontinuity_rows(AdcDims dm, float* __restrict__ disp, const uint8_t* __restrict__ edge,
                                     const float* __restrict__ vol) {
    const int pair = blockIdx.y;
    const int y = blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= dm.H) return;
    float* row = disp + (size_t)pair * dm.N + (size_t)y * dm.W;
    const uint8_t* erow = edge + (size_t)pair * dm.N + (size_t)y * dm.W;
    for (int x = 1; x < dm.W - 1; x++) {
        if (erow[x] != 1) continue;
        const float d = row[x];
        if (d == ADC_INVALID_F) continue;
        const float* cost = vol + (size_t)pair * dm.vol_stride + ((size_t)y * dm.W + x) * dm.Dp;
        const long di = lroundf(d);
        if (di < 0 || di >= dm.D) continue;
        float c0 = cost[di];
        for (int k = 0; k < 2; k++) {
            const float d2 = row[k == 0 ? x - 1 : x + 1];
            if (d2 == ADC_INVALID_F) continue;
            const long d2i = lroundf(d2);
            if (d2i < 0 || d2i >= dm.D) continue;
            const float cc = k == 0 ? cost[-dm.Dp + d2i] : cost[dm.Dp + d2i];
            if (cc < c0) { row[x] = d2; c0 = cc; }
        }
    }
}

void adc_launch_discontinuity(const AdcParams& P, const AdcWave& w, const float* vol, cudaStream_t st, unsigned long long* launches) {
    dim3 grid((P.dm.N + 255) / 256, w.S);
    k_edge_mask<<<grid, 256, 0, st>>>(P.dm, w.disp_l, w.flag);
    dim3 grid2((P.dm.H + 63) / 64, w.S);
    k_discontinuity_rows<<<grid2, 64, 0, st>>>(P.dm, w.disp_l, w.flag, vol);
    *launches += 2;
}

// =============================================================================================
// 5. In-place 3x3 median in raster order.  out(y,x) sees already-filtered values in row y-1 and
//    at (y,x-1), and original values elsewhere.  (y,x) depends on (y,x-1) and (y-1,x+1), so all
//    pixels with x + 2y = t are independent: a wavefront over t = 0 .. W+2H-3 with a CTA barrier
//    per step reproduces the sequential scan exactly (every window element of step t was produced
//    at a step != t).  Window = in-image neighbours, sorted, element n/2 (9->[4], 6->[3], 4->[2]);
//    realised as the median of 9 after padding with -inf/+inf so that the rank is preserved.
//    Data movement: one thread per row.  "Original" values come from the untouched input map
//    (read-only, so they cache in L1), "filtered" values of the row above come from a 4-deep
//    per-row ring in shared memory written by the neighbouring thread, the filtered left
//    neighbour is the thread's own previous result; the output goes to a second map.
// =============================================================================================
#define MED_THREADS 1024

__device__ __forceinline__ void cswap(float& a, float& b) { const float lo = fminf(a, b), hi = fmaxf(a, b); a = lo; b = hi; }

__device__ __forceinline__ float median9(float v[9]) {
    // 19-exchange median-of-9 selection network (Paeth / Smith)
    cswap(v[1], v[2]); cswap(v[4], v[5]); cswap(v[7], v[8]);
    cswap(v[0], v[1]); cswap(v[3], v[4]); cswap(v[6], v[7]);
    cswap(v[1], v[2]); cswap(v[4], v[5]); cswap(v[7], v[8]);
    cswap(v[0], v[3]); cswap(v[5], v[8]); cswap(v[4], v[7]);
    cswap(v[3], v[6]); cswap(v[1], v[4]); cswap(v[2], v[5]);
    cswap(v[4], v[7]); cswap(v[4], v[2]); cswap(v[6], v[4]);
    cswap(v[4], v[2]);
    return v[4];
}


__device__ __forceinline__ void med_cp4(float* smem_dst, const float* gmem_src) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem_src) : "memory");
}

template <int MED_ROWS, int MED_PF>   // rows per thread (1 for H <= 1024, 2 up to 2048, 4 up to 4096); wavefront steps between issuing a load and using it
__global__ void __launch_bounds__(MED_THREADS)
k_median_wavefront(AdcDims dm, const float* __restrict__ in, float* __restrict__ out) {
    extern __shared__ float med_smem[];
    const int MT = blockDim.x;   // threads actually launched (rows rounded up to whole warps)
    // [H][4]: filtered values of each row, indexed by column & 3
    // then per thread and row: MED_PF slots x 2 floats of ORIGINAL values (row y, row y+1) of the column that
    // enters the window at a given step, filled by 4-byte cp.async issued MED_PF steps ahead
    const int pair = blockIdx.x;
    const float* src = in + (size_t)pair * dm.N;
    float* dst = out + (size_t)pair * dm.N;
    const int W = dm.W, H = dm.H;
    float* med_ring = med_smem;
    float* stage = med_smem + (size_t)H * 4 + (size_t)threadIdx.x * (MED_ROWS * MED_PF * 2);
    (void)MT;
    const float NINF = __int_as_float(0xff800000), PINF = ADC_INVALID_F;
    const int n_steps = W + 2 * H - 2;
    float A0[MED_ROWS], A1[MED_ROWS], Bm[MED_ROWS], B0[MED_ROWS], B1[MED_ROWS], left_new[MED_ROWS];
    auto issue = [&](int r, int t, int slot) {   // originals of column x + 1 = (t - 2y) + 1, consumed at step t
        const int y = threadIdx.x + r * MT;
        const int c = t - 2 * y + 1;
        float* s2 = stage + (r * MED_PF + slot) * 2;
        const bool ok = y < H && c >= 0 && c < W;
        if (ok) med_cp4(s2, src + y * W + c); else s2[0] = PINF;
        if (ok && y + 1 < H) med_cp4(s2 + 1, src + (y + 1) * W + c); else s2[1] = PINF;
    };
#pragma unroll
    for (int r = 0; r < MED_ROWS; r++) { A0[r] = A1[r] = Bm[r] = B0[r] = B1[r] = PINF; left_new[r] = PINF; }
#pragma unroll
    for (int j = 0; j < MED_PF; j++) {
#pragma unroll
        for (int r = 0; r < MED_ROWS; r++) issue(r, j - 2, j);
        asm volatile("cp.async.commit_group;\n" ::: "memory");
    }
    for (int tb = -2; tb < n_steps; tb += MED_PF) {
#pragma unroll
        for (int j = 0; j < MED_PF; j++) {
            const int t = tb + j;
            asm volatile("cp.async.wait_group %0;\n" ::"n"(MED_PF - 1) : "memory");   // this thread's copies for step t
            float res[MED_ROWS];
            bool act[MED_ROWS];
#pragma unroll
            for (int r = 0; r < MED_ROWS; r++) {
                const int y = threadIdx.x + r * MT;
                const int x = t - 2 * y;
                act[r] = false;
                res[r] = 0.f;
                if (x < -2 - MED_PF || x >= W) continue;   // this row's turn is far away or over: nothing to shift, fetch or compute
                const float* s2 = stage + (r * MED_PF + j) * 2;
                A0[r] = A1[r]; A1[r] = s2[0];
                Bm[r] = B0[r]; B0[r] = B1[r]; B1[r] = s2[1];
                issue(r, t + MED_PF, j);
                act[r] = t < n_steps && y < H && x >= 0 && x < W;
                if (!act[r]) continue;
                const bool up = y > 0, dn = y + 1 < H, lf = x > 0, rt = x + 1 < W;
                float v[9];
                const float* ring_up = med_ring + (size_t)(y - 1) * 4;
                v[0] = (up && lf) ? ring_up[(x - 1) & 3] : PINF;
                v[1] = up ? ring_up[x & 3] : PINF;
                v[2] = (up && rt) ? ring_up[(x + 1) & 3] : PINF;
                v[3] = lf ? left_new[r] : PINF;
                v[4] = A0[r];
                v[5] = rt ? A1[r] : PINF;
                v[6] = (dn && lf) ? Bm[r] : PINF;
                v[7] = dn ? B0[r] : PINF;
                v[8] = (dn && rt) ? B1[r] : PINF;
                const int n = (1 + (int)up + (int)dn) * (1 + (int)lf + (int)rt);
                int need = 4 - n / 2;   // rank n/2 of n values == rank 4 of 9 with (4 - n/2) absent slots at -inf
                const bool present[9] = {up && lf, up, up && rt, lf, true, rt, dn && lf, dn, dn && rt};
#pragma unroll
                for (int q = 0; q < 9; q++)
                    if (!present[q] && need > 0) { v[q] = NINF; need--; }
                res[r] = median9(v);
            }
            asm volatile("cp.async.commit_group;\n" ::: "memory");
            // Publish the results of this step.  Row y writes ring slot (x & 3); during this same step row y+1
            // (at column x-2) reads slots (x-3..x-1) & 3 of row y -- three slots that differ from x & 3 -- so the
            // writes need no barrier of their own; one barrier per step makes them visible to the next step.
#pragma unroll
            for (int r = 0; r < MED_ROWS; r++) {
                if (!act[r]) continue;
                const int y = threadIdx.x + r * MT;
                const int x = t - 2 * y;
                med_ring[(size_t)y * 4 + (x & 3)] = res[r];
                left_new[r] = res[r];
                dst[y * W + x] = res[r];
            }
            __syncthreads();
        }
    }
    asm volatile("cp.async.wait_group 0;\n" ::: "memory");
}

int adc_launch_median(const AdcParams& P, const AdcWave& w, const float* in, float* out, cudaStream_t st,
                      unsigned long long* launches) {
    if (P.dm.H > MED_THREADS * 4) return 1;        // (adc_create rejects such images: ADC_MAX_HEIGHT)
    const int rows = P.dm.H <= MED_THREADS ? 1 : (P.dm.H <= 2 * MED_THREADS ? 2 : 4);
    const int pf = rows == 4 ? 4 : 8;
    const int threads = std::min(MED_THREADS, ((P.dm.H + rows - 1) / rows + 31) / 32 * 32);
    const size_t smem = ((size_t)P.dm.H * 4 + (size_t)threads * rows * pf * 2) * sizeof(float);
    static AdcOnce attr_once;
    if (adc_once_needed(attr_once)) {
        cudaFuncSetAttribute(k_median_wavefront<1, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(k_median_wavefront<2, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(k_median_wavefront<4, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        adc_once_done(attr_once);
    }
    if (rows == 1)      k_median_wavefront<1, 8><<<w.S, threads, smem, st>>>(P.dm, in, out);
    else if (rows == 2) k_median_wavefront<2, 8><<<w.S, threads, smem, st>>>(P.dm, in, out);
    else                k_median_wavefront<4, 4><<<w.S, threads, smem, st>>>(P.dm, in, out);
    ++*launches;
    return 0;
}
