// k_confidence.cu -- cost-curve confidence of the left view: MIN_COST = c1 = C(d1) and PEAK_RATIO = c1 / c2 per pixel,
// from the scanline-optimised volume the WTA reads (definitions in include/adcensus_b200.h, ADC_MAP_*).
#include "adc_common.cuh"

// ---------------------------------------------------------------------------------------------
// One streaming reduction over d per pixel, the volume read once.  A CTA owns CF_PX neighbouring pixels of one image row
// and sweeps the disparity range in chunks of CF_DC, staging the chunk of its columns in shared memory with coalesced
// 128-bit loads (four lanes read the 64 contiguous bytes of one pixel's chunk) that are issued one chunk ahead, as in
// k_wta's left tile.  Shared memory is one chunk (8 KB), independent of the disparity range.
//
// Each thread keeps the four smallest (value, index) pairs of its pixel in registers, ordered by value and, among equal
// values, by index: d runs upwards and a cost enters only if it is strictly below the fourth, so an equal value never
// overtakes an earlier index.  Slot 0 is then the first minimum d1, the index the left WTA's strict '>' scan picks.
// At most three of the four lie in {d1 - 1, d1, d1 + 1}, so the first slot outside that set holds c2 = min C(d) over
// |d - d1| >= 2; if none does, no such d exists.
// ---------------------------------------------------------------------------------------------
#define CF_PX 128
#define CF_DC 16
#define CF_LS CF_DC            // row stride of the tile; quad k of column t is stored at quad k ^ ((t >> 1) & 3) (k_wta's swizzle:
                               // the eight threads of a 128-bit phase hit eight different 16-byte bank groups)

__global__ void __launch_bounds__(CF_PX)
k_confidence(AdcDims dm, const float* __restrict__ vol, float* __restrict__ min_cost, float* __restrict__ peak_ratio) {
    __shared__ __align__(16) float tl[CF_PX * CF_LS];
    const int pair = blockIdx.z, y = blockIdx.y, x0 = blockIdx.x * CF_PX;
    const int W = dm.W, D = dm.D, Dp = dm.Dp;
    const float* rowv = vol + (size_t)pair * dm.vol_stride + (size_t)y * W * Dp;
    const int t = threadIdx.x;
    const int kq = t & 3, cj = t >> 2;                  // staging role: float4 kq of the chunk, 32 columns per trip
    const float INF = __int_as_float(0x7f800000);
    float v0 = INF, v1 = INF, v2 = INF, v3 = INF;       // the four smallest costs, ascending
    int i0 = -1, i1 = -1, i2 = -1, i3 = -1;             // their indices d, -1 = slot empty
    float4 vl[CF_PX / 32];
    auto fetch = [&](int d0) {
        const bool qin = d0 + 4 * kq < Dp;              // this float4 exists (Dp is a multiple of 4)
        const float* cv = rowv + d0 + 4 * kq;
#pragma unroll
        for (int i = 0; i < CF_PX / 32; i++) {
            const int x = x0 + cj + 32 * i;
            vl[i] = (qin && x < W) ? __ldg(reinterpret_cast<const float4*>(cv + (size_t)x * Dp)) : make_float4(INF, INF, INF, INF);
        }
    };
    auto insert = [&](float c, int d) {
        if (c < v3) {
            v3 = c; i3 = d;
            if (v3 < v2) { v3 = v2; i3 = i2; v2 = c; i2 = d;
                if (v2 < v1) { v2 = v1; i2 = i1; v1 = c; i1 = d;
                    if (v1 < v0) { v1 = v0; i1 = i0; v0 = c; i0 = d; } } }
        }
    };
    fetch(0);
    for (int d0 = 0; d0 < D; d0 += CF_DC) {
        const int dn = min(CF_DC, D - d0);
#pragma unroll
        for (int i = 0; i < CF_PX / 32; i++)
            *reinterpret_cast<float4*>(tl + (cj + 32 * i) * CF_LS + 4 * (kq ^ ((cj >> 1) & 3))) = vl[i];
        __syncthreads();
        if (d0 + CF_DC < D) fetch(d0 + CF_DC);
        const float* pl = tl + t * CF_LS;
        const int sw = ((t >> 1) & 3) << 2;             // this column's quad swizzle, as a word offset
        if (dn == CF_DC) {
#pragma unroll
            for (int k4 = 0; k4 < CF_DC; k4 += 4) {
                const float4 a4 = *reinterpret_cast<const float4*>(pl + (k4 ^ sw));
                insert(a4.x, d0 + k4);
                insert(a4.y, d0 + k4 + 1);
                insert(a4.z, d0 + k4 + 2);
                insert(a4.w, d0 + k4 + 3);
            }
        } else {
            for (int k = 0; k < dn; k++) insert(pl[k ^ sw], d0 + k);
        }
        __syncthreads();
    }
    const int x = x0 + t;
    if (x >= W) return;
    const size_t o = (size_t)pair * dm.N + (size_t)y * W + x;
    if (min_cost) min_cost[o] = v0;
    if (peak_ratio) {
        // c2: the first slot (in value order) whose index is at least 2 away from d1
        float c2 = INF;
        bool found = false;
        if (i1 >= 0 && abs(i1 - i0) >= 2) { c2 = v1; found = true; }
        else if (i2 >= 0 && abs(i2 - i0) >= 2) { c2 = v2; found = true; }
        else if (i3 >= 0 && abs(i3 - i0) >= 2) { c2 = v3; found = true; }
        peak_ratio[o] = (found && c2 != 0.0f) ? __fdiv_rn(v0, c2) : 1.0f;
    }
}

void adc_launch_confidence(const AdcParams& P, const AdcWave& w, const float* vol, float* min_cost, float* peak_ratio,
                           cudaStream_t st, unsigned long long* launches) {
    dim3 grid((P.dm.W + CF_PX - 1) / CF_PX, P.dm.H, w.S);
    k_confidence<<<grid, CF_PX, 0, st>>>(P.dm, vol, min_cost, peak_ratio);
    ++*launches;
}
