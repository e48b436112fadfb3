// k_cost.cuh -- the AD-census matching cost of a block of four pixels x four disparities (cost_computor.cpp:58-121), the
// one definition of the cost arithmetic.  k_cost_volume (k_cost.cu) stores the block to the cost volume; the fused cost +
// first horizontal arm sum (k_cost_arm_sum_h, k_aggregate.cu) keeps it in shared memory and sums it there.
#pragma once
#include "adc_common.cuh"

// Row i of a block: left pixel i of the four (packed BGR cb, census words cl / ch) at disparity index d0 + j, matched against
// right-image entry 3 - j + i of the seven that the block touches (entries 0..3 in b0 / l0 / h0, 4..6 in b1 / l1 / h1;
// the 8th is not used).  An entry holding the marker 0xffffffff lies outside the image: its cost is 1.0
// (cost_computor.cpp:101-104).  Disparity indices >= D are padding (EXACT: D is a multiple of 4, there are none): 0.
// t_ad / t_ce point at this lane's replica of the AD table ([766] entries AD_REP floats apart) and of the census table
// ([64] entries 32 floats apart); both tables hold the host's expf factors, combined as ((1 - e_ad) + 1) - e_cen.
// Returns the costs of pixel i at disparity indices d0 .. d0 + 3; callers unroll i over 0..3.
template <bool EXACT, int AD_REP>
__device__ __forceinline__ float4 adc_cost_row(int i, const uint4& b0, const uint4& b1, const uint4& l0, const uint4& l1,
                                               const uint4& h0, const uint4& h1, const uint4& cb, const uint4& cl,
                                               const uint4& ch, const float* t_ad, const float* t_ce, int d0, int D) {
    const unsigned rb[7] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z};
    const unsigned rl[7] = {l0.x, l0.y, l0.z, l0.w, l1.x, l1.y, l1.z};
    const unsigned rh[7] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z};
    const unsigned lb[4] = {cb.x, cb.y, cb.z, cb.w}, ll[4] = {cl.x, cl.y, cl.z, cl.w}, lh[4] = {ch.x, ch.y, ch.z, ch.w};
    float out[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        // branch-free: padding disparities (di >= D) and out-of-image matches compute on whatever the entry holds and
        // are overwritten by selects -- the per-disparity branches used to cost more than the arithmetic
        const int c = 3 - j + i;
        const int sad = min((int)__vsadu4(lb[i], rb[c]), 765);     // |dB| + |dG| + |dR| (4th byte is 0 in both; the marker clamps)
        const int ham = (__popc(ll[i] ^ rl[c]) + __popc(lh[i] ^ rh[c])) & 63;
        float v = __fsub_rn(t_ad[sad * AD_REP], t_ce[ham * 32]);
        v = rb[c] == 0xffffffffu ? 1.0f : v;                        // out-of-image match: cost_computor.cpp:101-104
        out[j] = (EXACT || d0 + j < D) ? v : 0.0f;                  // padding disparity, never read as a cost
    }
    return make_float4(out[0], out[1], out[2], out[3]);
}
