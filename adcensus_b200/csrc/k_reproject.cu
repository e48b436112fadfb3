// k_reproject.cu -- reprojection to 3-D (adc_reproject, adc_reproject_batch_device).
//
// One pass over n disparity maps: each pixel's f32 value is read once, and only the requested outputs are written
// (include/adcensus_b200.h, DESIGN.md section 15):
//   POINTS    cv::reprojectImageTo3D bit for bit: h_i = (((+0.0 + Q[i][0]*x) + Q[i][1]*y) + Q[i][2]*d) + Q[i][3] in
//             double, P_c = (float)((double)(float)h_c * (1.0 / h_3)); P_z = 10000 where d is FLT_MAX
//   DEPTH     P_2 alone
//   DISP_S16  saturate_cast<short>(d * 16) as x86 computes it, (min_disparity - 1) * 16 for +inf
// The double arithmetic (q_row, coord) is in k_reproject.cuh, shared with the point clouds of k_cloud.cu.
// Each template instance computes only what its outputs need: the S16-only kernel does no double arithmetic, the
// depth-only kernel evaluates rows 2 and 3.
// Grid: blockIdx.x = a run of RP_PIX consecutive pixels of a map, blockIdx.y (striding by gridDim.y) = the map.  Offsets
// into the batch are 64-bit: n * H * W * 12 bytes of points pass 2^31 for about 90 maps of 1080p.  The 12-byte points
// of a CTA's run are staged in shared memory and leave it as consecutive 32-bit words, so every warp store is one
// contiguous 128-byte stretch; destinations need only 4-byte alignment.
#include <algorithm>

#include "adc_common.cuh"
#include "k_reproject.cuh"

#define RP_THREADS 256
#define RP_PER_THREAD 4
#define RP_PIX (RP_THREADS * RP_PER_THREAD)   // pixels per CTA and map

enum { RP_POINTS = 1, RP_DEPTH = 2, RP_S16 = 4 };

// cv::saturate_cast<short>(d * 16) on x86, the engine's invalid value for +inf
static __device__ __forceinline__ int16_t disp_s16(float d, int16_t invalid) {
    if (d == __int_as_float(0x7f800000)) return invalid;
    const float t = __fmul_rn(d, 16.0f);   // exact, or +-inf past FLT_MAX
    // NaN, +inf and every t at or above 2^31 convert to x86's integer indefinite, INT_MIN
    if (!(t < 2147483648.0f)) return -32768;
    // round half to even; -inf and t below -2^31 give INT_MIN here as on x86
    return (int16_t)min(max(__float2int_rn(t), -32768), 32767);
}

template <int K>
__global__ void __launch_bounds__(RP_THREADS)
k_reproject(int W, int N, long long n, const float* __restrict__ disp, const AdcReprojQ Q, float* __restrict__ points,
            float* __restrict__ depth, int16_t* __restrict__ s16, int16_t s16_invalid) {
    __shared__ float stage[(K & RP_POINTS) ? 3 * RP_PIX : 1];
    const int r0 = blockIdx.x * RP_PIX;
    const int cnt = min(RP_PIX, N - r0);
    for (long long m = blockIdx.y; m < n; m += gridDim.y) {
        const size_t base = (size_t)m * N + r0;
#pragma unroll
        for (int k = 0; k < RP_PER_THREAD; k++) {
            const int j = k * RP_THREADS + threadIdx.x;
            if (j >= cnt) break;
            const float d = __ldg(disp + base + j);
            if (K & RP_S16) s16[base + j] = disp_s16(d, s16_invalid);
            if (K & (RP_POINTS | RP_DEPTH)) {
                const int r = r0 + j, y = r / W, x = r - y * W;
                const double xd = x, yd = y, dd = d;
                const double ia = __drcp_rn(q_row(Q, 3, xd, yd, dd));
                const float z = coord_z(Q, xd, yd, d, ia);
                if (K & RP_DEPTH) depth[base + j] = z;
                if (K & RP_POINTS) {
                    stage[3 * j] = coord(q_row(Q, 0, xd, yd, dd), ia);
                    stage[3 * j + 1] = coord(q_row(Q, 1, xd, yd, dd), ia);
                    stage[3 * j + 2] = z;
                }
            }
        }
        if (K & RP_POINTS) {
            __syncthreads();
            float* o = points + 3 * base;
            for (int j = threadIdx.x; j < 3 * cnt; j += RP_THREADS) o[j] = stage[j];
            __syncthreads();   // the next map's pixels reuse the stage
        }
    }
}

template <int K>
static void launch(const AdcDims& dm, long long n, const float* disp, const AdcReprojQ& Q, float* points, float* depth,
                   int16_t* s16, int16_t s16_invalid, cudaStream_t st) {
    const dim3 grid((unsigned)((dm.N + RP_PIX - 1) / RP_PIX), (unsigned)std::min(n, 65535ll));
    k_reproject<K><<<grid, RP_THREADS, 0, st>>>(dm.W, dm.N, n, disp, Q, points, depth, s16, s16_invalid);
}

void adc_launch_reproject(const AdcDims& dm, long long n, const float* disp, const AdcReprojQ& Q, float* points,
                          float* depth, int16_t* s16, int16_t s16_invalid, cudaStream_t st, unsigned long long* launches) {
    const int k = (points ? RP_POINTS : 0) | (depth ? RP_DEPTH : 0) | (s16 ? RP_S16 : 0);
    switch (k) {
        case 1: launch<1>(dm, n, disp, Q, points, depth, s16, s16_invalid, st); break;
        case 2: launch<2>(dm, n, disp, Q, points, depth, s16, s16_invalid, st); break;
        case 3: launch<3>(dm, n, disp, Q, points, depth, s16, s16_invalid, st); break;
        case 4: launch<4>(dm, n, disp, Q, points, depth, s16, s16_invalid, st); break;
        case 5: launch<5>(dm, n, disp, Q, points, depth, s16, s16_invalid, st); break;
        case 6: launch<6>(dm, n, disp, Q, points, depth, s16, s16_invalid, st); break;
        default: launch<7>(dm, n, disp, Q, points, depth, s16, s16_invalid, st); break;
    }
    ++*launches;
}
