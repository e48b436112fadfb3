// k_render.cu -- the output side of the reference's demo program, SURVEY.md 8(f) rank 3 (reference: main.cpp:147-178
// ShowDisparityMap, :180-207 SaveDisparityMap, :209-230 SaveDisparityCloud): the 8-bit min/max-normalised disparity
// image, its cv::COLORMAP_JET colouring and the (x, y, disparity, r, g, b) cloud of the valid pixels.  Small kernels on
// one map; they exist so that a caller of the drop-in gets the demo's files without a round trip through OpenCV code.
#include "adc_common.cuh"
#include "jet_lut.h"

__constant__ unsigned char c_jet[256 * 3];
static AdcOnce g_jet_uploaded;   // per device

// min / max of |d| over the valid pixels; starting values float(width) / -float(width) as in main.cpp:151,185
__global__ void k_render_init(unsigned* mm, int width) {
    mm[0] = adc_f2key((float)width);
    mm[1] = adc_f2key(-(float)width);
}

__global__ void __launch_bounds__(256)
k_render_minmax(int n, const float* __restrict__ disp, unsigned* mm) {
    unsigned lo = 0xffffffffu, hi = 0u;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float d = fabsf(disp[i]);
        if (d != ADC_INVALID_F) { const unsigned k = adc_f2key(d); lo = min(lo, k); hi = max(hi, k); }
    }
    lo = __reduce_min_sync(0xffffffffu, lo);
    hi = __reduce_max_sync(0xffffffffu, hi);
    if ((threadIdx.x & 31) == 0) { atomicMin(mm + 0, lo); atomicMax(mm + 1, hi); }
}

// gray = uchar((|d| - min) / (max - min) * 255), 0 for invalid pixels (main.cpp:160-170); float32 arithmetic, truncation.
// A constant map (max == min) divides 0 by 0 in the reference (an undefined float -> uchar conversion); 0 is written here.
__global__ void __launch_bounds__(256)
k_render_gray_jet(int n, const float* __restrict__ disp, const unsigned* __restrict__ mm, uint8_t* __restrict__ gray,
                  uint8_t* __restrict__ jet, float* __restrict__ mm_out) {
    const float mn = adc_key2f(mm[0]), mx = adc_key2f(mm[1]);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 && mm_out) { mm_out[0] = mn; mm_out[1] = mx; }
    if (i >= n) return;
    const float d = fabsf(disp[i]);
    unsigned g = 0;
    if (d != ADC_INVALID_F) {
        const float range = __fsub_rn(mx, mn);
        if (range != 0.0f) {
            const float v = __fmul_rn(__fdiv_rn(__fsub_rn(d, mn), range), 255.0f);
            g = (unsigned)__float2int_rz(v) & 255u;
        }
    }
    if (gray) gray[i] = (uint8_t)g;
    if (jet) { jet[3 * i] = c_jet[3 * g]; jet[3 * i + 1] = c_jet[3 * g + 1]; jet[3 * i + 2] = c_jet[3 * g + 2]; }
}

__global__ void __launch_bounds__(256)
k_render_valid(int n, const float* __restrict__ disp, uint8_t* __restrict__ label) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) label[i] = fabsf(disp[i]) != ADC_INVALID_F ? 1 : 0;
}

// one record per valid pixel, raster order: x, y, |d|, r, g, b (main.cpp:219-225; the image is packed BGR)
__global__ void __launch_bounds__(256)
k_render_cloud(int W, const int* __restrict__ list, const int* __restrict__ counters, const float* __restrict__ disp,
               const uint8_t* __restrict__ bgr, float* __restrict__ cloud) {
    const int n = counters[0];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int p = list[i], y = p / W, x = p - y * W;
    float* o = cloud + (size_t)i * 6;
    o[0] = (float)x; o[1] = (float)y; o[2] = fabsf(disp[p]);
    o[3] = (float)bgr[3 * p + 2]; o[4] = (float)bgr[3 * p + 1]; o[5] = (float)bgr[3 * p];
}

int adc_launch_render(const AdcDims& dm, const float* d_disp, unsigned* d_mm, uint8_t* d_gray, uint8_t* d_jet, float* d_mm_out,
                      cudaStream_t st, unsigned long long* launches) {
    if (adc_once_needed(g_jet_uploaded)) {
        if (cudaMemcpyToSymbol(c_jet, ADC_JET_LUT, sizeof(ADC_JET_LUT)) != cudaSuccess) return 1;
        adc_once_done(g_jet_uploaded);
    }
    k_render_init<<<1, 1, 0, st>>>(d_mm, dm.W);
    k_render_minmax<<<adc_sm_count(), 256, 0, st>>>(dm.N, d_disp, d_mm);
    k_render_gray_jet<<<(dm.N + 255) / 256, 256, 0, st>>>(dm.N, d_disp, d_mm, d_gray, d_jet, d_mm_out);
    *launches += 3;
    return 0;
}

void adc_launch_cloud(const AdcParams& P, const AdcWave& w1 /* S = 1 */, const float* d_disp, const uint8_t* d_bgr, float* d_cloud,
                      cudaStream_t st, unsigned long long* launches) {
    k_render_valid<<<(P.dm.N + 255) / 256, 256, 0, st>>>(P.dm.N, d_disp, w1.label);
    adc_launch_build_lists(P, w1, st, launches);       // raster-ordered list of the pixels labelled 1 -> w1.pend, counters[0]
    k_render_cloud<<<(P.dm.N + 255) / 256, 256, 0, st>>>(P.dm.W, w1.pend, w1.counters, d_disp, d_bgr, d_cloud);
    *launches += 2;
}
