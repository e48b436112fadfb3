// k_rectify.cu -- rectification on the way in (adc_set_rectification): the conversion of remap tables.
//
// Set time: k_remap_convert turns a view's remap table, float (CV_32FC1 x / y planes) or fixed (CV_16SC2 + CV_16UC1),
// into the engine's one internal form (adc_common.cuh AdcRectGeom): per output pixel the integer source corner
// (x0, y0) and the two 5-bit fractions, 8 bytes.  The float rule is OpenCV's: X = round_half_even(x * 32) saturated to
// int32, x0 = sat_int16(X >> 5), ax = X & 31.  cvt.rni.s32.f32 differs from x86's conversion in two places, and both are
// resolved here so that the result does not change (DESIGN.md section 14):
//   - NaN converts to 0 on the GPU (pixel 0, a real sample) but to INT_MIN on x86 (the border value): NaN is mapped to
//     INT_MIN explicitly;
//   - values outside int32 saturate to INT_MAX / INT_MIN on the GPU but give INT_MIN on x86 either way.  Any X outside
//     [-2^20, 2^20] has x0 = +-32767 / -32768 after the int16 saturation, and since src_width, src_height <= 32767
//     both neighbours x0 and x0 + 1 lie outside the frame: the border value 0 whichever way X saturated.
//
// Per wave the raw frames are resampled through these maps by k_view_ingest's remap geometry (k_image.cuh,
// rectified_px).
#include <algorithm>

#include "adc_common.cuh"
#include "k_image.cuh"

#define RC_THREADS 256

static __device__ __forceinline__ int sat_int16(int v) { return min(max(v, -32768), 32767); }

// OpenCV's cvRound(v * 32) on x86 for a float map coordinate: round half to even, INT_MIN for NaN (see the top)
static __device__ __forceinline__ int coord_x32(float v) { return isnan(v) ? INT_MIN : __float2int_rn(v * 32.0f); }

static __device__ __forceinline__ uint2 internal_form(int x0, int y0, int a) {
    return make_uint2((unsigned)(uint16_t)x0 | (unsigned)(uint16_t)y0 << 16, (unsigned)a);
}

__global__ void __launch_bounds__(RC_THREADS)
k_remap_convert_f32(int W, int N, const uint8_t* __restrict__ mx, long long px, const uint8_t* __restrict__ my,
                    long long py, uint2* __restrict__ out) {
    const int p = blockIdx.x * RC_THREADS + threadIdx.x;
    if (p >= N) return;
    const int y = p / W, x = p - y * W;
    const int X = coord_x32(__ldg(reinterpret_cast<const float*>(mx + y * px) + x));
    const int Y = coord_x32(__ldg(reinterpret_cast<const float*>(my + y * py) + x));
    out[p] = internal_form(sat_int16(X >> 5), sat_int16(Y >> 5), (X & 31) | (Y & 31) << 5);
}

__global__ void __launch_bounds__(RC_THREADS)
k_remap_convert_fixed(int W, int N, const uint8_t* __restrict__ m1, long long p1, const uint8_t* __restrict__ m2,
                      long long p2, uint2* __restrict__ out) {
    const int p = blockIdx.x * RC_THREADS + threadIdx.x;
    if (p >= N) return;
    const int y = p / W, x = p - y * W;
    const short* xy = reinterpret_cast<const short*>(m1 + y * p1) + 2 * x;
    const unsigned a = __ldg(reinterpret_cast<const unsigned short*>(m2 + y * p2) + x) & 1023u;
    out[p] = internal_form(__ldg(xy), __ldg(xy + 1), (int)a);
}

void adc_launch_remap_convert(const AdcDims& dm, int map_type, const void* map1, long long pitch1, const void* map2,
                              long long pitch2, uint2* out, cudaStream_t st) {
    const int grid = (dm.N + RC_THREADS - 1) / RC_THREADS;
    const uint8_t* m1 = static_cast<const uint8_t*>(map1);
    const uint8_t* m2 = static_cast<const uint8_t*>(map2);
    if (map_type == ADC_REMAP_F32) k_remap_convert_f32<<<grid, RC_THREADS, 0, st>>>(dm.W, dm.N, m1, pitch1, m2, pitch2, out);
    else k_remap_convert_fixed<<<grid, RC_THREADS, 0, st>>>(dm.W, dm.N, m1, pitch1, m2, pitch2, out);
}
