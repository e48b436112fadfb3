// k_rectify.cu -- rectification on the way in (adc_set_rectification, adc_match_rectified*).
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
// Per wave: k_rectify_ingest<F> makes one launch over the wave's pairs x 2 views.  For each output pixel it gathers
// the four neighbours of (x0, y0) from the raw view through the format readers of k_image.cuh, weights them
// (32 - ax | ax) * (32 - ay | ay), and writes (sum + 512) >> 10 per channel with the store scheme of k_image.cuh.  When
// all four neighbours lie inside the frame (0 <= x0 < src_width - 1, 0 <= y0 < src_height - 1; never for a frame one
// pixel wide or high) the loads are unconditional; otherwise each neighbour is loaded only if it is inside, so nothing
// outside a view's frame is read, and alpha bytes never are.  Source offsets are 64-bit.
// Grid: blockIdx.x = tile * S + pair, blockIdx.y = view.  The S CTAs that read the same stretch of a view's map are
// adjacent in launch order and run at the same time, so a wave reads each map from HBM once and from L2 S - 1 times.
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

// One output pixel: the bilinear blend of the raw view `src` at map entry m, as B | G << 8 | R << 16.
template <int F>
static __device__ __forceinline__ unsigned rectified_px(uint2 m, const uint8_t* src, int sw, int sh, long long row_pitch,
                                                        long long plane_pitch) {
    const int x0 = (short)(m.x & 0xffffu), y0 = (short)(m.x >> 16);
    const int ax = m.y & 31, ay = m.y >> 5;
    unsigned s[4];   // (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1)
    if ((unsigned)x0 < (unsigned)(sw - 1) && (unsigned)y0 < (unsigned)(sh - 1)) {
        const uint8_t* r0 = src + y0 * row_pitch;
        s[0] = ImgIn<F>::px(r0, x0, plane_pitch);
        s[1] = ImgIn<F>::px(r0, x0 + 1, plane_pitch);
        s[2] = ImgIn<F>::px(r0 + row_pitch, x0, plane_pitch);
        s[3] = ImgIn<F>::px(r0 + row_pitch, x0 + 1, plane_pitch);
    } else {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int x = x0 + (k & 1), y = y0 + (k >> 1);
            s[k] = (unsigned)x < (unsigned)sw && (unsigned)y < (unsigned)sh ? ImgIn<F>::px(src + y * row_pitch, x, plane_pitch) : 0u;
        }
    }
    const int w[4] = {(32 - ax) * (32 - ay), ax * (32 - ay), (32 - ax) * ay, ax * ay};
    unsigned out = 0;
#pragma unroll
    for (int c = 0; c < 24; c += 8) {
        int v = 512;
#pragma unroll
        for (int k = 0; k < 4; k++) v += w[k] * (int)(s[k] >> c & 255u);
        out |= (unsigned)(v >> 10) << c;
    }
    return out;
}

template <int F>
__global__ void __launch_bounds__(II_THREADS)
k_rectify_ingest(int W, int N, int S, int sw, int sh, const uint2* __restrict__ map_l, const uint2* __restrict__ map_r,
                 const uint8_t* __restrict__ left, const uint8_t* __restrict__ right, long long row_pitch,
                 long long plane_pitch, long long image_stride, uint8_t* __restrict__ bgr) {
    const int pair = blockIdx.x % S, tile = blockIdx.x / S, view = blockIdx.y;
    const uint8_t* src = (view ? right : left) + (long long)pair * image_stride;
    const uint2* map = view ? map_r : map_l;
    uint8_t* o = bgr + ((size_t)pair * 2 + view) * 3 * (size_t)N;
    store_view_bgr(o, N, W, tile, [&](int p, int, int) {
        return rectified_px<F>(__ldg(map + p), src, sw, sh, row_pitch, plane_pitch);
    });
}

template <int F>
static void launch_rectify(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                           const AdcRectGeom& r, uint8_t* bgr, cudaStream_t st) {
    const int tiles = std::max(1, (dm.N / 4 + II_GROUPS - 1) / II_GROUPS);
    dim3 grid((unsigned)(tiles * S), 2);
    k_rectify_ingest<F><<<grid, II_THREADS, 0, st>>>(dm.W, dm.N, S, r.src_w, r.src_h, r.map[0], r.map[1], left, right,
                                                     g.row_pitch, g.plane_pitch, g.image_stride, bgr);
}

void adc_launch_rectify_ingest(const AdcParams& P, const AdcWave& w, const uint8_t* left, const uint8_t* right,
                               const AdcImageGeom& g, const AdcRectGeom& r, cudaStream_t st, unsigned long long* launches) {
    switch (g.format) {
        case ADC_IMG_BGR: launch_rectify<ADC_IMG_BGR>(P.dm, w.S, left, right, g, r, w.bgr, st); break;
        case ADC_IMG_RGB: launch_rectify<ADC_IMG_RGB>(P.dm, w.S, left, right, g, r, w.bgr, st); break;
        case ADC_IMG_BGRA: launch_rectify<ADC_IMG_BGRA>(P.dm, w.S, left, right, g, r, w.bgr, st); break;
        case ADC_IMG_RGBA: launch_rectify<ADC_IMG_RGBA>(P.dm, w.S, left, right, g, r, w.bgr, st); break;
        case ADC_IMG_GRAY: launch_rectify<ADC_IMG_GRAY>(P.dm, w.S, left, right, g, r, w.bgr, st); break;
        default: launch_rectify<ADC_IMG_RGB_PLANAR>(P.dm, w.S, left, right, g, r, w.bgr, st); break;
    }
    ++*launches;
}
