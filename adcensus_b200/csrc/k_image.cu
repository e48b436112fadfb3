// k_image.cu -- image ingestion (adc_match_images*): the caller's views, in any of the ADC_IMG_* formats and with any
// row, plane and image pitch, become the wave's packed BGR images ([S][2][H][W][3], what the rest of the pipeline reads)
// in one pass.  Channel order is resolved, alpha is skipped, a gray value v becomes (v, v, v); nothing else happens to a
// pixel, so the gray conversion, the census and every later stage see exactly the bytes a caller who packed the same
// pixels as BGR would have handed in.
//
// The output of one view is a contiguous run of 3*N bytes.  A thread takes four consecutive pixels of it at a time:
// 12 bytes, stored as three 32-bit words.  The view's run starts at an arbitrary byte phase (3*N*(2*pair + view) mod
// 4), so the groups start at the first pixel whose output address is a multiple of 4 (pixel a, for a run starting at
// a mod 4); the at most 3 pixels before it and 3 after the last whole group are written byte by byte.
// Source reads: pixel p of the view is (y, x) = divmod(p, W) at base + y*row_pitch + x*bytes_per_pixel (+ c*plane_pitch
// for planar images); neighbouring lanes take neighbouring groups, so a warp's loads cover one contiguous stretch of a
// row (of each plane): coalesced along x.  Every pixel is loaded by exactly one thread, alpha bytes are never loaded, and
// nothing past the last pixel of the last row is touched.  The loads are single bytes because the caller's bases and
// pitches may have any alignment.  All source offsets are 64-bit.
#include <algorithm>

#include "adc_common.cuh"
#include "../../include/adcensus_b200.h"

// One pixel of a format as B | G << 8 | R << 16.  `row` points at the pixel row (of the first plane).
template <int F> struct ImgIn;
template <> struct ImgIn<ADC_IMG_BGR> {
    static __device__ __forceinline__ unsigned px(const uint8_t* row, int x, long long) {
        const uint8_t* p = row + 3ll * x;
        return __ldg(p) | (unsigned)__ldg(p + 1) << 8 | (unsigned)__ldg(p + 2) << 16;
    }
};
template <> struct ImgIn<ADC_IMG_RGB> {
    static __device__ __forceinline__ unsigned px(const uint8_t* row, int x, long long) {
        const uint8_t* p = row + 3ll * x;
        return __ldg(p + 2) | (unsigned)__ldg(p + 1) << 8 | (unsigned)__ldg(p) << 16;
    }
};
template <> struct ImgIn<ADC_IMG_BGRA> {
    static __device__ __forceinline__ unsigned px(const uint8_t* row, int x, long long) {
        const uint8_t* p = row + 4ll * x;
        return __ldg(p) | (unsigned)__ldg(p + 1) << 8 | (unsigned)__ldg(p + 2) << 16;
    }
};
template <> struct ImgIn<ADC_IMG_RGBA> {
    static __device__ __forceinline__ unsigned px(const uint8_t* row, int x, long long) {
        const uint8_t* p = row + 4ll * x;
        return __ldg(p + 2) | (unsigned)__ldg(p + 1) << 8 | (unsigned)__ldg(p) << 16;
    }
};
template <> struct ImgIn<ADC_IMG_GRAY> {
    static __device__ __forceinline__ unsigned px(const uint8_t* row, int x, long long) { return __ldg(row + x) * 0x010101u; }
};
template <> struct ImgIn<ADC_IMG_RGB_PLANAR> {
    static __device__ __forceinline__ unsigned px(const uint8_t* row, int x, long long plane) {
        const uint8_t* p = row + x;
        return __ldg(p + 2 * plane) | (unsigned)__ldg(p + plane) << 8 | (unsigned)__ldg(p) << 16;
    }
};

#define II_THREADS 256
#define II_GROUPS 1024   // four-pixel groups per CTA

template <int F>
__global__ void __launch_bounds__(II_THREADS)
k_image_ingest(int W, int N, const uint8_t* __restrict__ left, const uint8_t* __restrict__ right, long long row_pitch,
               long long plane_pitch, long long image_stride, uint8_t* __restrict__ bgr) {
    const int view = blockIdx.y, pair = blockIdx.z;
    const uint8_t* src = (view ? right : left) + (long long)pair * image_stride;
    uint8_t* o = bgr + ((size_t)pair * 2 + view) * 3 * (size_t)N;
    const int head = min(N, (int)((uintptr_t)o & 3));
    const int G = (N - head) / 4, tail0 = head + 4 * G;
    const int g1 = min(G, (blockIdx.x + 1) * II_GROUPS);
    for (int g = blockIdx.x * II_GROUPS + threadIdx.x; g < g1; g += II_THREADS) {
        const int p = head + 4 * g;
        int y = p / W, x = p - y * W;
        unsigned c[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            c[j] = ImgIn<F>::px(src + y * row_pitch, x, plane_pitch);
            if (++x == W) { x = 0; ++y; }
        }
        unsigned* q = reinterpret_cast<unsigned*>(o + 3ll * p);
        q[0] = c[0] | c[1] << 24;
        q[1] = c[1] >> 8 | c[2] << 16;
        q[2] = c[2] >> 16 | c[3] << 8;
    }
    // CTA 0: threads 0..head-1 take the head, threads 32.. the tail (each fewer than 4 pixels)
    if (blockIdx.x == 0) {
        const int t = threadIdx.x;
        const int p = t < head ? t : (t >= 32 && tail0 + t - 32 < N ? tail0 + t - 32 : -1);
        if (p >= 0) {
            const int y = p / W, x = p - y * W;
            const unsigned c = ImgIn<F>::px(src + y * row_pitch, x, plane_pitch);
            o[3ll * p] = (uint8_t)c;
            o[3ll * p + 1] = (uint8_t)(c >> 8);
            o[3ll * p + 2] = (uint8_t)(c >> 16);
        }
    }
}

template <int F>
static void launch_image(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                         uint8_t* bgr, cudaStream_t st) {
    const int groups = dm.N / 4;
    dim3 grid(std::max(1, (groups + II_GROUPS - 1) / II_GROUPS), 2, S);
    k_image_ingest<F><<<grid, II_THREADS, 0, st>>>(dm.W, dm.N, left, right, g.row_pitch, g.plane_pitch, g.image_stride, bgr);
}

void adc_launch_image_ingest(const AdcParams& P, const AdcWave& w, const uint8_t* left, const uint8_t* right,
                             const AdcImageGeom& g, cudaStream_t st, unsigned long long* launches) {
    switch (g.format) {
        case ADC_IMG_BGR: launch_image<ADC_IMG_BGR>(P.dm, w.S, left, right, g, w.bgr, st); break;
        case ADC_IMG_RGB: launch_image<ADC_IMG_RGB>(P.dm, w.S, left, right, g, w.bgr, st); break;
        case ADC_IMG_BGRA: launch_image<ADC_IMG_BGRA>(P.dm, w.S, left, right, g, w.bgr, st); break;
        case ADC_IMG_RGBA: launch_image<ADC_IMG_RGBA>(P.dm, w.S, left, right, g, w.bgr, st); break;
        case ADC_IMG_GRAY: launch_image<ADC_IMG_GRAY>(P.dm, w.S, left, right, g, w.bgr, st); break;
        default: launch_image<ADC_IMG_RGB_PLANAR>(P.dm, w.S, left, right, g, w.bgr, st); break;
    }
    ++*launches;
}

int adc_image_bytes_per_pixel(int format) {
    switch (format) {
        case ADC_IMG_BGR: case ADC_IMG_RGB: return 3;
        case ADC_IMG_BGRA: case ADC_IMG_RGBA: return 4;
        default: return 1;   // gray, and each plane of a planar image
    }
}
