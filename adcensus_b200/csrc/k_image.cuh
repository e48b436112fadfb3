// k_image.cuh -- the pieces the two image ingestion kernels share (k_image.cu: images in any format / pitch,
// k_rectify.cu: raw frames resampled through remap tables): the per-format pixel readers and the store scheme that
// writes one view's packed BGR.
//
// The output of one view is a contiguous run of 3*N bytes.  A thread takes four consecutive pixels of it at a time:
// 12 bytes, stored as three 32-bit words.  The view's run starts at an arbitrary byte phase (3*N*(2*pair + view) mod
// 4), so the groups start at the first pixel whose output address is a multiple of 4 (pixel a, for a run starting at
// a mod 4); the at most 3 pixels before it and 3 after the last whole group are written byte by byte.
#pragma once

#include <stdint.h>

#include "../../include/adcensus_b200.h"

// One pixel of a format as B | G << 8 | R << 16.  `row` points at the pixel row (of the first plane).  Alpha bytes are
// never loaded.  The loads are single bytes because the caller's bases and pitches may have any alignment.
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

// CTA `cta`'s share of one view's packed BGR run o (N pixels of W per row): the four-pixel groups
// [cta*II_GROUPS, (cta+1)*II_GROUPS), and for CTA 0 the head and tail pixels (threads 0..head-1 the head, threads 32..
// the tail).  px(p, y, x) gives output pixel p = y*W + x as B | G << 8 | R << 16; neighbouring lanes take neighbouring
// groups, so whatever px reads per pixel, a warp's reads cover one contiguous stretch of p.
template <class Px>
__device__ __forceinline__ void store_view_bgr(uint8_t* __restrict__ o, int N, int W, int cta, Px px) {
    const int head = min(N, (int)((uintptr_t)o & 3));
    const int G = (N - head) / 4, tail0 = head + 4 * G;
    const int g1 = min(G, (cta + 1) * II_GROUPS);
    for (int g = cta * II_GROUPS + threadIdx.x; g < g1; g += II_THREADS) {
        const int p = head + 4 * g;
        int y = p / W, x = p - y * W;
        unsigned c[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            c[j] = px(p + j, y, x);
            if (++x == W) { x = 0; ++y; }
        }
        unsigned* q = reinterpret_cast<unsigned*>(o + 3ll * p);
        q[0] = c[0] | c[1] << 24;
        q[1] = c[1] >> 8 | c[2] << 16;
        q[2] = c[2] >> 16 | c[3] << 8;
    }
    if (cta == 0) {
        const int t = threadIdx.x;
        const int p = t < head ? t : (t >= 32 && tail0 + t - 32 < N ? tail0 + t - 32 : -1);
        if (p >= 0) {
            const int y = p / W, x = p - y * W;
            const unsigned c = px(p, y, x);
            o[3ll * p] = (uint8_t)c;
            o[3ll * p + 1] = (uint8_t)(c >> 8);
            o[3ll * p + 2] = (uint8_t)(c >> 16);
        }
    }
}
