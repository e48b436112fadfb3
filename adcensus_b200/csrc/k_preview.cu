// k_preview.cu -- disparity / depth previews (adc_preview, adc_preview_batch_device; include/adcensus_b200_preview.h,
// DESIGN.md section 23).
//
// Two kernels, a fixed number of launches per call:
//   k_preview_minmax  (MINMAX only) the ordered-integer keys (adc_f2key) of each map's smallest and largest finite
//                     value: each CTA reduces a slice of one map with a warp __reduce_max_sync, then one atomicMax per
//                     warp into the map's two workspace words, which a memset zeroed in stream order.  The minimum is
//                     kept as ~key so that both words start at 0 and take atomicMax; a finite value's key and ~key are
//                     never 0, so 0 means "no valid pixel".  Atomics of max commute: the result does not depend on order.
//   k_preview<F>      one thread per run of 4 output pixels of a row (packed formats) or per 4 x 2 block (4:2:0, so
//                     that each chroma pair is computed once): the nearest source pixel, g, the CTA's table entry, and
//                     whole-word stores where the address allows.
// The table (shared memory, 257 words) holds, for g = 0..255 and the invalid colour (entry 256), the output pixel in
// the call's format: B | G << 8 | R << 16 (| 255 << 24 for BGRA), R | G << 8 | B << 16 | 255 << 24 for RGBA, the gray
// value, or Y | U << 8 | V << 16 for the YUV formats.  A pixel's whole colour conversion is that lookup, and lanes that
// read different entries do not serialise as they would on a __constant__ table (the 22 colormaps themselves are in
// global memory for the same reason).  A CTA keeps its run of output pixels for a stride of maps (blockIdx.y), so that
// the table and the source columns are built once per CTA rather than once per map.  Offsets are 64-bit: n *
// image_stride passes 2^31 bytes for 256 BGRA frames of 1920 x 1200.
#include <float.h>

#include <algorithm>

#include "adc_common.cuh"
#include "colormap_lut.h"

#define PV_THREADS 256
#define PV_MM_PIX 4096   // pixels per CTA of the min / max pass
#define PV_RUN 4         // output pixels per thread along x

enum { PV_BGR, PV_BGRA, PV_RGBA, PV_GRAY, PV_NV12, PV_NV21, PV_I420, PV_YV12 };

__global__ void __launch_bounds__(PV_THREADS)
k_preview_minmax(int N, long long n, const float* __restrict__ maps, unsigned* __restrict__ work) {
    const int i0 = blockIdx.x * PV_MM_PIX, i1 = min(N, i0 + PV_MM_PIX);
    for (long long m = blockIdx.y; m < n; m += gridDim.y) {
        const float* p = maps + (size_t)m * N;
        unsigned lo = 0, hi = 0;   // lo = ~key of the minimum
        for (int i = i0 + threadIdx.x; i < i1; i += PV_THREADS) {
            const float v = __ldg(p + i);
            if (isfinite(v)) {
                const unsigned k = adc_f2key(v);
                lo = max(lo, ~k);
                hi = max(hi, k);
            }
        }
        lo = __reduce_max_sync(0xffffffffu, lo);
        hi = __reduce_max_sync(0xffffffffu, hi);
        if ((threadIdx.x & 31) == 0 && hi != 0) {
            atomicMax(work + 2 * m, lo);
            atomicMax(work + 2 * m + 1, hi);
        }
    }
}

// The table word of pixel colour (b, g, r) in format F.
template <int F>
__device__ __forceinline__ unsigned pv_word(int b, int g, int r) {
    if (F == PV_BGR) return b | g << 8 | r << 16;
    if (F == PV_BGRA) return b | g << 8 | r << 16 | 255u << 24;
    if (F == PV_RGBA) return r | g << 8 | b << 16 | 255u << 24;
    if (F == PV_GRAY) return (9798 * r + 19235 * g + 3735 * b + (1 << 14)) >> 15;
    const int y = min(max((269484 * r + 528482 * g + 102760 * b + (1 << 19) + (16 << 20)) >> 20, 0), 255);
    const int u = min(max((-155188 * r - 305135 * g + 460324 * b + (1 << 19) + (128 << 20)) >> 20, 0), 255);
    const int v = min(max((460324 * r - 385875 * g - 74448 * b + (1 << 19) + (128 << 20)) >> 20, 0), 255);
    return y | u << 8 | v << 16;
}

// g of a finite value: round_half_even(fmaf(v, a, b)) saturated to 0..255, 0 where it is outside int32 (x86's cvtps2dq
// gives INT_MIN there, which the saturating packs make 0).  __float2int_rn saturates to INT_MIN below -2^31 already.
__device__ __forceinline__ int pv_g(float v, float a, float b) {
    const float t = __fmaf_rn(v, a, b);
    if (!(t < 2147483648.0f)) return 0;
    return min(max(__float2int_rn(t), 0), 255);
}

// Table entry of a source value: g, or 256 for an invalid (non-finite) pixel.
__device__ __forceinline__ int pv_entry(float v, float a, float b) { return isfinite(v) ? pv_g(v, a, b) : 256; }

// cv::resize INTER_NEAREST's source index of destination index d: min(floor(d * inv), n_src - 1), inv = 1.0 /
// ((double)n_dst / n_src) computed on the host.
__device__ __forceinline__ int pv_src(int d, double inv, int n_src) {
    return min(__double2int_rd(__dmul_rn((double)d, inv)), n_src - 1);
}

// k bytes of `w` (little-endian) at p: one word store when p is aligned and the whole word is the frame's, else bytes.
__device__ __forceinline__ void pv_store4(uint8_t* p, unsigned w, int k) {
    if (k == 4 && ((uintptr_t)p & 3) == 0) {
        *reinterpret_cast<unsigned*>(p) = w;
    } else {
        for (int j = 0; j < k; j++) p[j] = (uint8_t)(w >> (8 * j));
    }
}
__device__ __forceinline__ void pv_store2(uint8_t* p, unsigned w, int k) {
    if (k == 2 && ((uintptr_t)p & 1) == 0) {
        *reinterpret_cast<unsigned short*>(p) = (unsigned short)w;
    } else {
        for (int j = 0; j < k; j++) p[j] = (uint8_t)(w >> (8 * j));
    }
}

template <int F>
__global__ void __launch_bounds__(PV_THREADS)
k_preview(AdcPreviewArgs a, int W, int H, long long n, const float* __restrict__ maps) {
    constexpr bool yuv = F >= PV_NV12;
    __shared__ unsigned tab[257];
    for (int k = threadIdx.x; k < 257; k += PV_THREADS) {
        int b, g, r;
        if (k == 256) {
            b = a.invalid[0]; g = a.invalid[1]; r = a.invalid[2];
        } else if (a.colormap < 0) {
            b = g = r = k;
        } else {
            const unsigned char* c = g_colormap_lut[a.colormap] + 3 * k;
            b = __ldg(c); g = __ldg(c + 1); r = __ldg(c + 2);
        }
        tab[k] = pv_word<F>(b, g, r);
    }
    __syncthreads();
    const int runs = (a.dst_w + PV_RUN - 1) / PV_RUN;
    const long long units = (long long)runs * (yuv ? a.dst_h / 2 : a.dst_h);
    const long long u = (long long)blockIdx.x * PV_THREADS + threadIdx.x;
    if (u >= units) return;
    const int ry = (int)(u / runs), x0 = (int)(u - (long long)ry * runs) * PV_RUN;
    const int y0 = yuv ? 2 * ry : ry;
    const int cnt = min(PV_RUN, a.dst_w - x0);
    int sx[PV_RUN];
#pragma unroll
    for (int j = 0; j < PV_RUN; j++) sx[j] = pv_src(min(x0 + j, a.dst_w - 1), a.inv_x, W);
    const int N = W * H;
    for (long long m = blockIdx.y; m < n; m += gridDim.y) {
        float sc = a.alpha, sh = a.beta;
        if (a.work) {   // MINMAX: cv::normalize's scale and shift from the map's keys, in double
            const unsigned lo = ~a.work[2 * m], hi = a.work[2 * m + 1];
            sc = sh = 0.0f;
            if (hi != 0) {
                const double smin = adc_key2f(lo), smax = adc_key2f(hi), range = __dsub_rn(smax, smin);
                const double s = __dmul_rn(255.0, range > DBL_EPSILON ? __ddiv_rn(1.0, range) : 0.0);
                sc = __double2float_rn(s);
                sh = __double2float_rn(__dsub_rn(0.0, __dmul_rn(smin, s)));
            }
        }
        const float* mp = maps + (size_t)m * N;
        uint8_t* frame = a.dst + (size_t)m * a.image_stride;
#pragma unroll
        for (int dy = 0; dy < (yuv ? 2 : 1); dy++) {
            const int y = y0 + dy;
            const float* row = mp + (size_t)pv_src(y, a.inv_y, H) * W;
            unsigned w[PV_RUN];
#pragma unroll
            for (int j = 0; j < PV_RUN; j++) w[j] = tab[pv_entry(__ldg(row + sx[j]), sc, sh)];
            uint8_t* p = frame + (size_t)y * a.row_pitch;
            if (F == PV_BGRA || F == PV_RGBA) {
#pragma unroll
                for (int j = 0; j < PV_RUN; j++)
                    if (j < cnt) pv_store4(p + 4 * (x0 + j), w[j], 4);
            } else if (F == PV_BGR) {
                uint8_t* q = p + 3 * x0;
                if (cnt == PV_RUN && ((uintptr_t)q & 3) == 0) {
                    unsigned* o = reinterpret_cast<unsigned*>(q);
                    o[0] = w[0] | w[1] << 24;
                    o[1] = w[1] >> 8 | w[2] << 16;
                    o[2] = w[2] >> 16 | w[3] << 8;
                } else {
                    for (int j = 0; j < cnt; j++) pv_store4(q + 3 * j, w[j], 3);
                }
            } else {   // one byte per pixel: gray, or the Y of the YUV formats
                pv_store4(p + x0, (w[0] & 255) | (w[1] & 255) << 8 | (w[2] & 255) << 16 | (w[3] & 255) << 24, cnt);
            }
            if (yuv && dy == 0) {   // chroma of the blocks at x0 and x0 + 2, from their top-left pixels
                const unsigned u0 = w[0] >> 8 & 255, v0 = w[0] >> 16 & 255, u1 = w[2] >> 8 & 255, v1 = w[2] >> 16 & 255;
                const int cy = y0 / 2;
                if (F == PV_NV12 || F == PV_NV21) {
                    const unsigned c = F == PV_NV12 ? (u0 | v0 << 8 | u1 << 16 | v1 << 24) : (v0 | u0 << 8 | v1 << 16 | u1 << 24);
                    pv_store4(frame + a.plane_pitch + (size_t)cy * a.row_pitch + x0, c, cnt);
                } else {
                    const long long cp = a.row_pitch / 2;
                    uint8_t* first = frame + a.plane_pitch + cy * cp + x0 / 2;
                    uint8_t* second = first + (long long)(a.dst_h / 2) * cp;
                    const unsigned us = u0 | u1 << 8, vs = v0 | v1 << 8;
                    pv_store2(first, F == PV_I420 ? us : vs, cnt / 2);
                    pv_store2(second, F == PV_I420 ? vs : us, cnt / 2);
                }
            }
        }
    }
}

template <int F>
static void launch(const AdcDims& dm, long long n, const float* maps, const AdcPreviewArgs& a, cudaStream_t st) {
    const long long units = (long long)((a.dst_w + PV_RUN - 1) / PV_RUN) * (F >= PV_NV12 ? a.dst_h / 2 : a.dst_h);
    const long long gx = (units + PV_THREADS - 1) / PV_THREADS;
    // about four waves of resident CTAs in all; each CTA walks n / gridDim.y maps
    const long long gy = std::max(1ll, std::min({n, 65535ll, 4ll * 8 * adc_sm_count() / gx}));
    const dim3 grid((unsigned)gx, (unsigned)gy);
    k_preview<F><<<grid, PV_THREADS, 0, st>>>(a, dm.W, dm.H, n, maps);
}

void adc_launch_preview(const AdcDims& dm, long long n, const float* maps, const AdcPreviewArgs& a, cudaStream_t st,
                        unsigned long long* launches) {
    if (a.work) {
        const dim3 grid((unsigned)((dm.N + PV_MM_PIX - 1) / PV_MM_PIX), (unsigned)std::min(n, 65535ll));
        k_preview_minmax<<<grid, PV_THREADS, 0, st>>>(dm.N, n, maps, a.work);
        ++*launches;
    }
    switch (a.format) {
        case ADC_IMG_BGR: launch<PV_BGR>(dm, n, maps, a, st); break;
        case ADC_IMG_BGRA: launch<PV_BGRA>(dm, n, maps, a, st); break;
        case ADC_IMG_RGBA: launch<PV_RGBA>(dm, n, maps, a, st); break;
        case ADC_IMG_GRAY: launch<PV_GRAY>(dm, n, maps, a, st); break;
        case ADC_IMG_NV12: launch<PV_NV12>(dm, n, maps, a, st); break;
        case ADC_IMG_NV21: launch<PV_NV21>(dm, n, maps, a, st); break;
        case ADC_IMG_I420: launch<PV_I420>(dm, n, maps, a, st); break;
        default: launch<PV_YV12>(dm, n, maps, a, st); break;
    }
    ++*launches;
}
