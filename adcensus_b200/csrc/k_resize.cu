// k_resize.cu -- resizing on the way in (adc_set_rectification with r->map_type ADC_RESIZE_AREA / _LINEAR_EXACT,
// adc_match_rectified*, adc_ingest_views(rectified = 1)).
//
// The raw views are src_w x src_h frames in any ADC_IMG_* format.  k_resize_ingest<F, I> converts each source pixel it
// needs with the format's reader (view_px, k_image.cuh: demosaic, YUV rule, depth reduction, gray -> (v, v, v)), so it
// resamples the 8-bit BGR frame the format rule gives, and writes the wave's packed BGR with the store scheme of
// k_image.cuh.  The two rules (include/adcensus_b200.h, DESIGN.md section 22) are cv::resize's:
//   - ADC_RESIZE_AREA, integer factors kx = src_w / W, ky = src_h / H (each exact in double as OpenCV computes it,
//     which the engine checks at set time): each output pixel sums its own kx x ky block, so every source pixel is
//     read by exactly one output pixel; (s + 2) >> 2 for 2 x 2, round_half_even((float)s * (1.0f / n)) otherwise
//     (n = kx * ky, the reciprocal rounded to float on the host);
//   - ADC_RESIZE_LINEAR_EXACT, any sizes: per axis f = (d + 0.5) * scale - 0.5 in IEEE double (__dmul_rn /
//     __dadd_rn: no fused multiply-add), scale = 1 / (n_dst / n_src) rounded on the host, i = floor(f), 8-bit
//     weights c1 = round_half_even((f - i) * 256), c0 = 256 - c1, the index clamped into the frame with c1 = 0 at
//     both borders; each thread computes its own taps, so there are no tables.  Four neighbours, all inside the
//     frame, are blended as (h0 * c0y + h1 * c1y + 2^15) >> 16 with h = p[i] * c0x + p[i + 1] * c1x.
// Grid: blockIdx.x = tile * S + pair, blockIdx.y = view, as k_rectify_ingest.  Source offsets are 64-bit.
#include <algorithm>

#include "adc_common.cuh"
#include "k_image.cuh"

// Per-channel sums of B | G << 8 | R << 16 pixels.
struct Bgr3 {
    int b = 0, g = 0, r = 0;
    __device__ __forceinline__ void add(unsigned c) {
        b += c & 255u;
        g += c >> 8 & 255u;
        r += c >> 16 & 255u;
    }
};

// ADC_RESIZE_AREA: output pixel (x, y) from its kx x ky block.
template <int F>
static __device__ __forceinline__ unsigned area_px(const uint8_t* src, long long row_pitch, long long plane_pitch, int sw,
                                                   int sh, int kx, int ky, float inv_n, int x, int y) {
    Bgr3 s;
    const int x0 = x * kx, y0 = y * ky;
    if constexpr (img_mosaic(F)) {
        // a 2 x 2 block of a mosaic away from the frame's edges: the four sites from one 4x4 window of samples
        // (mosaic_quad) instead of four 3x3 neighbourhoods
        if (kx == 2 && ky == 2 && x0 >= 1 && x0 <= sw - 3 && y0 >= 1 && y0 <= sh - 3) {
            unsigned q[4];
            mosaic_quad<F>(src, row_pitch, x0, y0, q);
#pragma unroll
            for (int k = 0; k < 4; k++) s.add(q[k]);
            return (unsigned)((s.b + 2) >> 2) | (unsigned)((s.g + 2) >> 2) << 8 | (unsigned)((s.r + 2) >> 2) << 16;
        }
    }
    for (int j = 0; j < ky; j++)
        for (int i = 0; i < kx; i++) s.add(view_px<F>(src, row_pitch, plane_pitch, sw, sh, x0 + i, y0 + j));
    if (kx == 2 && ky == 2)
        return (unsigned)((s.b + 2) >> 2) | (unsigned)((s.g + 2) >> 2) << 8 | (unsigned)((s.r + 2) >> 2) << 16;
    const auto q = [&](int v) { return (unsigned)min(255, __float2int_rn(__fmul_rn(__int2float_rn(v), inv_n))); };
    return q(s.b) | q(s.g) << 8 | q(s.r) << 16;
}

// ADC_RESIZE_LINEAR_EXACT: the taps of destination index d on an axis of n source samples.
struct Tap {
    int i0, i1, c1;
};
static __device__ __forceinline__ Tap linear_tap(int d, double scale, int n) {
    const double f = __dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
    const double fl = floor(f);
    int i = (int)fl, c1 = __double2int_rn(__dmul_rn(__dsub_rn(f, fl), 256.0));
    if (i < 0) i = 0, c1 = 0;
    if (i >= n - 1) i = n - 1, c1 = 0;
    return Tap{i, min(i + 1, n - 1), c1};
}

template <int F>
static __device__ __forceinline__ unsigned linear_px(const uint8_t* src, long long row_pitch, long long plane_pitch,
                                                     int sw, int sh, double sx, double sy, int x, int y) {
    const Tap tx = linear_tap(x, sx, sw), ty = linear_tap(y, sy, sh);
    const unsigned p00 = view_px<F>(src, row_pitch, plane_pitch, sw, sh, tx.i0, ty.i0);
    const unsigned p01 = view_px<F>(src, row_pitch, plane_pitch, sw, sh, tx.i1, ty.i0);
    const unsigned p10 = view_px<F>(src, row_pitch, plane_pitch, sw, sh, tx.i0, ty.i1);
    const unsigned p11 = view_px<F>(src, row_pitch, plane_pitch, sw, sh, tx.i1, ty.i1);
    const int c0x = 256 - tx.c1, c0y = 256 - ty.c1;
    unsigned out = 0;
#pragma unroll
    for (int c = 0; c < 24; c += 8) {
        const int h0 = (int)(p00 >> c & 255u) * c0x + (int)(p01 >> c & 255u) * tx.c1;
        const int h1 = (int)(p10 >> c & 255u) * c0x + (int)(p11 >> c & 255u) * tx.c1;
        out |= (unsigned)((h0 * c0y + h1 * ty.c1 + (1 << 15)) >> 16) << c;
    }
    return out;
}

// The parameters of one geometry: the AREA factors and reciprocal, the LINEAR_EXACT scales.
struct ResizeRule {
    int kx, ky;
    float inv_n;
    double sx, sy;
};

template <int F, int I>
__global__ void __launch_bounds__(II_THREADS)
k_resize_ingest(int W, int N, int S, int sw, int sh, ResizeRule rule, const uint8_t* __restrict__ left,
                const uint8_t* __restrict__ right, long long row_pitch, long long plane_pitch, long long image_stride,
                uint8_t* __restrict__ bgr) {
    const int pair = blockIdx.x % S, tile = blockIdx.x / S, view = blockIdx.y;
    const uint8_t* src = (view ? right : left) + (long long)pair * image_stride;
    uint8_t* o = bgr + ((size_t)pair * 2 + view) * 3 * (size_t)N;
    store_view_bgr(o, N, W, tile, [&](int, int y, int x) {
        if constexpr (I == ADC_RESIZE_AREA)
            return area_px<F>(src, row_pitch, plane_pitch, sw, sh, rule.kx, rule.ky, rule.inv_n, x, y);
        else
            return linear_px<F>(src, row_pitch, plane_pitch, sw, sh, rule.sx, rule.sy, x, y);
    });
}

template <int F, int I>
static void launch_resize(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                          const AdcRectGeom& r, const ResizeRule& rule, uint8_t* bgr, cudaStream_t st) {
    const int tiles = std::max(1, (dm.N / 4 + II_GROUPS - 1) / II_GROUPS);
    dim3 grid((unsigned)(tiles * S), 2);
    k_resize_ingest<F, I><<<grid, II_THREADS, 0, st>>>(dm.W, dm.N, S, r.src_w, r.src_h, rule, left, right, g.row_pitch,
                                                       g.plane_pitch, g.image_stride, bgr);
}

void adc_launch_resize_ingest(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                              const AdcRectGeom& r, uint8_t* bgr, cudaStream_t st, unsigned long long* launches) {
    ResizeRule rule{};
    if (r.type == ADC_RESIZE_AREA) {
        rule.kx = r.src_w / dm.W;
        rule.ky = r.src_h / dm.H;
        rule.inv_n = 1.0f / (float)(rule.kx * rule.ky);
    } else {
        rule.sx = 1.0 / ((double)dm.W / r.src_w);   // OpenCV's scale, the inverse of its inv_scale
        rule.sy = 1.0 / ((double)dm.H / r.src_h);
    }
    const bool area = r.type == ADC_RESIZE_AREA;
    switch (g.format) {
#define RS_CASE(F)                                                                                                     \
    case F:                                                                                                            \
        if (area) launch_resize<F, ADC_RESIZE_AREA>(dm, S, left, right, g, r, rule, bgr, st);                          \
        else launch_resize<F, ADC_RESIZE_LINEAR_EXACT>(dm, S, left, right, g, r, rule, bgr, st);                       \
        break;
        ADC_IMG_CODES(RS_CASE)
#undef RS_CASE
    }
    ++*launches;
}
