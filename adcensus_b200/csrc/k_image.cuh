// k_image.cuh -- the view ingestion kernel k_view_ingest<F, G>: a caller's views in format F (any ADC_IMG_* code) and
// source geometry G become packed BGR.  G says which source pixels an output pixel reads: its own pixel in place
// (plain), four neighbours through a remap table (remap), its block (resize AREA) or four taps (resize LINEAR_EXACT).
// Here are the per-format pixel readers, the one demosaic reader of the 8-bit and high-bit-depth mosaics, the YUV
// conversion, the 10- / 12- / 16-bit sample readers with their depth reduction, the pixel rule of each geometry, the
// store scheme that writes one view's packed BGR, and the kernel with its launcher.  The formats and their constants
// come from img_format.h; the launch and its dispatch are in k_image.cu.
//
// The output of one view is a contiguous run of 3*N bytes.  A thread takes four consecutive pixels of it at a time:
// 12 bytes, stored as three 32-bit words.  The view's run starts at an arbitrary byte phase (3*N*(2*pair + view) mod
// 4), so the groups start at the first pixel whose output address is a multiple of 4 (pixel a, for a run starting at
// a mod 4); the at most 3 pixels before it and 3 after the last whole group are written byte by byte.
#pragma once

#include <stdint.h>

#include <algorithm>

#include "../../include/adcensus_b200.h"
#include "adc_common.cuh"

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

// round_half_even(v / 2^S) saturated to 8 bits, the depth reduction of the high-bit-depth formats (S = depth - 8):
// cv::Mat::convertTo(CV_8U, 1.0 / (1 << S)).  S = 0: 8-bit samples as they are.
template <int S>
static __device__ __forceinline__ int to8(int v) {
    if constexpr (S == 0) return v;
    else return min(255, (v + (1 << (S - 1)) - 1 + (v >> S & 1)) >> S);
}

// The demosaic rule of Bayer pattern P (an ADC_IMG_BAYER_* code) at interior site (x, y) from the raw value c there and
// its eight neighbours, computed at the samples' own depth (8 + S bits) and then reduced to 8 bits.  The colour of a
// site comes from the parities of x and y against the pattern's R site.
template <int P, int S>
static __device__ __forceinline__ unsigned bayer_rule(int x, int y, int c, int n, int s, int wv, int e, int nw, int ne,
                                                      int sw, int se) {
    const int cross = (n + s + wv + e + 2) >> 2, diag = (nw + ne + sw + se + 2) >> 2;
    const int hor = (wv + e + 1) >> 1, ver = (n + s + 1) >> 1;
    const int dx = (x ^ img_r_site(P)) & 1, dy = (y ^ img_r_site(P) >> 1) & 1;
    int r, g, b;
    if (dx == dy) {   // an R (dy = 0) or B (dy = 1) site
        g = cross;
        r = dy ? diag : c;
        b = dy ? c : diag;
    } else {          // a G site in an R row (dy = 0: R left and right, B above and below) or in a B row
        g = c;
        r = dy ? ver : hor;
        b = dy ? hor : ver;
    }
    return (unsigned)to8<S>(b) | (unsigned)to8<S>(g) << 8 | (unsigned)to8<S>(r) << 16;
}

// YUV frames (ADC_IMG_NV12 ... ADC_IMG_P016, with or without the colour encoding flags): the conversion of one pixel's
// Y, U, V to B | G << 8 | R << 16 under encoding E (img_encoding: bit 0 BT.709, bit 1 full range; the rules and their
// constants are in include/adcensus_b200.h).  One constant row per encoding and two shift structures: limited range is
// OpenCV's 20-bit rule (E = 0 is cv::cvtColor's COLOR_YUV2BGR_*), full range its 14-bit YCrCb rule.
struct YuvCoef {
    int rv, gu, gv, bu;
};
__host__ __device__ constexpr YuvCoef yuv_coef(int e) {
    return e == 0 ? YuvCoef{1673527, -409993, -852492, 2116026} : e == 1 ? YuvCoef{1879825, -223607, -558796, 2215014}
         : e == 2 ? YuvCoef{22987, -5636, -11698, 29049} : YuvCoef{25802, -3069, -7670, 30402};
}

template <int E>
static __device__ __forceinline__ unsigned yuv_rule(int Y, int U, int V) {
    constexpr YuvCoef k = yuv_coef(E);
    const int u = U - 128, v = V - 128;
    int r, g, b;
    if constexpr (E & 2) {
        r = Y + ((k.rv * v + 8192) >> 14);
        g = Y + ((k.gu * u + k.gv * v + 8192) >> 14);
        b = Y + ((k.bu * u + 8192) >> 14);
    } else {
        const int y = max(Y - 16, 0) * 1220542 + (1 << 19);
        r = (y + k.rv * v) >> 20;
        g = (y + k.gv * v + k.gu * u) >> 20;
        b = (y + k.bu * u) >> 20;
    }
    r = min(max(r, 0), 255);
    g = min(max(g, 0), 255);
    b = min(max(b, 0), 255);
    return (unsigned)b | (unsigned)g << 8 | (unsigned)r << 16;
}

// Pixel (x, y) of the YUV view at src (h rows) in format F.  One luma and two chroma loads; neighbouring pixels share
// their chroma, so L1 serves that reuse.  8-bit samples are single bytes (any alignment); P016's are whole 16-bit words
// (2-byte aligned: the device entries require it, the host entries stage tightly), reduced to 8 bits before the rule.
template <int F>
static __device__ __forceinline__ unsigned yuv_px(const uint8_t* src, long long row_pitch, long long plane_pitch, int h,
                                                  int x, int y) {
    constexpr int C = img_base(F), E = img_encoding(F);
    if constexpr (C == ADC_IMG_P016) {
        const unsigned short* l = reinterpret_cast<const unsigned short*>(src + (long long)y * row_pitch);
        const unsigned short* c =
            reinterpret_cast<const unsigned short*>(src + plane_pitch + (long long)(y >> 1) * row_pitch) + (x & ~1);
        return yuv_rule<E>(to8<8>(__ldg(l + x)), to8<8>(__ldg(c)), to8<8>(__ldg(c + 1)));
    } else if constexpr (img_yuv_planar(F)) {
        const long long cp = row_pitch >> 1;
        const uint8_t* c0 = src + plane_pitch + (long long)(y >> 1) * cp + (x >> 1);
        const uint8_t* c1 = c0 + (long long)((h + 1) >> 1) * cp;
        const int s0 = __ldg(c0), s1 = __ldg(c1);
        return yuv_rule<E>(__ldg(src + (long long)y * row_pitch + x), C == ADC_IMG_I420 ? s0 : s1,
                           C == ADC_IMG_I420 ? s1 : s0);
    } else if constexpr (img_yuv420(F)) {
        const uint8_t* c = src + plane_pitch + (long long)(y >> 1) * row_pitch + (x & ~1);
        const int c0 = __ldg(c), c1 = __ldg(c + 1);
        return yuv_rule<E>(__ldg(src + (long long)y * row_pitch + x), C == ADC_IMG_NV12 ? c0 : c1,
                           C == ADC_IMG_NV12 ? c1 : c0);
    } else {
        // byte offsets of Y0, U and V in the 4-byte macropixel; Y1 is Y0 + 2
        constexpr int oy = C == ADC_IMG_UYVY ? 1 : 0;
        constexpr int ou = C == ADC_IMG_YUYV ? 1 : C == ADC_IMG_UYVY ? 0 : 3;
        constexpr int ov = C == ADC_IMG_YUYV ? 3 : C == ADC_IMG_UYVY ? 2 : 1;
        const uint8_t* m = src + (long long)y * row_pitch + 2ll * (x & ~1);
        return yuv_rule<E>(__ldg(m + oy + 2 * (x & 1)), __ldg(m + ou), __ldg(m + ov));
    }
}

// High-bit-depth frames (ADC_IMG_MONO10 ... ADC_IMG_BAYER_GB12P; rules in include/adcensus_b200.h, container and bits
// in img_format.h): sample x of the row at `row`.  A 16-bit container is read as the whole word (bits above the nominal
// depth are kept and saturate in to8); the words are 2-byte aligned (the device entries require it, the host entries
// stage tightly).  A packed row is a little-endian bit stream from its first byte: the field of sample x starts at bit
// x * b and, b being 10 or 12, always spans exactly two bytes, the second of which is for x = W - 1 the row's last byte.
template <int F>
static __device__ __forceinline__ int rd_sample(const uint8_t* row, int x) {
    if constexpr (img_words(F)) {
        return __ldg(reinterpret_cast<const unsigned short*>(row) + x);
    } else {
        constexpr int b = img_bits(F);
        const int o = x * b;
        const uint8_t* p = row + (o >> 3);
        return ((__ldg(p) | (int)__ldg(p + 1) << 8) >> (o & 7)) & ((1 << b) - 1);
    }
}

// Sample x + dx of a mosaic row: a byte for an 8-bit Bayer mosaic, a full-depth sample for a high-bit-depth one.  The
// neighbour offset dx is a constant, which an 8-bit load takes as its immediate offset.
template <int F>
static __device__ __forceinline__ int mosaic_sample(const uint8_t* row, int x, int dx) {
    if constexpr (img_family(F) == IMG_BAYER) return __ldg(row + x + dx);
    else return rd_sample<F>(row, x + dx);
}

// Mosaics (ADC_IMG_BAYER_* and the high-bit-depth Bayer formats): the demosaiced pixel (x, y) of a w x h mosaic at src
// as B | G << 8 | R << 16, equal to cv::cvtColor(mosaic, COLOR_Bayer*2BGR) (the rule is in include/adcensus_b200.h) on
// the full-depth samples, then reduced to 8 bits.  Frames narrower or lower than 3 pixels are all zero.  The position is
// clamped to [1, w - 2] x [1, h - 2] first, which is the border rule and also keeps all nine loads of the 3x3
// neighbourhood inside the frame, so none of them needs a predicate.
template <int F>
static __device__ __forceinline__ unsigned mosaic_px(const uint8_t* src, long long row_pitch, int w, int h, int x, int y) {
    if (w < 3 || h < 3) return 0u;
    x = min(max(x, 1), w - 2);
    y = min(max(y, 1), h - 2);
    const uint8_t* m = src + (long long)y * row_pitch;
    const uint8_t* u = m - row_pitch;
    const uint8_t* d = m + row_pitch;
    return bayer_rule<img_pattern(F), img_shift(F)>(
        x, y, mosaic_sample<F>(m, x, 0), mosaic_sample<F>(u, x, 0), mosaic_sample<F>(d, x, 0), mosaic_sample<F>(m, x, -1),
        mosaic_sample<F>(m, x, 1), mosaic_sample<F>(u, x, -1), mosaic_sample<F>(u, x, 1), mosaic_sample<F>(d, x, -1),
        mosaic_sample<F>(d, x, 1));
}

// Mosaics: the demosaiced pixels (x0 + (k & 1), y0 + (k >> 1)), k = 0..3, into s[k], where no clamp applies
// (1 <= x0 <= w - 3, 1 <= y0 <= h - 3): their four 3x3 neighbourhoods are one 4x4 window of full-depth samples, loaded
// once; each demosaic is reduced to 8 bits.
template <int F>
static __device__ __forceinline__ void mosaic_quad(const uint8_t* src, long long row_pitch, int x0, int y0,
                                                   unsigned s[4]) {
    int v[4][4];
    const uint8_t* r0 = src + (long long)(y0 - 1) * row_pitch;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) v[i][j] = mosaic_sample<F>(r0 + i * row_pitch, x0 - 1, j);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int dx = k & 1, dy = k >> 1;
        s[k] = bayer_rule<img_pattern(F), img_shift(F)>(
            x0 + dx, y0 + dy, v[1 + dy][1 + dx], v[dy][1 + dx], v[2 + dy][1 + dx], v[1 + dy][dx],
            v[1 + dy][2 + dx], v[dy][dx], v[dy][2 + dx], v[2 + dy][dx], v[2 + dy][2 + dx]);
    }
}

// Pixel (x, y) of a w x h view at src in format F as B | G << 8 | R << 16: the demosaic of a mosaic, the conversion of
// a YUV frame, a high-bit-depth mono sample reduced and repeated, or one of the one-pixel readers above.
template <int F>
static __device__ __forceinline__ unsigned view_px(const uint8_t* src, long long row_pitch, long long plane_pitch, int w,
                                                   int h, int x, int y) {
    if constexpr (img_mosaic(F)) return mosaic_px<F>(src, row_pitch, w, h, x, y);
    else if constexpr (img_family(F) == IMG_YUV) return yuv_px<F>(src, row_pitch, plane_pitch, h, x, y);
    else if constexpr (img_family(F) == IMG_RAWDEPTH)
        return to8<img_shift(F)>(rd_sample<F>(src + (long long)y * row_pitch, x)) * 0x010101u;
    else return ImgIn<F>::px(src + y * row_pitch, x, plane_pitch);
}

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

// ---- the source geometries: which source pixels an output pixel (x, y), p = y*W + x, reads ----

// Plain: pixel (x, y) of the view, read in place (view_px).

// Remap (ADC_REMAP_*): the bilinear blend of the raw view `src` at map entry m (k_rectify.cu's internal form), as
// B | G << 8 | R << 16: the four neighbours of (x0, y0) weighted (32 - ax | ax) * (32 - ay | ay), (sum + 512) >> 10 per
// channel.  When all four lie inside the frame (0 <= x0 < sw - 1, 0 <= y0 < sh - 1; never for a frame one pixel wide
// or high) the loads are unconditional; otherwise each is loaded only if it is inside, so nothing outside a view's
// frame is read.
template <int F>
static __device__ __forceinline__ unsigned rectified_px(uint2 m, const uint8_t* src, int sw, int sh, long long row_pitch,
                                                        long long plane_pitch) {
    const int x0 = (short)(m.x & 0xffffu), y0 = (short)(m.x >> 16);
    const int ax = m.y & 31, ay = m.y >> 5;
    unsigned s[4];   // (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1)
    // neighbour by neighbour: each one inside the frame through view_px (a mosaic site demosaiced from its clamped 3x3
    // neighbourhood, a YUV pixel from its own luma and nearest chroma), one outside the frame BGR 0, not the
    // conversion of zero samples
    const auto each = [&] {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int x = x0 + (k & 1), y = y0 + (k >> 1);
            s[k] = (unsigned)x < (unsigned)sw && (unsigned)y < (unsigned)sh
                       ? view_px<F>(src, row_pitch, plane_pitch, sw, sh, x, y) : 0u;
        }
    };
    if constexpr (img_mosaic(F)) {
        // when no clamp applies (1 <= x0, x0 + 1 <= sw - 2, likewise y0), one 4x4 window serves all four
        // neighbours; each demosaic is reduced to 8 bits before the blend
        if (x0 >= 1 && x0 <= sw - 3 && y0 >= 1 && y0 <= sh - 3) {
            mosaic_quad<F>(src, row_pitch, x0, y0, s);
        } else {
            each();
        }
    } else if constexpr (img_family(F) == IMG_PACKED) {
        if ((unsigned)x0 < (unsigned)(sw - 1) && (unsigned)y0 < (unsigned)(sh - 1)) {
            const uint8_t* r0 = src + y0 * row_pitch;
            s[0] = ImgIn<F>::px(r0, x0, plane_pitch);
            s[1] = ImgIn<F>::px(r0, x0 + 1, plane_pitch);
            s[2] = ImgIn<F>::px(r0 + row_pitch, x0, plane_pitch);
            s[3] = ImgIn<F>::px(r0 + row_pitch, x0 + 1, plane_pitch);
        } else {
            each();
        }
    } else {
        each();
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

// The two resize rules are cv::resize's (include/adcensus_b200.h, DESIGN.md section 22):
//   - ADC_RESIZE_AREA, integer factors kx = sw / W, ky = sh / H (each exact in double as OpenCV computes it, which the
//     engine checks at set time): each output pixel sums its own kx x ky block, so every source pixel is read by
//     exactly one output pixel; (s + 2) >> 2 for 2 x 2, round_half_even((float)s * (1.0f / n)) otherwise (n = kx * ky,
//     the reciprocal rounded to float on the host);
//   - ADC_RESIZE_LINEAR_EXACT, any sizes: per axis f = (d + 0.5) * scale - 0.5 in IEEE double (__dmul_rn / __dadd_rn:
//     no fused multiply-add), scale = 1 / (n_dst / n_src) rounded on the host, i = floor(f), 8-bit weights
//     c1 = round_half_even((f - i) * 256), c0 = 256 - c1, the index clamped into the frame with c1 = 0 at both
//     borders; each thread computes its own taps, so there are no tables.  Four neighbours, all inside the frame, are
//     blended as (h0 * c0y + h1 * c1y + 2^15) >> 16 with h = p[i] * c0x + p[i + 1] * c1x.

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

// The source geometries of k_view_ingest.
enum { VG_PLAIN, VG_REMAP, VG_AREA, VG_LINEAR };

// Grid: blockIdx.y = view.  The resampling geometries take blockIdx.x = tile * S + pair: the S CTAs that read the same
// stretch of a view's map are adjacent in launch order and run at the same time, so a wave reads each map from HBM once
// and from L2 S - 1 times.  Plain reads nothing that pairs share and takes blockIdx.x = tile, blockIdx.z = pair: no
// division in the block-index mapping, and a pair's views one after the other (the tile-outermost order measured gray
// 23 % slower on H100).  Source offsets are 64-bit.
// S pairs of views of sw x sh pixels at left / right (pair i at byte i*image_stride; plain views are the engine's
// W x H, sh = H) -> bgr [S][2][N*3].  map_l / map_r are read by VG_REMAP only, `rule` by VG_AREA and VG_LINEAR only.
template <int F, int G>
__global__ void __launch_bounds__(II_THREADS)
k_view_ingest(int W, int N, int S, int sw, int sh, ResizeRule rule, const uint2* __restrict__ map_l,
              const uint2* __restrict__ map_r, const uint8_t* __restrict__ left, const uint8_t* __restrict__ right,
              long long row_pitch, long long plane_pitch, long long image_stride, uint8_t* __restrict__ bgr) {
    const bool plain = G == VG_PLAIN;
    const int pair = plain ? blockIdx.z : blockIdx.x % S, tile = plain ? blockIdx.x : blockIdx.x / S, view = blockIdx.y;
    const uint8_t* src = (view ? right : left) + (long long)pair * image_stride;
    const uint2* map = view ? map_r : map_l;
    uint8_t* o = bgr + ((size_t)pair * 2 + view) * 3 * (size_t)N;
    store_view_bgr(o, N, W, tile, [&](int p, int y, int x) {
        if constexpr (G == VG_PLAIN) return view_px<F>(src, row_pitch, plane_pitch, W, sh, x, y);
        else if constexpr (G == VG_REMAP) return rectified_px<F>(__ldg(map + p), src, sw, sh, row_pitch, plane_pitch);
        else if constexpr (G == VG_AREA)
            return area_px<F>(src, row_pitch, plane_pitch, sw, sh, rule.kx, rule.ky, rule.inv_n, x, y);
        else return linear_px<F>(src, row_pitch, plane_pitch, sw, sh, rule.sx, rule.sy, x, y);
    });
}

// The arguments of one k_view_ingest launch, in the kernel's order.
struct ViewIngest {
    int W, N, S, sw, sh;
    ResizeRule rule;
    const uint2* map_l;
    const uint2* map_r;
    const uint8_t* left;
    const uint8_t* right;
    long long row_pitch, plane_pitch, image_stride;
    uint8_t* bgr;
};

template <int F>
void launch_view_ingest(int G, dim3 grid, const ViewIngest& a, cudaStream_t st) {
#define VI_LAUNCH(G)                                                                                                   \
    k_view_ingest<F, G><<<grid, II_THREADS, 0, st>>>(a.W, a.N, a.S, a.sw, a.sh, a.rule, a.map_l, a.map_r, a.left,     \
                                                     a.right, a.row_pitch, a.plane_pitch, a.image_stride, a.bgr)
    switch (G) {
        case VG_PLAIN: VI_LAUNCH(VG_PLAIN); break;
        case VG_REMAP: VI_LAUNCH(VG_REMAP); break;
        case VG_AREA: VI_LAUNCH(VG_AREA); break;
        default: VI_LAUNCH(VG_LINEAR); break;
    }
#undef VI_LAUNCH
}

// The kernels of format F, all four geometries, are instantiated in the file of F's family (img_format.h):
// II_VIEWS(F) there, and nowhere else, so each file compiles only its own formats' kernels.
#define II_VIEWS(F) template void launch_view_ingest<F>(int, dim3, const ViewIngest&, cudaStream_t);
#define II_EXTERN(F) extern II_VIEWS(F)
ADC_IMG_CODES(II_EXTERN)
#undef II_EXTERN
