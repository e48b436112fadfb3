// k_image.cu -- image ingestion (adc_match_images*): the caller's views, in any of the ADC_IMG_* formats and with any
// row, plane and image pitch, become the wave's packed BGR images ([S][2][H][W][3], what the rest of the pipeline reads)
// in one pass.  Channel order is resolved, alpha is skipped, a gray value v becomes (v, v, v); nothing else happens to a
// pixel, so the gray conversion, the census and every later stage see exactly the bytes a caller who packed the same
// pixels as BGR would have handed in.
//
// Stores: store_view_bgr (k_image.cuh), four pixels as three aligned words per thread, byte-wise heads and tails.
// Source reads: pixel p of the view is (y, x) = divmod(p, W) at base + y*row_pitch + x*bytes_per_pixel (+ c*plane_pitch
// for planar images); neighbouring lanes take neighbouring groups, so a warp's loads cover one contiguous stretch of a
// row (of each plane): coalesced along x.  Every pixel is loaded by exactly one thread, alpha bytes are never loaded, and
// nothing past the last pixel of the last row is touched.  All source offsets are 64-bit.
// The kernel template (k_image_ingest) is in k_image.cuh; this file instantiates it for the six formats above, and
// k_bayer.cu for the Bayer mosaics, k_yuv.cu for the YUV formats, k_rawdepth.cu for the high-bit-depth formats.
#include <algorithm>

#include "adc_common.cuh"
#include "k_image.cuh"

void adc_launch_image_ingest(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                             uint8_t* bgr, cudaStream_t st, unsigned long long* launches) {
    switch (g.format) {
        case ADC_IMG_BGR: launch_image<ADC_IMG_BGR>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_RGB: launch_image<ADC_IMG_RGB>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_BGRA: launch_image<ADC_IMG_BGRA>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_RGBA: launch_image<ADC_IMG_RGBA>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_GRAY: launch_image<ADC_IMG_GRAY>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_BAYER_RGGB: case ADC_IMG_BAYER_GRBG: case ADC_IMG_BAYER_BGGR: case ADC_IMG_BAYER_GBRG:
            adc_launch_bayer_image(dm, S, left, right, g, bgr, st);
            break;
        case ADC_IMG_NV12: case ADC_IMG_NV21: case ADC_IMG_YUYV: case ADC_IMG_UYVY: case ADC_IMG_YVYU:
            adc_launch_yuv_image(dm, S, left, right, g, bgr, st);
            break;
        case ADC_IMG_RGB_PLANAR: launch_image<ADC_IMG_RGB_PLANAR>(dm, S, left, right, g, bgr, st); break;
        default: adc_launch_rawdepth_image(dm, S, left, right, g, bgr, st); break;
    }
    ++*launches;
}

AdcImageGeom adc_image_tight(int format, long long w, long long h) {
    long long rp = w;   // gray, Bayer, and each plane of a planar image
    switch (format) {
        case ADC_IMG_BGR: case ADC_IMG_RGB: rp = 3 * w; break;
        case ADC_IMG_BGRA: case ADC_IMG_RGBA: rp = 4 * w; break;
        case ADC_IMG_NV12: case ADC_IMG_NV21: rp = 2 * ((w + 1) / 2); break;
        case ADC_IMG_YUYV: case ADC_IMG_UYVY: case ADC_IMG_YVYU: rp = 4 * ((w + 1) / 2); break;
        default: break;
    }
    // high bit depth: one 16-bit word per sample, or the whole bytes of a row's 10- / 12-bit stream
    if (is_rawdepth(format)) rp = rd_container(format) <= 2 ? 2 * w : (rd_bits(format) * w + 7) / 8;
    const long long plane = h * rp;
    if (format == ADC_IMG_RGB_PLANAR) return AdcImageGeom{format, rp, plane, 3 * plane};
    if (format == ADC_IMG_NV12 || format == ADC_IMG_NV21) return AdcImageGeom{format, rp, plane, plane + (h + 1) / 2 * rp};
    return AdcImageGeom{format, rp, 0, plane};
}

long long adc_image_read_bytes(int format, long long w, long long h) {
    if (format == ADC_IMG_NV12 || format == ADC_IMG_NV21) return w * h + 2 * ((w + 1) / 2) * ((h + 1) / 2);
    return adc_image_tight(format, w, h).image_stride;   // 4:2:2: 4 * ceil(W/2) * H
}
