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
// The kernel template (k_image_ingest) is in k_image.cuh.  This file holds the one dispatch over every format of
// img_format.h and instantiates the six formats above; k_bayer.cu, k_yuv.cu, k_yuv_video.cu, k_yuv_encodings.cu and
// k_rawdepth.cu instantiate the others.
#include <algorithm>

#include "adc_common.cuh"
#include "k_image.cuh"

void adc_launch_image_ingest(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                             uint8_t* bgr, cudaStream_t st, unsigned long long* launches) {
    switch (g.format) {
#define II_CASE(F) case F: launch_image<F>(dm, S, left, right, g, bgr, st); break;
        ADC_IMG_CODES(II_CASE)
#undef II_CASE
    }
    ++*launches;
}

ADC_IMG_PACKED_FORMATS(II_IMAGE)
