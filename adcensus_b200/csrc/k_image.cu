// k_image.cu -- image ingestion (adc_match_images*, adc_match_rectified*, adc_ingest_views*): the caller's views, in
// any of the ADC_IMG_* formats and with any row, plane and image pitch, become the wave's packed BGR images
// ([S][2][H][W][3], what the rest of the pipeline reads) in one pass.  Channel order is resolved, alpha is skipped, a
// gray value v becomes (v, v, v); nothing else happens to a pixel, so the gray conversion, the census and every later
// stage see exactly the bytes a caller who packed the same pixels as BGR would have handed in.
//
// Stores: store_view_bgr (k_image.cuh), four pixels as three aligned words per thread, byte-wise heads and tails.
// Source reads: pixel p of the view is (y, x) = divmod(p, W) at base + y*row_pitch + x*bytes_per_pixel (+ c*plane_pitch
// for planar images); neighbouring lanes take neighbouring groups, so a warp's loads cover one contiguous stretch of a
// row (of each plane): coalesced along x.  Every pixel is loaded by exactly one thread, alpha bytes are never loaded, and
// nothing past the last pixel of the last row is touched.  All source offsets are 64-bit.
// The kernel template (k_view_ingest) and the pixel rules of the other source geometries are in k_image.cuh.  This file
// holds the one launcher, whose dispatch covers every format of img_format.h x every geometry, and instantiates the
// six formats above in all four geometries; k_bayer.cu, k_yuv.cu, k_yuv_video.cu, k_yuv_encodings.cu and
// k_rawdepth.cu instantiate the others.
#include <limits.h>

#include <algorithm>

#include "adc_common.cuh"
#include "k_image.cuh"

static int view_tiles(const AdcDims& dm) { return std::max(1, (dm.N / 4 + II_GROUPS - 1) / II_GROUPS); }

int adc_view_ingest_max_pairs(const AdcDims& dm) { return std::min(65535, INT_MAX / view_tiles(dm)); }

void adc_launch_view_ingest(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                            const AdcRectGeom* r, uint8_t* bgr, cudaStream_t st, unsigned long long* launches) {
    ViewIngest a{dm.W, dm.N, S, dm.W, dm.H, {}, nullptr, nullptr,
                 left, right, g.row_pitch, g.plane_pitch, g.image_stride, bgr};
    int geom = VG_PLAIN;
    if (r) {
        a.sw = r->src_w;
        a.sh = r->src_h;
        if (r->type == ADC_RESIZE_AREA) {
            geom = VG_AREA;
            a.rule.kx = r->src_w / dm.W;
            a.rule.ky = r->src_h / dm.H;
            a.rule.inv_n = 1.0f / (float)(a.rule.kx * a.rule.ky);
        } else if (r->type == ADC_RESIZE_LINEAR_EXACT) {
            geom = VG_LINEAR;
            a.rule.sx = 1.0 / ((double)dm.W / r->src_w);   // OpenCV's scale, the inverse of its inv_scale
            a.rule.sy = 1.0 / ((double)dm.H / r->src_h);
        } else {
            geom = VG_REMAP;
            a.map_l = r->map[0];
            a.map_r = r->map[1];
        }
    }
    const int tiles = view_tiles(dm);
    const dim3 grid = geom == VG_PLAIN ? dim3(tiles, 2, S) : dim3((unsigned)(tiles * S), 2);
    switch (g.format) {
#define II_CASE(F) case F: launch_view_ingest<F>(geom, grid, a, st); break;
        ADC_IMG_CODES(II_CASE)
#undef II_CASE
    }
    ++*launches;
}

ADC_IMG_PACKED_FORMATS(II_VIEWS)
