// k_bayer.cu -- the Bayer-mosaic instantiations of the two image ingestion kernels (k_image.cuh): k_image_ingest for
// adc_match_images* and k_rectify_ingest for adc_match_rectified*, one per pattern, both reading through bayer_px.
//
// Plain ingestion: each thread demosaics four consecutive output pixels, nine byte loads each from the clamped 3x3
// neighbourhood; neighbouring lanes take neighbouring pixels, so a warp's loads hit the same three stretches of rows and
// L1 serves the 9x reuse.  Rectified ingestion: each of the four bilinear neighbours inside the frame is demosaiced the
// same way (a 4x4 raw window per output pixel), a neighbour outside the frame is 0.  A frame narrower or lower than 3
// pixels gives all-zero views without a load.  No shared memory: see DESIGN.md section 17 for the measurements.
#include "k_image.cuh"

void adc_launch_bayer_image(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                            uint8_t* bgr, cudaStream_t st) {
    switch (g.format) {
        case ADC_IMG_BAYER_RGGB: launch_image<ADC_IMG_BAYER_RGGB>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_BAYER_GRBG: launch_image<ADC_IMG_BAYER_GRBG>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_BAYER_BGGR: launch_image<ADC_IMG_BAYER_BGGR>(dm, S, left, right, g, bgr, st); break;
        default: launch_image<ADC_IMG_BAYER_GBRG>(dm, S, left, right, g, bgr, st); break;
    }
}

void adc_launch_bayer_rectify(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                              const AdcRectGeom& r, uint8_t* bgr, cudaStream_t st) {
    switch (g.format) {
        case ADC_IMG_BAYER_RGGB: launch_rectify<ADC_IMG_BAYER_RGGB>(dm, S, left, right, g, r, bgr, st); break;
        case ADC_IMG_BAYER_GRBG: launch_rectify<ADC_IMG_BAYER_GRBG>(dm, S, left, right, g, r, bgr, st); break;
        case ADC_IMG_BAYER_BGGR: launch_rectify<ADC_IMG_BAYER_BGGR>(dm, S, left, right, g, r, bgr, st); break;
        default: launch_rectify<ADC_IMG_BAYER_GBRG>(dm, S, left, right, g, r, bgr, st); break;
    }
}
