// k_yuv.cu -- the YUV instantiations of the two image ingestion kernels (k_image.cuh): k_image_ingest for
// adc_match_images* and k_rectify_ingest for adc_match_rectified*, one per format (NV12, NV21, YUYV, UYVY, YVYU), both
// reading through yuv_px.
//
// Plain ingestion: each thread converts four consecutive output pixels, one luma and two chroma byte loads each;
// neighbouring lanes take neighbouring pixels, so a warp's luma loads cover one contiguous stretch of a row and its
// chroma loads a stretch half as long (NV12 / NV21) or interleaved with the luma (4:2:2), served from L1.  Rectified
// ingestion: each of the four bilinear neighbours inside the frame is converted from its own luma and chroma, a
// neighbour outside the frame is 0.  No shared memory: see DESIGN.md section 18.
#include "k_image.cuh"

void adc_launch_yuv_image(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                          uint8_t* bgr, cudaStream_t st) {
    switch (g.format) {
        case ADC_IMG_NV12: launch_image<ADC_IMG_NV12>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_NV21: launch_image<ADC_IMG_NV21>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_YUYV: launch_image<ADC_IMG_YUYV>(dm, S, left, right, g, bgr, st); break;
        case ADC_IMG_UYVY: launch_image<ADC_IMG_UYVY>(dm, S, left, right, g, bgr, st); break;
        default: launch_image<ADC_IMG_YVYU>(dm, S, left, right, g, bgr, st); break;
    }
}

void adc_launch_yuv_rectify(const AdcDims& dm, int S, const uint8_t* left, const uint8_t* right, const AdcImageGeom& g,
                            const AdcRectGeom& r, uint8_t* bgr, cudaStream_t st) {
    switch (g.format) {
        case ADC_IMG_NV12: launch_rectify<ADC_IMG_NV12>(dm, S, left, right, g, r, bgr, st); break;
        case ADC_IMG_NV21: launch_rectify<ADC_IMG_NV21>(dm, S, left, right, g, r, bgr, st); break;
        case ADC_IMG_YUYV: launch_rectify<ADC_IMG_YUYV>(dm, S, left, right, g, r, bgr, st); break;
        case ADC_IMG_UYVY: launch_rectify<ADC_IMG_UYVY>(dm, S, left, right, g, r, bgr, st); break;
        default: launch_rectify<ADC_IMG_YVYU>(dm, S, left, right, g, r, bgr, st); break;
    }
}
