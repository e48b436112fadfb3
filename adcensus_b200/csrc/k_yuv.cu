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

ADC_IMG_YUV_FORMATS(II_IMAGE)
ADC_IMG_YUV_FORMATS(II_RECTIFY)
