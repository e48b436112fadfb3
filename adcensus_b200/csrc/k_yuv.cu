// k_yuv.cu -- the YUV instantiations of the view ingestion kernel k_view_ingest (k_image.cuh): one per format (NV12,
// NV21, YUYV, UYVY, YVYU) x source geometry, all reading through yuv_px.
//
// Plain ingestion: each thread converts four consecutive output pixels, one luma and two chroma byte loads each;
// neighbouring lanes take neighbouring pixels, so a warp's luma loads cover one contiguous stretch of a row and its
// chroma loads a stretch half as long (NV12 / NV21) or interleaved with the luma (4:2:2), served from L1.  Rectified
// ingestion: each of the four bilinear neighbours inside the frame is converted from its own luma and chroma, a
// neighbour outside the frame is 0.  No shared memory: see DESIGN.md section 18.
#include "k_image.cuh"

ADC_IMG_YUV_FORMATS(II_VIEWS)
