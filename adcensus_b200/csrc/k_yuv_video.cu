// k_yuv_video.cu -- the instantiations of the view ingestion kernel (k_image.cuh, every source geometry) for the YUV
// containers of video decoders that k_yuv.cu does not hold: I420 and YV12 (a luma plane and two chroma planes of half
// its row pitch) and P016 (NV12's geometry in 16-bit words), each in all four colour encodings (no flag,
// ADC_IMG_YUV_BT709, ADC_IMG_YUV_FULL_RANGE, both), all reading through yuv_px.
//
// Plain ingestion: each thread converts four consecutive output pixels, one luma and two chroma loads each (bytes for
// I420 / YV12, whole words for P016, reduced to 8 bits before the rule); neighbouring lanes take neighbouring pixels,
// so a warp's luma loads cover one contiguous stretch of a row and its chroma loads stretches half (P016) or a quarter
// (each I420 plane) as long, served from L1.  Rectified ingestion: each of the four bilinear neighbours inside the frame
// is converted from its own samples, a neighbour outside the frame is 0.  See DESIGN.md section 21.
#include "k_image.cuh"

ADC_IMG_YUV_VIDEO_FORMATS(II_VIEWS) ADC_IMG_YUV_VIDEO_FLAGGED_FORMATS(II_VIEWS)
