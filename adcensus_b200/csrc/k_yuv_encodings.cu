// k_yuv_encodings.cu -- the instantiations of the view ingestion kernel (k_image.cuh, every source geometry) for the
// YUV formats of k_yuv.cu (NV12, NV21, YUYV, UYVY, YVYU) under the three colour encodings that need a flag:
// ADC_IMG_YUV_BT709, ADC_IMG_YUV_FULL_RANGE and both.  The readers are k_yuv.cu's; only the constants and the shift structure of yuv_rule
// differ.  See DESIGN.md section 21.
#include "k_image.cuh"

ADC_IMG_YUV_FLAGGED_FORMATS(II_VIEWS)
