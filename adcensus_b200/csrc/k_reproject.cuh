// k_reproject.cuh -- the reprojection arithmetic shared by k_reproject.cu (adc_reproject*) and k_cloud.cu
// (adc_point_cloud*), so that both compute cv::reprojectImageTo3D with the same instructions:
//   h_i = (((+0.0 + Q[i][0]*x) + Q[i][1]*y) + Q[i][2]*d) + Q[i][3] in double, P_c = (float)((double)(float)h_c * (1.0 / h_3))
// The double arithmetic is written with the _rn intrinsics, so nvcc can neither contract a multiply and an add into a
// DFMA nor fold the +0.0 that turns a -0 first product into +0 (OpenCV's sum starts at +0.0).  Q[i][3] is added as it
// is: OpenCV multiplies it by 1.0, which changes no value.
#pragma once

#include "adc_common.cuh"

// h_i of pixel (x, y) with value d, one rounding per operation
static __device__ __forceinline__ double q_row(const AdcReprojQ& Q, int i, double x, double y, double d) {
    double h = __dadd_rn(0.0, __dmul_rn(Q.q[4 * i], x));
    h = __dadd_rn(h, __dmul_rn(Q.q[4 * i + 1], y));
    h = __dadd_rn(h, __dmul_rn(Q.q[4 * i + 2], d));
    return __dadd_rn(h, Q.q[4 * i + 3]);
}

// OpenCV's double-rounded coordinate: (float)((double)(float)h * ia)
static __device__ __forceinline__ float coord(double h, double ia) {
    return __double2float_rn(__dmul_rn((double)__double2float_rn(h), ia));
}

// Z: cv::reprojectImageTo3D replaces it by bigZ = 10000 wherever |d - minDisparity| <= FLT_EPSILON, and without
// handleMissingValues its minDisparity is FLT_MAX, so a disparity of exactly FLT_MAX gets Z = 10000 whatever Q is
static __device__ __forceinline__ float coord_z(const AdcReprojQ& Q, double x, double y, float d, double ia) {
    return d == 3.40282347e+38f ? 10000.0f : coord(q_row(Q, 2, x, y, (double)d), ia);
}
