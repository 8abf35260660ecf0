// bicubic.cuh — ATen's non-antialiased bicubic sample arithmetic (upsample_bicubic2d, align_corners=False, A = -0.75;
// ATen/native/UpSample.h cubic_convolution1/2, get_cubic_upsample_coefficients, cubic_interp1d;
// ATen/native/cuda/UpSampleBicubic2d.cu upsample_bicubic2d_out_frame), shared by resize_noaa_kernel (resize.cu) and the
// keypoint kernels (keypoints.cu).  Parity rests on these expressions as written: nvcc contracts them into FMAs the
// same way it contracts ATen's, so they are kept in the reference's form and order rather than spelled out with
// round-to-nearest intrinsics.
#pragma once
#include "common.cuh"

namespace vb200 {

__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }

// One axis of a sample, in three steps: area_pixel_compute_source_index (cubic: no clamp at 0) with `scale` =
// (float)in_size / out_size computed on the host; floorf and the fraction; the four coefficients of taps in - 1 .. in + 2.
__device__ __forceinline__ float cubic_source(float scale, int dst) { return scale * ((float)dst + 0.5f) - 0.5f; }

__device__ __forceinline__ float cubic_frac(float real, int* in) {
  const int i = (int)floorf(real);
  *in = i;
  return real - (float)i;
}

__device__ __forceinline__ void cubic_coeffs(float t, float c[4]) {
  const float A = -0.75f;
  c[0] = cubic2(t + 1.f, A);
  c[1] = cubic1(t, A);
  c[2] = cubic1(1.f - t, A);
  c[3] = cubic2(1.f - t + 1.f, A);
}

// cubic_interp1d: the four taps combined in the reference's order.  Rows first (x coefficients), then the four row
// values with the y coefficients.
__device__ __forceinline__ float cubic_interp(float x0, float x1, float x2, float x3, const float c[4]) {
  return x0 * c[0] + x1 * c[1] + x2 * c[2] + x3 * c[3];
}

// upsample_get_value_bounded's index clamp
__device__ __forceinline__ int cubic_clamp(int i, int size) { return max(min(i, size - 1), 0); }

}  // namespace vb200
