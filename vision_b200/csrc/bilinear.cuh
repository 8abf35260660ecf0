// bilinear.cuh — ATen's non-antialiased bilinear sample arithmetic (upsample_bilinear2d, align_corners=False;
// ATen/native/UpSample.h area_pixel_compute_source_index, ATen/native/cuda/UpSampleBilinear2d.cu
// upsample_bilinear2d_out_frame), shared by resize_noaa_kernel and resize_crop_norm_kernel (resize.cu) and
// rcnn_batch_kernel (rcnn_transform.cu).  As in bicubic.cuh, parity rests on the expressions as written: nvcc contracts
// the blend into FMAs the same way it contracts ATen's.
#pragma once
#include "common.cuh"

namespace vb200 {

// Output pixel (oy, ox) of an in_h x in_w plane: area_pixel_compute_source_index (clamped at 0) with sh / sw =
// (float)in / out computed by the caller, the second tap of each axis clamped to the last row / column, and
// h0 * (w0 * v00 + w1 * v01) + h1 * (w0 * v10 + w1 * v11) in the reference's form, rows first.  load(y, x) returns the
// input value at (y, x) in fp32.  A zero weight is still multiplied, so an infinite tap with weight 0 gives NaN.
template <typename Load>
__device__ __forceinline__ float bilinear_sample(float sh, float sw, int oy, int ox, int in_h, int in_w, Load load) {
  float ry = sh * ((float)oy + 0.5f) - 0.5f; if (ry < 0.f) ry = 0.f;
  float rx = sw * ((float)ox + 0.5f) - 0.5f; if (rx < 0.f) rx = 0.f;
  const int y0 = min((int)ry, in_h - 1), x0 = min((int)rx, in_w - 1);
  const int y1 = y0 + (y0 < in_h - 1 ? 1 : 0), x1 = x0 + (x0 < in_w - 1 ? 1 : 0);
  const float l1y = fminf(fmaxf(ry - (float)y0, 0.f), 1.f), l1x = fminf(fmaxf(rx - (float)x0, 0.f), 1.f);
  const float l0y = 1.f - l1y, l0x = 1.f - l1x;
  const float v00 = load(y0, x0), v01 = load(y0, x1);
  const float v10 = load(y1, x0), v11 = load(y1, x1);
  return l0y * (l0x * v00 + l1x * v01) + l1y * (l0x * v10 + l1x * v11);
}

}  // namespace vb200
