// dcn_geometry.cuh — the reference's deformable sampling arithmetic, shared by the deform_conv2d forward (deform_conv2d.cu,
// deform_conv2d_tc.cu) and backward (deform_conv2d_bwd.cu) kernels.  Parity with the reference rests on these rules, so they
// live here only:
//   * the sample position of tap (i, j) of output pixel (oy, ox): (oy * stride - pad + i * dilation) + offset, and the mask
//     value (deformable_im2col, deform_conv2d_kernel.cu:136-209);
//   * bilinear_interpolate's outer test, cell (floor y, floor x), clamped corners with their validity flags, corner weights
//     and four-corner blend (deform_conv2d_kernel.cu:97-134);
//   * the shared-memory sampling table of the SIMT and tensor-core forward kernels;
//   * host: DcnParams, the geometry checks of deform_conv2d_kernel.cu:1056-1150 and the dtype dispatch.
#pragma once
#include "common.cuh"

namespace vb200 {

struct DcnParams {
  int batch, c_in, in_h, in_w, c_out, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w;
  int groups, offset_groups, use_mask, out_h, out_w;
  // fused all-gather (vb200_deform_conv2d_forward): the epilogue also stores every output element to the same slot of
  // the peers' gathered buffers (peer-mapped device pointers; NVLink stores)
  void* peer_out[7];
  int n_peer;
};
// optional: pre-packed weights / channels-last input (no staging pass) / peer destinations of the fused all-gather.
// peers_done (may be NULL) is set when the launched kernel wrote the peer destinations itself.
struct DcnHints { const void* packed_weight; int input_is_nhwc; void* const* peer_out; int n_peer; bool* peers_done; };

// Sample position (y, x) and mask value m (1 without a mask) of tap `tap` of output pixel `pix`.  off / msk point at the
// (image, offset group)'s first offset / mask channel; msk is read only with a mask.
template <typename A, typename T>
__device__ __forceinline__ void sample_position(const T* __restrict__ off, const T* __restrict__ msk, const DcnParams& p, int tap,
                                                int pix, A& y, A& x, A& m) {
  const int HWo = p.out_h * p.out_w;
  const int oy = pix / p.out_w, ox = pix - oy * p.out_w;
  const int i = tap / p.kw, j = tap - i * p.kw;
  y = add_rn((A)(oy * p.stride_h - p.pad_h + i * p.dil_h), (A)to_acc(off[(int64_t)(2 * tap) * HWo + pix]));
  x = add_rn((A)(ox * p.stride_w - p.pad_w + j * p.dil_w), (A)to_acc(off[(int64_t)(2 * tap + 1) * HWo + pix]));
  m = p.use_mask ? (A)to_acc(msk[(int64_t)tap * HWo + pix]) : (A)1;
}

// bilinear_interpolate's geometry of the sample (y, x) in an H x W image.  The flags and clamps are two-sided because the
// backward's get_coordinate_weight reads the corners of samples outside the image too.  When `inside` holds, hl >= -1 and
// hl + 1 <= H (likewise for x), so they reduce to the reference's one-sided form (hl >= 0, hl + 1 <= H - 1, max(hl, 0),
// min(hl + 1, H - 1)).
template <typename A>
struct Sample {
  int o[4];          // y*W + x of the four corners (clamped into the image)
  bool ok[4];        // corner inside the image
  A lh, lw;          // fractional parts
  bool inside;       // bilinear_interpolate's outer test: -1 < y < H and -1 < x < W
  int hl, wl;        // the sample's cell: floor(y), floor(x)
};

// A position past +-2^31 saturates the conversion to INT_MAX / INT_MIN, and hl + 1 then overflows.  By default the next row /
// column is a wrapping add (INT_MAX + 1 = INT_MIN, outside the image like the sample).  As a signed add the overflow is
// undefined and the compiler folds the corner tests through it (hh >= 0 into hl > -2), which passed a corner of such a
// sample as live: the backward's grad_offset, which has no outer test, then summed it with a fraction y - hl of up to 1e12.
// INSIDE_ONLY keeps the signed add for callers that read the corners of `inside` samples alone (hl in [-1, H - 1], no
// overflow; an outside sample's flags are never read): the forward, whose tensor-core kernel measured 2% slower with the
// wrapping add (the folded tests are shorter in its table fill).
template <typename A, bool INSIDE_ONLY = false>
__device__ __forceinline__ Sample<A> make_sample(A y, A x, int H, int W) {
  Sample<A> s;
  const int hl = (int)floor(y), wl = (int)floor(x);
  const int hh = INSIDE_ONLY ? hl + 1 : (int)((unsigned)hl + 1u), wh = INSIDE_ONLY ? wl + 1 : (int)((unsigned)wl + 1u);
  s.hl = hl; s.wl = wl;
  s.lh = y - (A)hl; s.lw = x - (A)wl;
  s.inside = !(y <= (A)-1 || (A)H <= y || x <= (A)-1 || (A)W <= x);
  const bool t0 = hl >= 0 && hl < H, t1 = hh >= 0 && hh < H, l0 = wl >= 0 && wl < W, l1 = wh >= 0 && wh < W;
  const int hlc = min(max(hl, 0), H - 1), hhc = min(max(hh, 0), H - 1), wlc = min(max(wl, 0), W - 1), whc = min(max(wh, 0), W - 1);
  s.o[0] = hlc * W + wlc; s.ok[0] = t0 && l0;
  s.o[1] = hlc * W + whc; s.ok[1] = t0 && l1;
  s.o[2] = hhc * W + wlc; s.ok[2] = t1 && l0;
  s.o[3] = hhc * W + whc; s.ok[3] = t1 && l1;
  return s;
}

// Corner weights hh * hw, hh * lw, lh * hw, lh * lw with hh = 1 - lh, hw = 1 - lw.
template <typename A>
__device__ __forceinline__ void corner_weights(const Sample<A>& s, A w[4]) {
  const A hh = (A)1 - s.lh, hw = (A)1 - s.lw;
  w[0] = hh * hw; w[1] = hh * s.lw; w[2] = s.lh * hw; w[3] = s.lh * s.lw;
}

// The four corner values of one plane, a dead corner read as 0.
template <typename T, typename A>
__device__ __forceinline__ void corner_values(const T* __restrict__ plane, const Sample<A>& s, A v[4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = s.ok[k] ? (A)to_acc(plane[s.o[k]]) : (A)0;
}

// w1 v1 + w2 v2 + w3 v3 + w4 v4 in the reference's order; the caller applies the `inside` test.
template <typename A>
__device__ __forceinline__ A blend(const A w[4], const A v[4]) {
  return w[0] * v[0] + w[1] * v[1] + w[2] * v[2] + w[3] * v[3];
}

// Entry (tap, output pixel) of the forward kernels' shared-memory sampling table: the four clamped corner offsets times the
// caller's scale (1: element index into a plane; c_in * element size: byte offset into a channels-last image) and the weights
// m * corner weight, 0 for a dead corner.  The entry is all zero past the last pixel and for a sample outside the image.
// Tables start 16-byte aligned and are filled with two 16-byte stores per entry.  The type itself carries no alignment: with
// it, the SIMT kernel loads its entries as vectors and needs 103 registers instead of 80.
struct DcnTabEnt { int o[4]; float w[4]; };

// Fills tab[tl * WIDTH + px] for the taps t0 + tl (tl < nt) and the pixels pix0 + px (px < WIDTH) of one offset group (off /
// msk as for sample_position); thread tid of nthreads.
template <int WIDTH, typename T>
__device__ __forceinline__ void fill_sample_table(DcnTabEnt* tab, const T* __restrict__ off, const T* __restrict__ msk,
                                                  const DcnParams& p, int t0, int nt, int pix0, int scale, int tid, int nthreads) {
  const int HWo = p.out_h * p.out_w;
  for (int e = tid; e < nt * WIDTH; e += nthreads) {
    const int tl = e / WIDTH, px = e - tl * WIDTH;
    const int pix = pix0 + px;
    DcnTabEnt se;
#pragma unroll
    for (int q = 0; q < 4; ++q) { se.o[q] = 0; se.w[q] = 0.f; }
    if (pix < HWo) {
      float y, x, m;
      sample_position<float>(off, msk, p, t0 + tl, pix, y, x, m);
      const Sample<float> s = make_sample<float, true>(y, x, p.in_h, p.in_w);
      if (s.inside) {
        float w[4];
        corner_weights(s, w);
#pragma unroll
        for (int q = 0; q < 4; ++q) { se.o[q] = s.o[q] * scale; se.w[q] = s.ok[q] ? m * w[q] : 0.f; }
      }
    }
    reinterpret_cast<int4*>(tab + e)[0] = make_int4(se.o[0], se.o[1], se.o[2], se.o[3]);
    reinterpret_cast<float4*>(tab + e)[1] = make_float4(se.w[0], se.w[1], se.w[2], se.w[3]);
  }
}

// ---- host ------------------------------------------------------------------------------------------------------------
// Fills p for one call and checks its geometry with the reference's messages (deform_conv2d_kernel.cu:1056-1150): kernel,
// stride and dilation > 0, padding >= 0, groups and offset groups > 0 dividing the channels, output at least 1 x 1.  Returns
// 0, or VB200_EINVAL with the error set.  The backward has no weight groups: it passes groups 1 and c_out 0.
inline int dcn_params(DcnParams& p, int batch, int c_in, int in_h, int in_w, int c_out, int kh, int kw, int stride_h, int stride_w,
                      int pad_h, int pad_w, int dil_h, int dil_w, int groups, int offset_groups, int use_mask) {
  VB200_REQUIRE(kh > 0 && kw > 0, "weight_h: %d weight_w: %d", kh, kw);
  VB200_REQUIRE(stride_h > 0 && stride_w > 0, "stride_h: %d stride_w: %d", stride_h, stride_w);
  VB200_REQUIRE(pad_h >= 0 && pad_w >= 0, "pad_h: %d pad_w: %d", pad_h, pad_w);
  VB200_REQUIRE(dil_h > 0 && dil_w > 0, "dilation_h: %d dilation_w: %d", dil_h, dil_w);
  VB200_REQUIRE(groups > 0 && offset_groups > 0 && c_in % groups == 0 && c_out % groups == 0 && c_in % offset_groups == 0,
                "deform_conv2d: channels not divisible by groups");
  p = DcnParams{batch, c_in, in_h, in_w, c_out, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w,
                groups, offset_groups, use_mask, 0, 0};
  p.out_h = (in_h + 2 * pad_h - (dil_h * (kh - 1) + 1)) / stride_h + 1;
  p.out_w = (in_w + 2 * pad_w - (dil_w * (kw - 1) + 1)) / stride_w + 1;
  VB200_REQUIRE(p.out_h > 0 && p.out_w > 0, "Calculated output size too small - out_h: %d out_w: %d", p.out_h, p.out_w);
  return 0;
}

// Calls launch(T()) for the element type of dtype: float, double, half and bfloat16.  Any other dtype sets `unsupported` (a
// format taking the dtype) as the error and returns VB200_EUNSUPPORTED.
template <typename F>
int dispatch_dcn_dtype(int dtype, const char* unsupported, F&& launch) {
  switch (dtype) {
    case VB200_F32: return launch(float());
    case VB200_F64: return launch(double());
    case VB200_F16: return launch(__half());
    case VB200_BF16: return launch(__nv_bfloat16());
  }
  set_error(unsupported, dtype);
  return VB200_EUNSUPPORTED;
}

}  // namespace vb200
