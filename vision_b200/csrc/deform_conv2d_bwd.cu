// deform_conv2d_bwd.cu — backward of deform_conv2d for sm_90a (SURVEY.md §8f1).
//
// Reference: csrc/ops/cuda/deform_conv2d_kernel.cu:319-1033 — backward_gradient_inputs (GEMM weight^T x grad_out into a
// columns buffer, then deformable_col2im_coord_kernel for grad_offset / grad_mask and deformable_col2im_kernel for
// grad_input) and backward_gradient_parameters (deformable_im2col + GEMM for grad_weight).
//
// Here the two dense contractions stay plain library GEMMs (issued by the torch shim: cuBLAS through at::matmul, as the
// brief allows for plain GEMMs), and everything around them is two kernels instead of three:
//   * dcn_sample_columns_kernel: the sampled, mask-modulated columns [n, C_in*KK, HWo] for the grad_weight GEMM.  One
//     thread per (image, offset group, tap, output pixel): the sampling geometry (4 clamped corner offsets + weights) is
//     derived ONCE and reused for every channel of the group (the reference re-derives it per channel), column writes
//     are coalesced over pixels;
//   * dcn_backward_inputs_kernel: FUSES the reference's col2im and col2im_coord passes - the same thread walks the
//     group's channels once, reads dcol = (W^T grad_out)[c, tap, pixel] and the four corner pixels once, and produces
//     grad_mask (sum dcol * bilinear), grad_offset (sum dcol * mask * d bilinear / d{y, x}) - written once, no atomics,
//     deterministic - and scatters grad_input with atomics (as the reference does).
// Arithmetic follows bilinear_interpolate (:97-134) and get_coordinate_weight (:503-536).
#include "common.cuh"
#include "dcn_params.h"

namespace vb200 {
namespace {

template <typename A>
struct Sample {
  int o[4];          // y*W + x of the four corners (clamped into the image)
  bool ok[4];        // corner inside the image
  A lh, lw;          // fractional parts
  bool inside;       // bilinear_interpolate's outer test: -1 < y < H and -1 < x < W
};

template <typename A>
__device__ __forceinline__ Sample<A> make_sample(A y, A x, int H, int W) {
  Sample<A> s;
  const int hl = (int)floor(y), wl = (int)floor(x);
  const int hh = hl + 1, wh = wl + 1;
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

// columns[n][(c * KK + tap)][pix] = mask * bilinear(input[n][c], y, x)
template <typename T>
__global__ void __launch_bounds__(256)
dcn_sample_columns_kernel(const T* __restrict__ input, const T* __restrict__ offset, const T* __restrict__ mask, T* __restrict__ columns,
                          DcnParams p, int n_imgs) {
  using A = typename Acc<T>::type;
  const int HWo = p.out_h * p.out_w, HWi = p.in_h * p.in_w, KK = p.kh * p.kw;
  const int c_per_off = p.c_in / p.offset_groups;
  const int64_t total = (int64_t)n_imgs * p.offset_groups * KK * HWo;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int pix = (int)(idx % HWo);
    const int tap = (int)((idx / HWo) % KK);
    const int og = (int)((idx / HWo / KK) % p.offset_groups);
    const int b = (int)(idx / HWo / KK / p.offset_groups);
    const int oy = pix / p.out_w, ox = pix - oy * p.out_w;
    const int i = tap / p.kw, j = tap - i * p.kw;
    const int64_t ob = ((int64_t)b * p.offset_groups + og) * 2 * KK;
    const A y = (A)(oy * p.stride_h - p.pad_h + i * p.dil_h) + (A)to_acc(offset[(ob + 2 * tap) * HWo + pix]);
    const A x = (A)(ox * p.stride_w - p.pad_w + j * p.dil_w) + (A)to_acc(offset[(ob + 2 * tap + 1) * HWo + pix]);
    const A m = p.use_mask ? (A)to_acc(mask[(((int64_t)b * p.offset_groups + og) * KK + tap) * HWo + pix]) : (A)1;
    const Sample<A> s = make_sample<A>(y, x, p.in_h, p.in_w);
    const A hh = (A)1 - s.lh, hw = (A)1 - s.lw;
    const A w1 = hh * hw, w2 = hh * s.lw, w3 = s.lh * hw, w4 = s.lh * s.lw;
    for (int cl = 0; cl < c_per_off; ++cl) {
      const int c = og * c_per_off + cl;
      const T* __restrict__ plane = input + ((int64_t)b * p.c_in + c) * HWi;
      A val = 0;
      if (s.inside) {
        const A v1 = s.ok[0] ? (A)to_acc(plane[s.o[0]]) : (A)0, v2 = s.ok[1] ? (A)to_acc(plane[s.o[1]]) : (A)0;
        const A v3 = s.ok[2] ? (A)to_acc(plane[s.o[2]]) : (A)0, v4 = s.ok[3] ? (A)to_acc(plane[s.o[3]]) : (A)0;
        val = w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4;
      }
      columns[((int64_t)b * p.c_in * KK + (int64_t)c * KK + tap) * HWo + pix] = from_acc<T, A>(m * val);
    }
  }
}

// dcol [n][(c * KK + tap)][pix] = (weight^T x grad_out); writes grad_offset / grad_mask, scatters grad_input (pre-zeroed).
template <typename T>
__global__ void __launch_bounds__(256)
dcn_backward_inputs_kernel(const T* __restrict__ dcol, const T* __restrict__ input, const T* __restrict__ offset, const T* __restrict__ mask,
                           T* __restrict__ grad_input, T* __restrict__ grad_offset, T* __restrict__ grad_mask, DcnParams p, int n_imgs) {
  using A = typename Acc<T>::type;
  const int HWo = p.out_h * p.out_w, HWi = p.in_h * p.in_w, KK = p.kh * p.kw;
  const int c_per_off = p.c_in / p.offset_groups;
  const int64_t total = (int64_t)n_imgs * p.offset_groups * KK * HWo;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int pix = (int)(idx % HWo);
    const int tap = (int)((idx / HWo) % KK);
    const int og = (int)((idx / HWo / KK) % p.offset_groups);
    const int b = (int)(idx / HWo / KK / p.offset_groups);
    const int oy = pix / p.out_w, ox = pix - oy * p.out_w;
    const int i = tap / p.kw, j = tap - i * p.kw;
    const int64_t ob = ((int64_t)b * p.offset_groups + og) * 2 * KK;
    const A y = (A)(oy * p.stride_h - p.pad_h + i * p.dil_h) + (A)to_acc(offset[(ob + 2 * tap) * HWo + pix]);
    const A x = (A)(ox * p.stride_w - p.pad_w + j * p.dil_w) + (A)to_acc(offset[(ob + 2 * tap + 1) * HWo + pix]);
    const A m = p.use_mask ? (A)to_acc(mask[(((int64_t)b * p.offset_groups + og) * KK + tap) * HWo + pix]) : (A)1;
    const Sample<A> s = make_sample<A>(y, x, p.in_h, p.in_w);
    const A hh = (A)1 - s.lh, hw = (A)1 - s.lw;
    const A w1 = hh * hw, w2 = hh * s.lw, w3 = s.lh * hw, w4 = s.lh * s.lw;
    A gy = 0, gx = 0, gm = 0;
    for (int cl = 0; cl < c_per_off; ++cl) {
      const int c = og * c_per_off + cl;
      const int64_t plane_off = ((int64_t)b * p.c_in + c) * HWi;
      const T* __restrict__ plane = input + plane_off;
      const A d = (A)to_acc(dcol[((int64_t)b * p.c_in * KK + (int64_t)c * KK + tap) * HWo + pix]);
      const A v1 = s.ok[0] ? (A)to_acc(plane[s.o[0]]) : (A)0, v2 = s.ok[1] ? (A)to_acc(plane[s.o[1]]) : (A)0;
      const A v3 = s.ok[2] ? (A)to_acc(plane[s.o[2]]) : (A)0, v4 = s.ok[3] ? (A)to_acc(plane[s.o[3]]) : (A)0;
      // get_coordinate_weight (:503-536): d val / dy and d val / dx of the bilinear sample
      gy += m * (s.lw * (v4 - v2) + hw * (v3 - v1)) * d;
      gx += m * (s.lh * (v4 - v3) + hh * (v2 - v1)) * d;
      if (s.inside) {
        gm += d * (w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4);
        const A md = m * d;
        T* __restrict__ gi = grad_input + plane_off;
        if (s.ok[0] && w1 != (A)0) atomic_add<T>(gi + s.o[0], md * w1);
        if (s.ok[1] && w2 != (A)0) atomic_add<T>(gi + s.o[1], md * w2);
        if (s.ok[2] && w3 != (A)0) atomic_add<T>(gi + s.o[2], md * w3);
        if (s.ok[3] && w4 != (A)0) atomic_add<T>(gi + s.o[3], md * w4);
      }
    }
    grad_offset[(ob + 2 * tap) * HWo + pix] = from_acc<T, A>(gy);
    grad_offset[(ob + 2 * tap + 1) * HWo + pix] = from_acc<T, A>(gx);
    if (p.use_mask) grad_mask[(((int64_t)b * p.offset_groups + og) * KK + tap) * HWo + pix] = from_acc<T, A>(gm);
  }
}

template <typename T>
int launch_columns(const void* input, const void* offset, const void* mask, void* columns, const DcnParams& p, int n_imgs, cudaStream_t st) {
  const int64_t total = (int64_t)n_imgs * p.offset_groups * p.kh * p.kw * p.out_h * p.out_w;
  if (total == 0) return 0;
  const int grid = (int)(ceil_div64(total, 256) < (int64_t)sm_count() * 32 ? ceil_div64(total, 256) : (int64_t)sm_count() * 32);
  dcn_sample_columns_kernel<T><<<grid, 256, 0, st>>>((const T*)input, (const T*)offset, (const T*)mask, (T*)columns, p, n_imgs);
  return check_launch("dcn_sample_columns_kernel");
}
template <typename T>
int launch_bwd_inputs(const void* dcol, const void* input, const void* offset, const void* mask, void* gi, void* go, void* gm,
                      const DcnParams& p, int n_imgs, cudaStream_t st) {
  const int64_t total = (int64_t)n_imgs * p.offset_groups * p.kh * p.kw * p.out_h * p.out_w;
  if (total == 0) return 0;
  const int grid = (int)(ceil_div64(total, 256) < (int64_t)sm_count() * 32 ? ceil_div64(total, 256) : (int64_t)sm_count() * 32);
  dcn_backward_inputs_kernel<T><<<grid, 256, 0, st>>>((const T*)dcol, (const T*)input, (const T*)offset, (const T*)mask, (T*)gi, (T*)go,
                                                     (T*)gm, p, n_imgs);
  return check_launch("dcn_backward_inputs_kernel");
}

int fill_params(DcnParams& p, int c_in, int in_h, int in_w, int kh, int kw, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h,
                int dil_w, int offset_groups, int use_mask) {
  p = DcnParams{0, c_in, in_h, in_w, 0, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, 1, offset_groups, use_mask, 0, 0};
  p.out_h = (in_h + 2 * pad_h - (dil_h * (kh - 1) + 1)) / stride_h + 1;
  p.out_w = (in_w + 2 * pad_w - (dil_w * (kw - 1) + 1)) / stride_w + 1;
  return (p.out_h > 0 && p.out_w > 0 && offset_groups > 0 && c_in % offset_groups == 0) ? 0 : -1;
}

}  // namespace
}  // namespace vb200

using namespace vb200;

extern "C" int vb200_deform_conv2d_sample_columns(const void* input, const void* offset, const void* mask, void* columns, int dtype,
                                                  int n_imgs, int c_in, int in_h, int in_w, int kh, int kw, int stride_h, int stride_w,
                                                  int pad_h, int pad_w, int dil_h, int dil_w, int offset_groups, int use_mask,
                                                  vb200_stream stream) {
  DcnParams p;
  VB200_REQUIRE(kh > 0 && kw > 0 && stride_h > 0 && stride_w > 0 && dil_h > 0 && dil_w > 0 && pad_h >= 0 && pad_w >= 0,
                "deform_conv2d_sample_columns: bad geometry");
  VB200_REQUIRE(fill_params(p, c_in, in_h, in_w, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, offset_groups, use_mask) == 0,
                "deform_conv2d_sample_columns: bad sizes");
  if (n_imgs == 0 || c_in == 0) return 0;
  VB200_REQUIRE(input && offset && columns && (!use_mask || mask), "deform_conv2d_sample_columns: null pointer");
  VB200_REQUIRE((int64_t)in_h * in_w < (1ll << 31), "deform_conv2d_sample_columns: image too large");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case VB200_F32: return launch_columns<float>(input, offset, mask, columns, p, n_imgs, st);
    case VB200_F64: return launch_columns<double>(input, offset, mask, columns, p, n_imgs, st);
    case VB200_F16: return launch_columns<__half>(input, offset, mask, columns, p, n_imgs, st);
    case VB200_BF16: return launch_columns<__nv_bfloat16>(input, offset, mask, columns, p, n_imgs, st);
  }
  set_error("deform_conv2d_sample_columns: unsupported dtype %d", dtype);
  return VB200_EUNSUPPORTED;
}

extern "C" int vb200_deform_conv2d_backward_inputs(const void* dcol, const void* input, const void* offset, const void* mask,
                                                   void* grad_input, void* grad_offset, void* grad_mask, int dtype, int n_imgs, int c_in,
                                                   int in_h, int in_w, int kh, int kw, int stride_h, int stride_w, int pad_h, int pad_w,
                                                   int dil_h, int dil_w, int offset_groups, int use_mask, vb200_stream stream) {
  DcnParams p;
  VB200_REQUIRE(kh > 0 && kw > 0 && stride_h > 0 && stride_w > 0 && dil_h > 0 && dil_w > 0 && pad_h >= 0 && pad_w >= 0,
                "deform_conv2d_backward_inputs: bad geometry");
  VB200_REQUIRE(fill_params(p, c_in, in_h, in_w, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, offset_groups, use_mask) == 0,
                "deform_conv2d_backward_inputs: bad sizes");
  if (n_imgs == 0 || c_in == 0) return 0;
  VB200_REQUIRE(dcol && input && offset && grad_input && grad_offset && (!use_mask || (mask && grad_mask)), "deform_conv2d_backward_inputs: null pointer");
  VB200_REQUIRE((int64_t)in_h * in_w < (1ll << 31), "deform_conv2d_backward_inputs: image too large");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case VB200_F32: return launch_bwd_inputs<float>(dcol, input, offset, mask, grad_input, grad_offset, grad_mask, p, n_imgs, st);
    case VB200_F64: return launch_bwd_inputs<double>(dcol, input, offset, mask, grad_input, grad_offset, grad_mask, p, n_imgs, st);
    case VB200_F16: return launch_bwd_inputs<__half>(dcol, input, offset, mask, grad_input, grad_offset, grad_mask, p, n_imgs, st);
    case VB200_BF16: return launch_bwd_inputs<__nv_bfloat16>(dcol, input, offset, mask, grad_input, grad_offset, grad_mask, p, n_imgs, st);
  }
  set_error("deform_conv2d_backward_inputs: unsupported dtype %d", dtype);
  return VB200_EUNSUPPORTED;
}
