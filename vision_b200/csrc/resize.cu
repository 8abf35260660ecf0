// resize.cu — bilinear / bicubic resize (antialias on/off) with fused dtype casts, sm_90a.
//
// Replaces the interpolate leg of torchvision.transforms.v2.functional.resize_image
// (torchvision/transforms/v2/functional/_geometry.py:340-360): the reference casts
// fp16/bf16/uint8 -> fp32 (full-size pass), calls aten::upsample_bi{linear,cubic}2d[_aa]
// and casts back.  Here one kernel reads the storage dtype, accumulates in fp32
// and writes the storage dtype.  Arithmetic restates ATen's (torch 2.11:
// ATen/native/UpSample.h:259-315,398-424; ATen/native/cuda/UpSample.cuh:262-362):
// same source-index / weight formulas, weights normalised by their float sum,
// "rows then columns" accumulation per output pixel.
//
// Kernels:
//   resize_aa_generic_kernel   any scale / filter: CTA = 32x8 output tile of one
//                              plane, per-tile weight tables in shared memory.
//   resize_aa_stream_kernel    bilinear-AA downscale fast path (see below).
//   resize_noaa_kernel         antialias=False bilinear / bicubic gather.
#include "bicubic.cuh"
#include "bilinear.cuh"
#include "common.cuh"

namespace vb200 {
namespace {

__device__ __forceinline__ float aa_filter(int mode, float x) {
  if (x < 0.f) x = -x;
  if (mode == VB200_RESIZE_BILINEAR) return x < 1.f ? 1.f - x : 0.f;
  const float a = -0.5f;
  if (x < 1.f) return ((a + 2.f) * x - (a + 3.f)) * x * x + 1.f;
  if (x < 2.f) return (((x - 5.f) * x + 8.f) * x - 4.f) * a;
  return 0.f;
}

struct AxisAA { float scale, support, invscale; int ksize; };

inline AxisAA make_axis(int in_size, int out_size, int mode) {
  AxisAA a;
  a.scale = (float)in_size / (float)out_size;            // compute_scales_value<float>
  const float interp = mode == VB200_RESIZE_BILINEAR ? 2.f : 4.f;
  a.support = (a.scale >= 1.f) ? (interp * 0.5f) * a.scale : interp * 0.5f;
  a.invscale = (a.scale >= 1.f) ? 1.f / a.scale : 1.f;
  a.ksize = (int)ceilf(a.support) * 2 + 1;
  return a;
}

// _compute_weights_span + _compute_weights (UpSample.cuh:303-343) for output index i.
__device__ __forceinline__ void aa_weights(int mode, int i, int in_size, AxisAA ax, int* xmin_o, int* xsize_o,
                                           float* w /*[ksize]*/) {
  const float center = ax.scale * ((float)i + 0.5f);
  const int xmin = max((int)(center - ax.support + 0.5f), 0);
  int xsize = min((int)(center + ax.support + 0.5f), in_size) - xmin;
  xsize = min(max(xsize, 0), ax.ksize);
  const float xmc = (float)xmin - center;
  float total = 0.f;
  for (int j = 0; j < xsize; ++j) {
    const float wt = aa_filter(mode, ((float)j + xmc + 0.5f) * ax.invscale);
    w[j] = wt;
    total += wt;
  }
  for (int j = 0; j < xsize; ++j)
    if (total != 0.f) w[j] = __fdiv_rn(w[j], total);
  for (int j = xsize; j < ax.ksize; ++j) w[j] = 0.f;
  *xmin_o = xmin;
  *xsize_o = xsize;
}

template <typename T> __device__ __forceinline__ T store_cast(float v, int mode);
template <> __device__ __forceinline__ float store_cast<float>(float v, int) { return v; }
template <> __device__ __forceinline__ __half store_cast<__half>(float v, int) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 store_cast<__nv_bfloat16>(float v, int) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ uint8_t store_cast<uint8_t>(float v, int) {
  // _geometry.py:352-359: clamp (bicubic) -> round_ (half to even) -> to(uint8)
  v = fminf(fmaxf(v, 0.f), 255.f);
  return (uint8_t)(int)rintf(v);
}

constexpr int kTileX = 32, kTileY = 8;

template <typename T>
__global__ void __launch_bounds__(kTileX * kTileY)
resize_aa_generic_kernel(const T* __restrict__ in, T* __restrict__ out, int in_h, int in_w, int out_h, int out_w,
                         int mode, AxisAA ax, AxisAA ay) {
  extern __shared__ float smem[];
  float* wx = smem;                                   // [kTileX][kx]
  float* wy = wx + kTileX * ax.ksize;                 // [kTileY][ky]
  int* xmin = reinterpret_cast<int*>(wy + kTileY * ay.ksize);   // [kTileX]
  int* xsize = xmin + kTileX;
  int* ymin = xsize + kTileX;
  int* ysize = ymin + kTileY;

  const int tx = threadIdx.x % kTileX, ty = threadIdx.x / kTileX;
  const int ox0 = blockIdx.x * kTileX, oy0 = blockIdx.y * kTileY;
  const int64_t plane = blockIdx.z;
  if (threadIdx.x < kTileX) {
    const int ox = ox0 + threadIdx.x;
    if (ox < out_w) aa_weights(mode, ox, in_w, ax, &xmin[threadIdx.x], &xsize[threadIdx.x], wx + threadIdx.x * ax.ksize);
  } else if (threadIdx.x < kTileX + kTileY) {
    const int t = threadIdx.x - kTileX, oy = oy0 + t;
    if (oy < out_h) aa_weights(mode, oy, in_h, ay, &ymin[t], &ysize[t], wy + t * ay.ksize);
  }
  __syncthreads();
  const int ox = ox0 + tx, oy = oy0 + ty;
  if (ox >= out_w || oy >= out_h) return;
  const T* __restrict__ src = in + plane * (int64_t)in_h * in_w;
  const float* __restrict__ wxp = wx + tx * ax.ksize;
  const float* __restrict__ wyp = wy + ty * ay.ksize;
  const int x0 = xmin[tx], xs = xsize[tx], y0 = ymin[ty], ys = ysize[ty];
  float acc = 0.f;
  for (int j = 0; j < ys; ++j) {
    const T* __restrict__ row = src + (int64_t)(y0 + j) * in_w + x0;
    float h = 0.f;
    if (xs > 0) {
      h = to_acc(row[0]) * wxp[0];
      for (int i = 1; i < xs; ++i) h += to_acc(row[i]) * wxp[i];
    }
    acc = (j == 0) ? h * wyp[0] : acc + h * wyp[j];
  }
  out[plane * (int64_t)out_h * out_w + (int64_t)oy * out_w + ox] = store_cast<T>(acc, mode);
}

// ---- fused inference preprocessing (SURVEY.md §8f4) --------------------------------------------------------------
// ImageClassification.forward (torchvision/transforms/_presets.py:57-64): resize -> center_crop -> convert_image_dtype(float)
// -> normalize, four full passes (five with the fp32 round trip of the uint8 resize) in the reference.  Here the resize
// kernel computes only the crop window of the virtual resized image and its epilogue applies the rest: round to the STORAGE
// dtype exactly where the reference materialises the resized image (uint8: rint + cast; fp16 / bf16: RNE), scale to
// [0, 1] as convert_image_dtype does for integer images, then (x - mean[c]) / std[c] in fp32.  One launch, the input
// is read once (only the rows / columns the window needs), the fp32 output is written once.
struct NormParams { float mean[8], std[8]; float int_scale; };   // int_scale = 1/255 for uint8 input, 1 otherwise

template <typename T> __device__ __forceinline__ float storage_round(float v, int mode) { return to_acc(store_cast<T>(v, mode)); }

template <typename T>
__global__ void __launch_bounds__(kTileX * kTileY)
resize_crop_norm_kernel(const T* __restrict__ in, float* __restrict__ out, int C, int in_h, int in_w, int rs_h, int rs_w,
                        int crop_top, int crop_left, int crop_h, int crop_w, int mode, int antialias, AxisAA ax, AxisAA ay,
                        NormParams np) {
  extern __shared__ float smem[];
  float* wx = smem;                                   // [kTileX][kx]
  float* wy = wx + kTileX * ax.ksize;                 // [kTileY][ky]
  int* xmin = reinterpret_cast<int*>(wy + kTileY * ay.ksize);
  int* xsize = xmin + kTileX;
  int* ymin = xsize + kTileX;
  int* ysize = ymin + kTileY;
  const int tx = threadIdx.x % kTileX, ty = threadIdx.x / kTileX;
  const int cx0 = blockIdx.x * kTileX, cy0 = blockIdx.y * kTileY;       // position inside the crop window
  const int64_t plane = blockIdx.z;
  const int c = (int)(plane % C);
  if (antialias) {
    if (threadIdx.x < kTileX) {
      const int cx = cx0 + threadIdx.x;
      if (cx < crop_w) aa_weights(mode, crop_left + cx, in_w, ax, &xmin[threadIdx.x], &xsize[threadIdx.x], wx + threadIdx.x * ax.ksize);
    } else if (threadIdx.x < kTileX + kTileY) {
      const int t = threadIdx.x - kTileX, cy = cy0 + t;
      if (cy < crop_h) aa_weights(mode, crop_top + cy, in_h, ay, &ymin[t], &ysize[t], wy + t * ay.ksize);
    }
    __syncthreads();
  }
  const int cx = cx0 + tx, cy = cy0 + ty;
  if (cx >= crop_w || cy >= crop_h) return;
  const int ox = crop_left + cx, oy = crop_top + cy;       // coordinates in the virtual resized image
  const T* __restrict__ src = in + plane * (int64_t)in_h * in_w;
  float acc = 0.f;
  if (antialias) {
    const float* __restrict__ wxp = wx + tx * ax.ksize;
    const float* __restrict__ wyp = wy + ty * ay.ksize;
    const int x0 = xmin[tx], xs = xsize[tx], y0 = ymin[ty], ys = ysize[ty];
    for (int j = 0; j < ys; ++j) {
      const T* __restrict__ row = src + (int64_t)(y0 + j) * in_w + x0;
      float h = 0.f;
      if (xs > 0) {
        h = to_acc(row[0]) * wxp[0];
        for (int i = 1; i < xs; ++i) h += to_acc(row[i]) * wxp[i];
      }
      acc = (j == 0) ? h * wyp[0] : acc + h * wyp[j];
    }
  } else {
    // upsample_bilinear2d (align_corners=False), as resize_noaa_kernel
    const float sh = (float)in_h / (float)rs_h, sw = (float)in_w / (float)rs_w;
    acc = bilinear_sample(sh, sw, oy, ox, in_h, in_w, [=](int y, int x) { return to_acc(src[(int64_t)y * in_w + x]); });
  }
  float v = storage_round<T>(acc, mode);                       // the resized image exists in the storage dtype in the reference
  v = __fmul_rn(v, np.int_scale);                              // convert_image_dtype: uint8 -> x / 255 (CUDA tensor / scalar = x * (1/255))
  v = __fdiv_rn(__fsub_rn(v, np.mean[c]), np.std[c]);          // normalize: sub_(mean).div_(std), mean / std as fp32 tensors
  out[plane * (int64_t)crop_h * crop_w + (int64_t)cy * crop_w + cx] = v;
}

template <typename T>
__global__ void __launch_bounds__(256)
resize_noaa_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t total, int in_h, int in_w, int out_h,
                   int out_w, int mode, float sh, float sw) {
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int ox = (int)(idx % out_w);
    const int oy = (int)((idx / out_w) % out_h);
    const int64_t plane = idx / out_w / out_h;
    const T* __restrict__ src = in + plane * (int64_t)in_h * in_w;
    float r;
    if (mode == VB200_RESIZE_BILINEAR) {
      // upsample_bilinear2d: area_pixel_compute_source_index (align_corners=False, clamp at 0)
      r = bilinear_sample(sh, sw, oy, ox, in_h, in_w, [=](int y, int x) { return to_acc(src[(int64_t)y * in_w + x]); });
    } else {
      const float ry = cubic_source(sh, oy), rx = cubic_source(sw, ox);
      int iy, ix;
      const float ty = cubic_frac(ry, &iy), tx = cubic_frac(rx, &ix);
      float cy[4], cx[4];
      cubic_coeffs(ty, cy);
      cubic_coeffs(tx, cx);
      r = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int yy = cubic_clamp(iy - 1 + k, in_h);
        float v[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) v[m] = to_acc(src[(int64_t)yy * in_w + cubic_clamp(ix - 1 + m, in_w)]);
        const float rowv = cubic_interp(v[0], v[1], v[2], v[3], cx);
        r = (k == 0) ? rowv * cy[0] : r + rowv * cy[k];
      }
    }
    out[idx] = store_cast<T>(r, mode);
  }
}

template <typename T>
int launch_resize(const void* in, void* out, int64_t planes, int in_h, int in_w, int out_h, int out_w, int mode,
                  int antialias, cudaStream_t st) {
  if (antialias) {
    const AxisAA ax = make_axis(in_w, out_w, mode), ay = make_axis(in_h, out_h, mode);
    const size_t smem = (size_t)(kTileX * ax.ksize + kTileY * ay.ksize) * 4 + (size_t)(2 * kTileX + 2 * kTileY) * 4;
    if (smem > (size_t)max_smem_optin() - 1024) {
      set_error("resize: antialias filter too wide for this build (ksize %d x %d)", ax.ksize, ay.ksize);
      return VB200_EUNSUPPORTED;
    }
    if (smem > 48 * 1024)
      VB200_CUDA_TRY(ensure_dyn_smem<resize_aa_generic_kernel<T>>(smem));
    int64_t done = 0;
    while (done < planes) {   // gridDim.z limit
      const int64_t chunk = planes - done < 65535 ? planes - done : 65535;
      dim3 grid((unsigned)ceil_div(out_w, kTileX), (unsigned)ceil_div(out_h, kTileY), (unsigned)chunk);
      resize_aa_generic_kernel<T><<<grid, kTileX * kTileY, smem, st>>>(
          (const T*)in + done * (int64_t)in_h * in_w, (T*)out + done * (int64_t)out_h * out_w, in_h, in_w, out_h, out_w,
          mode, ax, ay);
      int rc = check_launch("resize_aa_generic_kernel");
      if (rc) return rc;
      done += chunk;
    }
    return 0;
  }
  const int64_t total = planes * out_h * out_w;
  const int64_t want = ceil_div64(total, 256);
  const int grid = (int)(want < (int64_t)sm_count() * 16 ? want : (int64_t)sm_count() * 16);
  resize_noaa_kernel<T><<<grid, 256, 0, st>>>((const T*)in, (T*)out, total, in_h, in_w, out_h, out_w, mode,
                                             (float)in_h / (float)out_h, (float)in_w / (float)out_w);
  return check_launch("resize_noaa_kernel");
}

}  // namespace

// implemented in resize_stream.cu; returns 1 if it handled the request, 0 if not applicable, <0 / >1 on error
int resize_aa_stream_try(const void* in, void* const* outs, int ndst, int dtype, int64_t planes, int in_h, int in_w, int out_h,
                         int out_w, int mode, cudaStream_t st);

}  // namespace vb200

using namespace vb200;

template <typename T>
static int launch_crop_norm(const void* in, float* out, int64_t planes, int C, int in_h, int in_w, int rs_h, int rs_w, int crop_top,
                            int crop_left, int crop_h, int crop_w, int mode, int antialias, const NormParams& np, cudaStream_t st) {
  const AxisAA ax = make_axis(in_w, rs_w, mode), ay = make_axis(in_h, rs_h, mode);
  const size_t smem = (size_t)(kTileX * ax.ksize + kTileY * ay.ksize) * 4 + (size_t)(2 * kTileX + 2 * kTileY) * 4;
  if (smem > (size_t)max_smem_optin() - 1024) {
    set_error("resize_crop_normalize: antialias filter too wide for this build (ksize %d x %d)", ax.ksize, ay.ksize);
    return VB200_EUNSUPPORTED;
  }
  if (smem > 48 * 1024) VB200_CUDA_TRY(ensure_dyn_smem<resize_crop_norm_kernel<T>>(smem));
  int64_t done = 0;
  while (done < planes) {
    int64_t chunk = planes - done < 65535 ? planes - done : 65535;
    chunk -= chunk % C ? chunk % C : 0;                 // whole images per launch keep plane % C == channel
    if (chunk == 0) chunk = planes - done;
    dim3 grid((unsigned)ceil_div(crop_w, kTileX), (unsigned)ceil_div(crop_h, kTileY), (unsigned)chunk);
    resize_crop_norm_kernel<T><<<grid, kTileX * kTileY, smem, st>>>((const T*)in + done * (int64_t)in_h * in_w,
                                                                   out + done * (int64_t)crop_h * crop_w, C, in_h, in_w, rs_h, rs_w,
                                                                   crop_top, crop_left, crop_h, crop_w, mode, antialias, ax, ay, np);
    int rc = check_launch("resize_crop_norm_kernel");
    if (rc) return rc;
    done += chunk;
  }
  return 0;
}

extern "C" int vb200_resize_crop_normalize(const void* input, float* output, int dtype, int64_t batch, int channels, int in_h, int in_w,
                                           int resize_h, int resize_w, int crop_top, int crop_left, int crop_h, int crop_w, int mode,
                                           int antialias, const float* mean_host, const float* std_host, vb200_stream stream) {
  VB200_REQUIRE(batch >= 0 && channels > 0 && channels <= 8, "resize_crop_normalize: 1..8 channels");
  VB200_REQUIRE(in_h > 0 && in_w > 0 && resize_h > 0 && resize_w > 0 && crop_h > 0 && crop_w > 0, "resize_crop_normalize: bad sizes");
  VB200_REQUIRE(crop_top >= 0 && crop_left >= 0 && crop_top + crop_h <= resize_h && crop_left + crop_w <= resize_w,
                "resize_crop_normalize: the crop window must lie inside the resized image");
  VB200_REQUIRE(mode == VB200_RESIZE_BILINEAR || (mode == VB200_RESIZE_BICUBIC && antialias), "resize_crop_normalize: bilinear, or bicubic with antialias");
  VB200_REQUIRE(mean_host && std_host, "resize_crop_normalize: null mean / std");
  if (batch == 0) return 0;
  VB200_REQUIRE(input && output, "resize_crop_normalize: null pointer");
  NormParams np = {};
  for (int c = 0; c < channels; ++c) { np.mean[c] = mean_host[c]; np.std[c] = std_host[c]; }
  np.int_scale = dtype == VB200_U8 ? 1.0f / 255.0f : 1.0f;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t planes = batch * channels;
#define VB200_CROP_NORM(T) launch_crop_norm<T>(input, output, planes, channels, in_h, in_w, resize_h, resize_w, crop_top, crop_left, crop_h, \
                                              crop_w, mode, antialias, np, st)
  switch (dtype) {
    case VB200_F32: return VB200_CROP_NORM(float);
    case VB200_F16: return VB200_CROP_NORM(__half);
    case VB200_BF16: return VB200_CROP_NORM(__nv_bfloat16);
    case VB200_U8: return VB200_CROP_NORM(uint8_t);
  }
#undef VB200_CROP_NORM
  set_error("resize_crop_normalize: unsupported dtype %d", dtype);
  return VB200_EUNSUPPORTED;
}

extern "C" int vb200_resize(const void* input, void* output, int dtype, int64_t planes, int in_h, int in_w,
                            int out_h, int out_w, int mode, int antialias, vb200_stream stream) {
  VB200_REQUIRE(planes >= 0 && in_h > 0 && in_w > 0 && out_h > 0 && out_w > 0, "resize: bad sizes");
  VB200_REQUIRE(mode == VB200_RESIZE_BILINEAR || mode == VB200_RESIZE_BICUBIC, "resize: mode must be bilinear or bicubic");
  if (planes == 0) return 0;
  VB200_REQUIRE(input && output, "resize: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (antialias) {
    void* outs[1] = {output};
    const int rc = resize_aa_stream_try(input, outs, 1, dtype, planes, in_h, in_w, out_h, out_w, mode, st);
    if (rc != 0) return rc == 1 ? 0 : rc;
  }
  switch (dtype) {
    case VB200_F32: return launch_resize<float>(input, output, planes, in_h, in_w, out_h, out_w, mode, antialias, st);
    case VB200_F16: return launch_resize<__half>(input, output, planes, in_h, in_w, out_h, out_w, mode, antialias, st);
    case VB200_BF16: return launch_resize<__nv_bfloat16>(input, output, planes, in_h, in_w, out_h, out_w, mode, antialias, st);
    case VB200_U8: return launch_resize<uint8_t>(input, output, planes, in_h, in_w, out_h, out_w, mode, antialias, st);
  }
  set_error("resize: unsupported dtype %d", dtype);
  return VB200_EUNSUPPORTED;
}

// resize fused with the all-gather of its output: every finished pixel is stored to outputs[0] (the caller's own slot) and to
// the same slot of outputs[1..n) - peer-mapped buffers of the other ranks - so the exchange rides under the input stream.
extern "C" int vb200_resize_gather(const void* input, void* const* outputs, int n_outputs, int dtype, int64_t planes, int in_h,
                                   int in_w, int out_h, int out_w, int mode, int antialias, vb200_stream stream) {
  VB200_REQUIRE(n_outputs >= 1 && n_outputs <= 8 && outputs, "resize_gather: 1..8 destinations");
  for (int d = 0; d < n_outputs; ++d) VB200_REQUIRE(outputs[d] != nullptr, "resize_gather: null destination");
  VB200_REQUIRE(planes >= 0 && in_h > 0 && in_w > 0 && out_h > 0 && out_w > 0, "resize: bad sizes");
  if (planes == 0) return 0;
  VB200_REQUIRE(input, "resize: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (antialias) {
    const int rc = resize_aa_stream_try(input, outputs, n_outputs, dtype, planes, in_h, in_w, out_h, out_w, mode, st);
    if (rc != 0) return rc == 1 ? 0 : rc;
  }
  // other modes: the plain kernel into the caller's slot, then one copy per peer on the same stream
  const int rc = vb200_resize(input, outputs[0], dtype, planes, in_h, in_w, out_h, out_w, mode, antialias, stream);
  if (rc) return rc;
  const size_t esize = dtype == VB200_F32 ? 4 : dtype == VB200_U8 ? 1 : 2;
  const size_t bytes = (size_t)planes * out_h * out_w * esize;
  for (int d = 1; d < n_outputs; ++d) VB200_CUDA_TRY(cudaMemcpyAsync(outputs[d], outputs[0], bytes, cudaMemcpyDefault, st));
  return 0;
}
