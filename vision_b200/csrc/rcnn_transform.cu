// rcnn_transform.cu — GeneralizedRCNNTransform's inference path (torchvision/models/detection/transform.py), sm_90a.
//
// The reference, per image: normalize (two full passes, with a blocking host-to-device copy of mean and std), an
// F.interpolate(bilinear) resize, then batch_images' new_full(0) of the whole padded batch and one copy_ per image.  After
// the model, postprocess rescales each image's boxes and keypoints with a handful of tiny kernels behind blocking copies of
// 0-dim ratio tensors.  Here:
//   rcnn_batch_kernel<T>   one uniform grid over the padded canvas, 32 x 8 output tiles x (image, channel): each output
//                          element is either +0.0 (padding) or the bilinear sample of the normalized image, so the inputs
//                          are read once (in place, any strides) and the batch is written once.  The per-image
//                          descriptors travel as a __grid_constant__ kernel parameter: no host-to-device copy.
//   rcnn_rescale_kernel    every image's boxes and keypoints, one (item, element) grid.
#include "bilinear.cuh"
#include "common.cuh"

namespace vb200 {
namespace {

constexpr int kRcTX = 32, kRcTY = 8;

// an image descriptor with its two scales, (float)in / out as ATen's area_pixel_compute_scale computes them
struct RcnnImage { vb200_rcnn_image d; float sh, sw; };
struct RcnnImages { RcnnImage img[VB200_RCNN_MAX_IMAGES]; };
struct RcnnNorm { float mean[8], std[8]; };
struct RcnnRescaleItems { vb200_rcnn_rescale_item item[VB200_RCNN_MAX_RESCALE]; };

// normalize: (image - mean) and then / std are separate tensors of the image dtype in the reference, each op in fp32.  Not
// inlined: four inlined IEEE divisions each keep a call to their slow path, and the registers live across those calls spill.
template <typename T>
__device__ __noinline__ float rcnn_normalize(float v, float m, float s) {
  const float diff = to_acc(from_acc<T>(__fsub_rn(v, m)));
  return to_acc(from_acc<T>(__fdiv_rn(diff, s)));
}

template <typename T>
__global__ void __launch_bounds__(kRcTX * kRcTY)
rcnn_batch_kernel(const __grid_constant__ RcnnImages images, const __grid_constant__ RcnnNorm norm, int C, int pad_h, int pad_w,
                  T* __restrict__ out) {
  const int x = blockIdx.x * kRcTX + threadIdx.x % kRcTX, y = blockIdx.y * kRcTY + threadIdx.x / kRcTX;
  if (x >= pad_w || y >= pad_h) return;
  const int i = blockIdx.z / C, c = blockIdx.z % C;
  const vb200_rcnn_image& d = images.img[i].d;
  float v = 0.f;
  if (y < d.out_h && x < d.out_w) {
    const T* __restrict__ src = static_cast<const T*>(d.data) + c * d.stride_c;
    const int64_t sy = d.stride_h, sx = d.stride_w;
    const float m = norm.mean[c], s = norm.std[c];
    const auto load = [=](int yy, int xx) { return rcnn_normalize<T>(to_acc(src[yy * sy + xx * sx]), m, s); };
    // ATen's CUDA kernel copies an image whose size does not change (its NCHW and channels-last kernels alike) where a
    // blend would turn an infinite neighbour into NaN through a zero weight
    if (d.in_h == d.out_h && d.in_w == d.out_w) v = load(y, x);
    else v = bilinear_sample(images.img[i].sh, images.img[i].sw, y, x, d.in_h, d.in_w, load);
  }
  out[((int64_t)blockIdx.z * pad_h + y) * pad_w + x] = from_acc<T>(v);
}

__global__ void __launch_bounds__(256)
rcnn_rescale_kernel(const __grid_constant__ RcnnRescaleItems items) {
  const vb200_rcnn_rescale_item& it = items.item[blockIdx.y];
  const int64_t total = it.rows * it.cols * it.width;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(e % it.width);
    const int64_t rk = e / it.width, k = rk % it.cols, r = rk / it.cols;
    const float v = it.input[r * it.in_stride[0] + k * it.in_stride[1] + j * it.in_stride[2]];
    // boxes (x1, y1, x2, y2): even columns by ratio_w, odd by ratio_h; keypoints (x, y, visibility): the third copied
    const float o = (it.width == 3 && j == 2) ? v : __fmul_rn(v, (j & 1) ? it.ratio_h : it.ratio_w);
    it.output[r * it.out_stride[0] + k * it.out_stride[1] + j * it.out_stride[2]] = o;
  }
}

template <typename T>
int launch_batch(const vb200_rcnn_image* images, int n, int C, int pad_h, int pad_w, const RcnnNorm& norm, void* output,
                 cudaStream_t st) {
  const int64_t plane = (int64_t)pad_h * pad_w;
  for (int done = 0; done < n; done += VB200_RCNN_MAX_IMAGES) {
    const int chunk = n - done < VB200_RCNN_MAX_IMAGES ? n - done : VB200_RCNN_MAX_IMAGES;
    RcnnImages batch;
    for (int i = 0; i < chunk; ++i) {
      const vb200_rcnn_image& d = images[done + i];
      batch.img[i] = {d, (float)d.in_h / (float)d.out_h, (float)d.in_w / (float)d.out_w};
    }
    const dim3 grid((unsigned)ceil_div(pad_w, kRcTX), (unsigned)ceil_div(pad_h, kRcTY), (unsigned)(chunk * C));
    rcnn_batch_kernel<T><<<grid, kRcTX * kRcTY, 0, st>>>(batch, norm, C, pad_h, pad_w, static_cast<T*>(output) + (int64_t)done * C * plane);
    const int rc = check_launch("rcnn_batch_kernel");
    if (rc) return rc;
  }
  return 0;
}

}  // namespace
}  // namespace vb200

using namespace vb200;

extern "C" int vb200_rcnn_batch_images(const vb200_rcnn_image* images, int num_images, int channels, int dtype, int pad_h,
                                       int pad_w, const float* mean_host, const float* std_host, void* output,
                                       vb200_stream stream) {
  VB200_REQUIRE(num_images >= 0 && channels >= 1 && channels <= 8, "rcnn_batch_images: 1..8 channels");
  VB200_REQUIRE(pad_h > 0 && pad_w > 0 && pad_h <= 65535 * kRcTY, "rcnn_batch_images: padded size %d x %d out of range", pad_h, pad_w);
  VB200_REQUIRE(mean_host && std_host, "rcnn_batch_images: null mean / std");
  if (num_images == 0) return 0;
  VB200_REQUIRE(images && output, "rcnn_batch_images: null pointer");
  for (int i = 0; i < num_images; ++i) {
    const vb200_rcnn_image& d = images[i];
    VB200_REQUIRE(d.data, "rcnn_batch_images: image %d: null pointer", i);
    VB200_REQUIRE(d.in_h > 0 && d.in_w > 0 && d.out_h > 0 && d.out_w > 0 && d.out_h <= pad_h && d.out_w <= pad_w,
                  "rcnn_batch_images: image %d: %d x %d resized to %d x %d does not fit %d x %d", i, d.in_h, d.in_w, d.out_h, d.out_w,
                  pad_h, pad_w);
  }
  RcnnNorm norm = {};
  for (int c = 0; c < channels; ++c) { norm.mean[c] = mean_host[c]; norm.std[c] = std_host[c]; }
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case VB200_F32: return launch_batch<float>(images, num_images, channels, pad_h, pad_w, norm, output, st);
    case VB200_F16: return launch_batch<__half>(images, num_images, channels, pad_h, pad_w, norm, output, st);
    case VB200_BF16: return launch_batch<__nv_bfloat16>(images, num_images, channels, pad_h, pad_w, norm, output, st);
  }
  set_error("rcnn_batch_images: unsupported dtype %d", dtype);
  return VB200_EUNSUPPORTED;
}

extern "C" int vb200_rcnn_rescale(const vb200_rcnn_rescale_item* items, int num_items, vb200_stream stream) {
  VB200_REQUIRE(num_items >= 0, "rcnn_rescale: bad item count");
  if (num_items == 0) return 0;
  VB200_REQUIRE(items, "rcnn_rescale: null items");
  for (int k = 0; k < num_items; ++k) {
    const vb200_rcnn_rescale_item& it = items[k];
    VB200_REQUIRE(it.rows >= 0 && it.cols >= 1 && (it.width == 3 || it.width == 4), "rcnn_rescale: item %d: bad shape", k);
    VB200_REQUIRE(it.rows == 0 || (it.input && it.output), "rcnn_rescale: item %d: null pointer", k);
  }
  cudaStream_t st = (cudaStream_t)stream;
  for (int done = 0; done < num_items; done += VB200_RCNN_MAX_RESCALE) {
    const int chunk = num_items - done < VB200_RCNN_MAX_RESCALE ? num_items - done : VB200_RCNN_MAX_RESCALE;
    RcnnRescaleItems batch;
    int64_t most = 0;
    for (int k = 0; k < chunk; ++k) {
      batch.item[k] = items[done + k];
      const int64_t n = items[done + k].rows * items[done + k].cols * items[done + k].width;
      most = n > most ? n : most;
    }
    // at least one block per item: the launch count does not depend on how many detections there are
    const int64_t want = ceil_div64(most, 256);
    const unsigned gx = (unsigned)(want < 1 ? 1 : want < 1024 ? want : 1024);
    rcnn_rescale_kernel<<<dim3(gx, (unsigned)chunk), 256, 0, st>>>(batch);
    const int rc = check_launch("rcnn_rescale_kernel");
    if (rc) return rc;
  }
  return 0;
}
