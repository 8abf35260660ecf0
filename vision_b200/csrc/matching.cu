// matching.cu — training-target assignment of the detection models (torchvision/models/detection/rpn.py:193-229,
// roi_heads.py:580-613, retinanet.py:494-507), sm_90a.
//
// The reference, per image: box_iou(gt, predictions) materialises the M x N IoU matrix (ops/boxes.py:308-370, with [M, N, 2]
// intermediates), Matcher (_utils.py:313-416) reduces it over both axes, set_low_quality_matches_ runs a nonzero (a host
// sync), and a few masked writes build the caller's targets.  Here every image of a call is one grid layer and nothing of
// size M x N exists:
//   pass 1 (allow_low_quality_matches only)  every IoU once; each gt's max over the image's predictions, reduced as an
//            order-preserving integer key: redux.sync within a warp, one shared atomic per warp, one global atomicMax per
//            CTA and gt.  Max is order-independent, so the keys are the same whatever the schedule.
//   final    every IoU again (the same function, so the same bits): each prediction's best gt as Tensor.max(dim=0) picks it,
//            the thresholds, the low-quality rule against the pass-1 maxima, and the caller's epilogue.
// FCOS's centre-sampling matcher (fcos.py:440-487) is a different algorithm on the same layout: one pass, each anchor's
// best gt found while scanning the gt boxes, no N x M tensor (fcos_match_kernel below).
// The per-image descriptors travel as a __grid_constant__ kernel parameter.
#include <vector>

#include "common.cuh"

namespace vb200 {
namespace {

constexpr int kMatchThreads = 256;
constexpr int kPredsPerThread = 4;
constexpr int kMatchTile = kMatchThreads * kPredsPerThread;   // predictions per CTA
constexpr int kGtChunk = 256;                                  // gt boxes staged in shared memory at a time

struct MatchPlan {
  vb200_match_image img[VB200_MATCH_MAX_IMAGES];
  int64_t key_offset[VB200_MATCH_MAX_IMAGES];   // first gt-max key of each image in the workspace
  void* keys;
  int gt_dtype, pred_dtype, mode, allow_low_quality;
  float high_f, low_f;       // the thresholds as torch compares them with an fp32 tensor: rounded to float
  double high_d, low_d;      // ... and with an fp64 one
};

template <typename Acc> struct KeyOf { using type = uint32_t; };
template <> struct KeyOf<double> { using type = unsigned long long; };

// Order-preserving keys: NaN above everything (one key for every NaN), -0 equal to +0, negatives below positives.  Key 0 is
// below every value, so a zeroed key is the identity of the max.  decode(key(v)) == v for every non-NaN v up to the sign of
// zero, and is a NaN for a NaN.
__device__ __forceinline__ uint32_t order_key(float v) {
  if (v != v) return 0xFFFFFFFFu;
  const uint32_t u = v == 0.f ? 0u : __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ unsigned long long order_key(double v) {
  if (v != v) return ~0ull;
  const unsigned long long u = v == 0.0 ? 0ull : (unsigned long long)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | (1ull << 63));
}
__device__ __forceinline__ float decode_key(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }
__device__ __forceinline__ double decode_key(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & ~(1ull << 63)) : ~k));
}

__device__ __forceinline__ uint32_t warp_max(uint32_t k) { return __reduce_max_sync(0xFFFFFFFFu, k); }
__device__ __forceinline__ unsigned long long warp_max(unsigned long long k) {
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, k, s);
    k = o > k ? o : k;
  }
  return k;
}

// clamp(min=0), which keeps a NaN
template <typename A> __device__ __forceinline__ A clamp0(A v) { return v < A(0) ? A(0) : v; }

// A value computed in fp32 (as ATen computes fp16 / bf16 ops) and stored in a tensor of type S: rounded to S.  fp32 and fp64
// values are stored as computed.
template <typename S> __device__ __forceinline__ float round_as(float v) { return v; }
template <> __device__ __forceinline__ float round_as<__half>(float v) { return __half2float(__float2half_rn(v)); }
template <> __device__ __forceinline__ float round_as<__nv_bfloat16>(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
template <typename S> __device__ __forceinline__ double round_as(double v) { return v; }
// ... for a dtype known only at run time (one tensor of the call)
template <typename A> __device__ __forceinline__ A round_as(A v, int dtype) {
  return dtype == VB200_F16 ? round_as<__half>(v) : dtype == VB200_BF16 ? round_as<__nv_bfloat16>(v) : v;
}

// rb - lt: computed in the type of the operands.  When both sides are fp16 (or both bf16) lt and rb are fp16 tensors and the
// difference is rounded to fp16 before _upcast; every other mix promotes to fp32 (or is fp64 throughout).
template <typename S, typename A> __device__ __forceinline__ A round_sub(A a, A b) { return round_as<S>(sub_rn(a, b)); }

template <typename A> struct MBox { A x1, y1, x2, y2, area; };

// box_area: (x2 - x1) * (y2 - y1) of the upcast coordinates
template <typename A> __device__ __forceinline__ A box_area(A x1, A y1, A x2, A y2) { return mul_rn(sub_rn(x2, x1), sub_rn(y2, y1)); }

// box_iou(gt, pred) for one pair, op by op as _box_inter_union and box_iou compute it (ops/boxes.py:308-370): lt / rb by
// torch.max / torch.min, wh = clamp(rb - lt, min=0), inter = wh0 * wh1, union = (area1 + area2) - inter, inter / union.  Every
// pass calls this one function, so every pass sees the same bits.
template <typename A, typename S>
__device__ __forceinline__ A match_iou(const MBox<A>& g, const MBox<A>& p) {
  const A w = clamp0(round_sub<S>(nan_min(g.x2, p.x2), nan_max(g.x1, p.x1)));
  const A h = clamp0(round_sub<S>(nan_min(g.y2, p.y2), nan_max(g.y1, p.y1)));
  const A inter = mul_rn(w, h);
  return div_rn(inter, sub_rn(add_rn(g.area, p.area), inter));
}

template <typename A> __device__ __forceinline__ A load_coord(const void* base, int dtype, int64_t i) {
  switch (dtype) {
    case VB200_F16: return (A)__half2float(static_cast<const __half*>(base)[i]);
    case VB200_BF16: return (A)__bfloat162float(static_cast<const __nv_bfloat16*>(base)[i]);
    case VB200_F64: return (A) static_cast<const double*>(base)[i];
    default: return (A) static_cast<const float*>(base)[i];
  }
}

template <typename A> __device__ __forceinline__ MBox<A> load_box(const void* base, int dtype, int64_t row, const int64_t* stride) {
  MBox<A> b;
  b.x1 = load_coord<A>(base, dtype, row * stride[0]);
  b.y1 = load_coord<A>(base, dtype, row * stride[0] + stride[1]);
  b.x2 = load_coord<A>(base, dtype, row * stride[0] + 2 * stride[1]);
  b.y2 = load_coord<A>(base, dtype, row * stride[0] + 3 * stride[1]);
  b.area = box_area(b.x1, b.y1, b.x2, b.y2);
  return b;
}

template <typename E>
__device__ __forceinline__ void copy_row(const void* src, int64_t row, const int64_t* stride, void* dst, int64_t n) {
  const E* s = static_cast<const E*>(src) + row * stride[0];
  E* o = static_cast<E*>(dst) + n * 4;
#pragma unroll
  for (int j = 0; j < 4; ++j) o[j] = s[j * stride[1]];
}

// The caller's targets for prediction n from its Matcher value m (>= 0, -1 below low, -2 between thresholds).
__device__ __forceinline__ void match_epilogue(const MatchPlan& plan, const vb200_match_image& d, int64_t n, int m) {
  if (plan.mode == VB200_MATCH_RAW) {
    static_cast<int64_t*>(d.out0)[n] = d.num_gt == 0 ? -1 : m;                           // retinanet.py:498-505
  } else if (plan.mode == VB200_MATCH_RPN) {                                               // rpn.py:202-225
    if (d.num_gt == 0) {
      static_cast<float*>(d.out0)[n] = 0.f;
      *reinterpret_cast<float4*>(static_cast<float*>(d.out1) + n * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      return;
    }
    static_cast<float*>(d.out0)[n] = m >= 0 ? 1.f : m == -1 ? 0.f : -1.f;
    const int g = m < 0 ? 0 : m;
    switch (plan.gt_dtype) {
      case VB200_F64: copy_row<unsigned long long>(d.gt, g, d.gt_stride, d.out1, n); break;
      case VB200_F32: copy_row<uint32_t>(d.gt, g, d.gt_stride, d.out1, n); break;
      default: copy_row<uint16_t>(d.gt, g, d.gt_stride, d.out1, n); break;
    }
  } else {                                                                                 // roi_heads.py:586-609
    if (d.num_gt == 0) {
      static_cast<int64_t*>(d.out0)[n] = 0;
      static_cast<int64_t*>(d.out1)[n] = 0;
      return;
    }
    static_cast<int64_t*>(d.out0)[n] = m < 0 ? 0 : m;
    static_cast<int64_t*>(d.out1)[n] = m == -1 ? 0 : m == -2 ? -1 : d.gt_labels[(int64_t)m * d.label_stride];
  }
}

// One CTA: kMatchTile predictions of image blockIdx.y, kPredsPerThread per thread, against all of its gt boxes in chunks.
template <typename A, typename S, bool kFinal>
__global__ void __launch_bounds__(kMatchThreads)
match_kernel(const __grid_constant__ MatchPlan plan) {
  using Key = typename KeyOf<A>::type;
  const vb200_match_image& d = plan.img[blockIdx.y];
  const int M = d.num_gt;
  const int64_t N = d.num_pred, base = (int64_t)blockIdx.x * kMatchTile;
  if (base >= N || (!kFinal && M == 0)) return;     // uniform over the CTA
  __shared__ MBox<A> sg[kGtChunk];
  __shared__ Key skey[kGtChunk];                      // pass 1: this CTA's max per gt; final: the image's
  Key* __restrict__ keys = static_cast<Key*>(plan.keys) + plan.key_offset[blockIdx.y];
  const bool low_quality = kFinal && plan.allow_low_quality;

  MBox<A> p[kPredsPerThread];
  bool valid[kPredsPerThread];
  A best[kPredsPerThread];
  int best_idx[kPredsPerThread];
  bool lowq[kPredsPerThread];
#pragma unroll
  for (int k = 0; k < kPredsPerThread; ++k) {
    const int64_t n = base + threadIdx.x + k * kMatchThreads;
    valid[k] = n < N;
    p[k] = valid[k] ? load_box<A>(d.pred, plan.pred_dtype, n, d.pred_stride) : MBox<A>{};
    best[k] = A(0);
    best_idx[k] = -1;
    lowq[k] = false;
  }

  for (int c0 = 0; c0 < M; c0 += kGtChunk) {
    const int cnt = M - c0 < kGtChunk ? M - c0 : kGtChunk;
    __syncthreads();                                  // the previous chunk is consumed
    for (int j = threadIdx.x; j < cnt; j += kMatchThreads) {
      sg[j] = load_box<A>(d.gt, plan.gt_dtype, c0 + j, d.gt_stride);
      skey[j] = kFinal ? (low_quality ? keys[c0 + j] : Key(0)) : Key(0);
    }
    __syncthreads();
    for (int j = 0; j < cnt; ++j) {
      const MBox<A> g = sg[j];
      if (kFinal) {
        const A gmax = decode_key(skey[j]);
#pragma unroll
        for (int k = 0; k < kPredsPerThread; ++k) {
          const A v = match_iou<A, S>(g, p[k]);
          // Tensor.max(dim=0): ascending gt order, strict >, the first NaN wins and stays
          if (best_idx[k] < 0 || (best[k] == best[k] && (v != v || v > best[k]))) { best[k] = v; best_idx[k] = c0 + j; }
          if (low_quality) lowq[k] |= v == gmax;      // set_low_quality_matches_: an exact tie with the gt's max
        }
      } else {
        Key kmax = 0;
#pragma unroll
        for (int k = 0; k < kPredsPerThread; ++k)
          if (valid[k]) {
            const Key key = order_key(match_iou<A, S>(g, p[k]));
            kmax = key > kmax ? key : kmax;
          }
        kmax = warp_max(kmax);
        if ((threadIdx.x & 31) == 0) atomicMax(&skey[j], kmax);
      }
    }
    if (!kFinal) {
      __syncthreads();
      for (int j = threadIdx.x; j < cnt; j += kMatchThreads) atomicMax(&keys[c0 + j], skey[j]);
    }
  }

  if (kFinal) {
    const A low = sizeof(A) == 8 ? (A)plan.low_d : (A)plan.low_f, high = sizeof(A) == 8 ? (A)plan.high_d : (A)plan.high_f;
#pragma unroll
    for (int k = 0; k < kPredsPerThread; ++k) {
      if (!valid[k]) continue;
      // below_low_threshold, then between_thresholds (a NaN is neither), then the low-quality matches keep their argmax
      int m = best_idx[k];
      if (best[k] < low) m = -1;
      else if (best[k] < high) m = -2;
      if (lowq[k]) m = best_idx[k];
      match_epilogue(plan, d, base + threadIdx.x + k * kMatchThreads, m);
    }
  }
}

template <typename A, typename S>
int launch_matching(MatchPlan& plan, const vb200_match_image* images, int num_images, const int64_t* key_offset, cudaStream_t st) {
  for (int done = 0; done < num_images; done += VB200_MATCH_MAX_IMAGES) {
    const int chunk = num_images - done < VB200_MATCH_MAX_IMAGES ? num_images - done : VB200_MATCH_MAX_IMAGES;
    int64_t most = 0, gts = 0;
    for (int i = 0; i < chunk; ++i) {
      plan.img[i] = images[done + i];
      plan.key_offset[i] = key_offset[done + i];
      most = images[done + i].num_pred > most ? images[done + i].num_pred : most;
      gts += images[done + i].num_gt;
    }
    if (most == 0) continue;
    const dim3 grid((unsigned)ceil_div64(most, kMatchTile), (unsigned)chunk);
    if (plan.allow_low_quality && gts > 0) {
      match_kernel<A, S, false><<<grid, kMatchThreads, 0, st>>>(plan);
      const int rc = check_launch("match_kernel (gt max)");
      if (rc) return rc;
    }
    match_kernel<A, S, true><<<grid, kMatchThreads, 0, st>>>(plan);
    const int rc = check_launch("match_kernel");
    if (rc) return rc;
  }
  return 0;
}

size_t match_key_bytes(int64_t total_gt, int dtype) { return align256((size_t)total_gt * (dtype == VB200_F64 ? 8 : 4)); }

// ---- FCOS centre sampling (fcos.py:455-483) ------------------------------------------------------------------------------
// A thread holds kFcosAnchorsPerThread anchors' anchor-side values in registers and scans the image's gt boxes, staged in
// shared memory kGtChunk at a time with their gt-side values, in ascending index order: the running best is
// Tensor.max(dim=1)'s, so no N x M value is ever stored.
constexpr int kFcosThreads = 256;
constexpr int kFcosAnchorsPerThread = 2;
constexpr int kFcosTile = kFcosThreads * kFcosAnchorsPerThread;   // anchors per CTA

struct FcosPlan {
  vb200_fcos_image img[VB200_MATCH_MAX_IMAGES];
  int64_t lower_end[VB200_MATCH_MAX_IMAGES], upper_begin[VB200_MATCH_MAX_IMAGES];   // vb200_fcos_level_bounds of each image
  int gt_dtype, anchor_dtype;
  float radius_f;            // center_sampling_radius as ATen's CUDA scalar ops take it for a non-fp64 tensor
  double radius_d;
};

// The gt side, rounded to the gt dtype: gt_centers = (gt[:, :2] + gt[:, 2:]) / 2, the boxes, and 1e8 - gt_areas.
template <typename A> struct FcosGt { A cx, cy, x1, y1, x2, y2, term; };
// The anchor side, rounded to the anchor dtype: anchor_centers, center_sampling_radius * anchor_sizes and the level bounds.
template <typename A> struct FcosAnchor { A cx, cy, reach, lower, upper; };

// (a + b) / 2 of two coordinates of a tensor of `dtype`: the sum rounded to it, then the division, which ATen's CUDA kernel
// computes as a product with the scalar's reciprocal
template <typename A> __device__ __forceinline__ A fcos_center(A a, A b, int dtype) {
  return round_as(mul_rn(round_as(add_rn(a, b), dtype), A(0.5)), dtype);
}

// Run under S, the type anchor - gt differences are rounded to: the dtype when both sides share it, else fp32 (or fp64).
template <typename A, typename S>
__global__ void __launch_bounds__(kFcosThreads)
fcos_match_kernel(const __grid_constant__ FcosPlan plan) {
  const vb200_fcos_image& d = plan.img[blockIdx.y];
  const int M = d.num_gt;
  const int64_t N = d.num_anchors, base = (int64_t)blockIdx.x * kFcosTile;
  if (base >= N) return;                              // uniform over the CTA
  __shared__ FcosGt<A> sg[kGtChunk];
  const int ad = plan.anchor_dtype, gd = plan.gt_dtype;
  const A radius = sizeof(A) == 8 ? (A)plan.radius_d : (A)plan.radius_f;

  FcosAnchor<A> a[kFcosAnchorsPerThread];
  A best[kFcosAnchorsPerThread];
  int best_idx[kFcosAnchorsPerThread];
#pragma unroll
  for (int k = 0; k < kFcosAnchorsPerThread; ++k) {
    const int64_t n = base + threadIdx.x + k * kFcosThreads;
    const MBox<A> b = n < N ? load_box<A>(d.anchors, ad, n, d.anchor_stride) : MBox<A>{};    // (.area is box_iou's, unused)
    const A size = round_as(sub_rn(b.x2, b.x1), ad);                                           // anchor_sizes
    a[k].cx = fcos_center(b.x1, b.x2, ad);
    a[k].cy = fcos_center(b.y1, b.y2, ad);
    a[k].reach = round_as(mul_rn(radius, size), ad);
    a[k].lower = n < plan.lower_end[blockIdx.y] ? A(0) : round_as(mul_rn(size, A(4)), ad);
    a[k].upper = n >= plan.upper_begin[blockIdx.y] ? A(INFINITY) : round_as(mul_rn(size, A(8)), ad);
    best[k] = A(0);
    best_idx[k] = -1;
  }

  for (int c0 = 0; c0 < M; c0 += kGtChunk) {
    const int cnt = M - c0 < kGtChunk ? M - c0 : kGtChunk;
    __syncthreads();                                  // the previous chunk is consumed
    for (int j = threadIdx.x; j < cnt; j += kFcosThreads) {
      const MBox<A> b = load_box<A>(d.gt, gd, c0 + j, d.gt_stride);
      const A area = round_as(mul_rn(round_as(sub_rn(b.x2, b.x1), gd), round_as(sub_rn(b.y2, b.y1), gd)), gd);
      // 1e8 - gt_areas: the scalar as a float (exact), the difference rounded to the gt dtype (inf for fp16)
      sg[j] = FcosGt<A>{fcos_center(b.x1, b.x2, gd), fcos_center(b.y1, b.y2, gd), b.x1, b.y1, b.x2, b.y2,
                        round_as(sub_rn(A(1e8), area), gd)};
    }
    __syncthreads();
    for (int j = 0; j < cnt; ++j) {
      const FcosGt<A> g = sg[j];
#pragma unroll
      for (int k = 0; k < kFcosAnchorsPerThread; ++k) {
        // |anchor_centers - gt_centers|.max(dim=2) < radius * size; pairwise_dist's min > 0, its max in (lower, upper).
        // max / min over the stacked dimension propagate a NaN, and every comparison with a NaN is false.
        const A cdist = nan_max(fabs(round_sub<S>(a[k].cx, g.cx)), fabs(round_sub<S>(a[k].cy, g.cy)));
        const A l = round_sub<S>(a[k].cx, g.x1), t = round_sub<S>(a[k].cy, g.y1);
        const A r = round_sub<S>(g.x2, a[k].cx), btm = round_sub<S>(g.y2, a[k].cy);
        const A dmin = nan_min(nan_min(l, t), nan_min(r, btm)), dmax = nan_max(nan_max(l, t), nan_max(r, btm));
        const bool match = cdist < a[k].reach && dmin > A(0) && dmax > a[k].lower && dmax < a[k].upper;
        // match.to(float32) * (1e8 - area), multiplied literally: 0 * inf is NaN, 0 * a negative term is -0
        const A v = mul_rn(match ? A(1) : A(0), g.term);
        // Tensor.max(dim=1): ascending gt order, strict >, the first NaN wins and stays
        if (best_idx[k] < 0 || (best[k] == best[k] && (v != v || v > best[k]))) { best[k] = v; best_idx[k] = c0 + j; }
      }
    }
  }

  // matched_idx[min_values < 1e-5] = -1, the scalar rounded to the value's type; a NaN keeps its index.  An image without gt
  // keeps best 0 and index -1.
  const A min_value = sizeof(A) == 8 ? (A)1e-5 : (A)1e-5f;
#pragma unroll
  for (int k = 0; k < kFcosAnchorsPerThread; ++k) {
    const int64_t n = base + threadIdx.x + k * kFcosThreads;
    if (n < N) d.out[n] = best[k] < min_value ? -1 : best_idx[k];
  }
}

template <typename A, typename S>
int launch_fcos(FcosPlan& plan, const vb200_fcos_image* images, int num_images, int64_t first_level, int64_t last_level,
                cudaStream_t st) {
  for (int done = 0; done < num_images; done += VB200_MATCH_MAX_IMAGES) {
    const int chunk = num_images - done < VB200_MATCH_MAX_IMAGES ? num_images - done : VB200_MATCH_MAX_IMAGES;
    int64_t most = 0;
    for (int i = 0; i < chunk; ++i) {
      plan.img[i] = images[done + i];
      vb200_fcos_level_bounds(images[done + i].num_anchors, first_level, last_level, &plan.lower_end[i], &plan.upper_begin[i]);
      most = images[done + i].num_anchors > most ? images[done + i].num_anchors : most;
    }
    if (most == 0) continue;
    fcos_match_kernel<A, S><<<dim3((unsigned)ceil_div64(most, kFcosTile), (unsigned)chunk), kFcosThreads, 0, st>>>(plan);
    const int rc = check_launch("fcos_match_kernel");
    if (rc) return rc;
  }
  return 0;
}

}  // namespace
}  // namespace vb200

using namespace vb200;

extern "C" size_t vb200_match_boxes_workspace_bytes(int64_t total_gt, int dtype, int allow_low_quality) {
  if (!allow_low_quality || total_gt <= 0) return 0;
  return match_key_bytes(total_gt, dtype);
}

extern "C" int vb200_match_boxes(const vb200_match_image* images, int num_images, int gt_dtype, int pred_dtype, int mode,
                                 double high_threshold, double low_threshold, int allow_low_quality, void* workspace,
                                 size_t workspace_bytes, vb200_stream stream) {
  VB200_REQUIRE(num_images >= 0, "match_boxes: bad image count");
  VB200_REQUIRE(mode == VB200_MATCH_RAW || mode == VB200_MATCH_RPN || mode == VB200_MATCH_ROI_HEADS, "match_boxes: unknown mode %d", mode);
  const bool wide = gt_dtype == VB200_F64 && pred_dtype == VB200_F64;
  const auto narrow_float = [](int t) { return t == VB200_F32 || t == VB200_F16 || t == VB200_BF16; };
  VB200_REQUIRE(wide || (narrow_float(gt_dtype) && narrow_float(pred_dtype)),
                "match_boxes: gt and predictions must both be float64, or both float32 / float16 / bfloat16 (dtypes %d, %d)", gt_dtype,
                pred_dtype);
  if (num_images == 0) return 0;
  VB200_REQUIRE(images, "match_boxes: null images");
  int64_t total_gt = 0;
  std::vector<int64_t> key_offset((size_t)num_images);
  for (int i = 0; i < num_images; ++i) {
    const vb200_match_image& d = images[i];
    VB200_REQUIRE(d.num_gt >= 0 && d.num_pred >= 0 && d.num_pred < ((int64_t)1 << 31), "match_boxes: image %d: bad sizes", i);
    VB200_REQUIRE(d.num_gt == 0 || d.num_pred > 0, "match_boxes: image %d: no proposal boxes for %d gt boxes", i, d.num_gt);
    VB200_REQUIRE(d.num_pred == 0 || (d.pred && d.out0 && (mode == VB200_MATCH_RAW || d.out1)), "match_boxes: image %d: null pointer", i);
    VB200_REQUIRE(d.num_gt == 0 || d.num_pred == 0 || (d.gt && (mode != VB200_MATCH_ROI_HEADS || d.gt_labels)),
                  "match_boxes: image %d: null gt pointer", i);
    key_offset[i] = total_gt;
    total_gt += d.num_gt;
  }
  const size_t need = vb200_match_boxes_workspace_bytes(total_gt, wide ? VB200_F64 : VB200_F32, allow_low_quality);
  if (need && (!workspace || workspace_bytes < need)) {
    set_error("match_boxes: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    return VB200_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (need) VB200_CUDA_TRY(cudaMemsetAsync(workspace, 0, need, st));
  MatchPlan plan;
  plan.keys = workspace;
  plan.gt_dtype = gt_dtype;
  plan.pred_dtype = pred_dtype;
  plan.mode = mode;
  plan.allow_low_quality = allow_low_quality ? 1 : 0;
  plan.high_f = (float)high_threshold;
  plan.low_f = (float)low_threshold;
  plan.high_d = high_threshold;
  plan.low_d = low_threshold;
  if (wide) return launch_matching<double, double>(plan, images, num_images, key_offset.data(), st);
  if (gt_dtype == VB200_F16 && pred_dtype == VB200_F16) return launch_matching<float, __half>(plan, images, num_images, key_offset.data(), st);
  if (gt_dtype == VB200_BF16 && pred_dtype == VB200_BF16)
    return launch_matching<float, __nv_bfloat16>(plan, images, num_images, key_offset.data(), st);
  return launch_matching<float, float>(plan, images, num_images, key_offset.data(), st);
}

extern "C" void vb200_fcos_level_bounds(int64_t num_anchors, int64_t first_level, int64_t last_level, int64_t* lower_end_host,
                                        int64_t* upper_begin_host) {
  // Python's slice bounds: a negative index counts from the end, then both clamp to [0, num_anchors]
  const auto index = [num_anchors](int64_t i) {
    if (i < 0) i += num_anchors;
    return i < 0 ? 0 : i > num_anchors ? num_anchors : i;
  };
  *lower_end_host = index(first_level);     // lower_bound[:first_level]
  *upper_begin_host = index(-last_level);   // upper_bound[-last_level:]; [-0:] starts at 0
}

extern "C" int vb200_fcos_match(const vb200_fcos_image* images, int num_images, int gt_dtype, int anchor_dtype, double radius,
                                int64_t first_level, int64_t last_level, vb200_stream stream) {
  VB200_REQUIRE(num_images >= 0, "fcos_match: bad image count");
  const bool wide = gt_dtype == VB200_F64 && anchor_dtype == VB200_F64;
  const auto narrow_float = [](int t) { return t == VB200_F32 || t == VB200_F16 || t == VB200_BF16; };
  VB200_REQUIRE(wide || (narrow_float(gt_dtype) && narrow_float(anchor_dtype)),
                "fcos_match: gt and anchors must both be float64, or both float32 / float16 / bfloat16 (dtypes %d, %d)", gt_dtype,
                anchor_dtype);
  VB200_REQUIRE(first_level > INT64_MIN && last_level > INT64_MIN, "fcos_match: bad level sizes");
  if (num_images == 0) return 0;
  VB200_REQUIRE(images, "fcos_match: null images");
  for (int i = 0; i < num_images; ++i) {
    const vb200_fcos_image& d = images[i];
    VB200_REQUIRE(d.num_gt >= 0 && d.num_anchors >= 0 && d.num_anchors < ((int64_t)1 << 31), "fcos_match: image %d: bad sizes", i);
    VB200_REQUIRE(d.num_anchors == 0 || (d.anchors && d.out && (d.num_gt == 0 || d.gt)), "fcos_match: image %d: null pointer", i);
  }
  FcosPlan plan;
  plan.gt_dtype = gt_dtype;
  plan.anchor_dtype = anchor_dtype;
  plan.radius_f = (float)radius;
  plan.radius_d = radius;
  cudaStream_t st = (cudaStream_t)stream;
  if (wide) return launch_fcos<double, double>(plan, images, num_images, first_level, last_level, st);
  if (gt_dtype == VB200_F16 && anchor_dtype == VB200_F16) return launch_fcos<float, __half>(plan, images, num_images, first_level, last_level, st);
  if (gt_dtype == VB200_BF16 && anchor_dtype == VB200_BF16)
    return launch_fcos<float, __nv_bfloat16>(plan, images, num_images, first_level, last_level, st);
  return launch_fcos<float, float>(plan, images, num_images, first_level, last_level, st);
}
