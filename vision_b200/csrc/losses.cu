// losses.cu — RetinaNet's head losses (torchvision/models/detection/retinanet.py:158-189 and 272-302), forward and backward,
// sm_90a.
//
// The reference, per image: a full-size zeros_like target with the ones scattered in, boolean indexing of the logits and the
// target (a nonzero, a host sync), sigmoid_focal_loss (ops/focal_loss.py:41-56) as a chain of full-size elementwise kernels,
// max(1, num_foreground) on a CUDA tensor (another sync); the regression head adds a torch.where sync and encode_single on the
// gathered foreground rows.  Autograd keeps the full-size intermediates for a backward of the same shape.  Here every image of a
// call is one grid layer of (tile of kLossTile anchors, image):
//   forward   each CTA stages its anchors' codes (target class, background, ignored or bad) in shared memory, streams its
//             anchors' logits once with 16-byte loads and writes one partial sum and foreground count to a per-(image, tile)
//             slot; the box loss does the same per foreground anchor with the reference's encode_single restated op by op.
//   finalize  one CTA adds each image's partials in a fixed order, divides as the reference does and adds the images in
//             _sum's order.
//   backward  the dense gradient written exactly once: the analytic derivative times each image's scale, 0 where the
//             reference's indexing leaves it 0.
// No floating-point atomics and no launch parameter depends on the SM count, so every result is bit-reproducible run to run.
#include "common.cuh"

namespace vb200 {
namespace {

constexpr int kLossThreads = 256;
constexpr int kLossTile = 256;                      // anchors per CTA, both losses: one anchor per thread when staging
static_assert(kLossThreads == kLossTile, "the code staging and the box loss give each thread one anchor");
constexpr int kFinalizeThreads = 256;

// anchor codes; a code >= 0 is the anchor's target class
constexpr int kBad = -3;          // matched >= num_gt, or a label outside [-C, C): the reference raises, the loss is NaN
constexpr int kIgnored = -2;      // matched == Matcher.BETWEEN_THRESHOLDS: no loss, zero gradient
constexpr int kBackground = -1;   // every class's target is 0

struct LossPlan {
  vb200_retinanet_loss_image img[VB200_LOSS_MAX_IMAGES];
  int64_t num_anchors;
  int num_classes, tiles, first_image, num_images;     // img[0] is image first_image of the call's num_images
  double* partial;                                      // forward: [num_images, tiles]
  int* tile_fg;                                         // forward: [num_images, tiles]
  const float* grad_loss;                               // backward: the 0-dim incoming gradient
  const int64_t* num_fg;                                // backward: the forward's per-image foreground counts
  float weights[4];                                     // box loss: the coder's weights as fp32
};

__device__ __forceinline__ int anchor_code(const vb200_retinanet_loss_image& d, int64_t a, int C, bool& fg) {
  const int64_t m = d.matched[a * d.matched_stride];
  fg = m >= 0;                                          // num_foreground counts matched >= 0, bad indices included
  if (m == -2) return kIgnored;
  if (m < 0) return kBackground;
  if (m >= d.num_gt) return kBad;
  const int64_t l = d.labels[m * d.label_stride];
  if (l < -C || l >= C) return kBad;
  return (int)(l < 0 ? l + C : l);                      // advanced indexing wraps negative labels
}

// Stable forms of one element's sigmoid focal loss (alpha 0.25, gamma 2) and its derivative.  With p = σ(x), q = σ(-x):
// -log p = softplus(-x), -log(1 - p) = softplus(x), both max(±x, 0) + log1p(exp(-|x|)).  The two transcendentals are fp32
// (as the reference's own sigmoid); everything after them is fp64 with one rounding to fp32 at the end, so the gradient's
// error is that of the two fp32 functions plus one rounding (a pure fp32 chain of the same formulas adds several more).
struct Sig { double p, q, sp_pos, sp_neg; };
__device__ __forceinline__ Sig sig(float x) {
  const float ef = expf(-fabsf(x)), lf = log1pf(ef);
  const double e = ef, l = lf, d = 1.0 + e;
  double r = (double)__frcp_rn((float)d);
  r = fma(r, fma(-d, r, 1.0), r);                       // one Newton step: 1 / (1 + e) to about 2^-47
  const double big = r, small = e * r;                  // σ(|x|), σ(-|x|)
  const double xd = x;
  return Sig{x >= 0.f ? big : small, x >= 0.f ? small : big, fmax(xd, 0.0) + l, fmax(-xd, 0.0) + l};
}

// A non-finite logit gives what the reference's own arithmetic gives: +inf for t = 0 at x = +inf, NaN otherwise.
__device__ __forceinline__ double focal_loss(float x, bool pos) {
  if (!isfinite(x)) return !pos && x > 0.f ? (double)INFINITY : (double)NAN;
  const Sig s = sig(x);
  return pos ? 0.25 * (s.q * s.q) * s.sp_neg : 0.75 * (s.p * s.p) * s.sp_pos;
}

// t = 1: α(1-p)²(2p·log p - (1-p));  t = 0: (1-α)p²(p - 2(1-p)·log(1-p)); times the image's scale, rounded once.  NaN for a
// non-finite logit, as the reference's.
__device__ __forceinline__ float focal_grad(float x, bool pos, float scale) {
  if (!isfinite(x)) return NAN;
  const Sig s = sig(x);
  const double g = pos ? -0.25 * (s.q * s.q) * (s.q + 2.0 * s.p * s.sp_neg) : 0.75 * (s.p * s.p) * (s.p + 2.0 * s.q * s.sp_pos);
  return (float)((double)scale * g);
}

// The CTA's sum of v in a fixed order: a shuffle tree per warp, then the warps in index order.  Thread 0 holds the result.
__device__ __forceinline__ double block_sum(double v, double* scratch) {
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, s);
  __syncthreads();                                      // scratch is free
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += scratch[w];
  return t;
}

// ATen's division by a Python number on CUDA: a product with the number's fp32 reciprocal.
__device__ __forceinline__ float reciprocal(float d) { return __fdiv_rn(1.f, d); }

// The per-image scale of the backward, in the order autograd applies the two divisions: grad / len(targets) (a Python int),
// then / max(1, num_foreground) -- a CUDA int64 tensor in the classification head (a true division), a Python int in the
// regression head.
template <bool kBox> __device__ __forceinline__ float image_scale(const LossPlan& plan, int image) {
  const float g = __fmul_rn(*plan.grad_loss, reciprocal((float)plan.num_images));
  const int64_t n = plan.num_fg[image];
  const float d = (float)(n > 1 ? n : 1);
  return kBox ? __fmul_rn(g, reciprocal(d)) : __fdiv_rn(g, d);
}

// One CTA: kLossTile anchors of image blockIdx.y, all C classes.  The tile's elements [e0, e1) of the image's [A, C] block are
// taken in 16-byte groups aligned on the streamed array (the logits forward, the gradient backward); the first and last groups
// may be partial, since C need not be a multiple of 4.
template <bool kBackward>
__global__ void __launch_bounds__(kLossThreads)
focal_loss_kernel(const __grid_constant__ LossPlan plan) {
  const vb200_retinanet_loss_image& d = plan.img[blockIdx.y];
  const int image = plan.first_image + (int)blockIdx.y;
  const int C = plan.num_classes;
  const int64_t a0 = (int64_t)blockIdx.x * kLossTile;
  const int na = (int)(plan.num_anchors - a0 < kLossTile ? plan.num_anchors - a0 : kLossTile);
  __shared__ int s_code[kLossTile];
  __shared__ double scratch[kLossThreads / 32];

  bool fg = false;
  s_code[threadIdx.x] = threadIdx.x < na ? anchor_code(d, a0 + threadIdx.x, C, fg) : kIgnored;
  const int tile_fg = __syncthreads_count(fg);          // also the barrier after the staging

  const int64_t e0 = a0 * C, e1 = (a0 + na) * C;
  const float* __restrict__ x = d.pred;
  float* __restrict__ out = d.grad;
  const float* streamed = kBackward ? out : x;
  const int pad = (int)((reinterpret_cast<uintptr_t>(streamed + e0) >> 2) & 3);
  const bool vec_load = !kBackward || ((reinterpret_cast<uintptr_t>(x) ^ reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  const int64_t g0 = e0 - pad;                          // first element of the first group
  const int groups = (int)((e1 - g0 + 3) >> 2);
  const float scale = kBackward ? image_scale<false>(plan, image) : 0.f;
  double acc = 0.0;

  for (int gi = threadIdx.x; gi < groups; gi += kLossThreads) {
    const int64_t eb = g0 + 4 * (int64_t)gi;
    const bool full = eb >= e0 && eb + 4 <= e1;
    float v[4];
    if (full && vec_load) {
      const float4 f = __ldcs(reinterpret_cast<const float4*>(x + eb));
      v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = eb + k >= e0 && eb + k < e1 ? x[eb + k] : 0.f;
    }
    // (local anchor, class) of the group's first element inside the tile, then stepped element by element
    const int k0 = eb < e0 ? (int)(e0 - eb) : 0;
    const int off = (int)(eb + k0 - e0);
    int al = off / C, c = off - al * C;
    float gout[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      gout[k] = 0.f;
      if (k < k0 || eb + k >= e1) continue;
      const int code = s_code[al];
      if (kBackward) {
        gout[k] = code == kIgnored ? 0.f : code == kBad ? NAN : focal_grad(v[k], c == code, scale);
      } else if (code != kIgnored) {
        acc += code == kBad ? (double)NAN : focal_loss(v[k], c == code);
      }
      if (++c == C) { c = 0; ++al; }
    }
    if (kBackward) {
      if (full) {
        __stcs(reinterpret_cast<float4*>(out + eb), make_float4(gout[0], gout[1], gout[2], gout[3]));
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (eb + k >= e0 && eb + k < e1) out[eb + k] = gout[k];
      }
    }
  }
  if (!kBackward) {
    const double sum = block_sum(acc, scratch);
    if (threadIdx.x == 0) {
      plan.partial[(int64_t)image * plan.tiles + blockIdx.x] = sum;
      plan.tile_fg[(int64_t)image * plan.tiles + blockIdx.x] = tile_fg;
    }
  }
}

// encode_boxes (models/detection/_utils.py:103-118) for one anchor and its matched gt box, one rounding per tensor op and
// nothing contracted, so each target has the reference's bits.
__device__ __forceinline__ void encode_box(const float* w, const float a[4], const float g[4], float t[4]) {
  const float ew = __fsub_rn(a[2], a[0]), eh = __fsub_rn(a[3], a[1]);
  const float ecx = __fadd_rn(a[0], __fmul_rn(0.5f, ew)), ecy = __fadd_rn(a[1], __fmul_rn(0.5f, eh));
  const float gw = __fsub_rn(g[2], g[0]), gh = __fsub_rn(g[3], g[1]);
  const float gcx = __fadd_rn(g[0], __fmul_rn(0.5f, gw)), gcy = __fadd_rn(g[1], __fmul_rn(0.5f, gh));
  t[0] = __fdiv_rn(__fmul_rn(w[0], __fsub_rn(gcx, ecx)), ew);
  t[1] = __fdiv_rn(__fmul_rn(w[1], __fsub_rn(gcy, ecy)), eh);
  t[2] = __fmul_rn(w[2], logf(__fdiv_rn(gw, ew)));
  t[3] = __fmul_rn(w[3], logf(__fdiv_rn(gh, eh)));
}

__device__ __forceinline__ void load_row(const float* base, int64_t row, const int64_t* stride, float v[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = base[row * stride[0] + j * stride[1]];
}

// torch.sign: 0 for ±0 and for NaN
__device__ __forceinline__ float sign_of(float v) { return (float)((0.f < v) - (v < 0.f)); }

// One CTA: kLossTile anchors of image blockIdx.y, one per thread.  Only foreground anchors read their regression row.
template <bool kBackward>
__global__ void __launch_bounds__(kLossThreads)
box_loss_kernel(const __grid_constant__ LossPlan plan) {
  const vb200_retinanet_loss_image& d = plan.img[blockIdx.y];
  const int image = plan.first_image + (int)blockIdx.y;
  const int64_t a = (int64_t)blockIdx.x * kLossTile + threadIdx.x;
  const bool valid = a < plan.num_anchors;
  const int64_t m = valid ? d.matched[a * d.matched_stride] : -1;
  const bool fg = m >= 0;
  __shared__ double scratch[kLossThreads / 32];
  double acc = 0.0;
  float gout[4] = {0.f, 0.f, 0.f, 0.f};
  if (fg) {
    if (m >= d.num_gt) {
      acc = (double)NAN;
#pragma unroll
      for (int j = 0; j < 4; ++j) gout[j] = NAN;
    } else {
      float an[4], gt[4], t[4], pv[4];
      load_row(d.anchors, a, d.anchor_stride, an);
      load_row(d.gt, m, d.gt_stride, gt);
      encode_box(plan.weights, an, gt, t);
#pragma unroll
      for (int j = 0; j < 4; ++j) pv[j] = d.pred[a * 4 + j];
      if (kBackward) {
        const float scale = image_scale<true>(plan, image);
#pragma unroll
        for (int j = 0; j < 4; ++j) gout[j] = scale * sign_of(__fsub_rn(pv[j], t[j]));
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) acc += (double)fabsf(__fsub_rn(pv[j], t[j]));
      }
    }
  }
  if (kBackward) {
    if (valid) *reinterpret_cast<float4*>(d.grad + a * 4) = make_float4(gout[0], gout[1], gout[2], gout[3]);
  } else {
    const int tile_fg = __syncthreads_count(fg);
    const double sum = block_sum(acc, scratch);
    if (threadIdx.x == 0) {
      plan.partial[(int64_t)image * plan.tiles + blockIdx.x] = sum;
      plan.tile_fg[(int64_t)image * plan.tiles + blockIdx.x] = tile_fg;
    }
  }
}

// Per image: the partials in a fixed order, / max(1, n_fg) as the head divides (true division in the classification head,
// the reciprocal product in the regression head); then ((L0 + L1) + L2) ... as _sum adds them, times the fp32 reciprocal of
// len(targets).
template <bool kBox>
__global__ void __launch_bounds__(kFinalizeThreads)
loss_finalize_kernel(const double* __restrict__ partial, const int* __restrict__ tile_fg, int tiles, int num_images, float* loss,
                     int64_t* num_fg) {
  __shared__ double scratch[kFinalizeThreads / 32];
  float total = 0.f;
  for (int i = 0; i < num_images; ++i) {
    double s = 0.0, n = 0.0;                           // counts below 2^53 are exact in a double
    for (int j = threadIdx.x; j < tiles; j += kFinalizeThreads) {
      s += partial[(int64_t)i * tiles + j];
      n += (double)tile_fg[(int64_t)i * tiles + j];
    }
    s = block_sum(s, scratch);
    n = block_sum(n, scratch);
    if (threadIdx.x == 0) {
      const int64_t count = (int64_t)n;
      num_fg[i] = count;
      const float dv = (float)(count > 1 ? count : 1);
      const float li = kBox ? __fmul_rn((float)s, reciprocal(dv)) : __fdiv_rn((float)s, dv);
      total = i == 0 ? li : __fadd_rn(total, li);
    }
  }
  if (threadIdx.x == 0) *loss = __fmul_rn(total, reciprocal((float)num_images));
}

int check_call(const vb200_retinanet_loss_image* images, int num_images, int64_t num_anchors, int width, bool box, bool backward,
               const char* op) {
  VB200_REQUIRE(num_images >= 1 && images, "%s: at least one image", op);
  VB200_REQUIRE(num_anchors >= 0 && width >= 1 && num_anchors * width < ((int64_t)1 << 31), "%s: bad sizes (%lld anchors, width %d)", op,
                (long long)num_anchors, width);
  for (int i = 0; i < num_images; ++i) {
    const vb200_retinanet_loss_image& d = images[i];
    VB200_REQUIRE(d.num_gt >= 0, "%s: image %d: bad gt count", op, i);
    if (num_anchors == 0) continue;
    VB200_REQUIRE(d.pred && d.matched && (!backward || d.grad) && (!box || d.anchors), "%s: image %d: null pointer", op, i);
    VB200_REQUIRE(d.num_gt == 0 || (box ? d.gt != nullptr : d.labels != nullptr), "%s: image %d: null gt pointer", op, i);
    VB200_REQUIRE(!box || !backward || (reinterpret_cast<uintptr_t>(d.grad) & 15) == 0, "%s: image %d: gradient rows must be 16-byte aligned",
                  op, i);
  }
  return 0;
}

template <bool kBox, bool kBackward>
int launch_loss(LossPlan& plan, const vb200_retinanet_loss_image* images, int num_images, cudaStream_t st) {
  if (plan.tiles == 0) return 0;
  for (int done = 0; done < num_images; done += VB200_LOSS_MAX_IMAGES) {
    const int chunk = num_images - done < VB200_LOSS_MAX_IMAGES ? num_images - done : VB200_LOSS_MAX_IMAGES;
    for (int i = 0; i < chunk; ++i) plan.img[i] = images[done + i];
    plan.first_image = done;
    const dim3 grid((unsigned)plan.tiles, (unsigned)chunk);
    if (kBox) box_loss_kernel<kBackward><<<grid, kLossThreads, 0, st>>>(plan);
    else focal_loss_kernel<kBackward><<<grid, kLossThreads, 0, st>>>(plan);
    const int rc = check_launch(kBox ? "box_loss_kernel" : "focal_loss_kernel");
    if (rc) return rc;
  }
  return 0;
}

int tiles_of(int64_t num_anchors) { return (int)ceil_div64(num_anchors, kLossTile); }

size_t loss_workspace_bytes(int num_images, int64_t num_anchors) {
  if (num_images < 1 || num_anchors < 0) return 0;
  const size_t slots = (size_t)num_images * (size_t)tiles_of(num_anchors);
  return align256(slots * sizeof(double)) + align256(slots * sizeof(int));
}

template <bool kBox>
int loss_forward(const vb200_retinanet_loss_image* images, int num_images, int64_t num_anchors, int width, const float* weights,
                 float* loss, int64_t* num_fg, void* workspace, size_t workspace_bytes, cudaStream_t st, const char* op) {
  const int rc = check_call(images, num_images, num_anchors, width, kBox, false, op);
  if (rc) return rc;
  VB200_REQUIRE(loss && num_fg, "%s: null outputs", op);
  const size_t need = loss_workspace_bytes(num_images, num_anchors);
  if (need && (!workspace || workspace_bytes < need)) {
    set_error("%s: workspace of %zu bytes, %zu needed", op, workspace_bytes, need);
    return VB200_EWORKSPACE;
  }
  LossPlan plan;
  plan.num_anchors = num_anchors;
  plan.num_classes = width;
  plan.tiles = tiles_of(num_anchors);
  plan.num_images = num_images;
  Carver ws(workspace);
  plan.partial = ws.take<double>((size_t)num_images * plan.tiles);
  plan.tile_fg = ws.take<int>((size_t)num_images * plan.tiles);
  plan.grad_loss = nullptr;
  plan.num_fg = nullptr;
  for (int j = 0; j < 4; ++j) plan.weights[j] = weights ? weights[j] : 0.f;
  const int lrc = launch_loss<kBox, false>(plan, images, num_images, st);
  if (lrc) return lrc;
  loss_finalize_kernel<kBox><<<1, kFinalizeThreads, 0, st>>>(plan.partial, plan.tile_fg, plan.tiles, num_images, loss, num_fg);
  return check_launch("loss_finalize_kernel");
}

template <bool kBox>
int loss_backward(const vb200_retinanet_loss_image* images, int num_images, int64_t num_anchors, int width, const float* weights,
                  const float* grad_loss, const int64_t* num_fg, cudaStream_t st, const char* op) {
  const int rc = check_call(images, num_images, num_anchors, width, kBox, true, op);
  if (rc) return rc;
  VB200_REQUIRE(grad_loss && num_fg, "%s: null gradient or counts", op);
  LossPlan plan;
  plan.num_anchors = num_anchors;
  plan.num_classes = width;
  plan.tiles = tiles_of(num_anchors);
  plan.num_images = num_images;
  plan.partial = nullptr;
  plan.tile_fg = nullptr;
  plan.grad_loss = grad_loss;
  plan.num_fg = num_fg;
  for (int j = 0; j < 4; ++j) plan.weights[j] = weights ? weights[j] : 0.f;
  return launch_loss<kBox, true>(plan, images, num_images, st);
}

}  // namespace
}  // namespace vb200

using namespace vb200;

extern "C" size_t vb200_retinanet_cls_loss_workspace_bytes(int num_images, int64_t num_anchors) {
  return loss_workspace_bytes(num_images, num_anchors);
}

extern "C" int vb200_retinanet_cls_loss(const vb200_retinanet_loss_image* images, int num_images, int64_t num_anchors, int num_classes,
                                        float* loss, int64_t* num_foreground, void* workspace, size_t workspace_bytes,
                                        vb200_stream stream) {
  return loss_forward<false>(images, num_images, num_anchors, num_classes, nullptr, loss, num_foreground, workspace, workspace_bytes,
                             (cudaStream_t)stream, "retinanet_cls_loss");
}

extern "C" int vb200_retinanet_cls_loss_backward(const vb200_retinanet_loss_image* images, int num_images, int64_t num_anchors,
                                                 int num_classes, const float* grad_loss, const int64_t* num_foreground,
                                                 vb200_stream stream) {
  return loss_backward<false>(images, num_images, num_anchors, num_classes, nullptr, grad_loss, num_foreground, (cudaStream_t)stream,
                              "retinanet_cls_loss_backward");
}

extern "C" size_t vb200_retinanet_box_loss_workspace_bytes(int num_images, int64_t num_anchors) {
  return loss_workspace_bytes(num_images, num_anchors);
}

extern "C" int vb200_retinanet_box_loss(const vb200_retinanet_loss_image* images, int num_images, int64_t num_anchors,
                                        const float* weights_host, float* loss, int64_t* num_foreground, void* workspace,
                                        size_t workspace_bytes, vb200_stream stream) {
  VB200_REQUIRE(weights_host, "retinanet_box_loss: null weights");
  return loss_forward<true>(images, num_images, num_anchors, 4, weights_host, loss, num_foreground, workspace, workspace_bytes,
                            (cudaStream_t)stream, "retinanet_box_loss");
}

extern "C" int vb200_retinanet_box_loss_backward(const vb200_retinanet_loss_image* images, int num_images, int64_t num_anchors,
                                                 const float* weights_host, const float* grad_loss, const int64_t* num_foreground,
                                                 vb200_stream stream) {
  VB200_REQUIRE(weights_host, "retinanet_box_loss_backward: null weights");
  return loss_backward<true>(images, num_images, num_anchors, 4, weights_host, grad_loss, num_foreground, (cudaStream_t)stream,
                             "retinanet_box_loss_backward");
}
