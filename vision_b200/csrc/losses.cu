// losses.cu — the single-stage detectors' head losses, forward and backward, sm_90a: RetinaNet's
// (torchvision/models/detection/retinanet.py:158-189 and 272-302) and FCOS's (fcos.py:52-125).
//
// The reference, per image: a full-size zeros_like target with the ones scattered in, boolean indexing of the logits and the
// target (a nonzero, a host sync), sigmoid_focal_loss (ops/focal_loss.py:41-56) as a chain of full-size elementwise kernels,
// max(1, num_foreground) on a CUDA tensor or a .item() (another sync); the box terms add more syncs and chains of small
// kernels over the gathered foreground rows.  Autograd keeps the full-size intermediates for a backward of the same shape.
// Here every image of a call is one grid layer of (tile of kLossTile anchors, image):
//   forward   each CTA stages its anchors' codes (target class, background, ignored or bad) in shared memory, streams its
//             anchors' logits once with 16-byte loads and writes one partial sum and foreground count to a per-(image, tile)
//             slot; the box losses do the same per foreground anchor with the reference's box arithmetic restated op by op.
//   finalize  one CTA adds the partials in a fixed order and divides as the head does: per image then over the images
//             (RetinaNet), or once for the whole batch (FCOS).
//   backward  the dense gradient written exactly once: the analytic derivative times the head's scale, 0 where the
//             reference's indexing leaves it 0.
// No floating-point atomics and no launch parameter depends on the SM count, so every result is bit-reproducible run to run.
//
// Mask R-CNN's mask loss (roi_heads.py:85-129) follows the same plan over (RoI, bin) instead of (anchor, class): the
// forward projects each positive RoI's gt mask on its box with the generic roi_align kernel's own per-bin routine
// (roi_geometry.cuh), reading the uint8 / bool masks in place, and adds the BCE term of the RoI's label plane; the backward
// writes the dense [P, C, M, M] gradient once from the saved targets.
#include "common.cuh"
#include "roi_geometry.cuh"

namespace vb200 {
namespace {

constexpr int kLossThreads = 256;
constexpr int kLossTile = 256;                      // anchors per CTA, every loss: one anchor per thread when staging
static_assert(kLossThreads == kLossTile, "the code staging and the box losses give each thread one anchor");
constexpr int kFinalizeThreads = 256;

// anchor codes; a code >= 0 is the anchor's target class
constexpr int kBad = -3;          // an index the reference cannot gather with (it raises): the loss is NaN
constexpr int kIgnored = -2;      // RetinaNet's matched == Matcher.BETWEEN_THRESHOLDS: no loss, zero gradient
constexpr int kBackground = -1;   // every class's target is 0

// How a head turns its sum into the loss (and so the backward's scale):
//   kImageDiv    per image, a true division by max(1, n_i) (a CUDA tensor), the images summed, times fl(1 / B)
//   kImageRecip  per image, the product with fl(1 / max(1, n_i)) (a Python int), the images summed, times fl(1 / B)
//   kBatchRecip  once for the batch, the product with fl(1 / max(1, n)), n from .item()
enum class Norm { kImageDiv, kImageRecip, kBatchRecip };

struct LossPlan {
  vb200_loss_image img[VB200_LOSS_MAX_IMAGES];
  int64_t num_anchors;
  int num_classes, tiles, first_image, num_images;     // img[0] is image first_image of the call's num_images
  double* partial;                                      // forward: [num_images, tiles]
  double* partial2;                                     // FCOS box forward: the centre-ness partials, [num_images, tiles]
  int* tile_fg;                                         // forward: [num_images, tiles]
  const float* grad_loss;                               // backward: the 0-dim incoming gradient (FCOS box: of the GIoU loss)
  const float* grad_loss2;                              // FCOS box backward: of the centre-ness loss
  const int64_t* num_fg;                                // backward: the forward's foreground counts
  float weights[4];                                     // RetinaNet box loss: the coder's weights as fp32
  bool normalize;                                       // FCOS box loss: BoxLinearCoder.normalize_by_size
};

// RetinaNet: the Matcher's -2 is ignored; a label in [-C, 0) wraps as advanced indexing does.
struct RetinaNetCls {
  static constexpr Norm kNorm = Norm::kImageDiv;
  __device__ static __forceinline__ int code(const vb200_loss_image& d, int64_t a, int C, bool& fg) {
    const int64_t m = d.matched[a * d.matched_stride];
    fg = m >= 0;                                        // num_foreground counts matched >= 0, bad indices included
    if (m == -2) return kIgnored;
    if (m < 0) return kBackground;
    if (m >= d.num_gt) return kBad;
    const int64_t l = d.labels[m * d.label_stride];
    if (l < -C || l >= C) return kBad;
    return (int)(l < 0 ? l + C : l);
  }
};

// FCOS (fcos.py:64-90): every negative match is background; an image without gt gives a match the class 0 of new_zeros; a
// negative label is background (the mask is >= 0, nothing wraps).  `C` bounds the class: the box call passes INT64_MAX, as
// its reference reads no class.  m is the match, for the box call's gt row.
__device__ __forceinline__ int fcos_code(const vb200_loss_image& d, int64_t a, int64_t C, int64_t& m) {
  m = d.matched[a * d.matched_stride];
  if (m < 0) return kBackground;
  if (d.num_gt == 0) return 0;
  if (m >= d.num_gt) return kBad;
  const int64_t l = d.labels[m * d.label_stride];
  if (l < 0) return kBackground;
  return l >= C ? kBad : (int)l;
}

struct FcosCls {
  static constexpr Norm kNorm = Norm::kBatchRecip;
  __device__ static __forceinline__ int code(const vb200_loss_image& d, int64_t a, int C, bool& fg) {
    int64_t m;
    const int c = fcos_code(d, a, C, m);
    fg = c >= 0 || c == kBad;                           // the reference's mask is label >= 0, bad indices included
    return c;
  }
};

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

// t = 1: α(1-p)²(2p·log p - (1-p));  t = 0: (1-α)p²(p - 2(1-p)·log(1-p)); times the head's scale, rounded once.  NaN for a
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

__device__ __forceinline__ float max1(int64_t n) { return (float)(n > 1 ? n : 1); }

// The backward's scale of an image's elements, in the order autograd applies the head's divisions to the incoming g: for
// RetinaNet g / len(targets) (a Python int), then / max(1, num_foreground) -- a CUDA int64 tensor in the classification head
// (a true division), a Python int in the regression head; for FCOS g / max(1, n), a Python int.
template <Norm kNorm> __device__ __forceinline__ float loss_scale(const float* grad, const int64_t* num_fg, int num_images, int image) {
  if (kNorm == Norm::kBatchRecip) return __fmul_rn(*grad, reciprocal(max1(num_fg[0])));
  const float g = __fmul_rn(*grad, reciprocal((float)num_images));
  const float d = max1(num_fg[image]);
  return kNorm == Norm::kImageRecip ? __fmul_rn(g, reciprocal(d)) : __fdiv_rn(g, d);
}

// A forward CTA's results in its per-(image, tile) slots, stored by thread 0 (which holds the block sums); sum2 only for the
// FCOS box loss.
__device__ __forceinline__ void store_tile(const LossPlan& plan, int image, int tile_fg, double sum, const double* sum2 = nullptr) {
  if (threadIdx.x != 0) return;
  const int64_t slot = (int64_t)image * plan.tiles + blockIdx.x;
  plan.partial[slot] = sum;
  if (sum2) plan.partial2[slot] = *sum2;
  plan.tile_fg[slot] = tile_fg;
}

// One CTA: kLossTile anchors of image blockIdx.y, all C classes.  The tile's elements [e0, e1) of the image's [A, C] block are
// taken in 16-byte groups aligned on the streamed array (the logits forward, the gradient backward); the first and last groups
// may be partial, since C need not be a multiple of 4.  Rule gives each anchor its code and the head's division.
template <class Rule, bool kBackward>
__global__ void __launch_bounds__(kLossThreads)
focal_loss_kernel(const __grid_constant__ LossPlan plan) {
  const vb200_loss_image& d = plan.img[blockIdx.y];
  const int image = plan.first_image + (int)blockIdx.y;
  const int C = plan.num_classes;
  const int64_t a0 = (int64_t)blockIdx.x * kLossTile;
  const int na = (int)(plan.num_anchors - a0 < kLossTile ? plan.num_anchors - a0 : kLossTile);
  __shared__ int s_code[kLossTile];
  __shared__ double scratch[kLossThreads / 32];

  bool fg = false;
  s_code[threadIdx.x] = threadIdx.x < na ? Rule::code(d, a0 + threadIdx.x, C, fg) : kIgnored;
  const int tile_fg = __syncthreads_count(fg);          // also the barrier after the staging

  const int64_t e0 = a0 * C, e1 = (a0 + na) * C;
  const float* __restrict__ x = d.pred;
  float* __restrict__ out = d.grad;
  const float* streamed = kBackward ? out : x;
  const int pad = (int)((reinterpret_cast<uintptr_t>(streamed + e0) >> 2) & 3);
  const bool vec_load = !kBackward || ((reinterpret_cast<uintptr_t>(x) ^ reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  const int64_t g0 = e0 - pad;                          // first element of the first group
  const int groups = (int)((e1 - g0 + 3) >> 2);
  const float scale = kBackward ? loss_scale<Rule::kNorm>(plan.grad_loss, plan.num_fg, plan.num_images, image) : 0.f;
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
  if (!kBackward) store_tile(plan, image, tile_fg, block_sum(acc, scratch));
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

// BoxLinearCoder (models/detection/_utils.py:227-310), op by op in fp32 with nothing contracted.  decode: p = (cx - r0,
// cy - r1, cx + r2, cy + r3) with r = rel · (w, h, w, h) when normalising, else rel; the same decode in fp64 (for the
// gradient's values) and d p_j / d rel_j.  encode: the anchor centre's distances to the gt box's edges, / (w, h, w, h) when
// normalising.
__device__ __forceinline__ void linear_decode(const float rel[4], const float a[4], bool normalize, float p[4], double pd[4],
                                              double dp_drel[4]) {
  const float cx = __fmul_rn(0.5f, __fadd_rn(a[0], a[2])), cy = __fmul_rn(0.5f, __fadd_rn(a[1], a[3]));
  const float w = __fsub_rn(a[2], a[0]), h = __fsub_rn(a[3], a[1]);
  const double cxd = 0.5 * ((double)a[0] + a[2]), cyd = 0.5 * ((double)a[1] + a[3]);
  const double wd = normalize ? (double)a[2] - a[0] : 1.0, hd = normalize ? (double)a[3] - a[1] : 1.0;
  float r[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) r[j] = normalize ? __fmul_rn(rel[j], j & 1 ? h : w) : rel[j];
  p[0] = __fsub_rn(cx, r[0]);
  p[1] = __fsub_rn(cy, r[1]);
  p[2] = __fadd_rn(cx, r[2]);
  p[3] = __fadd_rn(cy, r[3]);
  pd[0] = cxd - rel[0] * wd;
  pd[1] = cyd - rel[1] * hd;
  pd[2] = cxd + rel[2] * wd;
  pd[3] = cyd + rel[3] * hd;
  dp_drel[0] = -wd;
  dp_drel[1] = -hd;
  dp_drel[2] = wd;
  dp_drel[3] = hd;
}

__device__ __forceinline__ void linear_encode(const float a[4], const float g[4], bool normalize, float t[4]) {
  const float cx = __fmul_rn(0.5f, __fadd_rn(a[0], a[2])), cy = __fmul_rn(0.5f, __fadd_rn(a[1], a[3]));
  t[0] = __fsub_rn(cx, g[0]);
  t[1] = __fsub_rn(cy, g[1]);
  t[2] = __fsub_rn(g[2], cx);
  t[3] = __fsub_rn(g[3], cy);
  if (normalize) {
    const float w = __fsub_rn(a[2], a[0]), h = __fsub_rn(a[3], a[1]);
#pragma unroll
    for (int j = 0; j < 4; ++j) t[j] = __fdiv_rn(t[j], j & 1 ? h : w);
  }
}

constexpr float kGiouEps = 1e-7f;                       // generalized_box_iou_loss's eps, as a fp32 tensor op rounds it

// generalized_box_iou_loss (ops/giou_loss.py) with _loss_inter_union (ops/_utils.py:87-105) for one box p against its gt g,
// op by op in fp32: the intersection only where (yk2 > yk1) & (xk2 > xk1) (strict, so NaN fails), else exactly 0;
// union = (a1 + a2) - inter; loss = 1 - (iou - (area_c - union) / (area_c + eps)).
__device__ __forceinline__ float giou_loss(const float p[4], const float g[4]) {
  const float xk1 = nan_max(p[0], g[0]), yk1 = nan_max(p[1], g[1]), xk2 = nan_min(p[2], g[2]), yk2 = nan_min(p[3], g[3]);
  const float inter = yk2 > yk1 && xk2 > xk1 ? __fmul_rn(__fsub_rn(xk2, xk1), __fsub_rn(yk2, yk1)) : 0.f;
  const float a1 = __fmul_rn(__fsub_rn(p[2], p[0]), __fsub_rn(p[3], p[1]));
  const float a2 = __fmul_rn(__fsub_rn(g[2], g[0]), __fsub_rn(g[3], g[1]));
  const float uni = __fsub_rn(__fadd_rn(a1, a2), inter);
  const float iou = __fdiv_rn(inter, __fadd_rn(uni, kGiouEps));
  const float xc1 = nan_min(p[0], g[0]), yc1 = nan_min(p[1], g[1]), xc2 = nan_max(p[2], g[2]), yc2 = nan_max(p[3], g[3]);
  const float area_c = __fmul_rn(__fsub_rn(xc2, xc1), __fsub_rn(yc2, yc1));
  return __fsub_rn(1.f, __fsub_rn(iou, __fdiv_rn(__fsub_rn(area_c, uni), __fadd_rn(area_c, kGiouEps))));
}

// autograd's share of torch.max(p, g) / torch.min(p, g) for p: half where they are equal, none where the other side wins
__device__ __forceinline__ double max_share(float p, float g) { return p == g ? 0.5 : p < g ? 0.0 : 1.0; }
__device__ __forceinline__ double min_share(float p, float g) { return p == g ? 0.5 : p > g ? 0.0 : 1.0; }

// d giou_loss / d p.  Every branch -- the overlap mask and which side of each min / max wins -- is the fp32 forward's
// decision on p; the values are fp64, from pd (p's fp64 decode).  With U = union + eps, C = area_c + eps, I = inter:
// dL/dI = -1/U - I/U² + 1/C, dL/d a1 = I/U² - 1/C, dL/d area_c = U/C².
__device__ __forceinline__ void giou_grad(const float p[4], const double pd[4], const float g[4], double dl[4]) {
  const bool overlap = nan_min(p[3], g[3]) > nan_max(p[1], g[1]) && nan_min(p[2], g[2]) > nan_max(p[0], g[0]);
  double gd[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) gd[j] = g[j];
  const double iw = nan_min(pd[2], gd[2]) - nan_max(pd[0], gd[0]), ih = nan_min(pd[3], gd[3]) - nan_max(pd[1], gd[1]);
  const double I = overlap ? iw * ih : 0.0;
  const double pw = pd[2] - pd[0], ph = pd[3] - pd[1];
  const double U = pw * ph + (gd[2] - gd[0]) * (gd[3] - gd[1]) - I + (double)kGiouEps;
  const double cw = nan_max(pd[2], gd[2]) - nan_min(pd[0], gd[0]), ch = nan_max(pd[3], gd[3]) - nan_min(pd[1], gd[1]);
  const double C = cw * ch + (double)kGiouEps;
  const double d_a1 = I / (U * U) - 1.0 / C, d_c = U / (C * C);
  dl[0] = -d_a1 * ph - d_c * ch * min_share(p[0], g[0]);
  dl[1] = -d_a1 * pw - d_c * cw * min_share(p[1], g[1]);
  dl[2] = d_a1 * ph + d_c * ch * max_share(p[2], g[2]);
  dl[3] = d_a1 * pw + d_c * cw * max_share(p[3], g[3]);
  if (overlap) {
    const double d_i = -1.0 / U - I / (U * U) + 1.0 / C;
    dl[0] -= d_i * ih * max_share(p[0], g[0]);
    dl[1] -= d_i * iw * max_share(p[1], g[1]);
    dl[2] += d_i * ih * min_share(p[2], g[2]);
    dl[3] += d_i * iw * min_share(p[3], g[3]);
  }
}

// The centre-ness target (fcos.py:105-115): sqrt(min(l, r) / max(l, r) · min(t, b) / max(t, b)) of encode(anchor, gt), with
// the NaN-propagating min and max of Tensor.min / .max(dim).
__device__ __forceinline__ float ctrness_target(const float a[4], const float g[4], bool normalize) {
  float t[4];
  linear_encode(a, g, normalize, t);
  const float lr = __fdiv_rn(nan_min(t[0], t[2]), nan_max(t[0], t[2]));
  const float tb = __fdiv_rn(nan_min(t[1], t[3]), nan_max(t[1], t[3]));
  return __fsqrt_rn(__fmul_rn(lr, tb));
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
  const vb200_loss_image& d = plan.img[blockIdx.y];
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
        const float scale = loss_scale<Norm::kImageRecip>(plan.grad_loss, plan.num_fg, plan.num_images, image);
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
    store_tile(plan, image, tile_fg, block_sum(acc, scratch));
  }
}

// FCOS's GIoU and centre-ness losses.  One CTA: kLossTile anchors of image blockIdx.y, one per thread; only foreground
// anchors read their regression row, centre-ness logit, anchor and gt box (the zero box for an image without gt).  The
// centre-ness term is binary_cross_entropy_with_logits, (1 - t) x - log σ(x) with -log σ(x) = softplus(-x) in the focal
// loss's stable form; its derivative σ(x) - t.
template <bool kBackward>
__global__ void __launch_bounds__(kLossThreads)
fcos_box_loss_kernel(const __grid_constant__ LossPlan plan) {
  const vb200_loss_image& d = plan.img[blockIdx.y];
  const int image = plan.first_image + (int)blockIdx.y;
  const int64_t a = (int64_t)blockIdx.x * kLossTile + threadIdx.x;
  const bool valid = a < plan.num_anchors;
  int64_t m = -1;
  const int code = valid ? fcos_code(d, a, INT64_MAX, m) : kBackground;
  const bool fg = code >= 0 || code == kBad;
  __shared__ double scratch[kLossThreads / 32];
  double giou = 0.0, bce = 0.0;
  float gbox[4] = {0.f, 0.f, 0.f, 0.f}, gctr = 0.f;
  if (code == kBad) {
    giou = bce = (double)NAN;
#pragma unroll
    for (int j = 0; j < 4; ++j) gbox[j] = NAN;
    gctr = NAN;
  } else if (fg) {
    float an[4], gt[4] = {0.f, 0.f, 0.f, 0.f}, rel[4], p[4];
    double pd[4], dp_drel[4];
    load_row(d.anchors, a, d.anchor_stride, an);
    if (d.num_gt > 0) load_row(d.gt, m, d.gt_stride, gt);
#pragma unroll
    for (int j = 0; j < 4; ++j) rel[j] = d.pred[a * 4 + j];
    const float x = d.ctrness[a * d.ctrness_stride];
    const float t = ctrness_target(an, gt, plan.normalize);
    linear_decode(rel, an, plan.normalize, p, pd, dp_drel);
    if (kBackward) {
      if (plan.grad_loss) {
        const double s = loss_scale<Norm::kBatchRecip>(plan.grad_loss, plan.num_fg, plan.num_images, image);
        double dl[4];
        giou_grad(p, pd, gt, dl);
#pragma unroll
        for (int j = 0; j < 4; ++j) gbox[j] = (float)(s * dl[j] * dp_drel[j]);
      }
      if (plan.grad_loss2) {
        const double s = loss_scale<Norm::kBatchRecip>(plan.grad_loss2, plan.num_fg, plan.num_images, image);
        gctr = (float)(s * (sig(x).p - (double)t));
      }
    } else {
      giou = (double)giou_loss(p, gt);
      bce = (1.0 - (double)t) * (double)x + sig(x).sp_neg;
    }
  }
  if (kBackward) {
    if (valid) {
      *reinterpret_cast<float4*>(d.grad + a * 4) = make_float4(gbox[0], gbox[1], gbox[2], gbox[3]);
      d.grad_ctrness[a] = gctr;
    }
  } else {
    const int tile_fg = __syncthreads_count(fg);
    const double sum = block_sum(giou, scratch);
    const double sum2 = block_sum(bce, scratch);
    store_tile(plan, image, tile_fg, sum, &sum2);
  }
}

// Each image's partials and counts in a fixed order.  Per image (RetinaNet): / max(1, n_i) as the head divides, then
// ((L0 + L1) + L2) ... as _sum adds them, times the fp32 reciprocal of len(targets); each image's count kept.  For the batch
// (FCOS, launched as one image of all the batch's slots): the sum rounded to fp32 once, times fl(1 / max(1, n)); the batch's
// count kept.  partial2 (may be null) gives loss2 the same way.
template <Norm kNorm>
__global__ void __launch_bounds__(kFinalizeThreads)
loss_finalize_kernel(const double* __restrict__ partial, const double* __restrict__ partial2, const int* __restrict__ tile_fg,
                     int tiles, int num_images, float* loss, float* loss2, int64_t* num_fg) {
  __shared__ double scratch[kFinalizeThreads / 32];
  float total = 0.f;
  for (int i = 0; i < num_images; ++i) {
    double s = 0.0, s2 = 0.0, n = 0.0;                 // counts below 2^53 are exact in a double
    for (int j = threadIdx.x; j < tiles; j += kFinalizeThreads) {
      s += partial[(int64_t)i * tiles + j];
      if (partial2) s2 += partial2[(int64_t)i * tiles + j];
      n += (double)tile_fg[(int64_t)i * tiles + j];
    }
    s = block_sum(s, scratch);
    if (partial2) s2 = block_sum(s2, scratch);
    n = block_sum(n, scratch);
    if (threadIdx.x == 0) {
      const int64_t count = (int64_t)n;
      num_fg[i] = count;
      if (kNorm == Norm::kBatchRecip) {
        const float r = reciprocal(max1(count));
        *loss = __fmul_rn((float)s, r);
        if (loss2) *loss2 = __fmul_rn((float)s2, r);
      } else {
        const float dv = max1(count);
        const float li = kNorm == Norm::kImageRecip ? __fmul_rn((float)s, reciprocal(dv)) : __fdiv_rn((float)s, dv);
        total = i == 0 ? li : __fadd_rn(total, li);
      }
    }
  }
  if (kNorm != Norm::kBatchRecip && threadIdx.x == 0) *loss = __fmul_rn(total, reciprocal((float)num_images));
}

// What each kind runs: its kernels, the division its finalize applies, its number of losses and its names in errors.
struct Head {
  void (*forward)(const LossPlan);
  void (*backward)(const LossPlan);
  const char* kernel;
  Norm norm;
  int terms;                                            // 2: FCOS's GIoU and centre-ness losses from one call
  const char *op, *op_backward;
};

Head head_of(int kind) {
  switch (kind) {
    case VB200_LOSS_RETINANET_CLS:
      return {focal_loss_kernel<RetinaNetCls, false>, focal_loss_kernel<RetinaNetCls, true>, "focal_loss_kernel", RetinaNetCls::kNorm, 1,
              "retinanet_cls_loss", "retinanet_cls_loss_backward"};
    case VB200_LOSS_RETINANET_BOX:
      return {box_loss_kernel<false>, box_loss_kernel<true>, "box_loss_kernel", Norm::kImageRecip, 1, "retinanet_box_loss",
              "retinanet_box_loss_backward"};
    case VB200_LOSS_FCOS_CLS:
      return {focal_loss_kernel<FcosCls, false>, focal_loss_kernel<FcosCls, true>, "focal_loss_kernel", FcosCls::kNorm, 1,
              "fcos_cls_loss", "fcos_cls_loss_backward"};
    case VB200_LOSS_FCOS_BOX:
      return {fcos_box_loss_kernel<false>, fcos_box_loss_kernel<true>, "fcos_box_loss_kernel", Norm::kBatchRecip, 2, "fcos_box_loss",
              "fcos_box_loss_backward"};
  }
  return {};                                            // forward null: an unknown kind
}

// The sizes, and every pointer of the descriptors that the kind reads.
int check_call(int kind, const vb200_loss_image* images, int num_images, int64_t num_anchors, int width, bool backward, const char* op) {
  const bool box = kind == VB200_LOSS_RETINANET_BOX || kind == VB200_LOSS_FCOS_BOX, ctrness = kind == VB200_LOSS_FCOS_BOX,
             labels = kind != VB200_LOSS_RETINANET_BOX;
  VB200_REQUIRE(num_images >= 1 && images, "%s: at least one image", op);
  VB200_REQUIRE(num_anchors >= 0 && width >= 1 && num_anchors * width < ((int64_t)1 << 31), "%s: bad sizes (%lld anchors, width %d)", op,
                (long long)num_anchors, width);
  VB200_REQUIRE(!box || width == 4, "%s: width %d, the box losses take 4", op, width);
  for (int i = 0; i < num_images; ++i) {
    const vb200_loss_image& d = images[i];
    VB200_REQUIRE(d.num_gt >= 0, "%s: image %d: bad gt count", op, i);
    if (num_anchors == 0) continue;
    VB200_REQUIRE(d.pred && d.matched && (!backward || d.grad) && (!box || d.anchors) && (!ctrness || (d.ctrness && (!backward || d.grad_ctrness))),
                  "%s: image %d: null pointer", op, i);
    VB200_REQUIRE(d.num_gt == 0 || ((!labels || d.labels) && (!box || d.gt)), "%s: image %d: null gt pointer", op, i);
    VB200_REQUIRE(!box || !backward || (reinterpret_cast<uintptr_t>(d.grad) & 15) == 0, "%s: image %d: gradient rows must be 16-byte aligned",
                  op, i);
  }
  return 0;
}

// One launch of `kernel` per VB200_LOSS_MAX_IMAGES images, each with its images' descriptors in the plan.
int launch_loss(void (*kernel)(const LossPlan), const char* name, LossPlan& plan, const vb200_loss_image* images, int num_images,
                cudaStream_t st) {
  if (plan.tiles == 0) return 0;
  for (int done = 0; done < num_images; done += VB200_LOSS_MAX_IMAGES) {
    const int chunk = num_images - done < VB200_LOSS_MAX_IMAGES ? num_images - done : VB200_LOSS_MAX_IMAGES;
    for (int i = 0; i < chunk; ++i) plan.img[i] = images[done + i];
    plan.first_image = done;
    const dim3 grid((unsigned)plan.tiles, (unsigned)chunk);
    kernel<<<grid, kLossThreads, 0, st>>>(plan);
    const int rc = check_launch(name);
    if (rc) return rc;
  }
  return 0;
}

int tiles_of(int64_t num_anchors) { return (int)ceil_div64(num_anchors, kLossTile); }

// the per-(image, tile) partials of `terms` losses and the foreground counts
size_t loss_workspace_bytes(int num_images, int64_t num_anchors, int terms) {
  if (num_images < 1 || num_anchors < 0) return 0;
  const size_t slots = (size_t)num_images * (size_t)tiles_of(num_anchors);
  return terms * align256(slots * sizeof(double)) + align256(slots * sizeof(int));
}

LossPlan make_plan(int kind, int num_images, int64_t num_anchors, int width, const float* weights_host, int normalize_by_size) {
  LossPlan plan;
  plan.num_anchors = num_anchors;
  plan.num_classes = width;
  plan.tiles = tiles_of(num_anchors);
  plan.first_image = 0;
  plan.num_images = num_images;
  plan.partial = plan.partial2 = nullptr;
  plan.tile_fg = nullptr;
  plan.grad_loss = plan.grad_loss2 = nullptr;
  plan.num_fg = nullptr;
  for (int j = 0; j < 4; ++j) plan.weights[j] = kind == VB200_LOSS_RETINANET_BOX ? weights_host[j] : 0.f;
  plan.normalize = kind == VB200_LOSS_FCOS_BOX && normalize_by_size != 0;
  return plan;
}

// ---- Mask R-CNN mask loss ------------------------------------------------------------------------------------------------
constexpr int kMaskThreads = 256;

struct MaskPlan {
  vb200_mask_image img[VB200_LOSS_MAX_IMAGES];
  int64_t roi_begin[VB200_LOSS_MAX_IMAGES];             // img[i]'s first RoI, counted from the chunk's first
  int images;                                           // in this chunk
  int num_classes, size;
  int64_t first_roi, num_rois;                          // the chunk's RoIs, counted in the call
  int64_t total_rois;                                   // the call's P
  int64_t first_partial;                                // forward: the chunk's first CTA slot
  const float* logits;
  float* targets;                                       // forward: written; backward: read
  double* partial;                                      // forward
  const float* grad_loss;                               // backward (null: a zero gradient)
  float* grad;                                          // backward
};

// A chunk RoI's gt index and class plane; bad as the loss's bad-index rule says.
struct MaskRoi {
  int image;
  int64_t row, m;
  int label;
  bool bad;
};

__device__ __forceinline__ MaskRoi mask_roi(const MaskPlan& plan, int64_t p) {
  int lo = 0, hi = plan.images - 1;                     // the last image starting at or before p holds it
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (plan.roi_begin[mid] <= p) lo = mid;
    else hi = mid - 1;
  }
  const vb200_mask_image& d = plan.img[lo];
  MaskRoi q;
  q.image = lo;
  q.row = p - plan.roi_begin[lo];
  q.m = d.matched[q.row * d.matched_stride];
  q.label = 0;
  q.bad = q.m < 0 || q.m >= d.num_gt;
  if (!q.bad) {
    const int64_t l = d.labels[q.m * d.label_stride];
    q.bad = l < -plan.num_classes || l >= plan.num_classes;
    q.label = (int)(l < 0 ? l + plan.num_classes : l);
  }
  return q;
}

// One thread per (RoI, bin) of the chunk: the bin's target, written, and its BCE term; one partial sum per CTA.
__global__ void __launch_bounds__(kMaskThreads)
mask_loss_kernel(const __grid_constant__ MaskPlan plan) {
  __shared__ double scratch[kMaskThreads / 32];
  const int M = plan.size, MM = M * M;
  const int64_t e = (int64_t)blockIdx.x * kMaskThreads + threadIdx.x;
  double term = 0.0;
  if (e < plan.num_rois * MM) {
    const int64_t pl = e / MM;
    const int bin = (int)(e - pl * MM);
    const MaskRoi q = mask_roi(plan, pl);
    const int64_t p = plan.first_roi + pl;
    float t = NAN;
    if (q.bad) {
      term = (double)NAN;
    } else {
      const vb200_mask_image& d = plan.img[q.image];
      float r[5];
      r[0] = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) r[1 + j] = d.proposals[q.row * d.proposal_stride[0] + j * d.proposal_stride[1]];
      const RoiGeom<float> g = roi_geometry<float, float>(r, 1.f, M, M, -1, false, false);
      const StridedPlane<uint8_t> mask{static_cast<const uint8_t*>(d.masks) + q.m * d.mask_stride[0], d.mask_stride[1], d.mask_stride[2]};
      t = roi_align_bin<float>(mask, (int)d.height, (int)d.width, g, bin / M, bin % M, false, nullptr, nullptr);
      const float x = __ldg(plan.logits + ((p * plan.num_classes + q.label) * MM + bin));
      term = (1.0 - (double)t) * (double)x + sig(x).sp_neg;
    }
    plan.targets[p * MM + bin] = t;
  }
  const double sum = block_sum(term, scratch);
  if (threadIdx.x == 0) plan.partial[plan.first_partial + blockIdx.x] = sum;
}

// The CTA partials in order; *loss = fl(S) * fl(1 / N).
__global__ void __launch_bounds__(kFinalizeThreads)
mask_loss_finalize_kernel(const double* __restrict__ partial, int64_t count, int64_t n, float* loss) {
  __shared__ double scratch[kFinalizeThreads / 32];
  double s = 0.0;
  for (int64_t j = threadIdx.x; j < count; j += kFinalizeThreads) s += partial[j];
  s = block_sum(s, scratch);
  if (threadIdx.x == 0) *loss = __fmul_rn((float)s, reciprocal((float)n));
}

// One thread per 16-byte group of the chunk's [P_chunk, C, M, M] gradient, groups aligned on the gradient's address (the
// first and last may be partial).  Flat element offsets are below 2^31, so the index arithmetic is 32-bit.
__global__ void __launch_bounds__(kMaskThreads)
mask_loss_backward_kernel(const __grid_constant__ MaskPlan plan) {
  const uint32_t MM = (uint32_t)(plan.size * plan.size), block = (uint32_t)plan.num_classes * MM;
  const int64_t e0 = plan.first_roi * block, e1 = (plan.first_roi + plan.num_rois) * block;
  float* __restrict__ out = plan.grad;
  const int pad = (int)((reinterpret_cast<uintptr_t>(out + e0) >> 2) & 3);
  const int64_t eb = e0 - pad + 4 * ((int64_t)blockIdx.x * kMaskThreads + threadIdx.x);
  if (eb >= e1) return;
  const float s = plan.grad_loss ? __fmul_rn(*plan.grad_loss, reciprocal((float)(plan.total_rois * MM))) : 0.f;
  // (RoI, class, bin) of the group's first element inside the chunk, then stepped element by element
  const uint32_t u = (uint32_t)(eb < e0 ? e0 : eb);
  uint32_t p = u / block, c = (u - p * block) / MM, bin = u - p * block - c * MM;
  MaskRoi q = mask_roi(plan, (int64_t)p - plan.first_roi);
  float gout[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    gout[k] = 0.f;
    const int64_t e = eb + k;
    if (e < e0 || e >= e1 || !plan.grad_loss) continue;
    if (q.bad) {
      gout[k] = NAN;
    } else if ((int)c == q.label) {
      const float x = __ldg(plan.logits + e), t = __ldg(plan.targets + (int64_t)p * MM + bin);
      gout[k] = (float)((double)s * (sig(x).p - (double)t));
    }
    if (++bin == MM) {
      bin = 0;
      if (++c == (uint32_t)plan.num_classes && k < 3 && e + 1 < e1) {
        c = 0;
        q = mask_roi(plan, (int64_t)++p - plan.first_roi);
      }
    }
  }
  if (eb >= e0 && eb + 4 <= e1) {
    __stcs(reinterpret_cast<float4*>(out + eb), make_float4(gout[0], gout[1], gout[2], gout[3]));
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (eb + k >= e0 && eb + k < e1) out[eb + k] = gout[k];
  }
}

// The sizes, and every pointer an image with RoIs reads (the backward reads neither masks nor proposals).
int check_mask_call(const vb200_mask_image* images, int num_images, int num_classes, int size, bool backward, int64_t& total_rois,
                    const char* op) {
  VB200_REQUIRE(num_images >= 1 && images, "%s: at least one image", op);
  VB200_REQUIRE(num_classes >= 1 && size >= 1 && size <= 4096, "%s: bad sizes (%d classes, size %d)", op, num_classes, size);
  total_rois = 0;
  for (int i = 0; i < num_images; ++i) {
    const vb200_mask_image& d = images[i];
    VB200_REQUIRE(d.num_rois >= 0 && d.num_gt >= 0 && d.height >= 0 && d.width >= 0 && d.height < ((int64_t)1 << 31) &&
                      d.width < ((int64_t)1 << 31),
                  "%s: image %d: bad sizes", op, i);
    VB200_REQUIRE(backward || d.mask_dtype == VB200_U8, "%s: image %d: masks must be uint8 (or bool as uint8), dtype %d given", op, i,
                  d.mask_dtype);
    total_rois += d.num_rois;
    VB200_REQUIRE(total_rois * num_classes * size * size < ((int64_t)1 << 31), "%s: 2^31 or more logits", op);
    if (d.num_rois == 0) continue;
    VB200_REQUIRE(d.matched && (backward || d.proposals), "%s: image %d: null pointer", op, i);
    VB200_REQUIRE(d.num_gt == 0 || (d.labels && (backward || (d.masks && d.height >= 1 && d.width >= 1))), "%s: image %d: null or empty gt",
                  op, i);
  }
  return 0;
}

// One launch of `kernel` per VB200_LOSS_MAX_IMAGES images holding RoIs; `grid(rois)` its CTA count for a chunk's RoIs, the
// CTA slots of the forward's partials handed out in order.
template <class Grid>
int launch_mask(void (*kernel)(const MaskPlan), const char* name, MaskPlan& plan, const vb200_mask_image* images, int num_images,
                Grid&& grid, cudaStream_t st) {
  int64_t roi = 0, slot = 0;
  for (int done = 0; done < num_images; done += VB200_LOSS_MAX_IMAGES) {
    const int chunk = num_images - done < VB200_LOSS_MAX_IMAGES ? num_images - done : VB200_LOSS_MAX_IMAGES;
    plan.images = chunk;
    plan.first_roi = roi;
    int64_t n = 0;
    for (int i = 0; i < chunk; ++i) {
      plan.img[i] = images[done + i];
      plan.roi_begin[i] = n;
      n += images[done + i].num_rois;
    }
    plan.num_rois = n;
    plan.first_partial = slot;
    roi += n;
    if (n == 0) continue;
    const int64_t ctas = grid(n);
    slot += ctas;
    kernel<<<(unsigned)ctas, kMaskThreads, 0, st>>>(plan);
    const int rc = check_launch(name);
    if (rc) return rc;
  }
  return 0;
}

// The forward's CTA slots: at most one partial CTA per chunk beyond the call's full ones.
int64_t mask_partials(int num_images, int64_t total_rois, int size) {
  return ceil_div64(total_rois * size * size, kMaskThreads) + ceil_div64(num_images, VB200_LOSS_MAX_IMAGES);
}

MaskPlan make_mask_plan(const float* logits, int num_classes, int size, int64_t total_rois) {
  MaskPlan plan;
  plan.num_classes = num_classes;
  plan.size = size;
  plan.total_rois = total_rois;
  plan.logits = logits;
  plan.targets = nullptr;
  plan.partial = nullptr;
  plan.grad_loss = nullptr;
  plan.grad = nullptr;
  return plan;
}

}  // namespace
}  // namespace vb200

using namespace vb200;

extern "C" size_t vb200_head_loss_workspace_bytes(int kind, int num_images, int64_t num_anchors) {
  const Head h = head_of(kind);
  return h.forward ? loss_workspace_bytes(num_images, num_anchors, h.terms) : 0;
}

// The partials of one loss (loss2 null) or two, then the finalize.
extern "C" int vb200_head_loss(int kind, const vb200_loss_image* images, int num_images, int64_t num_anchors, int width,
                               const float* weights_host, int normalize_by_size, float* loss, float* loss2, int64_t* num_foreground,
                               void* workspace, size_t workspace_bytes, vb200_stream stream) {
  const Head h = head_of(kind);
  VB200_REQUIRE(h.forward, "head_loss: unknown kind %d", kind);
  const char* op = h.op;
  VB200_REQUIRE(kind != VB200_LOSS_RETINANET_BOX || weights_host, "%s: null weights", op);
  VB200_REQUIRE(h.terms == 1 || loss2, "%s: null outputs", op);
  VB200_REQUIRE(h.terms == 2 || !loss2, "%s: loss2 is for the FCOS box loss only", op);
  int rc = check_call(kind, images, num_images, num_anchors, width, false, op);
  if (rc) return rc;
  VB200_REQUIRE(loss && num_foreground, "%s: null outputs", op);
  const size_t need = loss_workspace_bytes(num_images, num_anchors, h.terms);
  if (need && (!workspace || workspace_bytes < need)) {
    set_error("%s: workspace of %zu bytes, %zu needed", op, workspace_bytes, need);
    return VB200_EWORKSPACE;
  }
  LossPlan plan = make_plan(kind, num_images, num_anchors, width, weights_host, normalize_by_size);
  Carver ws(workspace);
  plan.partial = ws.take<double>((size_t)num_images * plan.tiles);
  if (loss2) plan.partial2 = ws.take<double>((size_t)num_images * plan.tiles);
  plan.tile_fg = ws.take<int>((size_t)num_images * plan.tiles);
  const cudaStream_t st = (cudaStream_t)stream;
  rc = launch_loss(h.forward, h.kernel, plan, images, num_images, st);
  if (rc) return rc;
  const bool batch = h.norm == Norm::kBatchRecip;     // the [num_images, tiles] slots as one image's
  const auto finalize = batch ? loss_finalize_kernel<Norm::kBatchRecip>
                        : h.norm == Norm::kImageRecip ? loss_finalize_kernel<Norm::kImageRecip> : loss_finalize_kernel<Norm::kImageDiv>;
  finalize<<<1, kFinalizeThreads, 0, st>>>(plan.partial, plan.partial2, plan.tile_fg, batch ? num_images * plan.tiles : plan.tiles,
                                          batch ? 1 : num_images, loss, loss2, num_foreground);
  return check_launch("loss_finalize_kernel");
}

extern "C" int vb200_head_loss_backward(int kind, const vb200_loss_image* images, int num_images, int64_t num_anchors, int width,
                                        const float* weights_host, int normalize_by_size, const float* grad_loss,
                                        const float* grad_loss2, const int64_t* num_foreground, vb200_stream stream) {
  const Head h = head_of(kind);
  VB200_REQUIRE(h.forward, "head_loss_backward: unknown kind %d", kind);
  const char* op = h.op_backward;
  VB200_REQUIRE(kind != VB200_LOSS_RETINANET_BOX || weights_host, "%s: null weights", op);
  VB200_REQUIRE(h.terms == 2 || !grad_loss2, "%s: grad_loss2 is for the FCOS box loss only", op);
  const int rc = check_call(kind, images, num_images, num_anchors, width, true, op);
  if (rc) return rc;
  VB200_REQUIRE(num_foreground && (grad_loss || grad_loss2), "%s: null gradient or counts", op);
  LossPlan plan = make_plan(kind, num_images, num_anchors, width, weights_host, normalize_by_size);
  plan.grad_loss = grad_loss;
  plan.grad_loss2 = grad_loss2;
  plan.num_fg = num_foreground;
  return launch_loss(h.backward, h.kernel, plan, images, num_images, (cudaStream_t)stream);
}

extern "C" size_t vb200_mask_loss_workspace_bytes(int num_images, int64_t total_rois, int size) {
  if (num_images < 1 || total_rois < 0 || size < 1) return 0;
  return align256((size_t)mask_partials(num_images, total_rois, size) * sizeof(double));
}

extern "C" int vb200_mask_loss(const vb200_mask_image* images, int num_images, const float* mask_logits, int num_classes, int size,
                               float* loss, float* targets, void* workspace, size_t workspace_bytes, vb200_stream stream) {
  const char* op = "maskrcnn_loss";
  int64_t total_rois = 0;
  int rc = check_mask_call(images, num_images, num_classes, size, false, total_rois, op);
  if (rc) return rc;
  VB200_REQUIRE(loss && (total_rois == 0 || (mask_logits && targets)), "%s: null logits or outputs", op);
  const size_t need = vb200_mask_loss_workspace_bytes(num_images, total_rois, size);
  if (!workspace || workspace_bytes < need) {
    set_error("%s: workspace of %zu bytes, %zu needed", op, workspace_bytes, need);
    return VB200_EWORKSPACE;
  }
  MaskPlan plan = make_mask_plan(mask_logits, num_classes, size, total_rois);
  plan.targets = targets;
  plan.partial = static_cast<double*>(workspace);
  const cudaStream_t st = (cudaStream_t)stream;
  const int64_t bins = (int64_t)size * size;
  int64_t slots = 0;
  rc = launch_mask(mask_loss_kernel, "mask_loss_kernel", plan, images, num_images,
                   [&](int64_t rois) {
                     const int64_t ctas = ceil_div64(rois * bins, kMaskThreads);
                     slots += ctas;
                     return ctas;
                   },
                   st);
  if (rc) return rc;
  mask_loss_finalize_kernel<<<1, kFinalizeThreads, 0, st>>>(plan.partial, slots, total_rois * bins, loss);
  return check_launch("mask_loss_finalize_kernel");
}

extern "C" int vb200_mask_loss_backward(const vb200_mask_image* images, int num_images, const float* mask_logits, const float* targets,
                                        int num_classes, int size, const float* grad_loss, float* grad_logits, vb200_stream stream) {
  const char* op = "maskrcnn_loss_backward";
  int64_t total_rois = 0;
  const int rc = check_mask_call(images, num_images, num_classes, size, true, total_rois, op);
  if (rc) return rc;
  VB200_REQUIRE(total_rois == 0 || (mask_logits && targets && grad_logits), "%s: null logits, targets or gradient", op);
  MaskPlan plan = make_mask_plan(mask_logits, num_classes, size, total_rois);
  plan.targets = const_cast<float*>(targets);
  plan.grad_loss = grad_loss;
  plan.grad = grad_logits;
  const int64_t block = (int64_t)num_classes * size * size;
  return launch_mask(mask_loss_backward_kernel, "mask_loss_backward_kernel", plan, images, num_images,
                     [&](int64_t rois) {
                       const int64_t e0 = plan.first_roi * block;
                       const int pad = (int)((reinterpret_cast<uintptr_t>(grad_logits + e0) >> 2) & 3);
                       return ceil_div64(ceil_div64(rois * block + pad, 4), kMaskThreads);
                     },
                     (cudaStream_t)stream);
}
