// nms.cu — nms and fused segmented batched_nms for sm_90a.
//
// Reference semantics (pytorch/vision):
//   nms           csrc/ops/cuda/nms_kernel.cu:42-148,166-258 ; csrc/ops/cpu/nms_kernel.cpp:17-95
//   batched_nms   torchvision/ops/boxes.py:57-126 (Python: per-class loop or coordinate trick)
//
// Design (not a port):
//   * order = stable radix sort of scores (descending);  batched: a second
//     stable sort by class id turns the score order into class-major segments
//     whose inner order is still score-descending;
//   * mask + scan (default): bnms_mask_kernel computes the IoU bit matrix of every class on all SMs
//     (64x64 tiles per warp, one vote per 32 tests, fp32 filter in front of the exact predicate),
//     bnms_scan_kernel walks each class's greedy chain on bit words (one CTA per class).  Plain nms
//     is the same pair with a single segment;
//   * "segment" kernel (classes longer than 2048 boxes): one CTA per class segment walks the segment
//     in blocks of 64 boxes: (1) the 64x64 diagonal IoU bit-matrix by warp ballot, (2) one thread
//     resolves the greedy chain inside the block on bit-words, (3) all threads test the still-alive
//     later boxes against the <=64 boxes kept in this block.  No mask memory, any segment length;
//   * kept indices are emitted in global score order by flag compaction.
// IoU arithmetic is written with explicit round-to-nearest intrinsics so that
// the selected semantics (compiled-CUDA-reference or CPU-reference) is
// reproduced bit for bit regardless of compiler contraction decisions.
#include <cub/cub.cuh>

#include <cmath>
#include <cstring>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace vb200 {
namespace {

constexpr int kSegThreads = 1024;

struct IouParams {
  float thr_f;
  double thr_d;
  int semantics;
  // division-free exact form of "RN_f32(inter / den) > threshold" (see make_iou_params)
  double mid;
  int s_even;
  int use_div;
  // fp32 filter in front of the exact test (bnms_mask_kernel): t = fma(-mid_f, den, inter) has the sign of
  // inter - mid*den whenever |t| > eps_f * den (see make_iou_params); anything else is re-tested exactly.
  float mid_f, eps_f;
  // boxes are exact widenings of fp16 values and the arithmetic is what nvcc made of devIoU<Half>
  // (csrc/ops/cuda/nms_kernel.cu:42-54; SASS of the wheel's cubin): min/max on the half values, the two
  // extents and the HEIGHT of each area rounded to half (F2FP.F16.F32), the WIDTH of each area kept in fp32, all
  // products in fp32, Sb's product contracted into Sa + Sb, IEEE fp32 division, float threshold.
  int half_mode;
};

// Both reference predicates have the form  q >= S  with q = RN_f32(inter/den) and S a float:
//   CUDA: q > (float)thr            -> S = nextafter((float)thr, +inf)
//   CPU : (double)q > thr (double)  -> S = smallest float whose double value exceeds thr
// q >= S  <=>  inter/den > m, or == m when the tie rounds up (S has an even mantissa), with
// m = (pred(S) + S) / 2.  For den > 0 that is  inter > m*den  evaluated EXACTLY in double
// (m has <= 25 significant bits, den 24: the product fits the 53-bit mantissa).  Verified against
// float32 division on 8 M borderline cases (tools note in DESIGN.md); den <= 0 / NaN and
// non-finite thresholds take the literal division path.
inline IouParams make_iou_params(double thr, int semantics) {
  IouParams p;
  p.thr_f = (float)thr;
  p.thr_d = thr;
  p.semantics = semantics;
  float S;
  if (semantics == VB200_NMS_CUDA) {
    S = nextafterf(p.thr_f, INFINITY);
  } else {
    const float c = (float)thr;
    S = ((double)c > thr) ? c : nextafterf(c, INFINITY);
  }
  const float T = nextafterf(S, -INFINITY);
  p.use_div = !(isfinite(S) && isfinite(T) && isfinite(thr));
  p.mid = ((double)T + (double)S) * 0.5;
  uint32_t bits;
  memcpy(&bits, &S, 4);
  p.s_even = (bits & 1u) == 0u;
  // v = inter - mid*den = (inter - mid_f*den) - (mid - mid_f)*den and t = RN(inter - mid_f*den):
  // |v - t| <= 2^-24 |t| + 2^-24 |mid| den, so |t| > 2^-21 |mid_f| den (four times the second term) fixes the sign
  // of v and rules out v == 0.  Tiny or non-finite operands never pass the filter (den > 1e-30 is required).
  p.mid_f = (float)p.mid;
  p.eps_f = p.use_div ? INFINITY : nextafterf(ldexpf(fabsf(p.mid_f), -21), INFINITY);
  p.half_mode = 0;
  return p;
}

// fp64 boxes (the reference instantiates nms for double; its tests compare CPU and CUDA in fp64)
struct alignas(16) double4a { double x, y, z, w; };
template <typename S> struct BoxOf;
template <> struct BoxOf<float> { using type = float4; };
template <> struct BoxOf<double> { using type = double4a; };
template <typename Box> struct ScalarOf;
template <> struct ScalarOf<float4> { using type = float; };
template <> struct ScalarOf<double4a> { using type = double; };
__device__ __forceinline__ float4 zero_box(float4*) { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ double4a zero_box(double4a*) { return double4a{0., 0., 0., 0.}; }
__device__ __forceinline__ float4 load_box(const float4* p) { return __ldg(p); }
__device__ __forceinline__ double4a load_box(const double4a* p) { return *p; }

// fp64: csrc/ops/cuda/nms_kernel.cu:42-54 instantiated for double compiles to the same shape as the float
// kernel (SASS of the wheel's cubin: Sa = DMUL, t = DFMA(bw, bh, Sa), den = t - inter, IEEE division, compare
// against the threshold narrowed to float and widened back); the CPU kernel rounds both areas and compares
// against the double threshold.
__device__ __forceinline__ bool iou_gt(const double4a a, const double area_a, const double4a b, const IouParams p) {
  const double left = fmax(a.x, b.x), right = fmin(a.z, b.z);
  const double top = fmax(a.y, b.y), bottom = fmin(a.w, b.w);
  const double w = fmax(sub_rn(right, left), 0.0), h = fmax(sub_rn(bottom, top), 0.0);
  const double inter = mul_rn(w, h);
  double den;
  if (p.semantics == VB200_NMS_CUDA) den = sub_rn(__fma_rn(sub_rn(b.z, b.x), sub_rn(b.w, b.y), area_a), inter);
  else den = sub_rn(add_rn(area_a, mul_rn(sub_rn(b.z, b.x), sub_rn(b.w, b.y))), inter);
  const double q = div_rn(inter, den);
  return p.semantics == VB200_NMS_CUDA ? (q > (double)p.thr_f) : (q > p.thr_d);
}

__device__ __forceinline__ float half_rn(float v) { return __half2float(__float2half_rn(v)); }

// Area of the suppressor box as the selected reference arithmetic forms it (the "Sa" of devIoU / `areas` of the CPU kernel).
__device__ __forceinline__ float box_area(const float4 a, const IouParams p) {
  const float w = sub_rn(a.z, a.x), h = sub_rn(a.w, a.y);
  return mul_rn(w, p.half_mode ? half_rn(h) : h);
}
__device__ __forceinline__ double box_area(const double4a a, const IouParams) { return mul_rn(sub_rn(a.z, a.x), sub_rn(a.w, a.y)); }

// a = higher-scoring (suppressor) box, b = candidate.  area_a precomputed = box_area(a).
__device__ __forceinline__ bool iou_gt(const float4 a, const float area_a, const float4 b, const IouParams p) {
  const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  float w = sub_rn(right, left), h = sub_rn(bottom, top);
  if (p.half_mode) { w = half_rn(w); h = half_rn(h); }
  w = fmaxf(w, 0.f); h = fmaxf(h, 0.f);
  const float inter = mul_rn(w, h);
  float den;
  if (p.half_mode) {
    den = sub_rn(__fmaf_rn(sub_rn(b.z, b.x), half_rn(sub_rn(b.w, b.y)), area_a), inter);
  } else if (p.semantics == VB200_NMS_CUDA) {
    // nms_kernel.cu:50-53 as compiled: Sb's product contracted into (Sa + Sb), float threshold
    den = sub_rn(__fmaf_rn(sub_rn(b.z, b.x), sub_rn(b.w, b.y), area_a), inter);
  } else {
    // cpu/nms_kernel.cpp:58,86-88: separately rounded areas, double threshold
    den = sub_rn(add_rn(area_a, mul_rn(sub_rn(b.z, b.x), sub_rn(b.w, b.y))), inter);
  }
  if (!p.use_div && den > 0.f) {
    const double di = (double)inter, rhs = p.mid * (double)den;     // exact
    return di > rhs || (p.s_even && di == rhs);
  }
  const float q = div_rn(inter, den);
  return p.semantics == VB200_NMS_CUDA ? (q > p.thr_f) : ((double)q > p.thr_d);
}

__global__ void iota_kernel(int* __restrict__ out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = i;
}

// boxes_sorted[p] = boxes[order[p]] (one 128-bit load per box)
template <typename Box>
__global__ void gather_boxes_kernel(const Box* __restrict__ boxes, const int* __restrict__ order,
                                    Box* __restrict__ out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = load_box(boxes + order[i]);
}

// class key of the box at score-rank r; flags ids outside [0, 2^16) (the narrow-key fast path is then invalid)
__global__ void gather_class_kernel(const int64_t* __restrict__ idxs, const int* __restrict__ order,
                                    int64_t* __restrict__ keys, int n, int* __restrict__ out_of_range) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const int64_t k = idxs[order[i]];
    keys[i] = k;
    if ((uint64_t)k >= 65536ull) *out_of_range = 1;        // benign race: every writer stores 1
  }
}

// *num_keep = -1 tells the caller to repeat the call with VB200_BNMS_WIDE_KEYS
__global__ void poison_count_kernel(const int* __restrict__ out_of_range, int64_t* __restrict__ num_keep) {
  if (*out_of_range) *num_keep = -1;
}

// class-major gather through two permutations + segment-start flags
template <typename Box>
__global__ void gather_boxes_cm_kernel(const Box* __restrict__ boxes, const int* __restrict__ order,
                                       const int* __restrict__ rank_cm, const int64_t* __restrict__ cls_sorted,
                                       Box* __restrict__ out, uint8_t* __restrict__ seg_flag, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    out[i] = load_box(boxes + order[rank_cm[i]]);
    seg_flag[i] = (i == 0 || cls_sorted[i] != cls_sorted[i - 1]) ? 1 : 0;
  }
}

// coordinate trick (boxes.py:103-107): boxes + float(idx) * (max + 1), each op rounded once
__device__ __forceinline__ float round_storage(float v, int half_mode) { return half_mode ? __half2float(__float2half_rn(v)) : v; }
__device__ __forceinline__ double round_storage(double v, int) { return v; }

// half_mode: the reference runs every step as a separate fp16 tensor op (boxes.py:103-107 on Half tensors):
// idxs.to(half), max + 1, the product and the sum are each computed in float and rounded to half.
template <typename Box>
__global__ void shift_boxes_kernel(const Box* __restrict__ boxes, const int64_t* __restrict__ idxs,
                                   const typename ScalarOf<Box>::type* __restrict__ max_coord, Box* __restrict__ out, int n,
                                   int half_mode) {
  using S = typename ScalarOf<Box>::type;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const S step = round_storage(add_rn(*max_coord, (S)1), half_mode);
    const S off = round_storage(mul_rn(round_storage((S)idxs[i], half_mode), step), half_mode);
    Box b = boxes[i];
    b.x = round_storage(add_rn(b.x, off), half_mode); b.y = round_storage(add_rn(b.y, off), half_mode);
    b.z = round_storage(add_rn(b.z, off), half_mode); b.w = round_storage(add_rn(b.w, off), half_mode);
    out[i] = b;
  }
}

// fp16 boxes / scores -> their exact fp32 widenings (the half arithmetic is reproduced on these, see IouParams::half_mode)
__global__ void widen_half_kernel(const uint2* __restrict__ boxes_h, const __half* __restrict__ scores_h,
                                  float4* __restrict__ boxes_f, float* __restrict__ scores_f, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const uint2 v = __ldg(boxes_h + i);
    const __half2 lo = *reinterpret_cast<const __half2*>(&v.x), hi = *reinterpret_cast<const __half2*>(&v.y);
    const float2 a = __half22float2(lo), b = __half22float2(hi);
    boxes_f[i] = make_float4(a.x, a.y, b.x, b.y);
    scores_f[i] = __half2float(scores_h[i]);
  }
}

// ---- segmented mask + scan (batched_nms, segments up to kBnmsMaxLen boxes) ----------------------
// The greedy chain of a class is short (n_c sequential decisions); the ~n_c^2/2 IoU tests are not, and
// with one CTA per class they keep only as many SMs busy as there are classes.  So the tests are done
// first, by every SM: row p (position in the class-major sorted order) gets `wpr` 64-bit words (stored
// word-major: word k of row p at mask[k * n + p]), word k covering positions [64 (p/64 + k), +64) - bit set <=> that later box of the same class has
// IoU(p, .) > threshold.  The per-class chain then only walks bit words.
constexpr int kBnmsWpr = 33;                         // words per row
constexpr int kBnmsMaxLen = 64 * (kBnmsWpr - 1);     // a segment this long spans at most kBnmsWpr position blocks

// Largest idx with seg_start[idx] <= p.
__device__ __forceinline__ int find_segment(const int* __restrict__ seg_start, int nseg, int p) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(seg_start + mid) <= p) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Column-side terms of the fp32 filter, fixed per lane for a whole tile.
template <typename Box> struct ColTerms;
template <> struct ColTerms<float4> {
  float4 b; float bw, bh, sb; bool bad;
  __device__ __forceinline__ void set(const float4 v) {
    b = v; bw = sub_rn(v.z, v.x); bh = sub_rn(v.w, v.y); sb = mul_rn(bw, bh);
    bad = !(bw >= 0.f) || !(bh >= 0.f) || !(sb <= 1e37f);   // inverted / NaN / huge boxes: exact test only
  }
};
template <> struct ColTerms<double4a> {
  double4a b; bool bad;
  __device__ __forceinline__ void set(const double4a v) { b = v; bad = true; }   // fp64 boxes: the exact test is the only test
};

// fp32 filter in front of the exact test.  For a proper row box (aw, ah >= 0, Sa > 1e-29) and a proper column
// box, inter <= min(Sa, Sb) up to rounding, so den > Sa / 2 > 1e-30: the den guard of make_iou_params holds
// without a per-test check.  Returns the decision; `unsure` when only the exact test may decide.
template <int SEM>
__device__ __forceinline__ bool iou_gt_filter(const float4 a, const float area_a, const ColTerms<float4>& c, const IouParams p,
                                              bool& unsure) {
  // Only one extent is clamped: with mid > 0 (required by the caller) a negative h makes inter <= 0 and the
  // decision "not greater", which is what the exact test returns for an empty intersection.
  const float w = fmaxf(sub_rn(fminf(a.z, c.b.z), fmaxf(a.x, c.b.x)), 0.f);
  const float h = sub_rn(fminf(a.w, c.b.w), fmaxf(a.y, c.b.y));
  const float inter = mul_rn(w, h);
  const float den = SEM == VB200_NMS_CUDA ? sub_rn(__fmaf_rn(c.bw, c.bh, area_a), inter) : sub_rn(add_rn(area_a, c.sb), inter);
  const float t = __fmaf_rn(-p.mid_f, den, inter);
  unsure = !(fabsf(t) > mul_rn(p.eps_f, den));
  return t > 0.f;
}
template <int SEM>
__device__ __forceinline__ bool iou_gt_filter(const double4a, const double, const ColTerms<double4a>&, const IouParams, bool& unsure) {
  unsure = true;
  return false;
}

// CTA = one block of 64 rows (positions), kMaskWarps warps; a warp owns whole 64x64 tiles (column block
// kb = i + warp, i + warp + kMaskWarps, ...): its lanes hold two column boxes each, the rows are broadcast from
// shared memory, and one vote per 32 IoU tests delivers the bits.  min/max, compares and votes share the
// half-rate ALU pipe, which is what bounds this kernel, so everything else (result capture, unsure flags, column
// validity) is kept off it or out of the loop.
constexpr int kMaskWarps = 8;
template <typename Box, int SEM>
__global__ void __launch_bounds__(kMaskWarps * 32)
bnms_mask_kernel(const Box* __restrict__ boxes, const int* __restrict__ seg_start, const int* __restrict__ num_seg_ptr,
                 int n, int wpr, int max_len, IouParams prm, unsigned long long* __restrict__ mask) {
  using S = typename ScalarOf<Box>::type;
  __shared__ Box rbx[64];
  __shared__ S rarea[64];
  __shared__ int rend[64];             // segment end of row r, or 0 when the row is not handled here
  __shared__ unsigned long long s_word[kMaskWarps][64];   // a warp's tile: row r's 64 column bits
  __shared__ int s_kmax, s_rowbad;
  const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nseg = seg_start ? *num_seg_ptr : 1;      // no table: one segment [0, n)
  if (tid == 0) { s_kmax = -1; s_rowbad = 0; }
  __syncthreads();
  if (tid < 64) {
    const int p = 64 * i + tid;
    int e = 0;
    Box a = zero_box((Box*)nullptr);
    if (p < n) {
      int s = 0, ee = n;
      if (seg_start) {
        const int sg = find_segment(seg_start, nseg, p);
        s = __ldg(seg_start + sg);
        ee = (sg + 1 < nseg) ? __ldg(seg_start + sg + 1) : n;
      }
      if (ee - s <= max_len) { e = ee; a = boxes[p]; }     // longer segments take the sequential path
    }
    const S aw = sub_rn(a.z, a.x), ah = sub_rn(a.w, a.y), sa = box_area(a, prm);
    rbx[tid] = a;
    rarea[tid] = sa;
    rend[tid] = e;
    if (e > 0) {
      atomicMax(&s_kmax, (e - 1) >> 6);
      if (!(aw >= (S)0) || !(ah >= (S)0) || !(sa > (S)1e-29) || !(sa <= (S)1e37)) s_rowbad = 1;   // the filter's den bound needs proper rows
    }
  }
  __syncthreads();
  const int kmax = s_kmax;
  const bool exact_only = s_rowbad != 0 || prm.use_div != 0 || !(prm.mid_f > 0.f) || prm.half_mode != 0;
  for (int kb = i + warp; kb <= kmax; kb += kMaskWarps) {
    const int col0 = kb * 64;
    ColTerms<Box> c0, c1;
    c0.set((col0 + lane < n) ? boxes[col0 + lane] : zero_box((Box*)nullptr));
    c1.set((col0 + 32 + lane < n) ? boxes[col0 + 32 + lane] : zero_box((Box*)nullptr));
    bool unsure = exact_only | c0.bad | c1.bad;
    if (!exact_only) {
#pragma unroll 8
      for (int r = 0; r < 64; ++r) {
        const Box a = rbx[r];
        const S aa = rarea[r];
        bool u0, u1;
        const bool p0 = iou_gt_filter<SEM>(a, aa, c0, prm, u0);
        const bool p1 = iou_gt_filter<SEM>(a, aa, c1, prm, u1);
        const unsigned int v0 = __ballot_sync(0xffffffffu, p0), v1 = __ballot_sync(0xffffffffu, p1);
        unsure |= u0 | u1;
        if (lane == 0) s_word[warp][r] = ((unsigned long long)v1 << 32) | v0;
      }
    }
    if (__any_sync(0xffffffffu, unsure)) {       // warp-uniform and rare: (re)do the tile with the exact predicate
      for (int r = 0; r < 64; ++r) {
        const Box a = rbx[r];
        const S aa = rarea[r];
        const unsigned int v0 = __ballot_sync(0xffffffffu, iou_gt(a, aa, c0.b, prm));
        const unsigned int v1 = __ballot_sync(0xffffffffu, iou_gt(a, aa, c1.b, prm));
        if (lane == 0) s_word[warp][r] = ((unsigned long long)v1 << 32) | v0;
      }
    }
    __syncwarp();
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = lane + 32 * hh;
      const int p = 64 * i + r, e = rend[r];
      if (e > 0 && col0 < e) {
        unsigned long long word = s_word[warp][r];
        // keep columns in (p, e): later positions of the same class
        const int first = p + 1 - col0, last = e - col0;         // valid bit range [first, last)
        if (first > 0) word &= first >= 64 ? 0ull : ~0ull << first;
        if (last < 64) word &= ~0ull >> (64 - last);
        mask[(size_t)(kb - i) * n + p] = word;          // word-major: the 64 rows of a tile are 512 contiguous bytes
      }
    }
    __syncwarp();              // s_word is rewritten by the next tile
  }
}

// Chain of one segment [s, e) over the mask, kScanThreads = 256 threads.  256 positions per step: their
// diagonal words (4 per row) are staged in shared memory one step ahead, warp 0 walks the 256 decisions, then
// warp j folds the rows that were kept into removed-word j for the blocks after the step.
__device__ __forceinline__ void segment_scan(const unsigned long long* __restrict__ mask, int wpr, int n, int s, int e,
                                             uint8_t* __restrict__ suppressed, unsigned long long* removed /* 2 (wpr + 4) */,
                                             unsigned long long (*dgbuf)[256][4] /* 2 */, unsigned long long* keptw /* 4 */) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int kfirst = s >> 6, klast = (e - 1) >> 6;
  unsigned long long* keptbits = removed + (wpr + 4);     // one bit per position of the segment, set when kept
  for (int t = tid; t < 2 * (wpr + 4); t += blockDim.x) removed[t] = 0ull;
  // thread t owns words (row t, 0..3) of a step
  auto fetch = [&](int kb0, unsigned long long (&v)[4]) {
    const int pos = 64 * kb0 + tid;
#pragma unroll
    for (int wq = 0; wq < 4; ++wq) {
      const int kb = kb0 + wq;
      v[wq] = 0ull;
      if (pos >= s && pos < e && kb <= klast && wq >= (tid >> 6)) v[wq] = mask[(size_t)(kb - (pos >> 6)) * n + pos];
    }
  };
  // Long segments (plain nms on tens of thousands of boxes) PULL: at the start of a step every thread folds the
  // four words of the step for some of the rows kept so far - independent, sector-sized loads, as many in
  // flight as there are threads x unroll - instead of pushing each step's kept rows into every later word.
  const bool pull = (klast - kfirst + 1) > 72;
  unsigned long long nxt[4];
  fetch(kfirst, nxt);
  int buf = 0;
  for (int kb0 = kfirst; kb0 <= klast; kb0 += 4, buf ^= 1) {
    unsigned long long (*dg)[4] = dgbuf[buf];
#pragma unroll
    for (int wq = 0; wq < 4; ++wq) dg[tid][wq] = nxt[wq];
    if (kb0 + 4 <= klast) fetch(kb0 + 4, nxt);         // in flight during the chain below
    if (pull && kb0 > kfirst) {
      unsigned long long acc[4] = {0ull, 0ull, 0ull, 0ull};
      const int r_end = 64 * kb0;
      const int nw = min(4, klast - kb0 + 1);       // words of this step that exist
      for (int r0 = s + tid; r0 < r_end; r0 += 8 * (int)blockDim.x) {
        // all loads are unconditional (suppressed rows are masked afterwards, rows past the end re-read the
        // last row), so the 8 flag loads and then the 32 word loads are in flight together
        unsigned long long keepm[8], v[8][4];
        int rr[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int r = r0 + u * (int)blockDim.x;
          rr[u] = min(r, r_end - 1);
          // kept bits of earlier steps live in shared memory (removed[] doubles as the bitmap once a block is decided)
          keepm[u] = (r < r_end && ((keptbits[(rr[u] >> 6) - kfirst] >> (rr[u] & 63)) & 1ull)) ? ~0ull : 0ull;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const unsigned long long* __restrict__ q = mask + (size_t)(kb0 - (rr[u] >> 6)) * n + rr[u];   // lanes = consecutive rows
#pragma unroll
          for (int wq = 0; wq < 4; ++wq) v[u][wq] = wq < nw ? q[(size_t)wq * n] : 0ull;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u)
#pragma unroll
          for (int wq = 0; wq < 4; ++wq) acc[wq] |= v[u][wq] & keepm[u];
      }
#pragma unroll
      for (int wq = 0; wq < 4; ++wq) {
        const unsigned int lo32 = __reduce_or_sync(0xffffffffu, (unsigned int)acc[wq]);
        const unsigned int hi32 = __reduce_or_sync(0xffffffffu, (unsigned int)(acc[wq] >> 32));
        if (lane == 0) atomicOr(&removed[kb0 - kfirst + wq], ((unsigned long long)hi32 << 32) | lo32);
      }
    }
    __syncthreads();
    if (warp == 0) {
      // Every lane runs the same chain on the block's diagonal words, which are pulled into registers first so
      // that no load sits between two decisions; then the lanes fold the kept rows' words of the later blocks.
      unsigned long long rem[4];
#pragma unroll
      for (int g = 0; g < 4; ++g) rem[g] = removed[kb0 - kfirst + g];
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const int base = 64 * (kb0 + g);
        unsigned long long kept = 0ull;
        if (base < e) {
          unsigned long long inseg = ~0ull;       // positions of this block inside [s, e)
          if (s > base) inseg &= ~0ull << (s - base);
          if (e - base < 64) inseg &= ~0ull >> (64 - (e - base));
          unsigned long long rg = rem[g] | ~inseg;
#pragma unroll
          for (int h0 = 0; h0 < 64; h0 += 32) {
            unsigned long long d[32];
#pragma unroll
            for (int b = 0; b < 32; ++b) d[b] = dg[g * 64 + h0 + b][g];
#pragma unroll
            for (int b = 0; b < 32; ++b)
              if (!((rg >> (h0 + b)) & 1ull)) { kept |= 1ull << (h0 + b); rg |= d[b]; }
          }
#pragma unroll
          for (int w2 = g + 1; w2 < 4; ++w2) {
            unsigned long long acc = 0ull;
            if ((kept >> lane) & 1ull) acc |= dg[g * 64 + lane][w2];
            if ((kept >> (lane + 32)) & 1ull) acc |= dg[g * 64 + 32 + lane][w2];
            const unsigned int lo32 = __reduce_or_sync(0xffffffffu, (unsigned int)acc);
            const unsigned int hi32 = __reduce_or_sync(0xffffffffu, (unsigned int)(acc >> 32));
            rem[w2] |= ((unsigned long long)hi32 << 32) | lo32;
          }
        }
        if (lane == 0) { keptw[g] = kept; if (kb0 + g <= klast) keptbits[kb0 - kfirst + g] = kept; }
      }
    }
    __syncthreads();
    {
      const int pos = 64 * kb0 + tid;
      if (pos >= s && pos < e) suppressed[pos] = ((keptw[tid >> 6] >> (tid & 63)) & 1ull) ? 0 : 1;
    }
    if (!pull) {   // push: warp j folds this step's kept rows into removed-word j (pull mode: later steps fetch what they need)
      for (int j = kb0 + 4 + warp; j <= klast; j += (int)(blockDim.x >> 5)) {
        unsigned long long acc = 0ull;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const unsigned long long kw = keptw[g];
          const int blk = kb0 + g;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int b = lane + 32 * hh;
            if ((kw >> b) & 1ull) acc |= mask[(size_t)(j - blk) * n + (64 * blk + b)];
          }
        }
        const unsigned int lo32 = __reduce_or_sync(0xffffffffu, (unsigned int)acc);
        const unsigned int hi32 = __reduce_or_sync(0xffffffffu, (unsigned int)(acc >> 32));
        if (lane == 0) removed[j - kfirst] |= ((unsigned long long)hi32 << 32) | lo32;
      }
    }
    __syncthreads();
  }
}

constexpr int kScanThreads = 256;
__global__ void __launch_bounds__(kScanThreads, 1)
bnms_scan_kernel(const unsigned long long* __restrict__ mask, int wpr, int max_len, const int* __restrict__ seg_start,
                 const int* __restrict__ num_seg_ptr, int n_total, uint8_t* __restrict__ suppressed) {
  extern __shared__ unsigned long long sc_removed[];          // 2 (wpr + 4) words: removed bits, kept bits
  __shared__ unsigned long long sc_dg[2][256][4], sc_keptw[4];
  const int nseg = seg_start ? *num_seg_ptr : 1;
  for (int seg = blockIdx.x; seg < nseg; seg += gridDim.x) {
    const int s = seg_start ? seg_start[seg] : 0;
    const int e = (seg_start && seg + 1 < nseg) ? seg_start[seg + 1] : n_total;
    if (e - s > 0 && e - s <= max_len) segment_scan(mask, wpr, n_total, s, e, suppressed, sc_removed, sc_dg, sc_keptw);
  }
}

// One CTA per segment; see file header.  `suppressed` (zero on entry) is indexed by
// position in the sorted order; on exit suppressed[p] == 0  <=>  box p is kept.
template <typename Box>
__global__ void __launch_bounds__(kSegThreads, 1)
nms_segment_kernel(const Box* __restrict__ boxes, const int* __restrict__ seg_start,
                   const int* __restrict__ num_seg_ptr, int n_total, IouParams prm,
                   uint8_t* __restrict__ suppressed, int min_len) {
  using S = typename ScalarOf<Box>::type;
  __shared__ Box sb[64];
  __shared__ S sarea[64];
  __shared__ unsigned long long diag[64];
  __shared__ unsigned long long s_removed, s_kept;
  __shared__ unsigned int s_rm[2];
  __shared__ Box ksb[64];           // the boxes kept in the current block, compacted
  __shared__ S karea[64];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nseg = num_seg_ptr ? *num_seg_ptr : 1;
  for (int seg = blockIdx.x; seg < nseg; seg += gridDim.x) {
    const int s = seg_start ? seg_start[seg] : 0;
    const int e = seg_start ? ((seg + 1 < nseg) ? seg_start[seg + 1] : n_total) : n_total;
    const int n = e - s;
    if (n <= min_len) continue;                     // short segments: bnms_mask_kernel + bnms_scan_kernel
    for (int b0 = 0; b0 < n; b0 += 64) {
      const int nb = min(64, n - b0);
      // stage the block's boxes; collect which of them are already suppressed
      bool sup = true;
      if (tid < 64) {
        Box b = zero_box((Box*)nullptr);
        if (tid < nb) { b = boxes[s + b0 + tid]; sup = suppressed[s + b0 + tid] != 0; }
        sb[tid] = b;
        sarea[tid] = box_area(b, prm);
        const unsigned int m = __ballot_sync(0xffffffffu, sup);
        if (lane == 0) s_rm[warp] = m;
      }
      __syncthreads();
      // (1) diagonal 64x64 bit-matrix: warp w owns rows 2w, 2w+1; lane owns cols lane, lane+32
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int row = warp * 2 + rr;
        const Box a = sb[row];
        const S aa = sarea[row];
        const bool p0 = (lane > row) && (lane < nb) && (row < nb) && iou_gt(a, aa, sb[lane], prm);
        const bool p1 = (lane + 32 > row) && (lane + 32 < nb) && (row < nb) && iou_gt(a, aa, sb[lane + 32], prm);
        const unsigned int lo = __ballot_sync(0xffffffffu, p0);
        const unsigned int hi = __ballot_sync(0xffffffffu, p1);
        if (lane == 0) diag[row] = ((unsigned long long)hi << 32) | lo;
      }
      __syncthreads();
      // (2) greedy chain inside the block (nms_kernel.cu:121-146 order), on registers
      if (tid == 0) {
        unsigned long long removed = ((unsigned long long)s_rm[1] << 32) | s_rm[0];
        unsigned long long kept = 0;
#pragma unroll 8
        for (int i = 0; i < 64; ++i) {
          const unsigned long long d = diag[i];
          if (!((removed >> i) & 1ull)) { kept |= 1ull << i; removed |= d; }
        }
        s_kept = kept;
        s_removed = removed;
      }
      __syncthreads();
      const unsigned long long kept = s_kept;
      const int nkept = __popcll(kept);
      if (tid < 64) {
        if (tid < nb) suppressed[s + b0 + tid] = ((kept >> tid) & 1ull) ? 0 : 1;
        if ((kept >> tid) & 1ull) {
          const int pos = __popcll(kept & ((1ull << tid) - 1ull));
          ksb[pos] = sb[tid];
          karea[pos] = sarea[tid];
        }
      }
      __syncthreads();
      // (3) later boxes vs. the boxes kept in this block.  Two threads per candidate (even / odd
      // entries of the compacted kept list), four independent IoU tests per trip.
      if (nkept > 0 && b0 + 64 < n) {
        const int half = tid & 1;
        for (int j = b0 + 64 + (tid >> 1); j < n; j += kSegThreads / 2) {
          if (suppressed[s + j]) continue;
          const Box bj = boxes[s + j];
          bool dead = false;
          for (int t = half; t < nkept && !dead; t += 8) {
            bool d[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const int tt = min(t + 2 * u, nkept - 1);         // clamped repeats are harmless
              d[u] = iou_gt(ksb[tt], karea[tt], bj, prm);
            }
            dead = d[0] | d[1] | d[2] | d[3];
          }
          if (dead) suppressed[s + j] = 1;
        }
      }
      __syncthreads();
    }
  }
}

struct NotZero {
  __host__ __device__ __forceinline__ bool operator()(const uint8_t v) const { return v == 0; }
};
struct ToI64 {
  __host__ __device__ __forceinline__ int64_t operator()(const int v) const { return (int64_t)v; }
};

size_t cub_temp_bytes(int64_t n) {
  // upper bound over every cub call below (queried with null storage); memoised per thread
  static thread_local int64_t cached_n = -1;
  static thread_local size_t cached_bytes = 0;
  if (n == cached_n) return cached_bytes;
  size_t mx = 0, b = 0;
  const int ni = (int)n;
  cub::DeviceRadixSort::SortPairsDescending(nullptr, b, (const float*)nullptr, (float*)nullptr, (const int*)nullptr, (int*)nullptr, ni);
  mx = b > mx ? b : mx;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const int64_t*)nullptr, (int64_t*)nullptr, (const int*)nullptr, (int*)nullptr, ni);
  mx = b > mx ? b : mx;
  cub::DeviceSelect::Flagged(nullptr, b, (const int*)nullptr, (const uint8_t*)nullptr, (int*)nullptr, (int*)nullptr, ni);
  mx = b > mx ? b : mx;
  cub::DeviceReduce::Max(nullptr, b, (const float*)nullptr, (float*)nullptr, ni * 4);
  mx = b > mx ? b : mx;
  cub::DeviceRadixSort::SortPairsDescending(nullptr, b, (const double*)nullptr, (double*)nullptr, (const int*)nullptr, (int*)nullptr, ni);
  mx = b > mx ? b : mx;
  cub::DeviceReduce::Max(nullptr, b, (const double*)nullptr, (double*)nullptr, ni * 4);
  mx = b > mx ? b : mx;
  cached_n = n;
  cached_bytes = mx + 4096;
  return cached_bytes;
}

// Workspaces are carved for the widest scalar (double): one size query serves both dtypes.
struct NmsWs {
  int* iota; int* order; void* scores_sorted; void* boxes_sorted; uint8_t* suppressed;
  unsigned long long* mask; void* cub_temp; size_t cub_bytes; size_t total;
};

// with_mask = false leaves out the n x n/64-bit IoU matrix (1.25 GB at n = 100 000): run_single_segment then takes
// the sequential chain kernel.
NmsWs carve_nms(void* base, int64_t n, bool with_mask = true) {
  Carver c(base);
  NmsWs w;
  w.iota = c.take<int>(n);
  w.order = c.take<int>(n);
  w.scores_sorted = c.take<double>(n);
  w.boxes_sorted = c.take<double4a>(n);
  w.suppressed = c.take<uint8_t>(n);
  w.cub_bytes = cub_temp_bytes(n);
  w.cub_temp = c.take<char>(w.cub_bytes);
  const int64_t cb = ceil_div64(n, 64);
  w.mask = with_mask ? c.take<unsigned long long>((size_t)n * cb) : nullptr;
  w.total = c.off;
  return w;
}

// Sorted-order suppression for ONE segment of n boxes (boxes_sorted), result in suppressed[].
template <typename Box>
int run_single_segment(const Box* boxes_sorted, int64_t n, IouParams prm, uint8_t* suppressed,
                       unsigned long long* mask, cudaStream_t st) {
  const char* force = env_override(ENV_NMS_PATH);      // "chain" | "mask" (testing / profiling)
  bool use_mask = true;            // measured faster at every size (0.09 vs 0.20 ms at n = 1000; 0.15 vs 0.87 ms at n = 3000)
  if (force && force[0] == 'c') use_mask = false;
  if (force && force[0] == 'm') use_mask = true;
  if (!use_mask || mask == nullptr) {
    VB200_CUDA_TRY(cudaMemsetAsync(suppressed, 0, (size_t)n, st));
    nms_segment_kernel<Box><<<1, kSegThreads, 0, st>>>(boxes_sorted, nullptr, nullptr, (int)n, prm, suppressed, 0);
    return check_launch("nms_segment_kernel");
  }
  // IoU bit matrix on every SM (row pitch = the number of 64-position blocks), then one CTA walks the chain
  const int cb = (int)ceil_div64(n, 64);
  if (prm.semantics == VB200_NMS_CUDA)
    bnms_mask_kernel<Box, VB200_NMS_CUDA><<<cb, kMaskWarps * 32, 0, st>>>(boxes_sorted, nullptr, nullptr, (int)n, cb, (int)n, prm, mask);
  else
    bnms_mask_kernel<Box, VB200_NMS_CPU><<<cb, kMaskWarps * 32, 0, st>>>(boxes_sorted, nullptr, nullptr, (int)n, cb, (int)n, prm, mask);
  int rc = check_launch("bnms_mask_kernel");
  if (rc) return rc;
  const size_t smem = 2 * (size_t)(cb + 4) * sizeof(unsigned long long);
  if (smem > 24 * 1024)
    VB200_CUDA_TRY(ensure_dyn_smem<bnms_scan_kernel>(smem));
  bnms_scan_kernel<<<1, kScanThreads, smem, st>>>(mask, cb, (int)n, nullptr, nullptr, (int)n, suppressed);
  return check_launch("bnms_scan_kernel");
}

template <typename S>
int nms_core(const typename BoxOf<S>::type* boxes, const S* scores, int64_t n, IouParams prm, void* workspace,
             size_t workspace_bytes, int64_t* keep_out, int64_t* num_keep_out, cudaStream_t st, bool with_mask = true) {
  using Box = typename BoxOf<S>::type;
  NmsWs w = carve_nms(workspace, n, with_mask);
  if (workspace_bytes < w.total) { set_error("nms: workspace too small (%zu < %zu)", workspace_bytes, w.total); return VB200_EWORKSPACE; }
  const int ni = (int)n, blk = 256, grd = ceil_div(ni, blk);
  iota_kernel<<<grd, blk, 0, st>>>(w.iota, ni);
  int rc = check_launch("iota_kernel");
  if (rc) return rc;
  size_t tb = w.cub_bytes;
  VB200_CUDA_TRY(cub::DeviceRadixSort::SortPairsDescending(w.cub_temp, tb, scores, (S*)w.scores_sorted, w.iota, w.order, ni, 0,
                                                           (int)sizeof(S) * 8, st));
  g_launch_count.fetch_add(3, std::memory_order_relaxed);
  gather_boxes_kernel<Box><<<grd, blk, 0, st>>>(boxes, w.order, (Box*)w.boxes_sorted, ni);
  rc = check_launch("gather_boxes_kernel");
  if (rc) return rc;
  rc = run_single_segment<Box>((const Box*)w.boxes_sorted, n, prm, w.suppressed, w.mask, st);
  if (rc) return rc;
  cub::TransformInputIterator<int64_t, ToI64, const int*> in_it(w.order, ToI64());
  cub::TransformInputIterator<bool, NotZero, const uint8_t*> flag_it(w.suppressed, NotZero());
  tb = w.cub_bytes;
  VB200_CUDA_TRY(cub::DeviceSelect::Flagged(w.cub_temp, tb, in_it, flag_it, keep_out, num_keep_out, ni, st));
  g_launch_count.fetch_add(2, std::memory_order_relaxed);
  return 0;
}

}  // namespace
}  // namespace vb200

using namespace vb200;

namespace {
// fp16 inputs: the exact fp32 widenings of boxes and scores live in front of the regular workspace
struct WideWs { float4* boxes; float* scores; size_t total; };
WideWs carve_wide(void* base, int64_t n) {
  Carver c(base);
  WideWs w;
  w.boxes = c.take<float4>(n);
  w.scores = c.take<float>(n);
  w.total = c.off;
  return w;
}
int widen_half(const void* boxes, const void* scores, const WideWs& w, int64_t n, cudaStream_t st) {
  widen_half_kernel<<<ceil_div((int)n, 256), 256, 0, st>>>((const uint2*)boxes, (const __half*)scores, w.boxes, w.scores, (int)n);
  return check_launch("widen_half_kernel");
}
}  // namespace

extern "C" size_t vb200_nms_workspace_bytes(int64_t n) {
  if (n <= 0) return 0;
  return carve_nms(nullptr, n).total + carve_wide(nullptr, n).total;
}

extern "C" int vb200_nms(const void* boxes, const void* scores, int dtype, int64_t n, double iou_threshold,
                         int semantics, void* workspace, size_t workspace_bytes, int64_t* keep_out,
                         int64_t* num_keep_out, vb200_stream stream) {
  VB200_REQUIRE(dtype == VB200_F32 || dtype == VB200_F64 || dtype == VB200_F16,
                "nms: boxes must be float32, float64 or float16 (got dtype %d)", dtype);
  VB200_REQUIRE(n >= 0 && n < (1ll << 31), "nms: bad box count");
  VB200_REQUIRE(semantics == VB200_NMS_CPU || semantics == VB200_NMS_CUDA, "nms: bad semantics selector");
  VB200_REQUIRE(num_keep_out != nullptr, "nms: null num_keep_out");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) { VB200_CUDA_TRY(cudaMemsetAsync(num_keep_out, 0, sizeof(int64_t), st)); return 0; }
  VB200_REQUIRE(boxes && scores && keep_out && workspace, "nms: null pointer");
  VB200_REQUIRE(((uintptr_t)boxes % (dtype == VB200_F16 ? 8 : 16)) == 0, "nms: boxes must be aligned to one box (4 scalars)");
  IouParams prm = make_iou_params(iou_threshold, semantics);
  if (dtype == VB200_F16) {
    // the reference has a Half kernel on CUDA only (the CPU kernel raises), so there is one fp16 arithmetic
    VB200_REQUIRE(semantics == VB200_NMS_CUDA, "nms: float16 boxes exist only with VB200_NMS_CUDA semantics");
    const WideWs ww = carve_wide(workspace, n);
    if (workspace_bytes < ww.total) { set_error("nms: workspace too small"); return VB200_EWORKSPACE; }
    const int rc = widen_half(boxes, scores, ww, n, st);
    if (rc) return rc;
    prm.half_mode = 1;
    return nms_core<float>(ww.boxes, ww.scores, n, prm, (char*)workspace + ww.total, workspace_bytes - ww.total, keep_out,
                           num_keep_out, st);
  }
  if (dtype == VB200_F64)
    return nms_core<double>((const double4a*)boxes, (const double*)scores, n, prm, workspace, workspace_bytes, keep_out,
                            num_keep_out, st);
  return nms_core<float>((const float4*)boxes, (const float*)scores, n, prm, workspace, workspace_bytes, keep_out,
                         num_keep_out, st);
}

namespace vb200 {
namespace {
struct BnmsWs {
  int* iota; int* order; void* scores_sorted; int64_t* cls_keys; int64_t* cls_sorted; int* rank_cm;
  void* boxes_cm; uint8_t* seg_flag; int* seg_start; int* num_seg; uint8_t* suppressed;
  uint8_t* keep_by_rank; void* max_coord; void* shifted; void* cub_temp; size_t cub_bytes;
  unsigned long long* mask; size_t nms_off; size_t total;
};
// The reference picks the coordinate trick only for numel <= 100 000 (boxes.py:86); a caller that forces it on a larger
// problem gets the sequential kernel instead of a gigabyte-sized bit matrix in every batched_nms workspace.
inline bool bnms_trick_with_mask(int64_t n) { return 4 * n <= 100000; }
BnmsWs carve_bnms(void* base, int64_t n) {
  Carver c(base);
  BnmsWs w;
  w.iota = c.take<int>(n);
  w.order = c.take<int>(n);
  w.scores_sorted = c.take<double>(n);
  w.cls_keys = c.take<int64_t>(n);
  w.cls_sorted = c.take<int64_t>(n);
  w.rank_cm = c.take<int>(n);
  w.boxes_cm = c.take<double4a>(n);
  w.seg_flag = c.take<uint8_t>(n);
  w.seg_start = c.take<int>(n + 1);
  w.num_seg = c.take<int>(64);
  w.suppressed = c.take<uint8_t>(n);
  w.keep_by_rank = c.take<uint8_t>(n);
  w.max_coord = c.take<double>(64);
  w.shifted = c.take<double4a>(n);
  w.cub_bytes = cub_temp_bytes(n);
  w.cub_temp = c.take<char>(w.cub_bytes);
  w.mask = c.take<unsigned long long>((size_t)n * kBnmsWpr);
  w.nms_off = c.off;                       // trick strategy reuses the plain-nms pipeline
  c.off += carve_nms(nullptr, n, bnms_trick_with_mask(n)).total;
  w.total = c.off;
  return w;
}

__global__ void scatter_keep_kernel(const uint8_t* __restrict__ suppressed, const int* __restrict__ rank_cm,
                                    uint8_t* __restrict__ keep_by_rank, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keep_by_rank[rank_cm[i]] = suppressed[i] ? 0 : 1;
}
}  // namespace
}  // namespace vb200

namespace vb200 {
namespace {
template <typename S>
int bnms_core(const void* boxes, const void* scores, const int64_t* idxs, int64_t n, double iou_threshold, int semantics,
              int strategy, bool wide_keys, void* workspace, size_t workspace_bytes, int64_t* keep_out,
              int64_t* num_keep_out, cudaStream_t st, int half_mode = 0) {
  using Box = typename BoxOf<S>::type;
  BnmsWs w = carve_bnms(workspace, n);
  if (workspace_bytes < w.total) { set_error("batched_nms: workspace too small (%zu < %zu)", workspace_bytes, w.total); return VB200_EWORKSPACE; }
  IouParams prm = make_iou_params(iou_threshold, semantics);
  prm.half_mode = half_mode;
  const int ni = (int)n, blk = 256, grd = ceil_div(ni, blk);
  if (strategy == VB200_BNMS_AUTO) strategy = (4 * n > 100000) ? VB200_BNMS_VANILLA : VB200_BNMS_TRICK;   // boxes.py:86

  if (strategy == VB200_BNMS_TRICK) {
    size_t tb = w.cub_bytes;
    VB200_CUDA_TRY(cub::DeviceReduce::Max(w.cub_temp, tb, (const S*)boxes, (S*)w.max_coord, ni * 4, st));
    g_launch_count.fetch_add(2, std::memory_order_relaxed);
    shift_boxes_kernel<Box><<<grd, blk, 0, st>>>((const Box*)boxes, idxs, (const S*)w.max_coord, (Box*)w.shifted, ni, half_mode);
    int rc = check_launch("shift_boxes_kernel");
    if (rc) return rc;
    return nms_core<S>((const Box*)w.shifted, (const S*)scores, n, prm, (char*)workspace + w.nms_off,
                       workspace_bytes - w.nms_off, keep_out, num_keep_out, st, bnms_trick_with_mask(n));
  }

  // ---- vanilla semantics, fused ------------------------------------------
  iota_kernel<<<grd, blk, 0, st>>>(w.iota, ni);
  int rc = check_launch("iota_kernel");
  if (rc) return rc;
  size_t tb = w.cub_bytes;
  VB200_CUDA_TRY(cub::DeviceRadixSort::SortPairsDescending(w.cub_temp, tb, (const S*)scores, (S*)w.scores_sorted, w.iota, w.order, ni, 0, (int)sizeof(S) * 8, st));
  g_launch_count.fetch_add(3, std::memory_order_relaxed);
  // num_seg[1] doubles as the "class id outside [0, 2^16)" flag of the narrow-key fast path
  VB200_CUDA_TRY(cudaMemsetAsync(w.num_seg, 0, 2 * sizeof(int), st));
  gather_class_kernel<<<grd, blk, 0, st>>>(idxs, w.order, w.cls_keys, ni, w.num_seg + 1);
  rc = check_launch("gather_class_kernel");
  if (rc) return rc;
  tb = w.cub_bytes;
  // Speculate that class ids fit 16 bits (2 radix passes instead of 8); the flag is checked on the
  // device after the pipeline and turns the result into "-1: call again with wide keys".
  VB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(w.cub_temp, tb, w.cls_keys, w.cls_sorted, w.iota, w.rank_cm, ni, 0,
                                                 wide_keys ? 64 : 16, st));
  g_launch_count.fetch_add(wide_keys ? 9 : 3, std::memory_order_relaxed);
  gather_boxes_cm_kernel<Box><<<grd, blk, 0, st>>>((const Box*)boxes, w.order, w.rank_cm, w.cls_sorted, (Box*)w.boxes_cm, w.seg_flag, ni);
  rc = check_launch("gather_boxes_cm_kernel");
  if (rc) return rc;
  tb = w.cub_bytes;
  VB200_CUDA_TRY(cub::DeviceSelect::Flagged(w.cub_temp, tb, w.iota, w.seg_flag, w.seg_start, w.num_seg, ni, st));
  g_launch_count.fetch_add(2, std::memory_order_relaxed);
  VB200_CUDA_TRY(cudaMemsetAsync(w.suppressed, 0, (size_t)n, st));
  const char* mp = env_override(ENV_BNMS_PATH);       // "chain": per-class sequential kernel only (testing / profiling)
  const bool use_mask = !(mp && mp[0] == 'c');
  if (use_mask) {
    if (semantics == VB200_NMS_CUDA)
      bnms_mask_kernel<Box, VB200_NMS_CUDA><<<ceil_div(ni, 64), kMaskWarps * 32, 0, st>>>(
          (const Box*)w.boxes_cm, w.seg_start, w.num_seg, ni, kBnmsWpr, kBnmsMaxLen, prm, w.mask);
    else
      bnms_mask_kernel<Box, VB200_NMS_CPU><<<ceil_div(ni, 64), kMaskWarps * 32, 0, st>>>(
          (const Box*)w.boxes_cm, w.seg_start, w.num_seg, ni, kBnmsWpr, kBnmsMaxLen, prm, w.mask);
    rc = check_launch("bnms_mask_kernel");
    if (rc) return rc;
  }
  const int grid = sm_count() * 1;
  if (use_mask) {
    bnms_scan_kernel<<<grid, kScanThreads, 2 * (kBnmsWpr + 4) * 8, st>>>(w.mask, kBnmsWpr, kBnmsMaxLen, w.seg_start, w.num_seg, ni, w.suppressed);
    rc = check_launch("bnms_scan_kernel");
    if (rc) return rc;
  }
  nms_segment_kernel<Box><<<grid, kSegThreads, 0, st>>>((const Box*)w.boxes_cm, w.seg_start, w.num_seg, ni, prm, w.suppressed,
                                                          use_mask ? kBnmsMaxLen : 0);
  rc = check_launch("nms_segment_kernel");
  if (rc) return rc;
  scatter_keep_kernel<<<grd, blk, 0, st>>>(w.suppressed, w.rank_cm, w.keep_by_rank, ni);
  rc = check_launch("scatter_keep_kernel");
  if (rc) return rc;
  cub::TransformInputIterator<int64_t, ToI64, const int*> in_it(w.order, ToI64());
  tb = w.cub_bytes;
  VB200_CUDA_TRY(cub::DeviceSelect::Flagged(w.cub_temp, tb, in_it, w.keep_by_rank, keep_out, num_keep_out, ni, st));
  g_launch_count.fetch_add(2, std::memory_order_relaxed);
  if (!wide_keys) {
    poison_count_kernel<<<1, 1, 0, st>>>(w.num_seg + 1, num_keep_out);
    rc = check_launch("poison_count_kernel");
    if (rc) return rc;
  }
  return 0;
}
}  // namespace
}  // namespace vb200

extern "C" size_t vb200_batched_nms_workspace_bytes(int64_t n) {
  if (n <= 0) return 0;
  return carve_bnms(nullptr, n).total + carve_wide(nullptr, n).total;
}

namespace {
int bnms_dispatch(const void* boxes, const void* scores, const int64_t* idxs, int dtype, int64_t n, double iou_threshold, int semantics,
                  int strategy, bool wide_keys, void* workspace, size_t workspace_bytes, int64_t* keep_out, int64_t* num_keep_out,
                  cudaStream_t st) {
  if (dtype == VB200_F16) {
    const WideWs ww = carve_wide(workspace, n);
    if (workspace_bytes < ww.total) { set_error("batched_nms: workspace too small"); return VB200_EWORKSPACE; }
    const int rc = widen_half(boxes, scores, ww, n, st);
    if (rc) return rc;
    return bnms_core<float>(ww.boxes, ww.scores, idxs, n, iou_threshold, semantics, strategy, wide_keys, (char*)workspace + ww.total,
                            workspace_bytes - ww.total, keep_out, num_keep_out, st, 1);
  }
  if (dtype == VB200_F64)
    return bnms_core<double>(boxes, scores, idxs, n, iou_threshold, semantics, strategy, wide_keys, workspace, workspace_bytes,
                             keep_out, num_keep_out, st);
  return bnms_core<float>(boxes, scores, idxs, n, iou_threshold, semantics, strategy, wide_keys, workspace, workspace_bytes,
                          keep_out, num_keep_out, st);
}

// The pipeline is ~25 launches (five of them CUB dispatches, each with its own attribute queries) for ~230 us of device
// work: launch-bound whenever the host is slower than usual (several ranks per host).  A call whose arguments - every
// pointer and size - repeat an earlier call's is replayed as a CUDA graph: the second identical call captures the pipeline
// (stream capture of exactly the launches above), later ones are one cudaGraphLaunch.  Contents may differ between calls,
// only the addresses must repeat - which is what a serving loop with a caching allocator produces.  VB200_BNMS_GRAPH=0 turns
// the cache off; a stream that is already being captured by the caller just records the plain launches.
struct BnmsKey {
  const void* boxes; const void* scores; const void* idxs; void* ws; void* keep; void* count;
  int64_t n; size_t wsb; double thr; int dtype, semantics, strategy, wide, device; cudaStream_t st; int env_gen;
  bool operator==(const BnmsKey& o) const {
    return boxes == o.boxes && scores == o.scores && idxs == o.idxs && ws == o.ws && keep == o.keep && count == o.count && n == o.n &&
           wsb == o.wsb && thr == o.thr && dtype == o.dtype && semantics == o.semantics && strategy == o.strategy && wide == o.wide &&
           device == o.device && st == o.st && env_gen == o.env_gen;
  }
};
struct BnmsGraph { BnmsKey key; cudaGraphExec_t exec; int hits; uint64_t stamp; };
constexpr int kBnmsGraphSlots = 16;
BnmsGraph g_bnms_graphs[kBnmsGraphSlots];
int g_bnms_used = 0;
uint64_t g_bnms_clock = 0;
std::mutex g_bnms_mu;
}  // namespace

extern "C" int vb200_batched_nms(const void* boxes, const void* scores, const int64_t* idxs, int dtype,
                                 int64_t n, double iou_threshold, int semantics, int strategy,
                                 void* workspace, size_t workspace_bytes, int64_t* keep_out,
                                 int64_t* num_keep_out, vb200_stream stream) {
  VB200_REQUIRE(dtype == VB200_F32 || dtype == VB200_F64 || dtype == VB200_F16,
                "batched_nms: boxes must be float32, float64 or float16 (got dtype %d)", dtype);
  VB200_REQUIRE(n >= 0 && n < (1ll << 31), "batched_nms: bad box count");
  VB200_REQUIRE(semantics == VB200_NMS_CPU || semantics == VB200_NMS_CUDA, "batched_nms: bad semantics selector");
  const bool wide_keys = (strategy & VB200_BNMS_WIDE_KEYS) != 0;
  strategy &= ~VB200_BNMS_WIDE_KEYS;
  VB200_REQUIRE(strategy >= VB200_BNMS_AUTO && strategy <= VB200_BNMS_TRICK, "batched_nms: bad strategy");
  VB200_REQUIRE(num_keep_out != nullptr, "batched_nms: null num_keep_out");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) { VB200_CUDA_TRY(cudaMemsetAsync(num_keep_out, 0, sizeof(int64_t), st)); return 0; }
  VB200_REQUIRE(boxes && scores && idxs && keep_out && workspace, "batched_nms: null pointer");
  VB200_REQUIRE(((uintptr_t)boxes % (dtype == VB200_F16 ? 8 : 16)) == 0, "batched_nms: boxes must be aligned to one box (4 scalars)");
  VB200_REQUIRE(dtype != VB200_F16 || semantics == VB200_NMS_CUDA, "batched_nms: float16 boxes exist only with VB200_NMS_CUDA semantics");

  const char* gsw = env_override(ENV_BNMS_GRAPH);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  bool use_graph = !(gsw && gsw[0] == '0') && n >= 4096 && cudaStreamIsCapturing(st, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone;
  if (!use_graph)
    return bnms_dispatch(boxes, scores, idxs, dtype, n, iou_threshold, semantics, strategy, wide_keys, workspace, workspace_bytes, keep_out,
                         num_keep_out, st);
  int dev = 0;
  cudaGetDevice(&dev);
  const BnmsKey key{boxes, scores, idxs, workspace, keep_out, num_keep_out, n, workspace_bytes, iou_threshold, dtype, semantics, strategy,
                    wide_keys ? 1 : 0, dev, st, env_generation()};
  std::lock_guard<std::mutex> lk(g_bnms_mu);
  BnmsGraph* slot = nullptr;
  for (int i = 0; i < g_bnms_used; ++i)
    if (g_bnms_graphs[i].key == key) { slot = &g_bnms_graphs[i]; break; }
  if (slot && slot->exec) {                       // replay
    slot->stamp = ++g_bnms_clock;
    VB200_CUDA_TRY(cudaGraphLaunch(slot->exec, st));
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    return 0;
  }
  if (!slot) {                                    // first sighting: run plainly, remember the arguments
    if (g_bnms_used < kBnmsGraphSlots) slot = &g_bnms_graphs[g_bnms_used++];
    else {
      slot = &g_bnms_graphs[0];
      for (int i = 1; i < kBnmsGraphSlots; ++i)
        if (g_bnms_graphs[i].stamp < slot->stamp) slot = &g_bnms_graphs[i];
      if (slot->exec) cudaGraphExecDestroy(slot->exec);
    }
    *slot = BnmsGraph{key, nullptr, 1, ++g_bnms_clock};
    return bnms_dispatch(boxes, scores, idxs, dtype, n, iou_threshold, semantics, strategy, wide_keys, workspace, workspace_bytes, keep_out,
                         num_keep_out, st);
  }
  // second identical call: capture the pipeline (on a private stream - the caller's may be the legacy default stream, which
  // cannot be captured; a graph does not remember the stream it was recorded on), instantiate, launch on the caller's stream
  slot->stamp = ++g_bnms_clock;
  cudaGraph_t graph = nullptr;
  static cudaStream_t cap_streams[64] = {nullptr};
  cudaStream_t& cs = cap_streams[dev < 0 || dev >= 64 ? 0 : dev];
  if (cs == nullptr && cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); cs = nullptr; }
  if (cs == nullptr || cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
    cudaGetLastError();
    slot->key.env_gen = -1;
    return bnms_dispatch(boxes, scores, idxs, dtype, n, iou_threshold, semantics, strategy, wide_keys, workspace, workspace_bytes, keep_out,
                         num_keep_out, st);
  }
  const uint64_t launches_before = g_launch_count.load();
  const int rc = bnms_dispatch(boxes, scores, idxs, dtype, n, iou_threshold, semantics, strategy, wide_keys, workspace, workspace_bytes, keep_out,
                               num_keep_out, cs);
  const cudaError_t ce = cudaStreamEndCapture(cs, &graph);
  g_launch_count.store(launches_before);          // the captured launches have not run yet
  if (rc != 0 || ce != cudaSuccess || graph == nullptr) {
    cudaGetLastError();
    if (graph) cudaGraphDestroy(graph);
    slot->hits = -1000000;                        // do not try again for these arguments
    slot->key.env_gen = -1;
    return bnms_dispatch(boxes, scores, idxs, dtype, n, iou_threshold, semantics, strategy, wide_keys, workspace, workspace_bytes, keep_out,
                         num_keep_out, st);
  }
  cudaGraphExec_t exec = nullptr;
  const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ie != cudaSuccess || exec == nullptr) {
    cudaGetLastError();
    slot->key.env_gen = -1;
    return bnms_dispatch(boxes, scores, idxs, dtype, n, iou_threshold, semantics, strategy, wide_keys, workspace, workspace_bytes, keep_out,
                         num_keep_out, st);
  }
  slot->exec = exec;
  VB200_CUDA_TRY(cudaGraphLaunch(exec, st));
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

// =====================================================================================================================
// Detection post-processing fused around batched_nms (SURVEY.md §8f3).
// Reference: torchvision/models/detection/roi_heads.py:700-737 (postprocess_detections, per image) and
// rpn.py:273-298 (filter_proposals, per image): clip_boxes_to_image -> score filter -> remove_small_boxes ->
// batched_nms -> keep[:top_k] -> index boxes / scores / labels.  The reference runs ~30 tiny tensor ops and 4-5 host
// synchronisations per image; here: one clip+filter kernel, one compaction, the fused batched_nms pipeline above and one
// gather - two synchronisations (candidate count: the reference's batched_nms strategy switch depends on it, boxes.py:86;
// output count).  Arithmetic: clamp / subtract / compare in fp32 exactly as the tensor ops do.
// =====================================================================================================================
namespace vb200 {
namespace {

__global__ void det_clip_filter_kernel(const float4* __restrict__ boxes, const float* __restrict__ scores, float4* __restrict__ clipped,
                                       uint8_t* __restrict__ flag, int n, float img_h, float img_w, float score_thresh,
                                       int score_inclusive, float min_size) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 b = __ldg(boxes + i);
  // boxes[..., 0::2].clamp(min=0, max=width), boxes[..., 1::2].clamp(min=0, max=height)  (ops/boxes.py clip_boxes_to_image)
  b.x = fminf(fmaxf(b.x, 0.f), img_w); b.z = fminf(fmaxf(b.z, 0.f), img_w);
  b.y = fminf(fmaxf(b.y, 0.f), img_h); b.w = fminf(fmaxf(b.w, 0.f), img_h);
  clipped[i] = b;
  const float s = scores[i];
  const bool score_ok = score_inclusive ? (s >= score_thresh) : (s > score_thresh);
  const bool size_ok = (sub_rn(b.z, b.x) >= min_size) && (sub_rn(b.w, b.y) >= min_size);     // remove_small_boxes
  flag[i] = (score_ok && size_ok) ? 1 : 0;
}

__global__ void det_gather_candidates_kernel(const float4* __restrict__ clipped, const float* __restrict__ scores,
                                             const int64_t* __restrict__ labels, const int* __restrict__ cand, const int* __restrict__ n_cand,
                                             float4* __restrict__ cb, float* __restrict__ cs, int64_t* __restrict__ cl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *n_cand) return;
  const int src = cand[i];
  cb[i] = clipped[src]; cs[i] = scores[src]; cl[i] = labels[src];
}

__global__ void det_gather_topk_kernel(const float4* __restrict__ cb, const float* __restrict__ cs, const int64_t* __restrict__ cl,
                                       const int64_t* __restrict__ keep, const int64_t* __restrict__ num_keep, int64_t topk,
                                       float4* __restrict__ boxes_out, float* __restrict__ scores_out, int64_t* __restrict__ labels_out,
                                       int64_t* __restrict__ count_out) {
  const int64_t k = min(*num_keep, topk);
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *count_out = k;
  if (i >= k) return;
  const int64_t src = keep[i];
  boxes_out[i] = cb[src]; scores_out[i] = cs[src]; labels_out[i] = cl[src];
}

struct DetWs { float4* clipped; uint8_t* flag; int* iota; int* cand; int* n_cand; float4* cb; float* cs; int64_t* cl; int64_t* keep;
               int64_t* num_keep; void* cub_temp; size_t cub_bytes; size_t bnms_off; size_t total; };
DetWs carve_det(void* base, int64_t n) {
  Carver c(base);
  DetWs w;
  w.clipped = c.take<float4>(n);
  w.flag = c.take<uint8_t>(n);
  w.iota = c.take<int>(n);
  w.cand = c.take<int>(n);
  w.n_cand = c.take<int>(64);
  w.cb = c.take<float4>(n);
  w.cs = c.take<float>(n);
  w.cl = c.take<int64_t>(n);
  w.keep = c.take<int64_t>(n);
  w.num_keep = c.take<int64_t>(32);
  w.cub_bytes = cub_temp_bytes(n);
  w.cub_temp = c.take<char>(w.cub_bytes);
  w.bnms_off = c.off;
  c.off += carve_bnms(nullptr, n).total;
  w.total = c.off;
  return w;
}
}  // namespace
}  // namespace vb200

extern "C" size_t vb200_detection_postprocess_workspace_bytes(int64_t n) {
  if (n <= 0) return 0;
  return carve_det(nullptr, n).total;
}

extern "C" int vb200_detection_postprocess(const void* boxes, const void* scores, const int64_t* labels, int dtype, int64_t n,
                                           double img_h, double img_w, double score_thresh, int score_inclusive, double min_size,
                                           double iou_threshold, int64_t topk, int semantics, void* workspace,
                                           size_t workspace_bytes, void* boxes_out, void* scores_out, int64_t* labels_out,
                                           int64_t* count_host, vb200_stream stream) {
  VB200_REQUIRE(dtype == VB200_F32, "detection_postprocess: float32 boxes only (got dtype %d)", dtype);
  VB200_REQUIRE(n >= 0 && n < (1ll << 31) && topk >= 0, "detection_postprocess: bad sizes");
  VB200_REQUIRE(count_host != nullptr, "detection_postprocess: null count_host");
  VB200_REQUIRE(semantics == VB200_NMS_CPU || semantics == VB200_NMS_CUDA, "detection_postprocess: bad semantics selector");
  *count_host = 0;
  if (n == 0 || topk == 0) return 0;
  VB200_REQUIRE(boxes && scores && labels && workspace && boxes_out && scores_out && labels_out, "detection_postprocess: null pointer");
  VB200_REQUIRE(((uintptr_t)boxes % 16) == 0 && ((uintptr_t)boxes_out % 16) == 0, "detection_postprocess: boxes must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const DetWs w = carve_det(workspace, n);
  if (workspace_bytes < w.total) { set_error("detection_postprocess: workspace too small (%zu < %zu)", workspace_bytes, w.total); return VB200_EWORKSPACE; }
  const int ni = (int)n, blk = 256, grd = ceil_div(ni, blk);
  det_clip_filter_kernel<<<grd, blk, 0, st>>>((const float4*)boxes, (const float*)scores, w.clipped, w.flag, ni, (float)img_h, (float)img_w,
                                             (float)score_thresh, score_inclusive, (float)min_size);
  int rc = check_launch("det_clip_filter_kernel");
  if (rc) return rc;
  iota_kernel<<<grd, blk, 0, st>>>(w.iota, ni);
  rc = check_launch("iota_kernel");
  if (rc) return rc;
  size_t tb = w.cub_bytes;
  VB200_CUDA_TRY(cub::DeviceSelect::Flagged(w.cub_temp, tb, w.iota, w.flag, w.cand, w.n_cand, ni, st));
  g_launch_count.fetch_add(2, std::memory_order_relaxed);
  det_gather_candidates_kernel<<<grd, blk, 0, st>>>(w.clipped, (const float*)scores, labels, w.cand, w.n_cand, w.cb, w.cs, w.cl);
  rc = check_launch("det_gather_candidates_kernel");
  if (rc) return rc;
  // the reference's strategy switch (boxes.py:86) looks at the number of candidates: one small read-back
  int n_cand = 0;
  VB200_CUDA_TRY(cudaMemcpyAsync(&n_cand, w.n_cand, sizeof(int), cudaMemcpyDeviceToHost, st));
  VB200_CUDA_TRY(cudaStreamSynchronize(st));
  if (n_cand == 0) return 0;
  for (int attempt = 0; attempt < 2; ++attempt) {
    rc = bnms_core<float>(w.cb, w.cs, w.cl, n_cand, iou_threshold, semantics, VB200_BNMS_AUTO, attempt == 1,
                          (char*)workspace + w.bnms_off, workspace_bytes - w.bnms_off, w.keep, w.num_keep, st);
    if (rc) return rc;
    const int64_t cap = topk < (int64_t)n_cand ? topk : (int64_t)n_cand;
    det_gather_topk_kernel<<<ceil_div((int)cap, blk), blk, 0, st>>>(w.cb, w.cs, w.cl, w.keep, w.num_keep, topk, (float4*)boxes_out,
                                                                   (float*)scores_out, labels_out, w.num_keep + 1);
    rc = check_launch("det_gather_topk_kernel");
    if (rc) return rc;
    int64_t hk[2] = {0, 0};
    VB200_CUDA_TRY(cudaMemcpyAsync(hk, w.num_keep, 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    VB200_CUDA_TRY(cudaStreamSynchronize(st));
    if (hk[0] >= 0) { *count_host = hk[1]; return 0; }        // -1: class ids outside [0, 65536) -> repeat with wide keys
  }
  set_error("detection_postprocess: internal error (negative kept count)");
  return VB200_EINVAL;
}

// =====================================================================================================================
// Single-stage detector post-processing: RetinaNet (retinanet.py:509-571), FCOS (fcos.py:489-556), SSD / SSDLite
// (ssd.py:414-463).  The reference loops over images and FPN levels (or foreground classes), writes a full score tensor
// and a full mask per level, compacts them and takes a topk - ~180 host synchronisations per SSD image.  Here every
// segment - an (image, level) slice of logits or an (image, class) column of probabilities - of every image is
// selected by one radix-select pipeline over the logits, read twice:
//   ss_hist_kernel     (read 1) per-segment histogram of the top 12 bits of key = bits(score) - bits(next float above
//                      the threshold).  Scores lie in [0, 1], so the key orders them and spans exactly the passing range
//                      (threshold, 1]: at a threshold of 0.05 the 4096 bins cover 2^14 ulps each (the top bits of the raw
//                      pattern would put all of (0.05, 1] into 37 bins);
//   ss_bound_kernel    boundary bucket B of each segment: fewer than k items lie above it, at least k at or above it;
//   ss_collect_kernel  (read 2) items above B are in the result; items in B are kept as (key, reversed index) pairs;
//   ss_final_kernel    one CTA per segment sorts the <= 4096 pairs (their significant bits only) by (score desc,
//                      index asc) and keeps the first k.
//                      When bucket B alone holds more items than fit, this CTA narrows it 12 bits at a time by
//                      re-reading its segment (the pairs are unique, so this ends) - only for such degenerate segments;
//   ss_decode_kernel   decode + clip of the selected items into each image's candidate list, in the reference's order.
// The per-image tail is bnms_core + det_gather_topk_kernel above; one concatenation kernel packs the images' results.
// Host synchronisations: two per call (candidate counts of all images, kept counts of all images).
// =====================================================================================================================
namespace vb200 {
namespace {

constexpr int kSelThreads = 256;
constexpr int kSelTile = 8192;                  // elements of one segment per CTA of the two passes over the logits
constexpr int kSelBits = 12;
constexpr int kSelBins = 1 << kSelBits;
constexpr int kSelSortThreads = 512, kSelSortItems = 8;
constexpr int kSelSortCap = kSelSortThreads * kSelSortItems;     // pairs sorted by one CTA
static_assert(2 * VB200_SS_MAX_TOPK <= kSelSortCap, "the boundary list needs at least as much room as the top-k");

struct SsSeg {                 // one segment
  const float* logit;          // element i: logit[(i / C) * lstride + i % C] (RetinaNet, FCOS), logit[i * lstride] (SSD)
  const float* ctr;            // FCOS: ctrness of anchor row a at ctr[a * cstride]
  const float* reg;            // regression row a at reg[a * rstride .. + 3]
  const float* anc;            // anchor row a at anc[a * astride .. + 3]
  int64_t n, lstride, cstride, rstride, astride;
  int label;                   // SSD: the class of this column
  float img_h, img_w;
};

struct SsParams {
  int kind, C;
  float thr;                   // float(score_thresh): the reference compares `scores > score_thresh` in fp32
  uint32_t base;               // bit pattern of the smallest passing score: key = bits(score) - base
  int shift0;                  // first digit = key >> shift0
  int ib;                      // pair = key << ib | (imask - index): ib bits hold any index of the largest segment
  unsigned long long imask;
  int sort_bits;               // significant bits of a pair
  int k, cap, spi, nmax;       // per-segment top-k, boundary-list capacity, segments per image, candidates per image
  float inv_w[4], clip;        // 1.0f / weight (torch divides a tensor by a Python float as a multiply by its reciprocal)
};

__device__ __forceinline__ float ss_sigmoid(float x) { return div_rn(1.f, add_rn(1.f, expf(-x))); }   // torch.sigmoid (fp32)

// Sigmoid, its square root and softmax probabilities lie in [+0, 1]; the clamp (NaN kept) only guarantees that every key
// of a passing score is at most bits(1.0f) - base, whatever the input holds.
__device__ __forceinline__ float ss_unit(float s) { return s > 1.f ? 1.f : (s <= 0.f ? 0.f : s); }

// Calls f(i, score) for i = i0 + t, i0 + t + stride, ... < i1 of segment g; four loads are issued before any use.
template <typename F>
__device__ __forceinline__ void ss_walk(const SsSeg& g, const SsParams& p, int64_t i0, int64_t i1, int t, int stride, F&& f) {
  constexpr int U = 4;
  if (p.kind == VB200_SS_SSD) {
    for (int64_t ib = i0 + t; ib < i1; ib += (int64_t)U * stride) {
      float x[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = ib + (int64_t)u * stride;
        x[u] = i < i1 ? __ldg(g.logit + i * g.lstride) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (ib + (int64_t)u * stride < i1) f(ib + (int64_t)u * stride, ss_unit(x[u]));
    }
    return;
  }
  // (anchor row, class) of the current index, advanced by `stride` elements per step
  const int C = p.C, sa = stride / C, sc = stride % C;
  int64_t a = (i0 + t) / C;
  int c = (int)(i0 + t - a * C);
  for (int64_t ib = i0 + t; ib < i1; ib += (int64_t)U * stride) {
    float x[U], y[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const bool in = ib + (int64_t)u * stride < i1;
      x[u] = in ? __ldg(g.logit + a * g.lstride + c) : 0.f;
      y[u] = (in && p.kind == VB200_SS_FCOS) ? __ldg(g.ctr + a * g.cstride) : 0.f;
      a += sa; c += sc;
      if (c >= C) { c -= C; ++a; }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (ib + (int64_t)u * stride >= i1) break;
      float s = ss_sigmoid(x[u]);
      if (p.kind == VB200_SS_FCOS) s = __fsqrt_rn(mul_rn(s, ss_sigmoid(y[u])));    // fcos.py:516-518
      f(ib + (int64_t)u * stride, ss_unit(s));
    }
  }
}

// key of a passing score (s > thr, so bits(s) >= base)
__device__ __forceinline__ uint32_t ss_key(float s, const SsParams& p) { return __float_as_uint(s) - p.base; }
// (key, reversed index): descending order of the pair is score descending, then index ascending
__device__ __forceinline__ unsigned long long ss_pair(float s, int64_t i, const SsParams& p) {
  return ((unsigned long long)ss_key(s, p) << p.ib) | (p.imask - (unsigned long long)i);
}

__device__ __forceinline__ int ss_tile_segment(const int* __restrict__ tile_off, int nseg, int b, int64_t& i0) {
  const int g = find_segment(tile_off, nseg, b);
  i0 = (int64_t)(b - __ldg(tile_off + g)) * kSelTile;
  return g;
}

__global__ void __launch_bounds__(kSelThreads) ss_hist_kernel(const SsSeg* __restrict__ segs, const int* __restrict__ tile_off,
                                                             int nseg, SsParams p, int* __restrict__ hist) {
  __shared__ int h[kSelBins];
  for (int b = threadIdx.x; b < kSelBins; b += kSelThreads) h[b] = 0;
  int64_t i0;
  const int g = ss_tile_segment(tile_off, nseg, blockIdx.x, i0);
  const SsSeg sg = segs[g];
  __syncthreads();
  ss_walk(sg, p, i0, min(sg.n, i0 + kSelTile), threadIdx.x, kSelThreads, [&](int64_t, float s) {
    if (s > p.thr) atomicAdd(&h[ss_key(s, p) >> p.shift0], 1);
  });
  __syncthreads();
  int* gh = hist + (size_t)g * kSelBins;
  for (int b = threadIdx.x; b < kSelBins; b += kSelThreads)
    if (h[b]) atomicAdd(gh + b, h[b]);
}

struct SsState {
  int B;           // boundary bucket, -1: every passing item is selected
  int n_bnd;       // items in bucket B
  int total;       // passing items
  int n_sure, n_list;   // pairs collected above B / in B
  int pad[3];
};

__global__ void __launch_bounds__(kSelThreads) ss_bound_kernel(const int* __restrict__ hist, SsParams p, SsState* __restrict__ st) {
  constexpr int per = kSelBins / kSelThreads;
  using Scan = cub::BlockScan<int, kSelThreads>;
  __shared__ typename Scan::TempStorage ts;
  const int g = blockIdx.x, hi = kSelBins - (int)threadIdx.x * per;     // thread 0 owns the top bins
  const int* h = hist + (size_t)g * kSelBins;
  int v[per], sum = 0;
#pragma unroll
  for (int j = 0; j < per; ++j) { v[j] = h[hi - 1 - j]; sum += v[j]; }
  int above, total;
  Scan(ts).ExclusiveSum(sum, above, total);
  if (threadIdx.x == 0) {
    st[g].total = total; st[g].n_sure = 0; st[g].n_list = 0;
    if (total <= p.k) { st[g].B = -1; st[g].n_bnd = 0; }
  }
  if (total > p.k) {
#pragma unroll
    for (int j = 0; j < per; ++j) {
      if (above < p.k && above + v[j] >= p.k) { st[g].B = hi - 1 - j; st[g].n_bnd = v[j]; }
      above += v[j];
    }
  }
}

__global__ void __launch_bounds__(kSelThreads) ss_collect_kernel(const SsSeg* __restrict__ segs, const int* __restrict__ tile_off,
                                                                int nseg, SsParams p, SsState* __restrict__ st,
                                                                unsigned long long* __restrict__ sure, unsigned long long* __restrict__ list) {
  int64_t i0;
  const int g = ss_tile_segment(tile_off, nseg, blockIdx.x, i0);
  const SsSeg sg = segs[g];
  const int B = st[g].B;
  const bool take_list = B >= 0 && st[g].n_bnd <= p.cap;       // otherwise ss_final_kernel narrows the bucket
  ss_walk(sg, p, i0, min(sg.n, i0 + kSelTile), threadIdx.x, kSelThreads, [&](int64_t i, float s) {
    if (!(s > p.thr)) return;
    const int d = (int)(ss_key(s, p) >> p.shift0);
    if (d > B) sure[(size_t)g * p.k + atomicAdd(&st[g].n_sure, 1)] = ss_pair(s, i, p);
    else if (d == B && take_list) list[(size_t)g * p.cap + atomicAdd(&st[g].n_list, 1)] = ss_pair(s, i, p);
  });
}

__global__ void __launch_bounds__(kSelSortThreads) ss_final_kernel(const SsSeg* __restrict__ segs, SsParams p, SsState* __restrict__ st,
                                                                  unsigned long long* __restrict__ sure, unsigned long long* __restrict__ list,
                                                                  unsigned long long* __restrict__ sel, int* __restrict__ sel_n) {
  using Sort = cub::BlockRadixSort<unsigned long long, kSelSortThreads, kSelSortItems>;
  __shared__ union { typename Sort::TempStorage sort; int hist[kSelBins]; } sm;
  __shared__ int s_sure, s_list, s_digit, s_above, s_count;
  const int g = blockIdx.x, t = threadIdx.x;
  const SsState S = st[g];
  unsigned long long* gs = sure + (size_t)g * p.k;
  unsigned long long* gl = list + (size_t)g * p.cap;
  if (t == 0) { s_sure = S.n_sure; s_list = S.n_list; }
  if (S.B >= 0 && S.n_bnd > p.cap) {
    // degenerate segment: narrow the boundary prefix 12 bits at a time over the (key, ~index) pair
    const SsSeg sg = segs[g];
    unsigned long long P = (unsigned long long)S.B;
    int pos = p.ib + p.shift0, need = p.k - S.n_sure, count = S.n_bnd;
    __syncthreads();
    while (count > p.cap) {
      const int npos = max(pos - kSelBits, 0), w = pos - npos;
      const unsigned long long mask = (1ull << w) - 1ull;
      for (int b = t; b < kSelBins; b += kSelSortThreads) sm.hist[b] = 0;
      __syncthreads();
      ss_walk(sg, p, 0, sg.n, t, kSelSortThreads, [&](int64_t i, float s) {
        if (!(s > p.thr)) return;
        const unsigned long long q = ss_pair(s, i, p);
        if ((q >> pos) == P) atomicAdd(&sm.hist[(q >> npos) & mask], 1);
      });
      __syncthreads();
      if (t == 0) {
        int run = 0;
        for (int b = (int)mask; b >= 0; --b) {
          if (run + sm.hist[b] >= need) { s_digit = b; s_above = run; s_count = sm.hist[b]; break; }
          run += sm.hist[b];
        }
      }
      __syncthreads();
      const unsigned long long D = (unsigned long long)s_digit;
      ss_walk(sg, p, 0, sg.n, t, kSelSortThreads, [&](int64_t i, float s) {
        if (!(s > p.thr)) return;
        const unsigned long long q = ss_pair(s, i, p);
        if ((q >> pos) == P && ((q >> npos) & mask) > D) gs[atomicAdd(&s_sure, 1)] = q;
      });
      need -= s_above;
      count = s_count;
      P = (P << w) | D;
      pos = npos;
      __syncthreads();
    }
    ss_walk(sg, p, 0, sg.n, t, kSelSortThreads, [&](int64_t i, float s) {
      if (!(s > p.thr)) return;
      const unsigned long long q = ss_pair(s, i, p);
      if ((q >> pos) == P) gl[atomicAdd(&s_list, 1)] = q;
    });
  }
  __syncthreads();
  const int ns = s_sure, nl = s_list;
  unsigned long long keys[kSelSortItems];
#pragma unroll
  for (int j = 0; j < kSelSortItems; ++j) {
    const int r = t * kSelSortItems + j;
    keys[j] = r < ns ? gs[r] : (r - ns < nl ? gl[r - ns] : 0ull);      // 0 sorts after every real pair
  }
  __syncthreads();
  Sort(sm.sort).SortDescending(keys, 0, p.sort_bits);
  const int m = min(p.k, S.total);
#pragma unroll
  for (int j = 0; j < kSelSortItems; ++j) {
    const int r = t * kSelSortItems + j;
    if (r < m) sel[(size_t)g * p.k + r] = keys[j];
  }
  if (t == 0) sel_n[g] = m;
}

// Decode + clip of the selected items.  Segment g of image g / spi lands after the items of the image's earlier segments
// (retinanet.py:555-557 concatenates the levels in order; ssd.py:448-450 the classes).
__global__ void ss_decode_kernel(const SsSeg* __restrict__ segs, SsParams p, const unsigned long long* __restrict__ sel,
                                 const int* __restrict__ sel_n, float4* __restrict__ cb, float* __restrict__ cs, int64_t* __restrict__ cl,
                                 int* __restrict__ n_img) {
  const int per = ceil_div(p.k, (int)blockDim.x);          // blocks per segment
  const int g = blockIdx.x / per, j = (blockIdx.x % per) * blockDim.x + threadIdx.x;
  const int img = g / p.spi, g0 = img * p.spi;
  const int m = sel_n[g];
  const bool last = g == g0 + p.spi - 1 && j == 0;
  if (j >= m && !last) return;
  int off = 0;
  for (int q = g0; q < g; ++q) off += sel_n[q];
  if (last) n_img[img] = off + m;
  if (j >= m) return;
  const unsigned long long q = sel[(size_t)g * p.k + j];
  const float s = __uint_as_float((uint32_t)(q >> p.ib) + p.base);
  const uint32_t i = (uint32_t)(p.imask - (q & p.imask));
  const SsSeg sg = segs[g];
  int64_t a, label;
  if (p.kind == VB200_SS_SSD) { a = i; label = sg.label; }
  else { a = i / (uint32_t)p.C; label = i % (uint32_t)p.C; }     // retinanet.py:543-544
  const float* r = sg.reg + a * sg.rstride;
  const float* an = sg.anc + a * sg.astride;
  const float x0 = an[0], y0 = an[1], x1 = an[2], y1 = an[3];
  const float r0 = r[0], r1 = r[1], r2 = r[2], r3 = r[3];
  float4 b;
  if (p.kind == VB200_SS_FCOS) {
    // BoxLinearCoder.decode, normalize_by_size=True (_utils.py:292-310)
    const float cx = mul_rn(0.5f, add_rn(x0, x1)), cy = mul_rn(0.5f, add_rn(y0, y1));
    const float w = sub_rn(x1, x0), h = sub_rn(y1, y0);
    b = make_float4(sub_rn(cx, mul_rn(r0, w)), sub_rn(cy, mul_rn(r1, h)), add_rn(cx, mul_rn(r2, w)), add_rn(cy, mul_rn(r3, h)));
  } else {
    // BoxCoder.decode_single (_utils.py:193-224): every tensor op rounded on its own
    const float w = sub_rn(x1, x0), h = sub_rn(y1, y0);
    const float cx = add_rn(x0, mul_rn(0.5f, w)), cy = add_rn(y0, mul_rn(0.5f, h));
    const float dx = mul_rn(r0, p.inv_w[0]), dy = mul_rn(r1, p.inv_w[1]);
    float dw = mul_rn(r2, p.inv_w[2]), dh = mul_rn(r3, p.inv_w[3]);
    dw = isnan(dw) ? dw : fminf(dw, p.clip);                      // torch.clamp(max=...) propagates NaN
    dh = isnan(dh) ? dh : fminf(dh, p.clip);
    const float pcx = add_rn(mul_rn(dx, w), cx), pcy = add_rn(mul_rn(dy, h), cy);
    const float hw = mul_rn(0.5f, mul_rn(expf(dw), w)), hh = mul_rn(0.5f, mul_rn(expf(dh), h));
    b = make_float4(sub_rn(pcx, hw), sub_rn(pcy, hh), add_rn(pcx, hw), add_rn(pcy, hh));
  }
  // clip_boxes_to_image, as det_clip_filter_kernel
  b.x = fminf(fmaxf(b.x, 0.f), sg.img_w); b.z = fminf(fmaxf(b.z, 0.f), sg.img_w);
  b.y = fminf(fmaxf(b.y, 0.f), sg.img_h); b.w = fminf(fmaxf(b.w, 0.f), sg.img_h);
  const size_t o = (size_t)img * p.nmax + off + j;
  cb[o] = b; cs[o] = s; cl[o] = label;
}

// image results at slot img * D -> packed one after another
__global__ void ss_concat_kernel(const float4* __restrict__ pb, const float* __restrict__ ps, const int64_t* __restrict__ pl,
                                 const int64_t* __restrict__ counts, int64_t D, float4* __restrict__ ob, float* __restrict__ os,
                                 int64_t* __restrict__ ol, int per) {
  const int img = blockIdx.x / per;
  const int64_t j = (int64_t)(blockIdx.x % per) * blockDim.x + threadIdx.x;
  if (j >= counts[img]) return;
  int64_t off = 0;
  for (int q = 0; q < img; ++q) off += counts[q];
  const int64_t src = (int64_t)img * D + j;
  ob[off + j] = pb[src]; os[off + j] = ps[src]; ol[off + j] = pl[src];
}

struct SsWs {
  SsSeg* segs; int* tile_off; int* hist; SsState* st; unsigned long long* sure; unsigned long long* list;
  unsigned long long* sel; int* sel_n; float4* cb; float* cs; int64_t* cl; int* n_img; int64_t* keep; int64_t* num_keep;
  float4* pb; float* ps; int64_t* pl; int64_t* counts; size_t bnms_off; size_t total;
};

// nmax candidates per image; the batched_nms workspace must hold any n <= nmax, and it shrinks where the plain-nms
// matrix leaves it (n above the coordinate-trick range), so both ends of that range are considered.
SsWs carve_ss(void* base, int N, int nseg, int k, int cap, int64_t nmax, int64_t D) {
  Carver c(base);
  SsWs w;
  w.segs = c.take<SsSeg>(nseg);
  w.tile_off = c.take<int>(nseg + 1);
  w.hist = c.take<int>((size_t)nseg * kSelBins);
  w.st = c.take<SsState>(nseg);
  w.sure = c.take<unsigned long long>((size_t)nseg * k);
  w.list = c.take<unsigned long long>((size_t)nseg * cap);
  w.sel = c.take<unsigned long long>((size_t)nseg * k);
  w.sel_n = c.take<int>(nseg);
  w.cb = c.take<float4>((size_t)N * nmax);
  w.cs = c.take<float>((size_t)N * nmax);
  w.cl = c.take<int64_t>((size_t)N * nmax);
  w.n_img = c.take<int>(N);
  w.keep = c.take<int64_t>(nmax);
  w.num_keep = c.take<int64_t>(32);
  w.pb = c.take<float4>((size_t)N * D);
  w.ps = c.take<float>((size_t)N * D);
  w.pl = c.take<int64_t>((size_t)N * D);
  w.counts = c.take<int64_t>(N);
  w.bnms_off = c.off;
  size_t bn = 0;
  if (nmax > 0) {
    bn = carve_bnms(nullptr, nmax).total;
    const int64_t n_trick = nmax < 25000 ? nmax : 25000;
    const size_t bt = carve_bnms(nullptr, n_trick).total;
    bn = bt > bn ? bt : bn;
  }
  c.off += bn;
  w.total = c.off;
  return w;
}

struct SsShape { int nseg, spi; int64_t tiles; int k, cap; int64_t nmax; };
SsShape ss_shape(int kind, int N, int L, const int64_t* level_anchors, int C, int64_t topk) {
  SsShape s;
  s.spi = kind == VB200_SS_SSD ? C - 1 : L;
  s.nseg = N * s.spi;
  s.k = (int)topk;
  s.cap = kSelSortCap - s.k;
  s.nmax = (int64_t)s.spi * s.k;
  int64_t per_image = 0;
  if (kind == VB200_SS_SSD) per_image = (int64_t)(C - 1) * ceil_div64(level_anchors[0], kSelTile);
  else for (int l = 0; l < L; ++l) per_image += ceil_div64(level_anchors[l] * C, kSelTile);
  s.tiles = per_image * N;
  return s;
}
}  // namespace
}  // namespace vb200

extern "C" size_t vb200_single_stage_postprocess_workspace_bytes(int kind, int num_images, int num_levels, const int64_t* level_anchors,
                                                                 int num_classes, int64_t topk_candidates, int64_t detections_per_img) {
  if (num_images <= 0 || num_levels <= 0 || !level_anchors || num_classes < 1 || topk_candidates <= 0 ||
      topk_candidates > VB200_SS_MAX_TOPK || detections_per_img <= 0)
    return 0;
  const SsShape s = ss_shape(kind, num_images, num_levels, level_anchors, num_classes, topk_candidates);
  if (s.nseg <= 0) return 0;
  return carve_ss(nullptr, num_images, s.nseg, s.k, s.cap, s.nmax, detections_per_img).total;
}

extern "C" int vb200_single_stage_postprocess(int kind, int num_images, int num_levels, const int64_t* level_anchors, int num_classes,
                                              const void* const* logits, const int64_t* logit_strides, const void* const* ctrness,
                                              const int64_t* ctrness_strides, const void* const* regression,
                                              const int64_t* regression_strides, const void* const* anchors, const int64_t* anchor_strides,
                                              const double* image_hw, double score_thresh, int64_t topk_candidates, double nms_thresh,
                                              int64_t detections_per_img, const double* weights, double bbox_xform_clip, int semantics,
                                              void* workspace, size_t workspace_bytes, void* boxes_out, void* scores_out,
                                              int64_t* labels_out, int64_t* counts_host, vb200_stream stream) {
  VB200_REQUIRE(kind == VB200_SS_RETINANET || kind == VB200_SS_FCOS || kind == VB200_SS_SSD, "single_stage_postprocess: bad kind %d", kind);
  VB200_REQUIRE(num_images >= 0 && num_levels >= 1 && num_levels <= 64 && (kind != VB200_SS_SSD || num_levels == 1),
                "single_stage_postprocess: bad image / level count");
  VB200_REQUIRE(num_classes >= 1 && topk_candidates >= 0 && topk_candidates <= VB200_SS_MAX_TOPK && detections_per_img >= 0,
                "single_stage_postprocess: bad sizes (topk_candidates must be <= %d)", VB200_SS_MAX_TOPK);
  VB200_REQUIRE(semantics == VB200_NMS_CPU || semantics == VB200_NMS_CUDA, "single_stage_postprocess: bad semantics selector");
  VB200_REQUIRE(counts_host != nullptr, "single_stage_postprocess: null counts_host");
  for (int i = 0; i < num_images; ++i) counts_host[i] = 0;
  if (num_images == 0 || topk_candidates == 0 || detections_per_img == 0 || (kind == VB200_SS_SSD && num_classes < 2)) return 0;
  VB200_REQUIRE(level_anchors && logits && logit_strides && regression && regression_strides && anchors && anchor_strides && image_hw &&
                    weights && workspace && boxes_out && scores_out && labels_out,
                "single_stage_postprocess: null pointer");
  VB200_REQUIRE(kind != VB200_SS_FCOS || (ctrness && ctrness_strides), "single_stage_postprocess: FCOS needs ctrness");
  const int N = num_images, L = num_levels, C = num_classes;
  const SsShape sh = ss_shape(kind, N, L, level_anchors, C, topk_candidates);
  VB200_REQUIRE(sh.tiles < (1ll << 31) && (int64_t)sh.nseg * ceil_div(sh.k, 128) < (1ll << 31), "single_stage_postprocess: too many segments");
  const SsWs w = carve_ss(workspace, N, sh.nseg, sh.k, sh.cap, sh.nmax, detections_per_img);
  if (workspace_bytes < w.total) {
    set_error("single_stage_postprocess: workspace too small (%zu < %zu)", workspace_bytes, w.total);
    return VB200_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;

  // segment table (image-major) and the first tile of every segment
  std::vector<SsSeg> segs((size_t)sh.nseg);
  std::vector<int> tile_off((size_t)sh.nseg + 1);
  int64_t tiles = 0, widest_seg = 1;
  for (int img = 0; img < N; ++img) {
    for (int q = 0; q < sh.spi; ++q) {
      const int l = kind == VB200_SS_SSD ? 0 : q;
      const int64_t A = level_anchors[l];
      VB200_REQUIRE(A >= 0 && A * C < (1ll << 31), "single_stage_postprocess: a segment must have fewer than 2^31 elements");
      SsSeg g;
      const float* lg = (const float*)logits[l] + img * logit_strides[2 * l];
      g.logit = kind == VB200_SS_SSD ? lg + (q + 1) : lg;
      g.lstride = logit_strides[2 * l + 1];
      g.ctr = kind == VB200_SS_FCOS ? (const float*)ctrness[l] + img * ctrness_strides[2 * l] : nullptr;
      g.cstride = kind == VB200_SS_FCOS ? ctrness_strides[2 * l + 1] : 0;
      g.reg = (const float*)regression[l] + img * regression_strides[2 * l];
      g.rstride = regression_strides[2 * l + 1];
      g.anc = (const float*)anchors[(size_t)img * L + l];
      g.astride = anchor_strides[(size_t)img * L + l];
      g.n = kind == VB200_SS_SSD ? A : A * C;
      g.label = q + 1;
      g.img_h = (float)image_hw[2 * img];
      g.img_w = (float)image_hw[2 * img + 1];
      segs[(size_t)img * sh.spi + q] = g;
      tile_off[(size_t)img * sh.spi + q] = (int)tiles;
      tiles += ceil_div64(g.n, kSelTile);
      widest_seg = g.n > widest_seg ? g.n : widest_seg;
    }
  }
  tile_off[sh.nseg] = (int)tiles;

  SsParams p;
  p.kind = kind;
  p.C = C;
  p.thr = (float)score_thresh;
  // Smallest passing bit pattern.  Scores lie in [+0, 1] (ss_unit), so for thr < 0 every score passes (base 0), and a
  // threshold of +0 or -0 passes every positive score (base = bits(+0) + 1).  A NaN threshold passes nothing.
  const float athr = fabsf(p.thr);
  uint32_t tb;
  memcpy(&tb, &athr, 4);
  p.base = (p.thr != p.thr || p.thr < 0.f) ? 0u : tb + 1u;
  const uint32_t one = 0x3f800000u;                       // bits(1.0f): keys of passing scores are <= one - base
  const uint32_t max_key = p.base <= one ? one - p.base : 0u;
  int bits = 0;
  while (bits < 32 && (max_key >> bits) != 0u) ++bits;
  p.shift0 = bits > kSelBits ? bits - kSelBits : 0;
  p.ib = 1;
  while ((1ll << p.ib) < widest_seg) ++p.ib;
  p.imask = (1ull << p.ib) - 1ull;
  p.sort_bits = bits + p.ib;
  p.k = sh.k;
  p.cap = sh.cap;
  p.spi = sh.spi;
  p.nmax = (int)sh.nmax;
  for (int j = 0; j < 4; ++j) p.inv_w[j] = 1.0f / (float)weights[j];
  p.clip = (float)bbox_xform_clip;

  VB200_CUDA_TRY(cudaMemcpyAsync(w.segs, segs.data(), segs.size() * sizeof(SsSeg), cudaMemcpyHostToDevice, st));
  VB200_CUDA_TRY(cudaMemcpyAsync(w.tile_off, tile_off.data(), tile_off.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  VB200_CUDA_TRY(cudaMemsetAsync(w.hist, 0, (size_t)sh.nseg * kSelBins * sizeof(int), st));
  VB200_CUDA_TRY(cudaMemsetAsync(w.counts, 0, (size_t)N * sizeof(int64_t), st));
  int rc = 0;
  if (tiles > 0) {
    ss_hist_kernel<<<(unsigned)tiles, kSelThreads, 0, st>>>(w.segs, w.tile_off, sh.nseg, p, w.hist);
    if ((rc = check_launch("ss_hist_kernel"))) return rc;
  }
  ss_bound_kernel<<<sh.nseg, kSelThreads, 0, st>>>(w.hist, p, w.st);
  if ((rc = check_launch("ss_bound_kernel"))) return rc;
  if (tiles > 0) {
    ss_collect_kernel<<<(unsigned)tiles, kSelThreads, 0, st>>>(w.segs, w.tile_off, sh.nseg, p, w.st, w.sure, w.list);
    if ((rc = check_launch("ss_collect_kernel"))) return rc;
  }
  ss_final_kernel<<<sh.nseg, kSelSortThreads, 0, st>>>(w.segs, p, w.st, w.sure, w.list, w.sel, w.sel_n);
  if ((rc = check_launch("ss_final_kernel"))) return rc;
  ss_decode_kernel<<<sh.nseg * ceil_div(sh.k, 128), 128, 0, st>>>(w.segs, p, w.sel, w.sel_n, w.cb, w.cs, w.cl, w.n_img);
  if ((rc = check_launch("ss_decode_kernel"))) return rc;

  // host read 1: every image's candidate count (the batched_nms strategy switch, boxes.py:86, looks at it)
  std::vector<int> n_img((size_t)N);
  VB200_CUDA_TRY(cudaMemcpyAsync(n_img.data(), w.n_img, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost, st));
  VB200_CUDA_TRY(cudaStreamSynchronize(st));
  const bool wide_keys = C > 65536;     // labels < C fit the 16-bit class keys otherwise
  const int blk = 256;
  for (int img = 0; img < N; ++img) {
    const int64_t n = n_img[img];
    if (n == 0) continue;
    const size_t o = (size_t)img * sh.nmax;
    rc = bnms_core<float>(w.cb + o, w.cs + o, w.cl + o, n, nms_thresh, semantics, VB200_BNMS_AUTO, wide_keys,
                          (char*)workspace + w.bnms_off, workspace_bytes - w.bnms_off, w.keep, w.num_keep, st);
    if (rc) return rc;
    const int64_t cap = detections_per_img < n ? detections_per_img : n;
    det_gather_topk_kernel<<<ceil_div((int)cap, blk), blk, 0, st>>>(w.cb + o, w.cs + o, w.cl + o, w.keep, w.num_keep, detections_per_img,
                                                                   w.pb + (size_t)img * detections_per_img, w.ps + (size_t)img * detections_per_img,
                                                                   w.pl + (size_t)img * detections_per_img, w.counts + img);
    if ((rc = check_launch("det_gather_topk_kernel"))) return rc;
  }
  // host read 2: every image's kept count
  VB200_CUDA_TRY(cudaMemcpyAsync(counts_host, w.counts, (size_t)N * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  VB200_CUDA_TRY(cudaStreamSynchronize(st));
  int64_t widest = 0;
  for (int img = 0; img < N; ++img) {
    VB200_REQUIRE(counts_host[img] >= 0, "single_stage_postprocess: internal error (negative kept count)");
    widest = counts_host[img] > widest ? counts_host[img] : widest;
  }
  if (widest == 0) return 0;
  const int per = ceil_div((int)widest, blk);
  ss_concat_kernel<<<(unsigned)((int64_t)N * per), blk, 0, st>>>(w.pb, w.ps, w.pl, w.counts, detections_per_img, (float4*)boxes_out,
                                                                 (float*)scores_out, labels_out, per);
  return check_launch("ss_concat_kernel");
}
