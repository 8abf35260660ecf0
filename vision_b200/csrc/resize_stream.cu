// resize_stream.cu — bilinear-antialias DOWNSCALE fast path (the cfg5 regime: 2160x3840 -> 224x224; fp16, bf16,
// uint8 and fp32 storage).
//
// Reference route (torchvision/transforms/v2/functional/_geometry.py:340-360): cast to fp32 (full
// size pass), aten::_upsample_bilinear2d_aa (one thread per output pixel looping over ~20x36 taps,
// ATen/native/cuda/UpSampleBilinear2d.cu), cast back: ~4x the algorithmic bytes and latency-bound.
//
// This kernel reads every input byte exactly once and is a single pass:
//   * the triangle filter of radius `scale` (>= 1) means every input pixel feeds at most TWO
//     neighbouring outputs per axis, so the separable filter is evaluated "input-driven":
//     thread i of a warp owns the pixels between output centres i-1 and i, forms the partial sums
//     A_i (-> output i) and B_i (-> output i-1) from registers-resident normalised weights, and
//     out[i] = A_i + B_{i+1} is one warp shuffle; warps overlap by one interval;
//   * input rows stream through a ring of shared-memory stages filled by 1-D bulk async copies
//     (TMA engine) issued by a producer warp; full/empty mbarriers, no block-wide barriers;
//   * vertically every row feeds two running accumulators per thread (outputs k-1 and k); a row
//     of outputs is written (storage dtype, round-to-nearest) the moment its last input row passed.
// Weights follow ATen's _compute_weights_span/_compute_weights (UpSample.cuh:303-343): same
// xmin/xsize, same filter argument, normalised by the sequential float sum.
#include "async_copy.cuh"
#include "common.cuh"

namespace vb200 {
namespace {

constexpr int kMaxConsumerWarps = 16;
constexpr int kMaxBandRows = 1024;   // upper bound on band_cap (keeps the per-row tables at 12 KB)

constexpr int kMaxResizeDst = 8;

struct StreamParams {
  int in_h, in_w, out_h, out_w;
  float scale_w, scale_h;
  int rows_out_per_cta, n_stages, row_pitch;   // row_pitch: bytes per stage (row + zeroed pad)
  int band_cap;                                // capacity of the per-row vertical tables
  // destinations: the caller's own output and, for the fused all-gather (vb200_resize_gather), the same slot of every
  // peer's gathered buffer (peer-mapped device memory: the stores travel over NVLink while the input streams from HBM)
  void* dst[kMaxResizeDst];
  int ndst;
};

__device__ __forceinline__ float centre(float scale, int m) { return scale * ((float)m + 0.5f); }
// P(x, m): centre(m) <= x + 0.5  — the one predicate every partition decision is derived from
__device__ __forceinline__ bool at_or_past(float scale, int m, int x) { return centre(scale, m) <= (float)x + 0.5f; }

// first input index belonging to interval i (pixels between centre i-1 and centre i); i in [0, O]
__device__ __forceinline__ int interval_lo(float scale, int i, int in_size) {
  if (i <= 0) return 0;
  int x = (int)ceilf(centre(scale, i - 1) - 0.5f);
  x = min(max(x, 0), in_size);
  while (x > 0 && at_or_past(scale, i - 1, x - 1)) --x;
  while (x < in_size && !at_or_past(scale, i - 1, x)) ++x;
  return x;
}

// ATen span + sequential total for output index o (UpSample.cuh:303-331), bilinear filter
__device__ __forceinline__ void aa_span(float scale, int o, int in_size, int* xmin_o, int* xend_o, float* xmc_o, float* total_o) {
  const float support = scale, invscale = 1.0f / scale;           // scale >= 1 on this path
  const float c = centre(scale, o);
  const int xmin = max((int)(c - support + 0.5f), 0);
  const int xsize = min((int)(c + support + 0.5f), in_size) - xmin;
  const float xmc = (float)xmin - c;
  float total = 0.f;
  for (int j = 0; j < xsize; ++j) {
    float a = ((float)j + xmc + 0.5f) * invscale;
    a = a < 0.f ? -a : a;
    total += a < 1.f ? 1.f - a : 0.f;
  }
  *xmin_o = xmin; *xend_o = xmin + xsize; *xmc_o = xmc; *total_o = total;
}

// weight of input x for an output with span [xmin, xend): ATen drops what its integer span excludes even when
// the filter argument is (just) inside the support
__device__ __forceinline__ float aa_weight(float scale, int x, int xmin, int xend, float xmc, float total) {
  float a = ((float)(x - xmin) + xmc + 0.5f) * (1.0f / scale);
  a = a < 0.f ? -a : a;
  const float w = a < 1.f ? 1.f - a : 0.f;
  const bool in_span = x >= xmin && x < xend;
  return (in_span && total != 0.f) ? __fdiv_rn(w, total) : (in_span ? w : 0.f);
}

// Storage types: PPW pixels per 32-bit shared-memory word; pair(rowp, q) = pixels 2q, 2q+1 of the thread's slot
// run as fp32 (q is a compile-time constant after unrolling, so the word loads are shared between pairs).
template <typename T> struct Px;
template <> struct Px<__half> {
  static constexpr int PPW = 2;
  static __device__ __forceinline__ float2 pair(const uint32_t* rowp, int q) {
    const uint32_t u = rowp[q];
    return __half22float2(*reinterpret_cast<const __half2*>(&u));
  }
};
template <> struct Px<__nv_bfloat16> {
  static constexpr int PPW = 2;
  static __device__ __forceinline__ float2 pair(const uint32_t* rowp, int q) {
    const uint32_t u = rowp[q];
    return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
  }
};
template <> struct Px<float> {
  static constexpr int PPW = 1;
  static __device__ __forceinline__ float2 pair(const uint32_t* rowp, int q) {
    const uint2 u = *reinterpret_cast<const uint2*>(rowp + 2 * q);      // the slot starts on an even pixel
    return make_float2(__uint_as_float(u.x), __uint_as_float(u.y));
  }
};
template <> struct Px<uint8_t> {
  static constexpr int PPW = 4;
  // byte b -> float without the conversion unit: 0x4B000000 | b is 2^23 + b exactly
  static __device__ __forceinline__ float2 pair(const uint32_t* rowp, int q) {
    const uint32_t u = rowp[q >> 1];
    const uint32_t lo = __byte_perm(u, 0x4B000000u, (q & 1) ? 0x7442 : 0x7440);
    const uint32_t hi = __byte_perm(u, 0x4B000000u, (q & 1) ? 0x7443 : 0x7441);
    return make_float2(__uint_as_float(lo) - 8388608.0f, __uint_as_float(hi) - 8388608.0f);
  }
};
template <typename T> __device__ __forceinline__ T store_px(float v) { return from_acc<T, float>(v); }
// _geometry.py:352-359 for integer images: round half to even, then the cast (bilinear weights are convex: no clamp needed,
// the saturating conversion is a guard only)
template <> __device__ __forceinline__ uint8_t store_px<uint8_t>(float v) { return (uint8_t)__float2uint_rn(fminf(fmaxf(v, 0.f), 255.f)); }

// T: storage type (fp16, bf16, fp32, uint8).  NP: pixel PAIRS each thread reads per row.
// NW: consumer warps the kernel is compiled for (block = (n_cwarps + 1) * 32 <= (NW + 1) * 32).
template <typename T, int NP, int NW>
__global__ void __launch_bounds__((NW + 1) * 32, (NW <= 8 && NP <= 12) ? 3 : 1)
resize_aa_stream_kernel(const T* __restrict__ in, StreamParams p, int n_cwarps) {
  extern __shared__ __align__(128) unsigned char smem[];
  // layout: [stages][row_pitch] | full[S] empty[S] | totx[OW] xmcx[OW] xminx[OW] xendx[OW] | toty.. | rowA[band] rowB[band] rowK[band]
  unsigned char* stages = smem;
  uint64_t* full = reinterpret_cast<uint64_t*>(stages + (size_t)p.n_stages * p.row_pitch);
  uint64_t* empty = full + p.n_stages;
  float* totx = reinterpret_cast<float*>(empty + p.n_stages);
  float* xmcx = totx + p.out_w;
  int* xminx = reinterpret_cast<int*>(xmcx + p.out_w);
  int* xendx = xminx + p.out_w;
  float* toty = reinterpret_cast<float*>(xendx + p.out_w);
  float* ymcy = toty + p.out_h;
  int* yminy = reinterpret_cast<int*>(ymcy + p.out_h);
  int* yendy = yminy + p.out_h;
  float* rowA = reinterpret_cast<float*>(yendy + p.out_h);
  float* rowB = rowA + p.band_cap;
  int* rowK = reinterpret_cast<int*>(rowB + p.band_cap);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nthreads = blockDim.x;
  const int64_t plane = blockIdx.y;
  const int oy0 = blockIdx.x * p.rows_out_per_cta;
  const int oy1 = min(oy0 + p.rows_out_per_cta, p.out_h);
  const int r0 = interval_lo(p.scale_h, oy0, p.in_h);
  const int r1 = (oy1 >= p.out_h) ? p.in_h : interval_lo(p.scale_h, oy1 + 1, p.in_h);
  const int nrows = min(r1 - r0, p.band_cap);
  const uint32_t row_bytes = (uint32_t)p.in_w * sizeof(T);

  // ---- setup: barriers, zeroed pads, per-output spans/totals, per-row vertical weights ----
  if (tid == 0) {
    for (int s = 0; s < p.n_stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], n_cwarps); }
    mbar_fence_init();
  }
  for (int s = 0; s < p.n_stages; ++s)
    for (int b = row_bytes + tid * 4; b < p.row_pitch; b += nthreads * 4)
      *reinterpret_cast<uint32_t*>(stages + (size_t)s * p.row_pitch + b) = 0u;
  for (int o = tid; o < p.out_w; o += nthreads) aa_span(p.scale_w, o, p.in_w, &xminx[o], &xendx[o], &xmcx[o], &totx[o]);
  for (int o = tid; o < p.out_h; o += nthreads) aa_span(p.scale_h, o, p.in_h, &yminy[o], &yendy[o], &ymcy[o], &toty[o]);
  __syncthreads();
  for (int rl = tid; rl < nrows; rl += nthreads) {
    const int r = r0 + rl;
    // interval index k of row r: number of centres at or before r + 0.5
    int k = (int)floorf(((float)r + 0.5f) / p.scale_h - 0.5f) + 1;
    k = min(max(k, 0), p.out_h);
    while (k > 0 && !at_or_past(p.scale_h, k - 1, r)) --k;
    while (k < p.out_h && at_or_past(p.scale_h, k, r)) ++k;
    rowK[rl] = k;
    rowA[rl] = (k < p.out_h) ? aa_weight(p.scale_h, r, yminy[k], yendy[k], ymcy[k], toty[k]) : 0.f;
    rowB[rl] = (k >= 1) ? aa_weight(p.scale_h, r, yminy[k - 1], yendy[k - 1], ymcy[k - 1], toty[k - 1]) : 0.f;
  }
  fence_proxy_async();
  __syncthreads();

  const T* __restrict__ src = in + plane * (int64_t)p.in_h * p.in_w + (int64_t)r0 * p.in_w;

  if (warp == n_cwarps) {
    // ===== producer warp: one elected lane streams the band's rows through the ring =====
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int rl = 0; rl < nrows; ++rl) {
        mbar_wait(&empty[s], ph ^ 1u);
        fence_proxy_async();      // consumers' generic-proxy reads of this stage (released by their arrive) before the async-proxy rewrite
        mbar_expect_tx(&full[s], row_bytes);
        bulk_g2s(stages + (size_t)s * p.row_pitch, src + (int64_t)rl * p.in_w, row_bytes, &full[s]);
        if (++s == p.n_stages) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }
  if (warp > n_cwarps) return;

  // ===== consumer warps =====
  const int i = warp * 31 + lane;                 // interval index owned by this thread (0 .. out_w)
  const bool have = i <= p.out_w;
  const int lo = have ? interval_lo(p.scale_w, i, p.in_w) : p.in_w;
  const int hi = have ? ((i >= p.out_w) ? p.in_w : interval_lo(p.scale_w, i + 1, p.in_w)) : p.in_w;
  constexpr int PPW = Px<T>::PPW;
  constexpr int ALIGN = PPW > 2 ? PPW : 2;        // the slot starts on a 32-bit word AND on a pixel pair
  const int e = lo & ~(ALIGN - 1);
  // weights kept as fp32 pairs: each step of the inner loop is two FMAs, one per pixel
  unsigned long long wA2[NP], wB2[NP];
#pragma unroll
  for (int t = 0; t < NP; ++t) {
    float wa[2], wb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int x = e + 2 * t + h;
      const bool in_iv = have && x >= lo && x < hi;
      wa[h] = (in_iv && i < p.out_w) ? aa_weight(p.scale_w, x, xminx[i], xendx[i], xmcx[i], totx[i]) : 0.f;
      wb[h] = (in_iv && i >= 1) ? aa_weight(p.scale_w, x, xminx[i - 1], xendx[i - 1], xmcx[i - 1], totx[i - 1]) : 0.f;
    }
    wA2[t] = pack2(wa[0], wa[1]);
    wB2[t] = pack2(wb[0], wb[1]);
  }
  const int word0 = min((int)((e * (int)sizeof(T)) >> 2), (int)(row_bytes >> 2));     // beyond the row: the zeroed pad
  const bool writer = have && lane < 31 && i < p.out_w;     // lane 31 only supplies B to lane 30
  const int64_t doff = plane * (int64_t)p.out_h * p.out_w + i;
  auto put = [&](int row, float v) {              // one finished output pixel -> every destination
    const T q = store_px<T>(v);
    const int64_t o = doff + (int64_t)row * p.out_w;
    for (int d = 0; d < p.ndst; ++d) reinterpret_cast<T*>(p.dst[d])[o] = q;
  };

  float acc_lo = 0.f, acc_hi = 0.f;
  int k_cur = oy0;
  int s = 0;
  uint32_t ph = 0;
  const unsigned char* stage_ptr = stages + (size_t)word0 * 4;
  const int n_stages = p.n_stages, row_pitch = p.row_pitch;      // registers, not a constant-bank load per row
  for (int rl = 0; rl < nrows; ++rl) {
    mbar_wait_hint(&full[s], ph, 2000u);
    const uint32_t* __restrict__ rowp = reinterpret_cast<const uint32_t*>(stage_ptr);
    unsigned long long accA = 0ull, accB = 0ull;             // (a0, a1), (b0, b1) as fp32 pairs
#pragma unroll
    for (int t = 0; t < NP; ++t) {
      const float2 v = Px<T>::pair(rowp, t);
      const unsigned long long v2 = pack2(v.x, v.y);
      accA = fma2(wA2[t], v2, accA);
      accB = fma2(wB2[t], v2, accB);
    }
    const float a0 = lo32(accA), a1 = hi32(accA), b0 = lo32(accB), b1 = hi32(accB);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
    if (++s == n_stages) { s = 0; ph ^= 1u; stage_ptr = stages + (size_t)word0 * 4; } else stage_ptr += row_pitch;
    const float A = a0 + a1, B = b0 + b1;
    const float h = A + __shfl_down_sync(0xffffffffu, B, 1);
    const int k = rowK[rl];
    if (k != k_cur) {                              // CTA-uniform: output row k_cur - 1 is complete
      if (writer && k_cur - 1 >= oy0) put(k_cur - 1, acc_lo);
      acc_lo = acc_hi; acc_hi = 0.f; k_cur = k;
    }
    acc_hi = fmaf(rowA[rl], h, acc_hi);
    acc_lo = fmaf(rowB[rl], h, acc_lo);
  }
  // rows of the band are exhausted: acc_lo holds output row k_cur - 1; a band that ended exactly on an
  // interval boundary (k_cur == oy1 - 1 cannot happen: the band includes interval oy1) -> k_cur == oy1
  if (writer && k_cur - 1 >= oy0 && k_cur - 1 < oy1) put(k_cur - 1, acc_lo);
  if (writer && k_cur < oy1 && k_cur >= oy0) put(k_cur, acc_hi);
}

template <typename T, int NP, int NW>
int launch_stream(const void* in, int64_t planes, const StreamParams& p0, cudaStream_t st) {
  constexpr int LW = (NP * 2 * (int)sizeof(T) + 3) / 4;       // 32-bit words a thread reads per row
  StreamParams p = p0;
  const int n_cwarps = ceil_div(p.out_w + 1, 31);
  const uint32_t row_bytes = (uint32_t)p.in_w * sizeof(T);
  p.row_pitch = (int)((row_bytes + LW * 4 + 4 + 127) & ~127u);
  // split the output rows so that the grid has a few waves of CTAs even for small batches
  const int64_t want_ctas = (int64_t)sm_count() * 3 * 2;
  int splits = (int)((want_ctas + planes - 1) / planes);
  splits = splits < 1 ? 1 : (splits > p.out_h ? p.out_h : splits);
  if (splits > 1 && p.out_h / splits < 8) splits = p.out_h / 8 > 0 ? p.out_h / 8 : 1;   // keep halo overhead <= ~12 %
  p.rows_out_per_cta = ceil_div(p.out_h, splits);
  splits = ceil_div(p.out_h, p.rows_out_per_cta);
  int band_rows = (int)((p.rows_out_per_cta + 2) * p.scale_h) + 4;
  if (band_rows > kMaxBandRows) {
    p.rows_out_per_cta = (int)((kMaxBandRows - 4) / p.scale_h) - 2;
    if (p.rows_out_per_cta < 1) return 0;
    splits = ceil_div(p.out_h, p.rows_out_per_cta);
    band_rows = (int)((p.rows_out_per_cta + 2) * p.scale_h) + 4;
  }
  p.band_cap = (band_rows + 31) & ~31;
  const size_t fixed = (size_t)(p.out_w + p.out_h) * 16 + (size_t)p.band_cap * 12 + 256;
  const int ctas_per_sm = (NW <= 8 && NP <= 12) ? 3 : 2;
  const size_t budget = ((size_t)max_smem_optin() - 3072) / ctas_per_sm - 1024;   // smem per CTA (1 KB reserved each)
  if (budget < fixed + 3 * (size_t)p.row_pitch) return 0;
  int stages = (int)((budget - fixed) / p.row_pitch);
  stages = stages > 8 ? 8 : stages;
  if (stages < 3) return 0;
  p.n_stages = stages;
  const size_t smem = (size_t)stages * p.row_pitch + (size_t)stages * 16 + fixed;
  VB200_CUDA_TRY(ensure_dyn_smem<resize_aa_stream_kernel<T, NP, NW>>(smem));
  int64_t done = 0;
  while (done < planes) {
    const int64_t chunk = planes - done < 65535 ? planes - done : 65535;
    dim3 grid((unsigned)splits, (unsigned)chunk);
    StreamParams pc = p;
    for (int d = 0; d < p.ndst; ++d) pc.dst[d] = (T*)p.dst[d] + done * (int64_t)p.out_h * p.out_w;
    resize_aa_stream_kernel<T, NP, NW><<<grid, (n_cwarps + 1) * 32, smem, st>>>((const T*)in + done * (int64_t)p.in_h * p.in_w, pc, n_cwarps);
    int rc = check_launch("resize_aa_stream_kernel");
    if (rc) return rc;
    done += chunk;
  }
  return 1;
}

template <typename T>
int dispatch_lw(const void* in, int64_t planes, const StreamParams& p, cudaStream_t st) {
  // a thread owns at most floor(scale)+1 pixels, + the slot alignment slack
  constexpr int ALIGN = Px<T>::PPW > 2 ? Px<T>::PPW : 2;
  const int need = ((int)floorf(p.scale_w) + 1 + (ALIGN - 1) + 1) / 2;     // pixel pairs
  const bool small = ceil_div(p.out_w + 1, 31) <= 8;
  if (small) {
    if (need <= 4) return launch_stream<T, 4, 8>(in, planes, p, st);
    if (need <= 6) return launch_stream<T, 6, 8>(in, planes, p, st);
    if (need <= 10) return launch_stream<T, 10, 8>(in, planes, p, st);
    if (need <= 12) return launch_stream<T, 12, 8>(in, planes, p, st);
    if (need <= 16) return launch_stream<T, 16, 8>(in, planes, p, st);
    return 0;
  }
  if (need <= 4) return launch_stream<T, 4, kMaxConsumerWarps>(in, planes, p, st);
  if (need <= 6) return launch_stream<T, 6, kMaxConsumerWarps>(in, planes, p, st);
  if (need <= 10) return launch_stream<T, 10, kMaxConsumerWarps>(in, planes, p, st);
  if (need <= 16) return launch_stream<T, 16, kMaxConsumerWarps>(in, planes, p, st);
  return 0;
}

}  // namespace

int resize_aa_stream_try(const void* in, void* const* outs, int ndst, int dtype, int64_t planes, int in_h, int in_w, int out_h,
                         int out_w, int mode, cudaStream_t st) {
  const char* force = env_override(ENV_RESIZE_PATH);            // "generic" disables the fast path
  if (force && force[0] == 'g') return 0;
  if (mode != VB200_RESIZE_BILINEAR) return 0;
  if (dtype != VB200_F16 && dtype != VB200_BF16 && dtype != VB200_U8 && dtype != VB200_F32) return 0;
  const size_t esize = dtype == VB200_F32 ? 4 : dtype == VB200_U8 ? 1 : 2;
  if (in_w <= out_w || in_h < out_h) return 0;                 // horizontal downscale, vertical scale >= 1
  if (out_w + 1 > 31 * kMaxConsumerWarps) return 0;
  if (((size_t)in_w * esize) % 16 != 0 || ((uintptr_t)in % 16) != 0) return 0;
  if (ndst < 1 || ndst > kMaxResizeDst) return 0;
  StreamParams p{};
  p.ndst = ndst;
  for (int d = 0; d < ndst; ++d) p.dst[d] = outs[d];
  p.in_h = in_h; p.in_w = in_w; p.out_h = out_h; p.out_w = out_w;
  p.scale_w = (float)in_w / (float)out_w;
  p.scale_h = (float)in_h / (float)out_h;
  if (p.scale_w < 2.0f) return 0;
  if (dtype == VB200_F16) return dispatch_lw<__half>(in, planes, p, st);
  if (dtype == VB200_U8) return dispatch_lw<uint8_t>(in, planes, p, st);
  if (dtype == VB200_F32) return dispatch_lw<float>(in, planes, p, st);
  return dispatch_lw<__nv_bfloat16>(in, planes, p, st);
}

}  // namespace vb200
