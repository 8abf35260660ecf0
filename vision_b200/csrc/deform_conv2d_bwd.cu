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
//
// Deterministic grad_input (torch.use_deterministic_algorithms): the scatter is turned into a gather.  A sample whose
// cell (hl, wl) = (floor y, floor x) is known writes exactly the four pixels (hl, wl), (hl, wl+1), (hl+1, wl), (hl+1, wl+1),
// so pixel (y, x) receives from the samples of the cells (y, x), (y, x-1), (y-1, x), (y-1, x-1) - as their corner 0, 1,
// 2, 3.  Per pass of images:
//   1. dcn_bin_samples_kernel: key = (image x offset group, cell) per sample; samples outside the image or with no
//      contributing corner get a sentinel key that sorts last;
//   2. cub::DeviceRadixSort::SortPairs(key, sample index): stable, so within a cell the samples keep ascending index;
//   3. dcn_cell_start_kernel (first sorted position of every key, by binary search) and dcn_cell_records_kernel (per
//      sorted sample: its dcol column tap*HWo + pix, the mask of contributing corners and mask * corner weight);
//   4. dcn_grad_input_gather_kernel: every grad_input element written once, no atomics.
// Summation order of grad_input[b, c, y, x]: cells (y, x), (y, x-1), (y-1, x), (y-1, x-1) in that order; inside a cell the
// samples in ascending ((offset group, tap), output pixel) index; one accumulator of Acc<T> (fp32, double for F64), rounded
// once to T.  It depends on image b's data alone, never on the other images of the call or on how they are split into passes.
#include <cub/cub.cuh>

#include <algorithm>

#include "common.cuh"
#include "dcn_geometry.cuh"

namespace vb200 {
namespace {

// One sample = (image b, offset group og, tap, output pixel pix), enumerated as idx = ((b * offset_groups + og) * KK + tap)
// * HWo + pix by every kernel of this file; this is its position, mask value and bilinear geometry.
template <typename A>
struct SamplePoint {
  int b, og, tap, pix;
  int64_t ob;        // (b * offset_groups + og) * 2 * KK: the (image, group)'s first offset channel
  A m;               // mask value (1 without a mask)
  Sample<A> s;
};

template <typename T>
__device__ __forceinline__ SamplePoint<typename Acc<T>::type> sample_point(int64_t idx, int HWo, int KK, const T* __restrict__ offset,
                                                                          const T* __restrict__ mask, const DcnParams& p) {
  using A = typename Acc<T>::type;
  SamplePoint<A> q;
  q.pix = (int)(idx % HWo);
  q.tap = (int)((idx / HWo) % KK);
  q.og = (int)((idx / HWo / KK) % p.offset_groups);
  q.b = (int)(idx / HWo / KK / p.offset_groups);
  q.ob = ((int64_t)q.b * p.offset_groups + q.og) * 2 * KK;
  A y, x;
  sample_position<A>(offset + q.ob * HWo, mask + q.ob / 2 * HWo, p, q.tap, q.pix, y, x, q.m);
  q.s = make_sample<A>(y, x, p.in_h, p.in_w);
  return q;
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
    const SamplePoint<A> q = sample_point<T>(idx, HWo, KK, offset, mask, p);
    const Sample<A>& s = q.s;
    const int b = q.b, og = q.og, tap = q.tap, pix = q.pix;
    const A m = q.m;
    A w[4];
    corner_weights(s, w);
    for (int cl = 0; cl < c_per_off; ++cl) {
      const int c = og * c_per_off + cl;
      const T* __restrict__ plane = input + ((int64_t)b * p.c_in + c) * HWi;
      A val = 0;
      if (s.inside) {
        A v[4];
        corner_values(plane, s, v);
        val = blend(w, v);
      }
      columns[((int64_t)b * p.c_in * KK + (int64_t)c * KK + tap) * HWo + pix] = from_acc<T, A>(m * val);
    }
  }
}

// dcol [n][(c * KK + tap)][pix] = (weight^T x grad_out); writes grad_offset / grad_mask and, with SCATTER, scatters
// grad_input (pre-zeroed).  The deterministic path instantiates it without the scatter and gathers grad_input instead.
template <typename T, bool SCATTER>
__global__ void __launch_bounds__(256)
dcn_backward_inputs_kernel(const T* __restrict__ dcol, const T* __restrict__ input, const T* __restrict__ offset, const T* __restrict__ mask,
                           T* __restrict__ grad_input, T* __restrict__ grad_offset, T* __restrict__ grad_mask, DcnParams p, int n_imgs) {
  using A = typename Acc<T>::type;
  const int HWo = p.out_h * p.out_w, HWi = p.in_h * p.in_w, KK = p.kh * p.kw;
  const int c_per_off = p.c_in / p.offset_groups;
  const int64_t total = (int64_t)n_imgs * p.offset_groups * KK * HWo;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const SamplePoint<A> q = sample_point<T>(idx, HWo, KK, offset, mask, p);
    const Sample<A>& s = q.s;
    const int b = q.b, og = q.og, tap = q.tap, pix = q.pix;
    const int64_t ob = q.ob;
    const A m = q.m;
    const A hh = (A)1 - s.lh, hw = (A)1 - s.lw;
    A w[4];
    corner_weights(s, w);
    A gy = 0, gx = 0, gm = 0;
    for (int cl = 0; cl < c_per_off; ++cl) {
      const int c = og * c_per_off + cl;
      const int64_t plane_off = ((int64_t)b * p.c_in + c) * HWi;
      const T* __restrict__ plane = input + plane_off;
      const A d = (A)to_acc(dcol[((int64_t)b * p.c_in * KK + (int64_t)c * KK + tap) * HWo + pix]);
      A v[4];
      corner_values(plane, s, v);
      // get_coordinate_weight (:503-536): d val / dy and d val / dx of the bilinear sample.  The fma is spelled out: left
      // to the compiler, which product it fuses changes with the surrounding code, and with it the last bit.
      gy += m * fma(hw, v[2] - v[0], s.lw * (v[3] - v[1])) * d;
      gx += m * fma(hh, v[1] - v[0], s.lh * (v[3] - v[2])) * d;
      if (s.inside) {
        gm += d * blend(w, v);
        if constexpr (SCATTER) {
          const A md = m * d;
          T* __restrict__ gi = grad_input + plane_off;
          // written out: as a loop over k, the channel loop is no longer unrolled (4 atomics in flight instead of 12)
          if (s.ok[0] && w[0] != (A)0) atomic_add<T>(gi + s.o[0], md * w[0]);
          if (s.ok[1] && w[1] != (A)0) atomic_add<T>(gi + s.o[1], md * w[1]);
          if (s.ok[2] && w[2] != (A)0) atomic_add<T>(gi + s.o[2], md * w[2]);
          if (s.ok[3] && w[3] != (A)0) atomic_add<T>(gi + s.o[3], md * w[3]);
        }
      }
    }
    grad_offset[(ob + 2 * tap) * HWo + pix] = from_acc<T, A>(gy);
    grad_offset[(ob + 2 * tap + 1) * HWo + pix] = from_acc<T, A>(gx);
    if (p.use_mask) grad_mask[(((int64_t)b * p.offset_groups + og) * KK + tap) * HWo + pix] = from_acc<T, A>(gm);
  }
}

// ---- deterministic grad_input: bin, sort, cell table, gather -------------------------------------------------------------
// Corner k of a sample contributes to grad_input when it lies in the image and its bilinear weight is not exactly 0 (the
// scatter's test).  Bit k of the result; w[k] = that weight.
template <typename A>
__device__ __forceinline__ int live_corners(const Sample<A>& s, A w[4]) {
  corner_weights(s, w);
  int bits = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) bits |= (s.ok[k] && w[k] != (A)0) ? (1 << k) : 0;
  return s.inside ? bits : 0;
}

// key = (b * offset_groups + og) * (H+1)(W+1) + (hl+1) * (W+1) + (wl+1); `sentinel` (= segments x cells) for a sample that
// contributes nothing.  vals = the sample index (the sort's payload).
template <typename T>
__global__ void __launch_bounds__(256)
dcn_bin_samples_kernel(const T* __restrict__ offset, const T* __restrict__ mask, uint32_t* __restrict__ keys, int* __restrict__ vals,
                       DcnParams p, int n_samples, uint32_t sentinel) {
  using A = typename Acc<T>::type;
  const int cw = p.in_w + 1, cells = (p.in_h + 1) * cw, HWo = p.out_h * p.out_w, KK = p.kh * p.kw;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n_samples; idx += gridDim.x * blockDim.x) {
    const SamplePoint<A> q = sample_point<T>(idx, HWo, KK, offset, mask, p);
    A w[4];
    const int bits = live_corners(q.s, w);
    keys[idx] = bits ? (uint32_t)(((int64_t)q.b * p.offset_groups + q.og) * cells + (q.s.hl + 1) * cw + (q.s.wl + 1)) : sentinel;
    vals[idx] = idx;
  }
}

// start[v] = first sorted position whose key is >= v, for v in [0, sentinel]: the samples of cell v are [start[v], start[v+1]).
__global__ void __launch_bounds__(256)
dcn_cell_start_kernel(const uint32_t* __restrict__ keys_sorted, int n_samples, int* __restrict__ start, uint32_t sentinel) {
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v <= (int64_t)sentinel; v += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = n_samples;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (keys_sorted[mid] < (uint32_t)v) lo = mid + 1; else hi = mid;
    }
    start[v] = lo;
  }
}

// One record per sorted sample: col = tap * HWo + pix (its dcol column inside the channel's KK x HWo block), the live-corner
// bits, and mw[k] = mask * corner weight k (0 for a dead corner; the bits, not the zero, decide whether it is added).
template <typename A>
struct alignas(4 * sizeof(A)) CornerW { A v[4]; };

template <typename T>
__global__ void __launch_bounds__(256)
dcn_cell_records_kernel(const uint32_t* __restrict__ keys_sorted, const int* __restrict__ vals_sorted, const T* __restrict__ offset,
                        const T* __restrict__ mask, int2* __restrict__ rec_col, CornerW<typename Acc<T>::type>* __restrict__ rec_w,
                        DcnParams p, int n_samples, uint32_t sentinel) {
  using A = typename Acc<T>::type;
  const int HWo = p.out_h * p.out_w;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_samples; i += gridDim.x * blockDim.x) {
    if (keys_sorted[i] == sentinel) continue;        // never read: the cell table ends before the first sentinel
    const SamplePoint<A> q = sample_point<T>(vals_sorted[i], HWo, p.kh * p.kw, offset, mask, p);
    A w[4];
    const int bits = live_corners(q.s, w);
    CornerW<A> r;
#pragma unroll
    for (int k = 0; k < 4; ++k) r.v[k] = (bits >> k & 1) ? q.m * w[k] : (A)0;
    rec_col[i] = make_int2(q.tap * HWo + q.pix, bits);
    rec_w[i] = r;
  }
}

// grad_input[b, c, y, x] = sum over the cells (y, x), (y, x-1), (y-1, x), (y-1, x-1) - the pixel is their corner 0, 1, 2, 3 -
// and over each cell's records in sorted order, of mw[k] * dcol[b, c * KK + tap, pix].  A CTA owns (image, offset group,
// CPB channels of the group, 256 pixels); a thread owns one pixel (lanes along x) and the CPB channels in registers, so
// each record is read once for CPB channels.  Every pixel is written, with 0 where nothing lands.
template <typename T, int CPB>
__global__ void __launch_bounds__(256)
dcn_grad_input_gather_kernel(const T* __restrict__ dcol, const int* __restrict__ cell_start, const int2* __restrict__ rec_col,
                             const CornerW<typename Acc<T>::type>* __restrict__ rec_w, T* __restrict__ grad_input, DcnParams p,
                             int n_tiles, int n_cchunks) {
  using A = typename Acc<T>::type;
  const int HWo = p.out_h * p.out_w, HWi = p.in_h * p.in_w, KK = p.kh * p.kw;
  const int c_per_off = p.c_in / p.offset_groups;
  const int cw = p.in_w + 1, cells = (p.in_h + 1) * cw;
  const int tile = (int)(blockIdx.x % n_tiles);
  const int cc = (int)((blockIdx.x / n_tiles) % n_cchunks);
  const int seg = (int)(blockIdx.x / n_tiles / n_cchunks);           // b * offset_groups + og
  const int b = seg / p.offset_groups, og = seg - b * p.offset_groups;
  const int pix = tile * 256 + threadIdx.x;
  if (pix >= HWi) return;
  const int y = pix / p.in_w, x = pix - y * p.in_w;
  const int c0 = og * c_per_off + cc * CPB, nc = min(CPB, c_per_off - cc * CPB);
  const T* __restrict__ dc = dcol + ((int64_t)b * p.c_in + c0) * KK * HWo;
  const int64_t cstride = (int64_t)KK * HWo;
  const int* __restrict__ cs = cell_start + (int64_t)seg * cells;
  const int cell0 = (y + 1) * cw + (x + 1);
  A acc[CPB];
#pragma unroll
  for (int j = 0; j < CPB; ++j) acc[j] = (A)0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int cell = cell0 - (k >> 1) * cw - (k & 1);
    const int beg = cs[cell], end = cs[cell + 1];
    for (int r = beg; r < end; ++r) {
      const int2 hdr = rec_col[r];
      if (!(hdr.y >> k & 1)) continue;
      const A mw = rec_w[r].v[k];
#pragma unroll
      for (int j = 0; j < CPB; ++j)
        if (j < nc) acc[j] += mw * (A)to_acc(dc[j * cstride + hdr.x]);
    }
  }
  T* __restrict__ gi = grad_input + ((int64_t)b * p.c_in + c0) * HWi + pix;
#pragma unroll
  for (int j = 0; j < CPB; ++j)
    if (j < nc) gi[(int64_t)j * HWi] = from_acc<T, A>(acc[j]);
}

// channels per gather thread: the accumulators stay in registers
template <typename T> struct GatherCpb { static constexpr int value = 16; };
template <> struct GatherCpb<double> { static constexpr int value = 8; };

// Images per pass of the deterministic path: sample indices and sorted positions are int, keys are 32-bit.  0 when one image
// alone exceeds that (the caller then reports the shape as unsupported).
int det_pass_imgs(const DcnParams& p, int n_imgs) {
  const int64_t spi = (int64_t)p.offset_groups * p.kh * p.kw * p.out_h * p.out_w;
  const int64_t kpi = (int64_t)p.offset_groups * (p.in_h + 1) * (p.in_w + 1);
  const int64_t by_samples = ((int64_t)INT32_MAX - 1) / spi, by_keys = ((int64_t)UINT32_MAX - 1) / kpi;
  return (int)std::min<int64_t>({(int64_t)n_imgs, by_samples, by_keys});
}

struct DetWs {
  uint32_t *keys_in, *keys_out; int *vals_in, *vals_out, *cell_start; int2* rec_col; void* rec_w;
  void* cub_temp; size_t cub_bytes; size_t total;
};

DetWs carve_det(void* base, const DcnParams& p, int pass_imgs, size_t acc_bytes) {
  const int n = (int)((int64_t)pass_imgs * p.offset_groups * p.kh * p.kw * p.out_h * p.out_w);
  const size_t nk = (size_t)pass_imgs * p.offset_groups * (p.in_h + 1) * (p.in_w + 1) + 1;
  Carver c(base);
  DetWs w;
  w.keys_in = c.take<uint32_t>(n);
  w.keys_out = c.take<uint32_t>(n);
  w.vals_in = c.take<int>(n);
  w.vals_out = c.take<int>(n);
  w.cell_start = c.take<int>(nk);
  w.rec_col = c.take<int2>(n);
  w.rec_w = c.take<char>((size_t)n * 4 * acc_bytes);
  w.cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, w.cub_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int*)nullptr, (int*)nullptr,
                                  n, 0, 32);
  w.cub_temp = c.take<char>(w.cub_bytes);
  w.total = c.off;
  return w;
}

int grid_for(int64_t total) {
  return (int)(ceil_div64(total, 256) < (int64_t)sm_count() * 32 ? ceil_div64(total, 256) : (int64_t)sm_count() * 32);
}

template <typename T>
int launch_columns(const void* input, const void* offset, const void* mask, void* columns, const DcnParams& p, int n_imgs, cudaStream_t st) {
  const int64_t total = (int64_t)n_imgs * p.offset_groups * p.kh * p.kw * p.out_h * p.out_w;
  if (total == 0) return 0;
  const int grid = grid_for(total);
  dcn_sample_columns_kernel<T><<<grid, 256, 0, st>>>((const T*)input, (const T*)offset, (const T*)mask, (T*)columns, p, n_imgs);
  return check_launch("dcn_sample_columns_kernel");
}
template <typename T, bool SCATTER = true>
int launch_bwd_inputs(const void* dcol, const void* input, const void* offset, const void* mask, void* gi, void* go, void* gm,
                      const DcnParams& p, int n_imgs, cudaStream_t st) {
  const int64_t total = (int64_t)n_imgs * p.offset_groups * p.kh * p.kw * p.out_h * p.out_w;
  if (total == 0) return 0;
  const int grid = grid_for(total);
  dcn_backward_inputs_kernel<T, SCATTER><<<grid, 256, 0, st>>>((const T*)dcol, (const T*)input, (const T*)offset, (const T*)mask, (T*)gi,
                                                              (T*)go, (T*)gm, p, n_imgs);
  return check_launch("dcn_backward_inputs_kernel");
}

// grad_offset / grad_mask by the scatter-free instantiation, then grad_input pass by pass (bin, sort, cell table, gather).
template <typename T>
int launch_bwd_inputs_det(const void* dcol, const void* input, const void* offset, const void* mask, void* gi, void* go, void* gm,
                          const DcnParams& p, int n_imgs, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  using A = typename Acc<T>::type;
  constexpr int CPB = GatherCpb<T>::value;
  const int pass = det_pass_imgs(p, n_imgs);
  const DetWs w = carve_det(workspace, p, pass, sizeof(A));
  if (workspace_bytes < w.total) {
    set_error("deform_conv2d_backward_inputs: workspace too small (%zu < %zu)", workspace_bytes, w.total);
    return VB200_EWORKSPACE;
  }
  int rc = launch_bwd_inputs<T, false>(dcol, input, offset, mask, nullptr, go, gm, p, n_imgs, st);
  if (rc) return rc;
  const int KK = p.kh * p.kw, HWo = p.out_h * p.out_w, HWi = p.in_h * p.in_w;
  const int64_t cells = (int64_t)(p.in_h + 1) * (p.in_w + 1);
  const int n_tiles = ceil_div(HWi, 256), n_cchunks = ceil_div(p.c_in / p.offset_groups, CPB);
  for (int b0 = 0; b0 < n_imgs; b0 += pass) {
    const int nb = std::min(pass, n_imgs - b0);
    const int n = (int)((int64_t)nb * p.offset_groups * KK * HWo);
    const uint32_t sentinel = (uint32_t)((int64_t)nb * p.offset_groups * cells);
    const T* off_b = (const T*)offset + (int64_t)b0 * p.offset_groups * 2 * KK * HWo;
    const T* mask_b = p.use_mask ? (const T*)mask + (int64_t)b0 * p.offset_groups * KK * HWo : nullptr;
    const T* dcol_b = (const T*)dcol + (int64_t)b0 * p.c_in * KK * HWo;
    T* gi_b = (T*)gi + (int64_t)b0 * p.c_in * HWi;
    dcn_bin_samples_kernel<T><<<grid_for(n), 256, 0, st>>>(off_b, mask_b, w.keys_in, w.vals_in, p, n, sentinel);
    if ((rc = check_launch("dcn_bin_samples_kernel"))) return rc;
    const int end_bit = 32 - __builtin_clz(sentinel | 1u);          // only the bits the key range needs
    size_t tb = w.cub_bytes;
    VB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(w.cub_temp, tb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, n, 0, end_bit, st));
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    dcn_cell_start_kernel<<<grid_for((int64_t)sentinel + 1), 256, 0, st>>>(w.keys_out, n, w.cell_start, sentinel);
    if ((rc = check_launch("dcn_cell_start_kernel"))) return rc;
    dcn_cell_records_kernel<T><<<grid_for(n), 256, 0, st>>>(w.keys_out, w.vals_out, off_b, mask_b, w.rec_col, (CornerW<A>*)w.rec_w, p, n,
                                                           sentinel);
    if ((rc = check_launch("dcn_cell_records_kernel"))) return rc;
    const int64_t blocks = (int64_t)nb * p.offset_groups * n_cchunks * n_tiles;
    dcn_grad_input_gather_kernel<T, CPB><<<(unsigned)blocks, 256, 0, st>>>(dcol_b, w.cell_start, w.rec_col, (const CornerW<A>*)w.rec_w, gi_b,
                                                                          p, n_tiles, n_cchunks);
    if ((rc = check_launch("dcn_grad_input_gather_kernel"))) return rc;
  }
  return 0;
}

}  // namespace
}  // namespace vb200

using namespace vb200;

extern "C" int vb200_deform_conv2d_sample_columns(const void* input, const void* offset, const void* mask, void* columns, int dtype,
                                                  int n_imgs, int c_in, int in_h, int in_w, int kh, int kw, int stride_h, int stride_w,
                                                  int pad_h, int pad_w, int dil_h, int dil_w, int offset_groups, int use_mask,
                                                  vb200_stream stream) {
  DcnParams p;
  if (const int rc = dcn_params(p, n_imgs, c_in, in_h, in_w, 0, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, 1, offset_groups,
                                use_mask))
    return rc;
  if (n_imgs == 0 || c_in == 0) return 0;
  VB200_REQUIRE(input && offset && columns && (!use_mask || mask), "deform_conv2d_sample_columns: null pointer");
  VB200_REQUIRE((int64_t)in_h * in_w < (1ll << 31), "deform_conv2d_sample_columns: image too large");
  return dispatch_dcn_dtype(dtype, "deform_conv2d_sample_columns: unsupported dtype %d", [&](auto t) {
    return launch_columns<decltype(t)>(input, offset, mask, columns, p, n_imgs, (cudaStream_t)stream);
  });
}

extern "C" size_t vb200_deform_conv2d_backward_inputs_workspace_bytes(int dtype, int n_imgs, int c_in, int in_h, int in_w, int kh, int kw,
                                                                     int stride_h, int stride_w, int pad_h, int pad_w, int dil_h,
                                                                     int dil_w, int offset_groups) {
  DcnParams p;
  if (n_imgs <= 0 || c_in <= 0 || in_h <= 0 || in_w <= 0 ||
      dcn_params(p, n_imgs, c_in, in_h, in_w, 0, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, 1, offset_groups, 0) != 0)
    return 0;
  const int pass = det_pass_imgs(p, n_imgs);
  if (pass == 0) return 0;
  return carve_det(nullptr, p, pass, dtype == VB200_F64 ? sizeof(double) : sizeof(float)).total;
}

extern "C" int vb200_deform_conv2d_backward_inputs(const void* dcol, const void* input, const void* offset, const void* mask,
                                                   void* grad_input, void* grad_offset, void* grad_mask, int dtype, int n_imgs, int c_in,
                                                   int in_h, int in_w, int kh, int kw, int stride_h, int stride_w, int pad_h, int pad_w,
                                                   int dil_h, int dil_w, int offset_groups, int use_mask, int deterministic, void* workspace,
                                                   size_t workspace_bytes, vb200_stream stream) {
  DcnParams p;
  if (const int rc = dcn_params(p, n_imgs, c_in, in_h, in_w, 0, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, 1, offset_groups,
                                use_mask))
    return rc;
  if (n_imgs == 0 || c_in == 0) return 0;
  VB200_REQUIRE(dcol && input && offset && grad_input && grad_offset && (!use_mask || (mask && grad_mask)), "deform_conv2d_backward_inputs: null pointer");
  VB200_REQUIRE((int64_t)in_h * in_w < (1ll << 31), "deform_conv2d_backward_inputs: image too large");
  cudaStream_t st = (cudaStream_t)stream;
  if (deterministic) {
    if (det_pass_imgs(p, n_imgs) == 0) {
      set_error("deform_conv2d_backward_inputs: one image has too many samples or cells for the deterministic grad_input");
      return VB200_EUNSUPPORTED;
    }
    VB200_REQUIRE(workspace, "deform_conv2d_backward_inputs: null workspace");
  }
  return dispatch_dcn_dtype(dtype, "deform_conv2d_backward_inputs: unsupported dtype %d", [&](auto t) {
    using T = decltype(t);
    if (deterministic)
      return launch_bwd_inputs_det<T>(dcol, input, offset, mask, grad_input, grad_offset, grad_mask, p, n_imgs, workspace, workspace_bytes, st);
    return launch_bwd_inputs<T>(dcol, input, offset, mask, grad_input, grad_offset, grad_mask, p, n_imgs, st);
  });
}
