// keypoints.cu — Keypoint R-CNN's heatmaps_to_keypoints (torchvision/models/detection/roi_heads.py:237-307) for every RoI
// of a call in one device pipeline, sm_90a.
//
// The reference, per RoI i: W_i = ceil(max(x2 - x1, 1)), H_i likewise; the N heatmaps resized to H_i x W_i by ATen's CUDA
// upsample_bicubic2d (align_corners=False); the argmax of each resized map; that position mapped back into the image.
// Here, three launches whatever the number of RoIs:
//   kp_geometry_kernel     one CTA: W_i, H_i and the tile count of every RoI, their prefix sum; the argmax keys cleared.
//   kp_sweep_kernel<T>     a persistent grid over (RoI, keypoint, 64 x 64 output tile) items, one contiguous range of items
//                          per CTA, so a large RoI spreads over many CTAs.  Per item: the heatmap staged in shared memory,
//                          a table of row values R[input row][output column] (a row value depends only on the input row and
//                          the output column, and the reference computes it in exactly that form, so reusing it across
//                          output rows is bit-identical), then per pixel the 4-term y combination, the rounding to the map
//                          dtype, and a (value, index) maximum, one 64-bit atomicMax per item.
//   kp_finalize_kernel<T>  per (RoI, keypoint): the winning position, its value recomputed from the heatmap (the key keeps
//                          neither -0.0 nor a NaN's payload), the reference's coordinate arithmetic.
#include "bicubic.cuh"
#include "common.cuh"

namespace vb200 {
namespace {

constexpr int kKpTX = 64, kKpTY = 64, kKpThreads = 256;

// One RoI's resized map and tiling; w = h = 0 for a box the pipeline does not take (non-finite size, or H_i * W_i >= 2^31).
struct KpGeo { int w, h, ntx, nty; };

// The reference's argmax order (ATen's ArgMaxOps): NaN above everything, the first NaN wins; ties go to the lowest index;
// -0.0 == +0.0.  The value as an order-preserving 32-bit key (NaN made +NaN, -0.0 made +0.0) above ~index: the largest
// 64-bit key is the argmax.  The maximum is associative and commutative, so any split across threads and CTAs agrees.
__device__ __forceinline__ unsigned long long kp_key(float v, uint32_t idx) {
  uint32_t u = __float_as_uint(v);
  if (v != v) u = 0x7fffffffu;
  else if (v == 0.f) u = 0u;
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | (uint32_t)~idx;
}

__global__ void __launch_bounds__(1024)
kp_geometry_kernel(const float* __restrict__ rois, int64_t K, int N, KpGeo* __restrict__ geo, int64_t* __restrict__ tile_start,
                   unsigned long long* __restrict__ keys) {
  __shared__ int64_t warp_sum[32];
  __shared__ int64_t carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t i = threadIdx.x; i < K * N; i += blockDim.x) keys[i] = 0ull;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < K; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    int64_t tiles = 0;
    if (i < K) {
      const float* b = rois + i * 4;
      // widths = (x2 - x1).clamp(min=1).ceil(): a NaN stays NaN and fails the range test below
      float w = __fsub_rn(b[2], b[0]), h = __fsub_rn(b[3], b[1]);
      w = ceilf(w < 1.f ? 1.f : w);
      h = ceilf(h < 1.f ? 1.f : h);
      KpGeo g = {0, 0, 0, 0};
      if (w <= 2147483648.f && h <= 2147483648.f && (int64_t)w * (int64_t)h < ((int64_t)1 << 31)) {
        g.w = (int)w;
        g.h = (int)h;
        g.ntx = ceil_div(g.w, kKpTX);
        g.nty = ceil_div(g.h, kKpTY);
        tiles = (int64_t)N * g.ntx * g.nty;
      }
      geo[i] = g;
    }
    int64_t incl = tiles;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      const int nw = blockDim.x >> 5;
      int64_t s = lane < nw ? warp_sum[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t v = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += v;
      }
      if (lane < nw) warp_sum[lane] = s;
    }
    __syncthreads();
    const int64_t before = carry + (warp ? warp_sum[warp - 1] : 0) + incl - tiles;
    if (i < K) tile_start[i] = before;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = before + tiles;
    __syncthreads();
  }
  if (threadIdx.x == 0) tile_start[K] = carry;
}

template <typename T>
__global__ void __launch_bounds__(kKpThreads)
kp_sweep_kernel(const T* __restrict__ maps, const KpGeo* __restrict__ geo, const int64_t* __restrict__ tile_start, int64_t K, int N,
                int H, int W, unsigned long long* __restrict__ keys) {
  extern __shared__ float4 kp_smem[];
  float4* colc = kp_smem;                                  // [kKpTX] x coefficients of the tile's columns
  float4* rowc = colc + kKpTX;                             // [kKpTY] y coefficients of the tile's rows
  int4* rowtap = reinterpret_cast<int4*>(rowc + kKpTY);    // [kKpTY] table offsets of each output row's four input rows
  int* colix = reinterpret_cast<int*>(rowtap + kKpTY);     // [kKpTX] floor of the source x
  int* rowiy = colix + kKpTX;                              // [kKpTY] floor of the source y
  float* plane = reinterpret_cast<float*>(rowiy + kKpTY);  // [H][W] the heatmap, widened to fp32
  float* table = plane + H * W;                            // [rows the tile reads][kKpTX] row values
  __shared__ unsigned long long red[kKpThreads / 32];

  const int tid = threadIdx.x;
  const int64_t total = tile_start[K];
  const int64_t chunk = ceil_div64(total, gridDim.x);
  const int64_t begin = (int64_t)blockIdx.x * chunk, end = begin + chunk < total ? begin + chunk : total;
  if (begin >= end) return;
  // the RoI holding item `begin`: tile_start[r] <= begin < tile_start[r + 1] (so RoI r has tiles)
  int64_t r = 0, hi = K;
  while (hi - r > 1) {
    const int64_t mid = (r + hi) >> 1;
    if (tile_start[mid] <= begin) r = mid; else hi = mid;
  }
  KpGeo g = geo[r];
  int64_t per = (int64_t)g.ntx * g.nty;
  int kp = (int)((begin - tile_start[r]) / per);
  int64_t t = (begin - tile_start[r]) % per;

  for (int64_t item = begin; item < end; ++item) {
    const int x0 = (int)(t % g.ntx) * kKpTX, y0 = (int)(t / g.ntx) * kKpTY;
    const int tw = min(kKpTX, g.w - x0), th = min(kKpTY, g.h - y0);
    const bool copy = g.h == H && g.w == W;   // upsample_bicubic2d_out_frame copies a same-size map unchanged
    const T* __restrict__ src = maps + (r * N + kp) * (int64_t)H * W;
    __syncthreads();   // the previous item's reads of shared memory are done
    for (int i = tid; i < H * W; i += kKpThreads) plane[i] = to_acc(src[i]);
    if (!copy) {
      if (tid < tw) {
        int ix;
        float c[4];
        cubic_coeffs(cubic_frac(cubic_source(__fdiv_rn((float)W, (float)g.w), x0 + tid), &ix), c);
        colix[tid] = ix;
        colc[tid] = make_float4(c[0], c[1], c[2], c[3]);
      } else if (tid >= kKpTX && tid - kKpTX < th) {
        const float sh = __fdiv_rn((float)H, (float)g.h);
        int iy, iy0;
        float c[4];
        cubic_coeffs(cubic_frac(cubic_source(sh, y0 + tid - kKpTX), &iy), c);
        cubic_frac(cubic_source(sh, y0), &iy0);
        // the source row index is monotone in the output row: the tile reads input rows lo = clamp(iy0 - 1) .. hi_row only
        const int base = cubic_clamp(iy0 - 1, H);
        rowiy[tid - kKpTX] = iy;
        rowc[tid - kKpTX] = make_float4(c[0], c[1], c[2], c[3]);
        rowtap[tid - kKpTX] = make_int4((cubic_clamp(iy - 1, H) - base) * kKpTX, (cubic_clamp(iy, H) - base) * kKpTX,
                                        (cubic_clamp(iy + 1, H) - base) * kKpTX, (cubic_clamp(iy + 2, H) - base) * kKpTX);
      }
      __syncthreads();
      const int lo = cubic_clamp(rowiy[0] - 1, H);
      const int hi_row = cubic_clamp(rowiy[th - 1] + 2, H);
      const int c = tid % kKpTX;
      if (c < tw) {
        const int ix = colix[c];
        const float4 q = colc[c];
        const float cx[4] = {q.x, q.y, q.z, q.w};
        const int i0 = cubic_clamp(ix - 1, W), i1 = cubic_clamp(ix, W), i2 = cubic_clamp(ix + 1, W), i3 = cubic_clamp(ix + 2, W);
        for (int row = lo + tid / kKpTX; row <= hi_row; row += kKpThreads / kKpTX) {
          const float* p = plane + row * W;
          table[(row - lo) * kKpTX + c] = cubic_interp(p[i0], p[i1], p[i2], p[i3], cx);
        }
      }
    }
    __syncthreads();

    // this thread's argmax: it visits its pixels in ascending flat index, so it takes a pixel only when it is strictly larger
    // (or the first NaN), which keeps the first of equal values
    uint32_t bi = 0xffffffffu;
    float bv = 0.f;
    const int c = tid % kKpTX;
    if (c < tw) {
      const float* tc = table + c;
      for (int rr = tid / kKpTX; rr < th; rr += kKpThreads / kKpTX) {
        float v;
        if (copy) {
          v = plane[(y0 + rr) * W + x0 + c];
        } else {
          const int4 o = rowtap[rr];
          const float4 q = rowc[rr];
          const float cy[4] = {q.x, q.y, q.z, q.w};
          v = to_acc(from_acc<T>(cubic_interp(tc[o.x], tc[o.y], tc[o.z], tc[o.w], cy)));   // the resized map is in the maps' dtype
        }
        // flat index into H_i x W_i: below 2^31, the geometry kernel takes no larger map
        const uint32_t idx = (uint32_t)((y0 + rr) * g.w + x0 + c);
        if (bi == 0xffffffffu || (!(v <= bv) && bv == bv)) {
          bv = v;
          bi = idx;
        }
      }
    }
    unsigned long long best = bi == 0xffffffffu ? 0ull : kp_key(bv, bi);   // 0 is below every key: -inf's is 0x007fffff'xxxxxxxx
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other > best ? other : best;
    }
    if ((tid & 31) == 0) red[tid >> 5] = best;
    __syncthreads();
    if (tid < 32) {
      best = tid < kKpThreads / 32 ? red[tid] : 0ull;
#pragma unroll
      for (int o = 4; o; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
        best = other > best ? other : best;
      }
      if (tid == 0) atomicMax(&keys[r * N + kp], best);
    }

    // next item: the next tile, keypoint, or RoI with tiles
    if (++t == per) {
      t = 0;
      if (++kp == N && item + 1 < end) {
        kp = 0;
        do ++r; while (tile_start[r + 1] == tile_start[r]);
        g = geo[r];
        per = (int64_t)g.ntx * g.nty;
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
kp_finalize_kernel(const T* __restrict__ maps, const float* __restrict__ rois, const KpGeo* __restrict__ geo,
                   const unsigned long long* __restrict__ keys, int64_t K, int N, int H, int W, float* __restrict__ xy,
                   float* __restrict__ scores) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= K * N) return;
  const int64_t r = i / N;
  const int kp = (int)(i - r * N);
  const KpGeo g = geo[r];
  float* __restrict__ xyr = xy + r * 3 * N;   // xy_preds [K, 3, N]: x, y, and the visibility row of ones
  xyr[2 * N + kp] = 1.f;
  if (g.w == 0) {
    xyr[kp] = xyr[N + kp] = scores[i] = __int_as_float(0x7fffffff);
    return;
  }
  const uint32_t idx = ~(uint32_t)keys[i];
  const int xi = (int)(idx % (uint32_t)g.w), yi = (int)(idx / (uint32_t)g.w);
  const T* __restrict__ src = maps + i * (int64_t)H * W;
  float v;
  if (g.h == H && g.w == W) {
    v = to_acc(src[yi * W + xi]);
  } else {
    // the same arithmetic as the sweep's table and pixel steps, for one pixel
    int iy, ix;
    float cy[4], cx[4];
    cubic_coeffs(cubic_frac(cubic_source(__fdiv_rn((float)H, (float)g.h), yi), &iy), cy);
    cubic_coeffs(cubic_frac(cubic_source(__fdiv_rn((float)W, (float)g.w), xi), &ix), cx);
    const int i0 = cubic_clamp(ix - 1, W), i1 = cubic_clamp(ix, W), i2 = cubic_clamp(ix + 1, W), i3 = cubic_clamp(ix + 2, W);
    float rowv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const T* __restrict__ p = src + cubic_clamp(iy - 1 + k, H) * W;
      rowv[k] = cubic_interp(to_acc(p[i0]), to_acc(p[i1]), to_acc(p[i2]), to_acc(p[i3]), cx);
    }
    v = to_acc(from_acc<T>(cubic_interp(rowv[0], rowv[1], rowv[2], rowv[3], cy)));
  }
  scores[i] = v;
  // width_correction = widths[i] / roi_map_width: torch's CUDA division by a Python scalar multiplies by the reciprocal it
  // computed on the host; then (x_int.float() + 0.5) * width_correction + offset_x, each op rounded on its own
  const float* b = rois + r * 4;
  float w = __fsub_rn(b[2], b[0]), h = __fsub_rn(b[3], b[1]);
  w = w < 1.f ? 1.f : w;
  h = h < 1.f ? 1.f : h;
  const float wc = __fmul_rn(w, __frcp_rn((float)g.w)), hc = __fmul_rn(h, __frcp_rn((float)g.h));
  xyr[kp] = __fadd_rn(__fmul_rn(__fadd_rn((float)xi, 0.5f), wc), b[0]);
  xyr[N + kp] = __fadd_rn(__fmul_rn(__fadd_rn((float)yi, 0.5f), hc), b[1]);
}

struct KpWorkspace {
  KpGeo* geo;
  int64_t* tile_start;
  unsigned long long* keys;
};

KpWorkspace carve_keypoints(void* base, int64_t K, int N, size_t* bytes) {
  Carver c(base);
  KpWorkspace ws;
  ws.geo = c.take<KpGeo>((size_t)K);
  ws.tile_start = c.take<int64_t>((size_t)K + 1);
  ws.keys = c.take<unsigned long long>((size_t)K * N);
  *bytes = c.off;
  return ws;
}

template <typename T>
int launch_keypoints(const void* maps, const float* rois, int64_t K, int N, int H, int W, float* xy, float* scores,
                     const KpWorkspace& ws, cudaStream_t st) {
  kp_geometry_kernel<<<1, 1024, 0, st>>>(rois, K, N, ws.geo, ws.tile_start, ws.keys);
  int rc = check_launch("kp_geometry_kernel");
  if (rc) return rc;
  const size_t smem = (size_t)(kKpTX + kKpTY) * sizeof(float4) + (size_t)kKpTY * sizeof(int4) + (size_t)(kKpTX + kKpTY) * sizeof(int) +
                      ((size_t)H * W + (size_t)H * kKpTX) * sizeof(float);
  if (smem > 48 * 1024) VB200_CUDA_TRY(ensure_dyn_smem<kp_sweep_kernel<T>>(smem));
  int per_sm = 0;
  VB200_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kp_sweep_kernel<T>, kKpThreads, smem));
  kp_sweep_kernel<T><<<sm_count() * (per_sm > 0 ? per_sm : 1), kKpThreads, smem, st>>>((const T*)maps, ws.geo, ws.tile_start, K, N, H,
                                                                                        W, ws.keys);
  rc = check_launch("kp_sweep_kernel");
  if (rc) return rc;
  kp_finalize_kernel<T><<<(unsigned)ceil_div64(K * N, 256), 256, 0, st>>>((const T*)maps, rois, ws.geo, ws.keys, K, N, H, W, xy, scores);
  return check_launch("kp_finalize_kernel");
}

}  // namespace
}  // namespace vb200

using namespace vb200;

extern "C" size_t vb200_heatmaps_to_keypoints_workspace_bytes(int64_t num_rois, int num_keypoints) {
  if (num_rois <= 0 || num_keypoints <= 0) return 0;
  size_t bytes = 0;
  carve_keypoints(nullptr, num_rois, num_keypoints, &bytes);
  return bytes;
}

extern "C" int vb200_heatmaps_to_keypoints(const void* maps, int dtype, const float* rois, int64_t num_rois, int num_keypoints,
                                           int height, int width, float* xy_out, float* scores_out, void* workspace,
                                           size_t workspace_bytes, vb200_stream stream) {
  const int64_t K = num_rois;
  const int N = num_keypoints, H = height, W = width;
  VB200_REQUIRE(K >= 0 && N > 0 && H > 0 && W > 0, "heatmaps_to_keypoints: bad sizes");
  VB200_REQUIRE(H <= VB200_KP_MAX_SIDE && W <= VB200_KP_MAX_SIDE, "heatmaps_to_keypoints: heatmaps of %d x %d exceed %d x %d", H, W,
                VB200_KP_MAX_SIDE, VB200_KP_MAX_SIDE);
  if (K == 0) return 0;
  VB200_REQUIRE(maps && rois && xy_out && scores_out, "heatmaps_to_keypoints: null pointer");
  size_t need = 0;
  carve_keypoints(nullptr, K, N, &need);
  if (!workspace || workspace_bytes < need) {
    set_error("heatmaps_to_keypoints: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    return VB200_EWORKSPACE;
  }
  const KpWorkspace ws = carve_keypoints(workspace, K, N, &need);
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case VB200_F32: return launch_keypoints<float>(maps, rois, K, N, H, W, xy_out, scores_out, ws, st);
    case VB200_F16: return launch_keypoints<__half>(maps, rois, K, N, H, W, xy_out, scores_out, ws, st);
    case VB200_BF16: return launch_keypoints<__nv_bfloat16>(maps, rois, K, N, H, W, xy_out, scores_out, ws, st);
  }
  set_error("heatmaps_to_keypoints: unsupported dtype %d", dtype);
  return VB200_EUNSUPPORTED;
}
