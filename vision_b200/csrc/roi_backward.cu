// roi_backward.cu — backward kernels of roi_align / roi_pool / ps_roi_align / ps_roi_pool for sm_90a.  The reference's
// RoI arithmetic they share with the forward kernels (roi_ops.cu) is in roi_geometry.cuh.
//
// Reference semantics (pytorch/vision; all four scatter with fastAtomicAdd into a zeroed grad_input and call
// alertNotDeterministic):
//   _roi_align_backward     csrc/ops/cuda/roi_align_kernel.cu:145-332 (host :396-468)
//   _roi_pool_backward      csrc/ops/cuda/roi_pool_kernel.cu:80-125
//   _ps_roi_align_backward  csrc/ops/cuda/ps_roi_align_kernel.cu:142-317
//   _ps_roi_pool_backward   csrc/ops/cuda/ps_roi_pool_kernel.cu:80-142
//
// Design (not a port).  grad_input is produced PLANE BY PLANE: a persistent CTA owns one (image, channel) plane of
// grad_input as an fp32 accumulator in shared memory, folds every RoI's contribution into it and writes the finished
// plane once - no zero-fill pass, no global atomics, each output byte written exactly once.  Determinism comes from
// ownership, not from ordering tricks: the rows of the plane are split into bands, band w belongs to warp w, and every
// warp walks ALL RoIs in index order and applies only the taps that land in its own rows.  A word of the accumulator
// is therefore only ever touched by one warp, in RoI order, then sample order - a fixed fp32 summation order, so
// two runs give identical bits (the reference's result depends on the atomics' arrival order).  The band test is
// vectorised: lane i checks RoI n0 + i against the band (one header load per lane), a ballot gives the RoIs that
// hit, and the warp processes those one after the other.  Lanes that would add into the same word inside one
// instruction (duplicate columns of very small RoIs, two bins with the same argmax) are merged first, in lane order.
// Shapes the plane path does not cover (plane larger than shared memory, adaptive sampling grids, fp16 / fp64) use
// a plain atomic scatter kernel organised per RoI with the sampling tables built once per CTA.  ps_roi_pool's backward is
// an atomic scatter only.
#include "common.cuh"
#include "roi_geometry.cuh"

namespace vb200 {
namespace {

constexpr int kBwdThreads = 1024;

struct BwdHdr { int batch, rmin, rmax, flags; };   // rows [rmin, rmax] receive contributions; flags bit 0: duplicate columns

// ---- geometry: one warp per RoI -----------------------------------------------------------------------------
// ys[n][PH*sr]      (lo | -1, l)                 one per y sample
// xe[n][2*PW*sr]    (col | pw << 16  or ~0, w)   one per x tap with non-zero weight
// The gradient's axis arithmetic is the forward's (roi_align_kernel.cu:146-203); `ps` selects the ps_roi_align variant of
// the box arithmetic.
__global__ void __launch_bounds__(256)
roi_bwd_geometry_kernel(const float* __restrict__ rois, BwdHdr* __restrict__ hdr, uint2* __restrict__ ys, uint2* __restrict__ xe,
                        int K, int H, int W, int PH, int PW, int sr, float scale, int aligned, int ps) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (n >= K) return;
  const RoiGeom<float> g = roi_geometry<float, float>(rois + (int64_t)n * 5, scale, PH, PW, sr, aligned != 0, ps != 0);
  const int NYS = PH * sr, NXS = PW * sr;
  int rmin = 0x7fffffff, rmax = -1;
  for (int j = lane; j < NYS; j += 32) {
    const AxisEnt<float> a = axis_entry<float>(sample_coord<float>(g.start_h, g.bin_h, j / sr, j % sr, sr), H);
    ys[(int64_t)n * NYS + j] = make_uint2((uint32_t)a.lo, __float_as_uint(a.l));     // lo = -1 outside
    if (a.lo >= 0) { rmin = min(rmin, a.lo); rmax = max(rmax, a.l > 0.f ? a.lo + 1 : a.lo); }
  }
  int dup = 0;
  for (int base = 0; base < 2 * NXS; base += 32) {      // chunks of 32 taps, as the accumulate kernel walks them
    const int k = base + lane;
    uint2 ent = make_uint2(0xffffffffu, 0u);
    if (k < 2 * NXS) {
      const int j = k >> 1, cx = k & 1;
      const AxisEnt<float> a = axis_entry<float>(sample_coord<float>(g.start_w, g.bin_w, j / sr, j % sr, sr), W);
      const float w = cx ? a.l : a.h;
      if (a.lo >= 0 && w != 0.f) ent = make_uint2((uint32_t)(a.lo + cx) | ((uint32_t)(j / sr) << 16), __float_as_uint(w));
      xe[(int64_t)n * 2 * NXS + k] = ent;
    }
    const bool v = ent.x != 0xffffffffu;
    const unsigned same = __match_any_sync(0xffffffffu, v ? (ent.x & 0xffffu) : 0x10000u + lane);
    if (v && (same & (same - 1))) dup = 1;
  }
  for (int o = 16; o; o >>= 1) {
    rmin = min(rmin, __shfl_xor_sync(0xffffffffu, rmin, o));
    rmax = max(rmax, __shfl_xor_sync(0xffffffffu, rmax, o));
    dup |= __shfl_xor_sync(0xffffffffu, dup, o);
  }
  if (lane == 0) {
    BwdHdr h;
    h.batch = g.batch; h.rmin = rmin; h.rmax = rmax; h.flags = dup;
    hdr[n] = h;
  }
}

// Sum of `a` over the lanes of `group` (same mask in every member), accumulated in ascending lane order; every
// lane of the warp must call it.  Non-members pass group == 0.
__device__ __forceinline__ float ordered_group_sum(float a, unsigned group) {
  float sum = 0.f;
  unsigned rem = group;
  while (__any_sync(0xffffffffu, rem != 0u)) {
    const int src = rem ? __ffs(rem) - 1 : 0;
    const float v = __shfl_sync(0xffffffffu, a, src);
    if (rem) { sum += v; rem &= rem - 1; }
  }
  return sum;
}

__device__ __forceinline__ void zero_plane(float* __restrict__ plane, int count) {
  float4* p4 = reinterpret_cast<float4*>(plane);
  const int n4 = (count + 3) >> 2;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) p4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

__device__ __forceinline__ void store_plane(float* __restrict__ dst, const float* __restrict__ plane, int count) {
  const int tid = threadIdx.x, NT = blockDim.x;
  if ((((uintptr_t)dst) & 15u) == 0) {
    const int nvec = count >> 2;
    const float4* s4 = reinterpret_cast<const float4*>(plane);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int i = tid; i < nvec; i += NT) d4[i] = s4[i];
    for (int i = (nvec << 2) + tid; i < count; i += NT) dst[i] = plane[i];
  } else {
    for (int i = tid; i < count; i += NT) dst[i] = plane[i];
  }
}

// ---- roi_align backward, plane-resident ----------------------------------------------------------------------
// grad [K, C, PH, PW] contiguous fp32; grad_input [B, C, H, W] written in full.
__global__ void __launch_bounds__(kBwdThreads, 1)
roi_align_bwd_plane_kernel(const float* __restrict__ grad, const BwdHdr* __restrict__ hdr, const uint2* __restrict__ ys,
                           const uint2* __restrict__ xe, float* __restrict__ grad_input, int B, int C, int H, int W, int K,
                           int PH, int PW, int sr, int band) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* plane = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NYS = PH * sr, NXE = 2 * PW * sr, NB = PH * PW;
  const float inv_count = 1.0f / (float)(sr * sr);         // exact for sr = 1, 2, 4; sr = 3 differs from /9 by one rounding
  const bool pow2 = (sr & (sr - 1)) == 0;
  const float count = (float)(sr * sr);
  const int r0 = warp * band, r1 = min(H, r0 + band);
  for (int pl = blockIdx.x; pl < B * C; pl += gridDim.x) {
    const int b = pl / C, c = pl - b * C;
    zero_plane(plane, H * W);
    __syncthreads();
    if (r0 < H) {
      for (int n0 = 0; n0 < K; n0 += 32) {
        const int nl = n0 + lane;
        bool hit = false;
        int flags_l = 0;
        if (nl < K) {
          const int4 h = __ldg(reinterpret_cast<const int4*>(hdr) + nl);
          hit = h.x == b && h.y < r1 && h.z >= r0;
          flags_l = h.w;
        }
        unsigned m = __ballot_sync(0xffffffffu, hit);
        while (m) {
          const int i = __ffs(m) - 1;
          m &= m - 1;
          const int n = n0 + i;
          const int flags = __shfl_sync(0xffffffffu, flags_l, i);
          const float* __restrict__ g = grad + ((int64_t)n * C + c) * NB;
          for (int yc = 0; yc < NYS; yc += 32) {
            uint2 yy = make_uint2(0xffffffffu, 0u);
            if (yc + lane < NYS) yy = __ldg(ys + (int64_t)n * NYS + yc + lane);
            const int lo = (int)yy.x;
            const float l = __uint_as_float(yy.y);
            const bool inb = lo >= 0 && lo < r1 && (lo + (l > 0.f ? 1 : 0)) >= r0;
            const unsigned ymask = __ballot_sync(0xffffffffu, inb);
            if (!ymask) continue;
            for (int xc = 0; xc < NXE; xc += 32) {
              uint2 e = make_uint2(0xffffffffu, 0u);
              if (xc + lane < NXE) e = __ldg(xe + (int64_t)n * NXE + xc + lane);
              const bool valid = e.x != 0xffffffffu;
              const int col = (int)(e.x & 0xffffu), pw = (int)(e.x >> 16);
              const float wx = __uint_as_float(e.y);
              bool leader = valid;
              unsigned group = 0u;
              if (flags & 1) {
                const unsigned same = __match_any_sync(0xffffffffu, valid ? col : 0x10000 + lane);
                group = valid ? same : 0u;
                leader = valid && (__ffs(same) - 1 == lane);
              }
              unsigned mm = ymask;
              int cur_ph = -1;
              float gv = 0.f;
              while (mm) {
                const int j = __ffs(mm) - 1;
                mm &= mm - 1;
                const int lo_j = __shfl_sync(0xffffffffu, lo, j);
                const float l_j = __shfl_sync(0xffffffffu, l, j);
                const int ph = (yc + j) / sr;
                if (ph != cur_ph) {
                  cur_ph = ph;
                  gv = valid ? __ldg(g + ph * PW + pw) : 0.f;
                  gv = pow2 ? gv * inv_count : __fdiv_rn(gv, count);
                }
                float a = wx * gv;
                if (flags & 1) a = ordered_group_sum(a, group);
                if (leader) {
                  if (lo_j >= r0) plane[lo_j * W + col] += (1.f - l_j) * a;               // lo_j < r1 holds for in-band samples
                  if (l_j > 0.f && lo_j + 1 >= r0 && lo_j + 1 < r1) plane[(lo_j + 1) * W + col] += l_j * a;
                }
              }
              __syncwarp();      // the next chunk's lanes may own the same words
            }
          }
        }
      }
    }
    __syncthreads();
    store_plane(grad_input + (int64_t)pl * H * W, plane, H * W);
    __syncthreads();
  }
}

// Same algorithm for the common shapes (PH*sr <= 32 y samples, 2*PW*sr <= 32 x taps, PH*PW <= 64 bins - e.g. 7x7 bins with
// sampling_ratio 2): a hit needs one table load per lane and two coalesced loads of the RoI's bin gradients, all
// independent of each other, so they are issued for hit i+1 BEFORE hit i is processed (the general kernel above chains
// three L2 round trips per hit and is latency-bound); the bin gradient of a (sample, tap) pair is then a shuffle.
struct HitLoads { uint2 yy, e; float gA, gB; };

__global__ void __launch_bounds__(kBwdThreads, 1)
roi_align_bwd_plane_fast_kernel(const float* __restrict__ grad, const BwdHdr* __restrict__ hdr, const uint2* __restrict__ ys,
                                const uint2* __restrict__ xe, float* __restrict__ grad_input, int B, int C, int H, int W, int K,
                                int PH, int PW, int sr, int band) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* plane = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NYS = PH * sr, NXE = 2 * PW * sr, NB = PH * PW;
  const float inv_count = 1.0f / (float)(sr * sr);
  const bool pow2 = (sr & (sr - 1)) == 0;
  const float count = (float)(sr * sr);
  const unsigned sr_recip = (65536u + (unsigned)sr - 1u) / (unsigned)sr;      // j / sr == (j * sr_recip) >> 16 for j < 32, sr <= 32
  const int r0 = warp * band, r1 = min(H, r0 + band);
  const int4* __restrict__ hdr4 = reinterpret_cast<const int4*>(hdr);
  for (int pl = blockIdx.x; pl < B * C; pl += gridDim.x) {
    const int b = pl / C, c = pl - b * C;
    zero_plane(plane, H * W);
    __syncthreads();
    if (r0 < H) {
      auto issue = [&](HitLoads& L, int n) {
        const float* __restrict__ g = grad + ((int64_t)n * C + c) * NB;
        L.yy = lane < NYS ? __ldg(ys + (int64_t)n * NYS + lane) : make_uint2(0xffffffffu, 0u);
        L.e = lane < NXE ? __ldg(xe + (int64_t)n * NXE + lane) : make_uint2(0xffffffffu, 0u);
        L.gA = lane < NB ? __ldg(g + lane) : 0.f;
        L.gB = lane + 32 < NB ? __ldg(g + 32 + lane) : 0.f;
      };
      int4 hnext = make_int4(-1, 0, -1, 0);
      if (lane < K) hnext = __ldg(hdr4 + lane);
      for (int n0 = 0; n0 < K; n0 += 32) {
        const int4 h = hnext;
        hnext = make_int4(-1, 0, -1, 0);
        if (n0 + 32 + lane < K) hnext = __ldg(hdr4 + n0 + 32 + lane);           // next chunk's headers travel under this chunk's hits
        const bool hit = (n0 + lane < K) && h.x == b && h.y < r1 && h.z >= r0;
        unsigned m = __ballot_sync(0xffffffffu, hit);
        HitLoads cur, nxt;
        if (m) issue(cur, n0 + __ffs(m) - 1);
        while (m) {
          const int i = __ffs(m) - 1;
          m &= m - 1;
          if (m) issue(nxt, n0 + __ffs(m) - 1);
          const int flags = __shfl_sync(0xffffffffu, h.w, i);
          const int lo = (int)cur.yy.x;
          const float l = __uint_as_float(cur.yy.y);
          const bool inb = lo >= 0 && lo < r1 && (lo + (l > 0.f ? 1 : 0)) >= r0;
          unsigned mm = __ballot_sync(0xffffffffu, inb);
          const bool valid = cur.e.x != 0xffffffffu;
          const int col = (int)(cur.e.x & 0xffffu), pw = (int)(cur.e.x >> 16);
          const float wx = __uint_as_float(cur.e.y);
          bool leader = valid;
          unsigned group = 0u;
          if (flags & 1) {
            const unsigned same = __match_any_sync(0xffffffffu, valid ? col : 0x10000 + lane);
            group = valid ? same : 0u;
            leader = valid && (__ffs(same) - 1 == lane);
          }
          while (mm) {
            const int j = __ffs(mm) - 1;
            mm &= mm - 1;
            const int lo_j = __shfl_sync(0xffffffffu, lo, j);
            const float l_j = __shfl_sync(0xffffffffu, l, j);
            const int ph = (int)(((unsigned)j * sr_recip) >> 16);
            const int t = valid ? ph * PW + pw : 0;
            const float ga = __shfl_sync(0xffffffffu, cur.gA, t & 31), gb = __shfl_sync(0xffffffffu, cur.gB, t & 31);
            float gv = t < 32 ? ga : gb;
            gv = pow2 ? gv * inv_count : __fdiv_rn(gv, count);
            float a = wx * gv;
            if (flags & 1) a = ordered_group_sum(a, group);
            if (leader) {
              if (lo_j >= r0) plane[lo_j * W + col] += (1.f - l_j) * a;
              if (l_j > 0.f && lo_j + 1 >= r0 && lo_j + 1 < r1) plane[(lo_j + 1) * W + col] += l_j * a;
            }
          }
          cur = nxt;
        }
      }
    }
    __syncthreads();
    store_plane(grad_input + (int64_t)pl * H * W, plane, H * W);
    __syncthreads();
  }
}

// Non-deterministic sibling of the two kernels above (the default unless the caller asks for determinism): the plane is
// still resident, but RoIs are dealt to the warps round-robin and every tap is a shared-memory atomic add, so no work is
// repeated per band (the ownership scheme pays ~10 band hits per RoI).  The shared-memory atomics are cheap while contention
// is low - a warp's 28 taps of one line hit distinct columns.  The result differs
// from run to run only in the summation order, as the reference's own atomic kernel does.
__global__ void __launch_bounds__(kBwdThreads, 1)
roi_align_bwd_plane_atomic_kernel(const float* __restrict__ grad, const BwdHdr* __restrict__ hdr, const uint2* __restrict__ ys,
                                  const uint2* __restrict__ xe, float* __restrict__ grad_input, int B, int C, int H, int W, int K,
                                  int PH, int PW, int sr) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* plane = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, NW = blockDim.x >> 5;
  const int NYS = PH * sr, NXE = 2 * PW * sr, NB = PH * PW;
  const float inv_count = 1.0f / (float)(sr * sr);
  const bool pow2 = (sr & (sr - 1)) == 0;
  const float count = (float)(sr * sr);
  const unsigned sr_recip = (65536u + (unsigned)sr - 1u) / (unsigned)sr;
  for (int pl = blockIdx.x; pl < B * C; pl += gridDim.x) {
    const int b = pl / C, c = pl - b * C;
    zero_plane(plane, H * W);
    __syncthreads();
    auto issue = [&](HitLoads& L, int& batch, int n) {
      const float* __restrict__ g = grad + ((int64_t)n * C + c) * NB;
      batch = __ldg(&hdr[n].batch);
      L.yy = lane < NYS ? __ldg(ys + (int64_t)n * NYS + lane) : make_uint2(0xffffffffu, 0u);
      L.e = lane < NXE ? __ldg(xe + (int64_t)n * NXE + lane) : make_uint2(0xffffffffu, 0u);
      L.gA = lane < NB ? __ldg(g + lane) : 0.f;
      L.gB = lane + 32 < NB ? __ldg(g + 32 + lane) : 0.f;
    };
    HitLoads cur, nxt;
    int cur_b = -1, nxt_b = -1;
    if (warp < K) issue(cur, cur_b, warp);
    for (int n = warp; n < K; n += NW) {
      if (n + NW < K) issue(nxt, nxt_b, n + NW);
      if (cur_b == b) {
        const int lo = (int)cur.yy.x;
        const float l = __uint_as_float(cur.yy.y);
        const bool valid = cur.e.x != 0xffffffffu;
        const int col = (int)(cur.e.x & 0xffffu), pw = (int)(cur.e.x >> 16);
        const float wx = __uint_as_float(cur.e.y);
        unsigned mm = __ballot_sync(0xffffffffu, lo >= 0);
        int cur_ph = -1;
        float a = 0.f;
        while (mm) {
          const int j = __ffs(mm) - 1;
          mm &= mm - 1;
          const int lo_j = __shfl_sync(0xffffffffu, lo, j);
          const float l_j = __shfl_sync(0xffffffffu, l, j);
          const int ph = (int)(((unsigned)j * sr_recip) >> 16);
          if (ph != cur_ph) {                       // warp-uniform: a new bin row
            cur_ph = ph;
            const int t = valid ? ph * PW + pw : 0;
            const float ga = __shfl_sync(0xffffffffu, cur.gA, t & 31), gb = __shfl_sync(0xffffffffu, cur.gB, t & 31);
            const float gv = t < 32 ? ga : gb;
            a = wx * (pow2 ? gv * inv_count : __fdiv_rn(gv, count));
          }
          if (valid) {
            atomicAdd(plane + lo_j * W + col, (1.f - l_j) * a);
            if (l_j > 0.f) atomicAdd(plane + (lo_j + 1) * W + col, l_j * a);
          }
        }
      }
      cur = nxt;
      cur_b = nxt_b;
    }
    __syncthreads();
    store_plane(grad_input + (int64_t)pl * H * W, plane, H * W);
    __syncthreads();
  }
}

// ---- roi_pool backward, plane-resident -----------------------------------------------------------------------
// Rows that can hold an argmax of RoI n: [clamp(rsh), clamp(reh + 1)) (roi_pool_kernel.cu:43-58).
__global__ void roi_pool_bwd_hdr_kernel(const float* __restrict__ rois, BwdHdr* __restrict__ hdr, int K, int H, int PH, int PW,
                                        float scale) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= K) return;
  const PoolGeom<float> g = pool_geometry<float, float, float>(rois + (int64_t)n * 5, scale, PH, PW, 1);
  BwdHdr h;
  h.batch = g.batch;
  h.rmin = min(max(g.rsh, 0), H);
  h.rmax = min(max(g.rsh + g.rh + 1, 0), H) - 1;  // hend <= ceil(PH * RN(rh / PH)) + rsh <= rh + 1 + rsh (conservative by one row)
  h.flags = 0;
  hdr[n] = h;
}

__global__ void __launch_bounds__(kBwdThreads, 1)
roi_pool_bwd_plane_kernel(const float* __restrict__ grad, const int32_t* __restrict__ argmax, const BwdHdr* __restrict__ hdr,
                          float* __restrict__ grad_input, int B, int C, int H, int W, int K, int NB, int band) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* plane = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r0 = warp * band, r1 = min(H, r0 + band);
  for (int pl = blockIdx.x; pl < B * C; pl += gridDim.x) {
    const int b = pl / C, c = pl - b * C;
    zero_plane(plane, H * W);
    __syncthreads();
    if (r0 < H) {
      const int lo_idx = r0 * W, hi_idx = r1 * W;          // flat argmax range of this band
      for (int n0 = 0; n0 < K; n0 += 32) {
        const int nl = n0 + lane;
        bool hit = false;
        if (nl < K) {
          const int4 h = __ldg(reinterpret_cast<const int4*>(hdr) + nl);
          hit = h.x == b && h.y < r1 && h.z >= r0;
        }
        unsigned m = __ballot_sync(0xffffffffu, hit);
        while (m) {
          const int i = __ffs(m) - 1;
          m &= m - 1;
          const int64_t base = ((int64_t)(n0 + i) * C + c) * NB;
          for (int k0 = 0; k0 < NB; k0 += 32) {
            int am = -1;
            float gv = 0.f;
            if (k0 + lane < NB) { am = __ldg(argmax + base + k0 + lane); gv = __ldg(grad + base + k0 + lane); }
            const bool mine = am >= lo_idx && am < hi_idx;
            // overlapping bin windows may share their maximum: merge equal targets in lane (= bin) order
            const unsigned same = __match_any_sync(0xffffffffu, mine ? am : -2 - lane);
            const float sum = ordered_group_sum(gv, mine ? same : 0u);
            if (mine && (__ffs(same) - 1 == lane)) plane[am] += sum;
            __syncwarp();
          }
        }
      }
    }
    __syncthreads();
    store_plane(grad_input + (int64_t)pl * H * W, plane, H * W);
    __syncthreads();
  }
}

// ---- ps_roi_align backward, plane-resident -------------------------------------------------------------------
// Input plane c_in receives gradient from ONE bin position (ph, pw) of output channel c_out = c_in / (PH * PW),
// for every RoI (ps_roi_align_kernel.cu:68-140: c_in = (c_out * PH + ph) * PW + pw).  Lanes = the bin's
// sr (y samples) x 2 sr (x taps); per-(RoI, bin row) headers give the rows touched.
__global__ void ps_roi_align_bwd_hdr_kernel(const BwdHdr* __restrict__ hdr, const uint2* __restrict__ ys, BwdHdr* __restrict__ hdr_ph,
                                            int K, int PH, int sr) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= K * PH) return;
  const int n = t / PH, ph = t - n * PH;
  int rmin = 0x7fffffff, rmax = -1;
  for (int iy = 0; iy < sr; ++iy) {
    const uint2 yy = ys[(int64_t)n * PH * sr + ph * sr + iy];
    const int lo = (int)yy.x;
    if (lo >= 0) { rmin = min(rmin, lo); rmax = max(rmax, __uint_as_float(yy.y) > 0.f ? lo + 1 : lo); }
  }
  BwdHdr h;
  h.batch = hdr[n].batch; h.rmin = rmin; h.rmax = rmax; h.flags = 0;
  hdr_ph[t] = h;
}

__global__ void __launch_bounds__(kBwdThreads, 1)
ps_roi_align_bwd_plane_kernel(const float* __restrict__ grad, const BwdHdr* __restrict__ hdr_ph, const uint2* __restrict__ ys,
                              const uint2* __restrict__ xe, float* __restrict__ grad_input, int B, int C, int H, int W, int K,
                              int PH, int PW, int Cout, int sr, int band) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* plane = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NYS = PH * sr, NXE = 2 * PW * sr;
  const int r0 = warp * band, r1 = min(H, r0 + band);
  const bool pow2 = (sr & (sr - 1)) == 0;
  const float inv_count = 1.0f / (float)(sr * sr), count = (float)(sr * sr);
  const int ntap = sr * 2 * sr;                 // lanes of one bin: (iy, k)
  for (int pl = blockIdx.x; pl < B * C; pl += gridDim.x) {
    const int b = pl / C, c_in = pl - b * C;
    const int pw = c_in % PW, ph = (c_in / PW) % PH, co = c_in / (PW * PH);
    zero_plane(plane, H * W);
    __syncthreads();
    if (r0 < H && co < Cout) {
      for (int n0 = 0; n0 < K; n0 += 32) {
        const int nl = n0 + lane;
        bool hit = false;
        if (nl < K) {
          const int4 h = __ldg(reinterpret_cast<const int4*>(hdr_ph) + (int64_t)nl * PH + ph);
          hit = h.x == b && h.y < r1 && h.z >= r0;
        }
        unsigned m = __ballot_sync(0xffffffffu, hit);
        while (m) {
          const int i = __ffs(m) - 1;
          m &= m - 1;
          const int n = n0 + i;
          float gv = __ldg(grad + (((int64_t)n * Cout + co) * PH + ph) * PW + pw);
          gv = pow2 ? gv * inv_count : __fdiv_rn(gv, count);
          for (int t0 = 0; t0 < ntap; t0 += 32) {
            const int t = t0 + lane;
            int lo = -1, col = 0;
            float l = 0.f, wx = 0.f;
            bool valid = false;
            if (t < ntap) {
              const int iy = t / (2 * sr), k = t - iy * 2 * sr;
              const uint2 yy = __ldg(ys + (int64_t)n * NYS + ph * sr + iy);
              const uint2 e = __ldg(xe + (int64_t)n * NXE + pw * 2 * sr + k);
              lo = (int)yy.x; l = __uint_as_float(yy.y);
              valid = lo >= 0 && e.x != 0xffffffffu;
              col = (int)(e.x & 0xffffu); wx = __uint_as_float(e.y);
            }
            const float a = wx * gv;
#pragma unroll
            for (int cy = 0; cy < 2; ++cy) {
              const int row = lo + cy;
              const float wy = cy ? l : 1.f - l;
              const bool mine = valid && wy != 0.f && row >= r0 && row < r1;
              const int addr = row * W + col;
              const unsigned same = __match_any_sync(0xffffffffu, mine ? addr : -2 - lane);
              const float sum = ordered_group_sum(wy * a, mine ? same : 0u);
              if (mine && (__ffs(same) - 1 == lane)) plane[addr] += sum;
              __syncwarp();
            }
          }
        }
      }
    }
    __syncthreads();
    store_plane(grad_input + (int64_t)pl * H * W, plane, H * W);
    __syncthreads();
  }
}

// ---- generic atomic scatter (any dtype / adaptive sampling / plane too large) ---------------------------------
// CTA = (RoI, channel chunk).  The RoI's axis tables are built once per CTA in shared memory; threads stride over
// (channel, bin) and scatter with atomicAdd.  Not deterministic (neither is the reference).
constexpr int kGenAxis = 512;
template <typename T>
__global__ void __launch_bounds__(256)
roi_align_bwd_atomic_kernel(const T* __restrict__ grad, const T* __restrict__ rois, T* __restrict__ grad_input, int C, int H, int W,
                            int PH, int PW, typename Acc<T>::type scale, int sampling_ratio, int aligned, int ps, int Cgrad,
                            int ch_per_cta) {
  using A = typename Acc<T>::type;
  __shared__ int row_lo[kGenAxis], col_lo[kGenAxis];
  __shared__ A row_l[kGenAxis], col_l[kGenAxis];
  const int n = blockIdx.x, c0 = blockIdx.y * ch_per_cta;
  const RoiGeom<A> g = roi_geometry<T, A>(rois + (int64_t)n * 5, scale, PH, PW, sampling_ratio, aligned != 0, ps != 0);
  const int batch = g.batch, gh = g.gh, gw = g.gw;
  const A count = (A)(gh * gw);      // ps: may be <= 0 -> no samples at all; roi_align backward divides by gh*gw as the reference does
  const int nrow = PH * gh, ncol = PW * gw;
  const bool tab = nrow <= kGenAxis && ncol <= kGenAxis && nrow > 0 && ncol > 0;
  if (tab) {
    for (int i = threadIdx.x; i < nrow; i += blockDim.x) axis_lo<A>(sample_coord<A>(g.start_h, g.bin_h, i / gh, i % gh, gh), H, row_lo[i], row_l[i]);
    for (int i = threadIdx.x; i < ncol; i += blockDim.x) axis_lo<A>(sample_coord<A>(g.start_w, g.bin_w, i / gw, i % gw, gw), W, col_lo[i], col_l[i]);
    __syncthreads();
  }
  const int nbins = PH * PW;
  const int nch = min(ch_per_cta, Cgrad - c0);
  for (int i = threadIdx.x; i < nch * nbins; i += blockDim.x) {
    const int cl = i / nbins, bin = i - cl * nbins;
    const int ph = bin / PW, pw = bin - ph * PW;
    const int cg = c0 + cl;                                  // channel of grad (= c_out for ps)
    const int c_in = ps ? (cg * PH + ph) * PW + pw : cg;
    const A gbin = to_acc(grad[((int64_t)n * Cgrad + cg) * nbins + bin]);
    T* __restrict__ gi = grad_input + ((int64_t)batch * C + c_in) * H * W;
    for (int iy = 0; iy < gh; ++iy) {
      int ylo; A yl;
      if (tab) { ylo = row_lo[ph * gh + iy]; yl = row_l[ph * gh + iy]; }
      else axis_lo<A>(sample_coord<A>(g.start_h, g.bin_h, ph, iy, gh), H, ylo, yl);
      if (ylo < 0) continue;
      const int yhi = min(ylo + 1, H - 1);
      const A hy = sub_rn((A)1, yl);
      for (int ix = 0; ix < gw; ++ix) {
        int xlo; A xl;
        if (tab) { xlo = col_lo[pw * gw + ix]; xl = col_l[pw * gw + ix]; }
        else axis_lo<A>(sample_coord<A>(g.start_w, g.bin_w, pw, ix, gw), W, xlo, xl);
        if (xlo < 0) continue;
        const int xhi = min(xlo + 1, W - 1);
        const A hx = sub_rn((A)1, xl);
        // g_k = grad * w_k / count (roi_align_kernel.cu:296-299)
        atomic_add<T>(gi + ylo * W + xlo, div_rn(mul_rn(gbin, mul_rn(hy, hx)), count));
        atomic_add<T>(gi + ylo * W + xhi, div_rn(mul_rn(gbin, mul_rn(hy, xl)), count));
        atomic_add<T>(gi + yhi * W + xlo, div_rn(mul_rn(gbin, mul_rn(yl, hx)), count));
        atomic_add<T>(gi + yhi * W + xhi, div_rn(mul_rn(gbin, mul_rn(yl, xl)), count));
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
roi_pool_bwd_atomic_kernel(const T* __restrict__ grad, const T* __restrict__ rois, const int32_t* __restrict__ argmax,
                           T* __restrict__ grad_input, int64_t total, int C, int HW, int NB) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int am = argmax[i];
    if (am < 0) continue;
    const int64_t nc = i / NB;
    const int64_t n = nc / C;
    const int c = (int)(nc - n * C);
    const int batch = (int)to_acc(rois[n * 5]);
    atomic_add<T>(grad_input + ((int64_t)batch * C + c) * HW + am, to_acc(grad[i]));
  }
}

// backward of ps_roi_pool (ps_roi_pool_kernel.cu:80-142): grad / bin_area spread over the bin window (clipped to the
// full size here, as the reference's backward does) - an atomic scatter, one thread per (RoI, output element).
template <typename T>
__global__ void __launch_bounds__(256)
ps_roi_pool_bwd_kernel(const T* __restrict__ grad, const T* __restrict__ rois, T* __restrict__ grad_input, int64_t total, int C,
                       int H, int W, int PH, int PW, int Cout, typename Acc<T>::type scale) {
  using A = typename Acc<T>::type;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int pw = (int)(i % PW), ph = (int)((i / PW) % PH), co = (int)((i / PW / PH) % Cout);
    const int64_t n = i / PW / PH / Cout;
    const PoolGeom<A> g = pool_geometry<T, A, float>(rois + n * 5, scale, PH, PW, 0);
    int hs, he, ws, we;
    bin_window<T>(ph, g.bh, g.rsh, H, hs, he);
    bin_window<T>(pw, g.bw, g.rsw, W, ws, we);
    if (he <= hs || we <= ws) continue;
    const int c_in = (co * PH + ph) * PW + pw;
    const A v = rnd<T>(div_rn((A)to_acc(grad[i]), rnd<T>((A)((he - hs) * (we - ws)))));
    T* __restrict__ gi = grad_input + ((int64_t)g.batch * C + c_in) * H * W;
    for (int h = hs; h < he; ++h)
      for (int x = ws; x < we; ++x) atomic_add<T>(gi + h * W + x, v);
  }
}

struct BwdWs { BwdHdr* hdr; BwdHdr* hdr_ph; uint2* ys; uint2* xe; size_t total; };
BwdWs carve_bwd(void* base, int K, int PH, int PW, int sr) {
  Carver c(base);
  const int s = sr > 0 ? sr : 1;
  BwdWs w;
  w.hdr = c.take<BwdHdr>(K);
  w.hdr_ph = c.take<BwdHdr>((size_t)K * PH);
  w.ys = c.take<uint2>((size_t)K * PH * s);
  w.xe = c.take<uint2>((size_t)K * 2 * PW * s);
  w.total = c.off;
  return w;
}

// plane path: fp32, fixed sampling grid, plane fits shared memory, 16-bit column / bin fields
bool bwd_plane_ok(int dtype, int H, int W, int PH, int PW, int sr, bool need_sr) {
  if (dtype != VB200_F32) return false;
  if ((size_t)(((size_t)H * W + 3) & ~(size_t)3) * 4 + 1024 > (size_t)max_smem_optin()) return false;
  if (W >= 65536 || PW >= 65536 || H < 1 || W < 1) return false;
  if (need_sr && (sr < 1 || sr > 8)) return false;
  const char* force = env_override(ENV_ROI_BWD_PATH);      // "atomic" pins the generic kernel (testing)
  if (force && force[0] == 'a') return false;
  return true;
}

int bwd_band(int H) { return ceil_div(H, kBwdThreads / 32); }

}  // namespace
}  // namespace vb200

using namespace vb200;

extern "C" size_t vb200_roi_backward_workspace_bytes(int num_rois, int pooled_h, int pooled_w, int sampling_ratio) {
  if (num_rois <= 0) return 0;
  return carve_bwd(nullptr, num_rois, pooled_h, pooled_w, sampling_ratio).total;
}

extern "C" int vb200_roi_align_backward(const void* grad, const void* rois, void* grad_input, int dtype, int batch,
                                        int channels, int height, int width, int num_rois, int pooled_h, int pooled_w,
                                        double spatial_scale, int sampling_ratio, int aligned, int deterministic,
                                        void* workspace, size_t workspace_bytes, vb200_stream stream) {
  VB200_REQUIRE(batch >= 0 && channels >= 0 && height >= 0 && width >= 0 && num_rois >= 0, "roi_align_backward: negative size");
  VB200_REQUIRE(pooled_h > 0 && pooled_w > 0, "roi_align_backward: pooled size must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t in_elems = (int64_t)batch * channels * height * width;
  if (in_elems == 0) return 0;
  VB200_REQUIRE(grad_input, "roi_align_backward: null grad_input");
  VB200_REQUIRE(in_elems < (1ll << 31) && (int64_t)num_rois * channels * pooled_h * pooled_w < (1ll << 31),
                "roi_align_backward: tensor too large for 32-bit indexing");
  const size_t esize = dtype == VB200_F64 ? 8 : dtype == VB200_F16 ? 2 : 4;
  VB200_REQUIRE(dtype == VB200_F32 || dtype == VB200_F64 || dtype == VB200_F16, "roi_align_backward: unsupported dtype %d", dtype);
  if (num_rois == 0) { VB200_CUDA_TRY(cudaMemsetAsync(grad_input, 0, (size_t)in_elems * esize, st)); return 0; }
  VB200_REQUIRE(grad && rois, "roi_align_backward: null pointer");
  const BwdWs ws = carve_bwd(workspace, num_rois, pooled_h, pooled_w, sampling_ratio);
  if (bwd_plane_ok(dtype, height, width, pooled_h, pooled_w, sampling_ratio, true) && workspace && workspace_bytes >= ws.total) {
    roi_bwd_geometry_kernel<<<ceil_div(num_rois * 32, 256), 256, 0, st>>>((const float*)rois, ws.hdr, ws.ys, ws.xe, num_rois, height,
                                                                           width, pooled_h, pooled_w, sampling_ratio,
                                                                           (float)spatial_scale, aligned, 0);
    int rc = check_launch("roi_bwd_geometry_kernel");
    if (rc) return rc;
    const size_t smem = (((size_t)height * width + 3) & ~(size_t)3) * 4;
    const int planes = batch * channels;
    const int grid = planes < sm_count() ? planes : sm_count();
    const bool small_tables = pooled_h * sampling_ratio <= 32 && 2 * pooled_w * sampling_ratio <= 32 && pooled_h * pooled_w <= 64;
    if (small_tables && !deterministic) {
      VB200_CUDA_TRY(ensure_dyn_smem<roi_align_bwd_plane_atomic_kernel>(smem));
      roi_align_bwd_plane_atomic_kernel<<<grid, kBwdThreads, smem, st>>>((const float*)grad, ws.hdr, ws.ys, ws.xe,
                                                                        (float*)grad_input, batch, channels, height, width, num_rois,
                                                                        pooled_h, pooled_w, sampling_ratio);
      return check_launch("roi_align_bwd_plane_atomic_kernel");
    }
    if (small_tables) {
      VB200_CUDA_TRY(ensure_dyn_smem<roi_align_bwd_plane_fast_kernel>(smem));
      roi_align_bwd_plane_fast_kernel<<<grid, kBwdThreads, smem, st>>>((const float*)grad, ws.hdr, ws.ys, ws.xe, (float*)grad_input,
                                                                      batch, channels, height, width, num_rois, pooled_h, pooled_w,
                                                                      sampling_ratio, bwd_band(height));
      return check_launch("roi_align_bwd_plane_fast_kernel");
    }
    VB200_CUDA_TRY(ensure_dyn_smem<roi_align_bwd_plane_kernel>(smem));
    roi_align_bwd_plane_kernel<<<grid, kBwdThreads, smem, st>>>((const float*)grad, ws.hdr, ws.ys, ws.xe, (float*)grad_input, batch,
                                                               channels, height, width, num_rois, pooled_h, pooled_w, sampling_ratio,
                                                               bwd_band(height));
    return check_launch("roi_align_bwd_plane_kernel");
  }
  VB200_CUDA_TRY(cudaMemsetAsync(grad_input, 0, (size_t)in_elems * esize, st));
  const int ch_per_cta = channels >= 64 ? 32 : (channels >= 16 ? 16 : channels);
  dim3 grid((unsigned)num_rois, (unsigned)ceil_div(channels, ch_per_cta));
  return dispatch_roi_dtype(dtype, "roi_align_backward: unsupported dtype %d", [&](auto t) {
    using T = decltype(t);
    roi_align_bwd_atomic_kernel<T><<<grid, 256, 0, st>>>((const T*)grad, (const T*)rois, (T*)grad_input, channels, height, width,
                                                        pooled_h, pooled_w, (typename Acc<T>::type)spatial_scale, sampling_ratio,
                                                        aligned, 0, channels, ch_per_cta);
    return check_launch("roi_align_bwd_atomic_kernel");
  });
}

extern "C" int vb200_ps_roi_align_backward(const void* grad, const void* rois, const int32_t* channel_mapping, void* grad_input,
                                           int dtype, int batch, int channels, int height, int width, int num_rois, int pooled_h,
                                           int pooled_w, double spatial_scale, int sampling_ratio, int deterministic,
                                           void* workspace, size_t workspace_bytes, vb200_stream stream) {
  (void)channel_mapping;   // c_in = (c_out * PH + ph) * PW + pw by construction (ps_roi_align_kernel.cu:95); not re-read
  VB200_REQUIRE(pooled_h > 0 && pooled_w > 0, "ps_roi_align_backward: pooled size must be positive");
  VB200_REQUIRE(batch >= 0 && channels >= 0 && height >= 0 && width >= 0 && num_rois >= 0, "ps_roi_align_backward: negative size");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t in_elems = (int64_t)batch * channels * height * width;
  if (in_elems == 0) return 0;
  VB200_REQUIRE(grad_input, "ps_roi_align_backward: null grad_input");
  VB200_REQUIRE(in_elems < (1ll << 31), "ps_roi_align_backward: tensor too large for 32-bit indexing");
  VB200_REQUIRE(dtype == VB200_F32 || dtype == VB200_F64 || dtype == VB200_F16, "ps_roi_align_backward: unsupported dtype %d", dtype);
  const size_t esize = dtype == VB200_F64 ? 8 : dtype == VB200_F16 ? 2 : 4;
  const int Cout = channels / (pooled_h * pooled_w);
  if (num_rois == 0 || Cout == 0) { VB200_CUDA_TRY(cudaMemsetAsync(grad_input, 0, (size_t)in_elems * esize, st)); return 0; }
  VB200_REQUIRE(grad && rois, "ps_roi_align_backward: null pointer");
  const BwdWs ws = carve_bwd(workspace, num_rois, pooled_h, pooled_w, sampling_ratio);
  // One bin per (RoI, plane): the atomic scatter is the faster kernel here (sr*sr*4 atomics per output); the plane kernel is
  // the bit-reproducible one and runs when the caller asks for determinism.
  if (deterministic && bwd_plane_ok(dtype, height, width, pooled_h, pooled_w, sampling_ratio, true) && workspace &&
      workspace_bytes >= ws.total) {
    roi_bwd_geometry_kernel<<<ceil_div(num_rois * 32, 256), 256, 0, st>>>((const float*)rois, ws.hdr, ws.ys, ws.xe, num_rois, height,
                                                                           width, pooled_h, pooled_w, sampling_ratio,
                                                                           (float)spatial_scale, 1, 1);
    int rc = check_launch("roi_bwd_geometry_kernel");
    if (rc) return rc;
    ps_roi_align_bwd_hdr_kernel<<<ceil_div(num_rois * pooled_h, 256), 256, 0, st>>>(ws.hdr, ws.ys, ws.hdr_ph, num_rois, pooled_h,
                                                                                    sampling_ratio);
    rc = check_launch("ps_roi_align_bwd_hdr_kernel");
    if (rc) return rc;
    const size_t smem = (((size_t)height * width + 3) & ~(size_t)3) * 4;
    VB200_CUDA_TRY(ensure_dyn_smem<ps_roi_align_bwd_plane_kernel>(smem));
    const int planes = batch * channels;
    ps_roi_align_bwd_plane_kernel<<<planes < sm_count() ? planes : sm_count(), kBwdThreads, smem, st>>>(
        (const float*)grad, ws.hdr_ph, ws.ys, ws.xe, (float*)grad_input, batch, channels, height, width, num_rois, pooled_h,
        pooled_w, Cout, sampling_ratio, bwd_band(height));
    return check_launch("ps_roi_align_bwd_plane_kernel");
  }
  VB200_CUDA_TRY(cudaMemsetAsync(grad_input, 0, (size_t)in_elems * esize, st));
  const int ch_per_cta = Cout >= 64 ? 32 : (Cout >= 16 ? 16 : Cout);
  dim3 grid((unsigned)num_rois, (unsigned)ceil_div(Cout, ch_per_cta));
  return dispatch_roi_dtype(dtype, "ps_roi_align_backward: unsupported dtype %d", [&](auto t) {
    using T = decltype(t);
    roi_align_bwd_atomic_kernel<T><<<grid, 256, 0, st>>>((const T*)grad, (const T*)rois, (T*)grad_input, channels, height, width,
                                                        pooled_h, pooled_w, (typename Acc<T>::type)spatial_scale, sampling_ratio,
                                                        1, 1, Cout, ch_per_cta);
    return check_launch("roi_align_bwd_atomic_kernel");
  });
}

extern "C" int vb200_roi_pool_backward(const void* grad, const void* rois, const int32_t* argmax, void* grad_input, int dtype,
                                       int batch, int channels, int height, int width, int num_rois, int pooled_h, int pooled_w,
                                       double spatial_scale, int deterministic, void* workspace, size_t workspace_bytes,
                                       vb200_stream stream) {
  VB200_REQUIRE(pooled_h > 0 && pooled_w > 0, "roi_pool_backward: pooled size must be positive");
  VB200_REQUIRE(batch >= 0 && channels >= 0 && height >= 0 && width >= 0 && num_rois >= 0, "roi_pool_backward: negative size");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t in_elems = (int64_t)batch * channels * height * width;
  if (in_elems == 0) return 0;
  VB200_REQUIRE(grad_input, "roi_pool_backward: null grad_input");
  VB200_REQUIRE(in_elems < (1ll << 31), "roi_pool_backward: tensor too large for 32-bit indexing");
  VB200_REQUIRE(dtype == VB200_F32 || dtype == VB200_F64 || dtype == VB200_F16, "roi_pool_backward: unsupported dtype %d", dtype);
  const size_t esize = dtype == VB200_F64 ? 8 : dtype == VB200_F16 ? 2 : 4;
  if (num_rois == 0) { VB200_CUDA_TRY(cudaMemsetAsync(grad_input, 0, (size_t)in_elems * esize, st)); return 0; }
  VB200_REQUIRE(grad && rois && argmax, "roi_pool_backward: null pointer");
  const BwdWs ws = carve_bwd(workspace, num_rois, pooled_h, pooled_w, 1);
  // one atomic per output element is hard to beat; the plane kernel is the bit-reproducible alternative
  if (deterministic && bwd_plane_ok(dtype, height, width, pooled_h, pooled_w, 1, false) && workspace && workspace_bytes >= ws.total) {
    roi_pool_bwd_hdr_kernel<<<ceil_div(num_rois, 256), 256, 0, st>>>((const float*)rois, ws.hdr, num_rois, height, pooled_h, pooled_w,
                                                                     (float)spatial_scale);
    int rc = check_launch("roi_pool_bwd_hdr_kernel");
    if (rc) return rc;
    const size_t smem = (((size_t)height * width + 3) & ~(size_t)3) * 4;
    VB200_CUDA_TRY(ensure_dyn_smem<roi_pool_bwd_plane_kernel>(smem));
    const int planes = batch * channels;
    roi_pool_bwd_plane_kernel<<<planes < sm_count() ? planes : sm_count(), kBwdThreads, smem, st>>>(
        (const float*)grad, argmax, ws.hdr, (float*)grad_input, batch, channels, height, width, num_rois, pooled_h * pooled_w,
        bwd_band(height));
    return check_launch("roi_pool_bwd_plane_kernel");
  }
  VB200_CUDA_TRY(cudaMemsetAsync(grad_input, 0, (size_t)in_elems * esize, st));
  const int64_t total = (int64_t)num_rois * channels * pooled_h * pooled_w;
  const int grid = (int)(ceil_div64(total, 256) < (int64_t)sm_count() * 16 ? ceil_div64(total, 256) : (int64_t)sm_count() * 16);
  return dispatch_roi_dtype(dtype, "roi_pool_backward: unsupported dtype %d", [&](auto t) {
    using T = decltype(t);
    roi_pool_bwd_atomic_kernel<T><<<grid, 256, 0, st>>>((const T*)grad, (const T*)rois, argmax, (T*)grad_input, total, channels,
                                                       height * width, pooled_h * pooled_w);
    return check_launch("roi_pool_bwd_atomic_kernel");
  });
}

extern "C" int vb200_ps_roi_pool_backward(const void* grad, const void* rois, void* grad_input, int dtype, int batch, int channels,
                                          int height, int width, int num_rois, int pooled_h, int pooled_w, double spatial_scale,
                                          vb200_stream stream) {
  VB200_REQUIRE(pooled_h > 0 && pooled_w > 0, "ps_roi_pool_backward: pooled size must be positive");
  const int64_t in_elems = (int64_t)batch * channels * height * width;
  if (in_elems == 0) return 0;
  VB200_REQUIRE(grad_input, "ps_roi_pool_backward: null grad_input");
  VB200_REQUIRE(in_elems < (1ll << 31), "ps_roi_pool_backward: tensor too large for 32-bit indexing");
  VB200_REQUIRE(dtype == VB200_F32 || dtype == VB200_F64 || dtype == VB200_F16, "ps_roi_pool_backward: unsupported dtype %d", dtype);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t esize = dtype == VB200_F64 ? 8 : dtype == VB200_F16 ? 2 : 4;
  VB200_CUDA_TRY(cudaMemsetAsync(grad_input, 0, (size_t)in_elems * esize, st));
  const int Cout = channels / (pooled_h * pooled_w);
  const int64_t total = (int64_t)num_rois * Cout * pooled_h * pooled_w;
  if (total == 0) return 0;
  VB200_REQUIRE(grad && rois, "ps_roi_pool_backward: null pointer");
  const int grid = (int)(ceil_div64(total, 256) < (int64_t)sm_count() * 16 ? ceil_div64(total, 256) : (int64_t)sm_count() * 16);
  return dispatch_roi_dtype(dtype, "ps_roi_pool_backward: unsupported dtype %d", [&](auto t) {
    using T = decltype(t);
    ps_roi_pool_bwd_kernel<T><<<grid, 256, 0, st>>>((const T*)grad, (const T*)rois, (T*)grad_input, total, channels, height, width,
                                                   pooled_h, pooled_w, Cout, (typename Acc<T>::type)spatial_scale);
    return check_launch("ps_roi_pool_bwd_kernel");
  });
}
