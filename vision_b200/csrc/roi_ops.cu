// roi_ops.cu — roi_align (plain, fused all-gather, MultiScaleRoIAlign) / roi_pool / ps_roi_align / ps_roi_pool forward
// for sm_90a.  The backward kernels are in roi_backward.cu, the reference's RoI arithmetic both share in roi_geometry.cuh.
//
// Reference semantics (pytorch/vision):
//   roi_align     csrc/ops/cuda/roi_align_kernel.cu:14-143   (CPU: cpu/roi_align_kernel.cpp:18-115,
//                                                             cpu/roi_align_common.h:32-124)
//   roi_pool      csrc/ops/cuda/roi_pool_kernel.cu:15-78     (CPU: cpu/roi_pool_kernel.cpp:24-92)
//   ps_roi_align  csrc/ops/cuda/ps_roi_align_kernel.cu:68-140 (CPU: cpu/ps_roi_align_kernel.cpp:73-151)
//   ps_roi_pool   csrc/ops/cuda/ps_roi_pool_kernel.cu:15-78
//
// Design (not a port — the reference runs one thread per output element and
// recomputes the RoI geometry K*C*PH*PW times):
//   * bilinear sampling is separable, so the geometry of a RoI is PH*gh row
//     entries + PW*gw column entries; it is computed ONCE per RoI with the
//     reference's exact (uncontracted, round-to-nearest) coordinate arithmetic;
//   * generic kernel: CTA = (RoI, channel chunk), geometry table in shared
//     memory, threads stride over (channel, bin) so output stores are coalesced;
//   * plane-resident kernels (fp32, fixed sampling_ratio, plane <= ~220 KB):
//     persistent CTAs hold one whole H*W channel plane in shared memory, every
//     gather is an LDS, each input byte leaves HBM once and each output byte is
//     written once.  Two lane mappings: thread-per-bin (any pooled size,
//     sampling_ratio 1..4; bank-conflict bound) and line-wise (7x7 bins,
//     sampling_ratio 2: a warp owns one RoI, its lanes are the taps of one line
//     of the sampling grid, so an LDS reads one image row or column).
#include "async_copy.cuh"
#include "common.cuh"
#include "roi_geometry.cuh"

namespace vb200 {
namespace {

constexpr int kMaxAxisEnt = 512;   // per-axis table capacity of the generic kernel

template <typename T>
__global__ void __launch_bounds__(256)
roi_align_generic_kernel(const T* __restrict__ input, const T* __restrict__ rois, T* __restrict__ output,
                         int C, int H, int W, int PH, int PW, typename Acc<T>::type scale,
                         int sampling_ratio, int aligned, int ch_per_cta) {
  using A = typename Acc<T>::type;
  __shared__ AxisEnt<A> rowtab[kMaxAxisEnt];
  __shared__ AxisEnt<A> coltab[kMaxAxisEnt];

  const int n = blockIdx.x;
  const int c0 = blockIdx.y * ch_per_cta;
  const int nch = min(ch_per_cta, C - c0);
  const RoiGeom<A> g = roi_geometry<T, A>(rois + (int64_t)n * 5, scale, PH, PW, sampling_ratio, aligned != 0, false);
  const int nrow = PH * g.gh, ncol = PW * g.gw;
  const bool tab = nrow <= kMaxAxisEnt && ncol <= kMaxAxisEnt;   // CTA-uniform
  if (tab) {
    for (int i = threadIdx.x; i < nrow; i += blockDim.x)
      rowtab[i] = axis_entry<A>(sample_coord<A>(g.start_h, g.bin_h, i / g.gh, i % g.gh, g.gh), H);
    for (int i = threadIdx.x; i < ncol; i += blockDim.x)
      coltab[i] = axis_entry<A>(sample_coord<A>(g.start_w, g.bin_w, i / g.gw, i % g.gw, g.gw), W);
    __syncthreads();
  }
  const int nbins = PH * PW;
  const int64_t plane = (int64_t)H * W;
  for (int i = threadIdx.x; i < nch * nbins; i += blockDim.x) {
    const int cl = i / nbins, bin = i - cl * nbins;
    const int ph = bin / PW, pw = bin - ph * PW;
    const DensePlane<T> in{input + ((int64_t)g.batch * C + (c0 + cl)) * plane, W};
    const A sum = roi_align_bin<A>(in, H, W, g, ph, pw, tab, rowtab, coltab);
    output[((int64_t)n * C + (c0 + cl)) * nbins + bin] = from_acc<T, A>(sum);
  }
}

// ---------------------------------------------------------------------------
// Plane-resident fp32 path.
// ---------------------------------------------------------------------------
// Shared-memory image of one channel plane: rows at a padded pitch (a multiple of 4 floats whose
// quarter is odd, so consecutive rows rotate through all eight 16-byte bank groups), pad columns
// and two extra rows are zero.  Geometry entries are (offset, l) only, encoded by packed_axis.
struct PackedEnt { uint32_t off; float l; };   // off in floats (row entries: row * pitch)

__host__ __device__ inline int plane_pitch(int W) {
  int p = (W + 2 + 3) & ~3;
  if (((p >> 2) & 1) == 0) p += 4;
  return p;
}

__global__ void roi_align_geometry_kernel(const float* __restrict__ rois, PackedEnt* __restrict__ geo,
                                          int32_t* __restrict__ roi_batch, int K, int H, int W, int PH,
                                          int PW, float scale, int sr, int aligned, int pitch) {
  const int ent_per_roi = (PH + PW) * sr;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= K * ent_per_roi) return;
  const int n = t / ent_per_roi, e = t - n * ent_per_roi;
  const RoiGeom<float> g = roi_geometry<float, float>(rois + (int64_t)n * 5, scale, PH, PW, sr, aligned != 0, false);
  if (e == 0) roi_batch[n] = g.batch;
  const bool is_row = e < PH * sr;
  const int f = is_row ? e : e - PH * sr;
  const int size = is_row ? H : W;
  const AxisEnt<float> a = is_row ? axis_entry<float>(sample_coord<float>(g.start_h, g.bin_h, f / sr, f % sr, sr), H)
                                  : axis_entry<float>(sample_coord<float>(g.start_w, g.bin_w, f / sr, f % sr, sr), W);
  int lo; float l;
  packed_axis(a, size, lo, l);
  PackedEnt pe;
  pe.off = (uint32_t)(is_row ? lo * pitch : lo);
  pe.l = l;
  geo[t] = pe;
}

constexpr int kPlaneMaxThreads = 1024;

// A thread's SR row entries and SR column entries of one RoI.  Entries of one bin row / column are
// adjacent, and for even SR their group is 16-byte aligned (ent_per_roi * 8 B and SR * 8 B are
// multiples of 16): two 128-bit loads instead of four 64-bit ones for the common SR = 2.
template <int SR>
__device__ __forceinline__ void load_entries(const PackedEnt* __restrict__ ge_, int gy, int gx, uint2 (&ey)[SR], uint2 (&ex)[SR]) {
  if constexpr (SR % 2 == 0) {
    const uint4* gy4 = reinterpret_cast<const uint4*>(ge_ + gy);
    const uint4* gx4 = reinterpret_cast<const uint4*>(ge_ + gx);
#pragma unroll
    for (int i = 0; i < SR / 2; ++i) {
      const uint4 a = __ldg(gy4 + i), b = __ldg(gx4 + i);
      ey[2 * i] = make_uint2(a.x, a.y); ey[2 * i + 1] = make_uint2(a.z, a.w);
      ex[2 * i] = make_uint2(b.x, b.y); ex[2 * i + 1] = make_uint2(b.z, b.w);
    }
  } else {
    const uint2* ge = reinterpret_cast<const uint2*>(ge_);
#pragma unroll
    for (int i = 0; i < SR; ++i) { ey[i] = __ldg(ge + gy + i); ex[i] = __ldg(ge + gx + i); }
  }
}

// Plane-major work split of the plane kernels: all (plane, RoI) pairs in plane-major order, cut evenly over the persistent
// CTAs.  A CTA walks its spans, one per plane it enters - RoIs [r0, r1) of plane pl = b * C + c - so it stages a plane only
// when its range enters it.  roi_align_plane_kernel splits the same way inline: through this helper it compiles to 2 more
// registers for sampling_ratio 2.
struct PlaneSpans {
  int64_t w, w1;
  int K, pl, r0, r1;
  __device__ __forceinline__ PlaneSpans(int B, int C, int K_) : K(K_) {
    const int64_t total = (int64_t)B * C * K;
    const int64_t per = (total + gridDim.x - 1) / gridDim.x;
    w = (int64_t)blockIdx.x * per;
    w1 = min(total, w + per);
  }
  __device__ __forceinline__ bool more() {
    if (w >= w1) return false;
    pl = (int)(w / K);
    r0 = (int)(w - (int64_t)pl * K);
    r1 = (int)min((int64_t)K, r0 + (w1 - w));
    return true;
  }
  __device__ __forceinline__ void advance() { w += r1 - r0; }
};

// Work split as PlaneSpans.  blockDim.x = NT = a multiple of nbins, so a thread keeps ONE bin position (ph, pw) for its
// whole life and walks RoIs with a fixed stride: no index arithmetic in the loop, geometry for the next RoI is prefetched.
template <int SR>
__global__ void __launch_bounds__(kPlaneMaxThreads, 1)
roi_align_plane_kernel(const float* __restrict__ input, const PackedEnt* __restrict__ geo,
                       const int32_t* __restrict__ roi_batch, float* __restrict__ output,
                       int B, int C, int H, int W, int K, int PH, int PW, int pitch) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* plane = reinterpret_cast<float*>(smem_raw);
  __shared__ uint64_t bar;

  const int tid = threadIdx.x, NT = blockDim.x;
  const int nbins = PH * PW;
  const int ent_per_roi = (PH + PW) * SR;
  const int bin = tid % nbins, rl0 = tid / nbins, rstep = NT / nbins;
  const int ph = bin / PW, pw = bin - ph * PW;
  const int gy = ph * SR, gx = PH * SR + pw * SR;
  const float inv_count = 1.0f / (float)(SR * SR);
  const float count = (float)(SR * SR);
  const bool pow2 = (SR & (SR - 1)) == 0;
  const int64_t total = (int64_t)B * C * K;
  const int64_t per = (total + gridDim.x - 1) / gridDim.x;
  const int64_t w0 = (int64_t)blockIdx.x * per;
  const int64_t w1 = min(total, w0 + per);

  // zero the pad columns and the two zero rows once (bulk copies only ever write [0, W) of rows < H)
  for (int r = tid; r < H; r += NT)
    for (int c = W; c < pitch; ++c) plane[r * pitch + c] = 0.f;
  for (int i = H * pitch + tid; i < (H + 2) * pitch + 2; i += NT) plane[i] = 0.f;
  if (tid == 0) { mbar_init(&bar, 1); mbar_fence_init(); }
  fence_proxy_async();
  __syncthreads();
  uint32_t parity = 0;
  const uint32_t row_bytes = (uint32_t)W * 4u;

  int64_t w = w0;
  while (w < w1) {
    const int pl = (int)(w / K);              // plane index = b * C + c
    const int r0 = (int)(w - (int64_t)pl * K);
    const int r1 = (int)min((int64_t)K, r0 + (w1 - w));
    const int b = pl / C;
    // ---- stage plane `pl`: one bulk copy per row, issued by warp 0, all completing on `bar` ----
    if (tid < 32) {
      if (tid == 0) { fence_proxy_async(); mbar_expect_tx(&bar, row_bytes * (uint32_t)H); }
      __syncwarp();
      const float* src = input + (int64_t)pl * H * W;
      for (int r = tid; r < H; r += 32) bulk_g2s(plane + r * pitch, src + (int64_t)r * W, row_bytes, &bar);
    }
    mbar_wait(&bar, parity);
    parity ^= 1u;

    int n = r0 + rl0;
    uint2 ey[SR], ex[SR];
    if (n < r1) load_entries<SR>(geo + (int64_t)n * ent_per_roi, gy, gx, ey, ex);
    float* __restrict__ outp = output + ((int64_t)n * C + (pl - b * C)) * nbins + bin;
    const int64_t ostep = (int64_t)rstep * C * nbins;
    for (; n < r1; n += rstep, outp += ostep) {
      uint2 cy[SR], cx[SR];
#pragma unroll
      for (int i = 0; i < SR; ++i) { cy[i] = ey[i]; cx[i] = ex[i]; }
      const int nn = n + rstep;
      if (nn < r1) load_entries<SR>(geo + (int64_t)nn * ent_per_roi, gy, gx, ey, ex);   // prefetch next RoI
      if (B > 1 && __ldg(roi_batch + n) != b) continue;
      float sum = 0.f;
#pragma unroll
      for (int iy = 0; iy < SR; ++iy) {
        const float ly = __uint_as_float(cy[iy].y), hy = 1.f - ly;
        const float* __restrict__ rowp = plane + cy[iy].x;
#pragma unroll
        for (int ix = 0; ix < SR; ++ix) {
          const float lx = __uint_as_float(cx[ix].y), hx = 1.f - lx;
          const float* __restrict__ q = rowp + cx[ix].x;
          const float v1 = q[0], v2 = q[1];
          const float v3 = q[pitch], v4 = q[pitch + 1];
          const float top = fmaf(lx, v2, hx * v1);
          const float bot = fmaf(lx, v4, hx * v3);
          sum = fmaf(hy, top, sum);
          sum = fmaf(ly, bot, sum);
        }
      }
      *outp = pow2 ? sum * inv_count : __fdiv_rn(sum, count);
    }
    __syncthreads();   // plane buffer may be overwritten by the next bulk copies
    w += (r1 - r0);
  }
}

// ---------------------------------------------------------------------------
// Plane-resident path, line-wise lanes (P x P bins, SR x SR samples, P*SR*2 <= 32).
// ---------------------------------------------------------------------------
// The thread-per-bin kernel above is bound by shared-memory bank conflicts: its 32 lanes read
// ~5 bin rows x 7 bin columns, i.e. random banks (3.2 wavefronts per LDS).  Here a warp owns one
// (RoI, plane) pair and its lanes are the P*SR*2 taps of ONE line of the sampling grid: lane
// (j, c) = tap c of sample j along the "lane axis".  The other ("loop") axis is walked by all
// lanes together, so one LDS reads 28 words of a single image row (lane axis = x) or a single
// image column (lane axis = y, conflict-free over any 32 consecutive rows because the pitch is
// odd).  The geometry kernel picks, per RoI, the axis with fewer conflicts (simulation on cfg2:
// 1.39 wavefronts per LDS vs 3.1).  Weights factor the same way: the lane-axis weight is a lane
// constant, the loop-axis pair (1-l, l) is warp-uniform.  The P*SR*2 lanes of a bin column are
// folded with a 2-step exchange that leaves each lane with two finished bins, stored directly.
struct LineTab {            // per RoI, 96 words
  uint2 lane[32];           // (BYTE offset | lane_is_y, weight) of this lane's tap; lanes >= P*SR*2: (lane 0's, 0)
  uint2 loop[14];           // (BYTE offset of the low tap, l) per loop-axis sample
  uint32_t lane_is_y;       // 0: lanes walk x, loop walks y (neighbour at +pitch); 1: the transpose
  int32_t batch;
  uint32_t pad[2];
};
static_assert(sizeof(LineTab) == 384, "LineTab layout");

__host__ __device__ inline int line_pitch(int W) { return (W + 2) | 1; }   // odd, >= W + 2 zero columns

// Max number of DISTINCT addresses of the active lanes that share a bank.
__device__ __forceinline__ int bank_multiplicity(uint32_t addr, bool active, int lane) {
  const unsigned same = __match_any_sync(0xffffffffu, active ? addr : 0xffffffffu - lane);
  const bool leader = active && (__ffs(same) - 1 == lane);
  const unsigned bank = __match_any_sync(0xffffffffu, leader ? (addr & 31u) : 64u + lane);
  int m = leader ? __popc(bank) : 0;
#pragma unroll
  for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  return m;
}

// Feature levels of the fused MultiScaleRoIAlign (torchvision/ops/poolers.py:147-228): passed by value.
constexpr int kMaxLevels = 8;
struct LevelDesc { const float* base; int H, W, pitch; float scale; };
struct LevelSet {
  LevelDesc lv[kMaxLevels];
  int num_levels;
  // LevelMapper (poolers.py:47-84): floor(lvl0 + log2(sqrt(area) / s0) + eps) clamped to [k_min, k_max], minus k_min
  int k_min, k_max;
  float inv_s0, lvl0, eps;
};

// The reference evaluates the mapper as a chain of fp32 tensor ops; each step below is one of them, rounded once.
__device__ __forceinline__ int map_level(const float* __restrict__ box /* x1 y1 x2 y2 */, const LevelSet& L) {
  const float area = mul_rn(sub_rn(box[2], box[0]), sub_rn(box[3], box[1]));    // box_area (boxes.py: (x2-x1)*(y2-y1))
  const float sq = sqrtf(area);                                                   // correctly rounded
  float t = add_rn(add_rn(L.lvl0, log2f(mul_rn(sq, L.inv_s0))), L.eps);   // torch's CUDA tensor / python-scalar is a * (1 / b)
  t = floorf(t);
  if (t != t) return -1;        // inverted box: NaN level matches no `levels == level` test in the reference -> its row stays zero
  t = fminf(fmaxf(t, (float)L.k_min), (float)L.k_max);
  return min(max((int)t - L.k_min, 0), L.num_levels - 1);
}

template <int P, int SR, bool MULTI>
__global__ void __launch_bounds__(256)
roi_align_line_geometry_kernel(const float* __restrict__ rois, LineTab* __restrict__ tab, int K, int H, int W,
                               float scale, int aligned, int pitch, int B, LevelSet L,
                               int* __restrict__ lvl_count, int* __restrict__ bucket, int32_t* __restrict__ lvl_out) {
  constexpr int NS = P * SR, NL = NS * 2;
  asm volatile("griddepcontrol.launch_dependents;");   // the gather kernel may start staging its first plane
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (n >= K) return;
  bool dead = false;        // RoIs the reference leaves at zero (no level) or reads out of bounds for (bad batch index): all-zero weights
  if (MULTI) {
    int lvl = map_level(rois + (int64_t)n * 5 + 1, L);
    if (lvl < 0) { dead = true; lvl = 0; }
    H = L.lv[lvl].H; W = L.lv[lvl].W; pitch = L.lv[lvl].pitch; scale = L.lv[lvl].scale;
    if (lane == 0) {
      bucket[(int64_t)lvl * K + atomicAdd(lvl_count + lvl, 1)] = n;     // order inside a level is irrelevant: outputs are addressed by RoI id
      lvl_out[n] = lvl;
    }
  }
  RoiGeom<float> g = roi_geometry<float, float>(rois + (int64_t)n * 5, scale, P, P, SR, aligned != 0, false);
  if (g.batch < 0 || g.batch >= B) { dead = true; g.batch = 0; }
  const bool act = lane < NL;
  const int j = act ? lane >> 1 : 0, c = lane & 1;
  int xlo, ylo; float xl, yl;
  packed_axis(axis_entry<float>(sample_coord<float>(g.start_w, g.bin_w, j / SR, j % SR, SR), W), W, xlo, xl);
  packed_axis(axis_entry<float>(sample_coord<float>(g.start_h, g.bin_h, j / SR, j % SR, SR), H), H, ylo, yl);
  const uint32_t ax = (uint32_t)(xlo + c), ay = (uint32_t)((ylo + c) * pitch);
  const int mx = bank_multiplicity(ax, act, lane), my = bank_multiplicity(ay, act, lane);
  const bool lane_is_y = my < mx;
  LineTab* t = tab + n;
  const float l = lane_is_y ? yl : xl;
  // lanes beyond the taps repeat lane 0's address with weight 0: a broadcast, never an extra bank conflict
  const uint32_t my_off = (lane_is_y ? ay : ax) * 4u + (lane_is_y ? 1u : 0u);   // bit 0: lane axis
  const uint32_t off0 = __shfl_sync(0xffffffffu, my_off, 0);
  t->lane[lane] = (act && !dead) ? make_uint2(my_off, __float_as_uint(c ? l : 1.f - l)) : make_uint2(act ? my_off : off0, 0u);
  if (lane < NS) {   // loop-axis sample `lane`
    int lo; float ll;
    if (lane_is_y) packed_axis(axis_entry<float>(sample_coord<float>(g.start_w, g.bin_w, lane / SR, lane % SR, SR), W), W, lo, ll);
    else packed_axis(axis_entry<float>(sample_coord<float>(g.start_h, g.bin_h, lane / SR, lane % SR, SR), H), H, lo, ll);
    t->loop[lane] = make_uint2((uint32_t)(lane_is_y ? lo : lo * pitch) * 4u, __float_as_uint(ll));
  }
  if (lane == 0) { t->lane_is_y = lane_is_y; t->batch = g.batch; }
}

__device__ __forceinline__ void cp_async4(uint32_t dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint4 lds_u128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

// Destinations of the fused all-gather (vb200_roi_align_forward_gather): besides `output` (the caller's slot of its own gathered
// buffer) every finished bin is stored to the same slot of the peers' buffers - `n` peer-mapped pointers, or ONE NVSwitch
// multicast address `mc` (multimem.st: the switch replicates the store to every rank, the local one included).
struct PeerDst { float* dst[7]; float* mc; int n; };

// Which of those destinations the line kernel stores to, fixed at compile time so the single-GPU kernel carries no
// per-item destination tests and no PeerDst array: `output` alone, `output` plus the pd.n peer copies, or pd.mc alone.
enum LineDst { kLineLocal = 0, kLinePeers = 1, kLineMulticast = 2 };

constexpr int kLineThreads = 1024;
constexpr int kLineStageBytes = (kLineThreads / 32) * 2 * 128;   // per warp: two 128-byte slots (loop entries + header)

__host__ __device__ inline size_t line_plane_bytes(int H, int pitch) { return (((size_t)(H + 2) * pitch * 4) + 15) & ~(size_t)15; }

// MULTI: fused MultiScaleRoIAlign - the work list runs over the planes of ALL feature levels (each level has its own
// H, W, pitch and RoI bucket, filled by the geometry kernel's device-side LevelMapper); outputs are addressed by RoI id,
// so there is no per-level gather / scatter / zero-fill pass.
template <int P, int SR, bool MULTI, int DST>
__global__ void __launch_bounds__(kLineThreads, 1)
roi_align_line_kernel(const float* __restrict__ input, const LineTab* __restrict__ tab, float* __restrict__ output,
                      int B, int C, int H, int W, int K, int pitch, LevelSet L, const int* __restrict__ lvl_count,
                      const int* __restrict__ bucket, PeerDst pd) {
  constexpr int NS = P * SR, NL = NS * 2, NB = P * P;
  static_assert(NL <= 32 && SR == 2 && P <= 8 && NS == 14, "lane mapping: 4 lanes per bin column, two finished bins per lane");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* plane = reinterpret_cast<float*>(smem_raw);
  const uint32_t plane_s = smem_u32(plane);

  // blockDim.x == kLineThreads.  The warp index is read through a shuffle from lane 0 so that the compiler knows it is
  // warp-uniform: the item loop's trip count then is too, and its __syncwarp / shuffles need no divergence checks.
  constexpr int NW = kLineThreads / 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  // the per-warp staging slots sit behind the LARGEST plane of the call
  int Hmax = H, pmax = pitch;
  if (MULTI) {
    size_t best = 0;
    for (int l = 0; l < L.num_levels; ++l) {
      const size_t bts = line_plane_bytes(L.lv[l].H, L.lv[l].pitch);
      if (bts > best) { best = bts; Hmax = L.lv[l].H; pmax = L.lv[l].pitch; }
    }
  }
  // this warp's two 128-byte staging slots; `slot` is the current one, slot ^ slot_x the other
  const uint32_t stage_s = plane_s + (uint32_t)line_plane_bytes(Hmax, pmax) + (uint32_t)warp * 256u;
  const uint32_t slot_x = stage_s ^ (stage_s + 128u);
  const uint32_t lane4 = __shfl_sync(0xffffffffu, (uint32_t)lane * 4u, lane);   // opaque for the same reason as lane_code
  const bool multi_batch = B > 1;

  const int q = lane & 3, grp = lane >> 2;
  const bool hi = (q & 2) != 0, lo = (q & 1) != 0;
  const float inv_count = 1.0f / (float)(SR * SR);
  // output offsets of this lane's two finished bins (loop-axis bins 2q, 2q+1 of lane group grp)
  const uint32_t off_x = 2 * q * P + grp, off_y = 2 * q + grp * P;   // lane axis x: bin = k * P + grp; y: the transpose
  const bool st0 = grp < P && 2 * q < P, st1 = grp < P && 2 * q + 1 < P;
  // ... packed into one register, which the item loop keeps instead of re-deriving them from the lane index per item:
  // byte 0 / 1 = the first bin's offset with the lanes along x / y, bit 16 / 17 = the lane stores its first / second bin
  // (passed through an identity shuffle: otherwise the compiler re-derives it from threadIdx.x in every item)
  const uint32_t lane_code = __shfl_sync(0xffffffffu, off_x | off_y << 8 | (uint32_t)st0 << 16 | (uint32_t)st1 << 17, lane);

  // Work is split evenly in COST units.  Single level: cost = (plane, RoI) pairs.  MULTI: a plane of level l costs
  // K_l + O_l, O_l = the fixed price of switching to it (two barriers, the load latency, its bytes) expressed in pairs -
  // without it a level that holds a dozen RoIs hands one CTA ~150 plane switches and the whole launch waits for it
  // (measured: 362 us instead of ~100 us for 1000 boxes over four levels).
  int64_t total = (int64_t)B * C * K;
  int Kl[kMaxLevels], Ol[kMaxLevels];
  if (MULTI) {
    asm volatile("griddepcontrol.wait;" ::: "memory");      // the level counts come from the geometry kernel
    total = 0;
#pragma unroll
    for (int l = 0; l < kMaxLevels; ++l) {
      Kl[l] = l < L.num_levels ? __ldg(lvl_count + l) : 0;
      Ol[l] = Kl[l] > 0 ? 48 + ((L.lv[l].H * L.lv[l].W) >> 9) : 0;
      total += (int64_t)B * C * (Kl[l] + Ol[l]);
    }
  }
  const int64_t per = (total + gridDim.x - 1) / gridDim.x;
  const int64_t w0 = (int64_t)blockIdx.x * per;
  const int64_t w1 = min(total, w0 + per);

  int cur_H = -1, cur_pitch = -1;
  int64_t w = w0;
  while (w < w1) {
    // ---- locate the (level, plane, first RoI) of work item w ----
    int lvl = 0, Kc = K;
    int64_t wl = w;
    const int* __restrict__ ids = nullptr;
    int cost_c = K, ovh = 0;
    if (MULTI) {
#pragma unroll
      for (int l = 0; l < kMaxLevels; ++l) {
        const int64_t pl_ = (int64_t)B * C * (Kl[l] + Ol[l]);
        if (lvl == l && wl >= pl_) { wl -= pl_; lvl = l + 1; }
      }
      Kc = Kl[lvl]; ovh = Ol[lvl]; cost_c = Kc + ovh;
      H = L.lv[lvl].H; W = L.lv[lvl].W; pitch = L.lv[lvl].pitch; input = L.lv[lvl].base;
      ids = bucket + (int64_t)lvl * K;
    }
    const int pl = (int)(wl / cost_c);              // plane index = b * C + c
    const int f = (int)(wl - (int64_t)pl * cost_c);  // position inside the plane's cost span: [0, ovh) switch, [ovh, ovh + Kc) RoIs
    const int span = (int)min((int64_t)(cost_c - f), w1 - w);
    const int r0 = max(0, f - ovh);
    const int r1 = min(Kc, f + span - ovh);
    const int b = pl / C;
    if (r1 <= r0) { w += span; continue; }          // this CTA's share of the plane is switch cost only
    // output element offsets fit 32 bits: the launchers require K * C * P * P < 2^31
    const uint32_t ostep = (uint32_t)(NW * C * NB), oplane = (uint32_t)((pl - b * C) * NB);
    __syncthreads();                           // everyone is done with the previous plane
    if (H != cur_H || pitch != cur_pitch) {    // (re)zero the pads: columns [W, pitch) of every row and the two zero rows
      for (int r = warp; r < H; r += NW)
        for (int col = W + lane; col < pitch; col += 32) plane[r * pitch + col] = 0.f;
      for (int i = H * pitch + tid; i < (H + 2) * pitch; i += blockDim.x) plane[i] = 0.f;
      cur_H = H; cur_pitch = pitch;
    }
    {
      const float* src = input + (int64_t)pl * H * W;
      for (int r = warp; r < H; r += NW) {
        const float* s = src + (int64_t)r * W;
        const uint32_t d = plane_s + (uint32_t)(r * pitch) * 4u;
        for (int col = lane; col < W; col += 32) cp_async4(d + col * 4u, s + col);
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    // The geometry of the next RoI travels one iteration ahead: the lane entry in registers, the
    // 14 loop entries + header (128 B) by cp.async into this warp's staging slot.
    if (!MULTI) asm volatile("griddepcontrol.wait;" ::: "memory");   // the table is complete from here on (no-op after the first time)
    int n = r0 + warp;
    int id = 0, id_next = 0;
    uint2 le = make_uint2(0u, 0u);
    uint32_t slot = stage_s;
    if (n < r1) {
      id = MULTI ? __ldg(ids + n) : n;
      if (n + NW < r1) id_next = MULTI ? __ldg(ids + n + NW) : n + NW;
      le = __ldg(&tab[id].lane[lane]);
      cp_async4(slot + lane4, reinterpret_cast<const float*>(tab + id) + 64 + lane);
    }
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 1;" ::: "memory");   // the plane has landed
    __syncthreads();

    uint32_t o_lin = (uint32_t)n * (uint32_t)(C * NB) + oplane;   // single level: RoI id == n, rows advance by a fixed step
    const char* __restrict__ tab_lin = reinterpret_cast<const char*>(tab + (n + NW));   // ... and so does the next RoI's table
    for (; n < r1; n += NW, o_lin += ostep, tab_lin += NW * sizeof(LineTab)) {
      const int nn = n + NW;
      const uint32_t slot_next = slot ^ slot_x;
      uint2 le_next = make_uint2(0u, 0u);
      int id_next2 = 0;
      __syncwarp();
      if (nn < r1) {
        if (MULTI && nn + NW < r1) id_next2 = __ldg(ids + nn + NW);
        const char* __restrict__ tn = MULTI ? reinterpret_cast<const char*>(tab + id_next) : tab_lin;
        le_next = __ldg(reinterpret_cast<const uint2*>(tn + 2 * lane4));                          // lane[lane]
        cp_async4(slot_next + lane4, reinterpret_cast<const float*>(tn + offsetof(LineTab, loop) + lane4));
      }
      asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 1;" ::: "memory");
      __syncwarp();
      const uint32_t st = slot;
      const bool lane_is_y = (le.x & 1u) != 0;             // bit 0 of every lane offset carries the lane axis
      // header word 1: the RoI's batch index (the same word in every lane, taken from lane 0 as above)
      const bool skip = multi_batch && __shfl_sync(0xffffffffu, (int)lds_u32(st + 116u), 0) != b;
      if (!skip) {
        const uint32_t obase = MULTI ? (uint32_t)id * (uint32_t)(C * NB) + oplane : o_lin;
        const uint32_t base0 = plane_s + (le.x & ~3u);
        const uint32_t base1 = base0 + (lane_is_y ? 4u : (uint32_t)pitch * 4u);
        const float wl_ = __uint_as_float(le.y);
        float acc[8];
        acc[7] = 0.f;
#pragma unroll
        for (int p = 0; p < P; ++p) {
          const uint4 ee = lds_u128(st + p * 16u);     // the two samples of loop-axis bin p
          const float a0 = lds_f32(base0 + ee.x), a1 = lds_f32(base1 + ee.x);
          const float b0 = lds_f32(base0 + ee.z), b1 = lds_f32(base1 + ee.z);
          const float ta = fmaf(__uint_as_float(ee.y), a1 - a0, a0);
          const float tb = fmaf(__uint_as_float(ee.w), b1 - b0, b0);
          acc[p] = (ta + tb) * wl_;
        }
        // fold the 4 lanes of a bin column: after two exchanges lane q holds loop-axis bins 2q, 2q+1
        float r4[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const float send = hi ? acc[m] : acc[4 + m], keep = hi ? acc[4 + m] : acc[m];
          r4[m] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
        }
        float s2[2];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          const float send = lo ? r4[m] : r4[2 + m], keep = lo ? r4[2 + m] : r4[m];
          s2[m] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
        }
        const uint32_t o0 = obase + __byte_perm(lane_code, 0u, 0x4440u | (le.x & 1u));   // byte 0 (x) or 1 (y)
        const uint32_t o1 = o0 + (lane_is_y ? 1u : (uint32_t)P);
        const bool st0 = (lane_code & 0x10000u) != 0, st1 = (lane_code & 0x20000u) != 0;
        const float v0 = s2[0] * inv_count, v1 = s2[1] * inv_count;
        if (DST == kLineMulticast) {         // one store each, replicated by the switch into every rank's buffer
          if (st0) asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(pd.mc + o0), "f"(v0) : "memory");
          if (st1) asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(pd.mc + o1), "f"(v1) : "memory");
        } else {
          if (st0) output[o0] = v0;
          if (st1) output[o1] = v1;
          if (DST == kLinePeers) {
#pragma unroll
            for (int d = 0; d < 7; ++d) {    // peer-mapped copies of the same slot (NVLink stores)
              if (d < pd.n && st0) pd.dst[d][o0] = v0;
              if (d < pd.n && st1) pd.dst[d][o1] = v1;
            }
          }
        }
      }
      slot = slot_next;
      le = le_next;
      id = id_next;
      id_next = id_next2;
    }
    w += span;
  }
}

// ---------------------------------------------------------------------------
// roi_pool / ps_roi_align / ps_roi_pool: work split by PlaneSpans, the plane staged into shared memory
// (RESIDENT) or read through L1/L2.
// ---------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void stage_plane_flat(T* __restrict__ dst, const T* __restrict__ src, int count) {
  // flat copy of one contiguous H*W plane: 16-byte vectors when source and element count allow it
  const int tid = threadIdx.x, NT = blockDim.x;
  if ((((uintptr_t)src) & 15u) == 0) {
    const int nvec = (int)(((size_t)count * sizeof(T)) / 16);
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    for (int i = tid; i < nvec; i += NT) d4[i] = __ldg(s4 + i);
    for (int i = (int)((size_t)nvec * 16 / sizeof(T)) + tid; i < count; i += NT) dst[i] = src[i];
  } else {
    for (int i = tid; i < count; i += NT) dst[i] = src[i];
  }
}

// ---------------------------------------------------------------------------
// roi_pool (reference semantics: csrc/ops/cuda/roi_pool_kernel.cu:15-78, cpu/roi_pool_kernel.cpp:24-92).
// Not the reference's thread-per-output design: a WARP owns one (RoI, plane) pair and its lanes are the
// bin columns x Q sub-lanes; it walks the bin rows once, every lane scanning its own columns of the bin window
// top to bottom (so each input word of the RoI is read about once per plane instead of once per overlapping
// output thread), then the Q sub-lanes of a bin combine (value, index) pairs with the reference's tie rule
// (strict '>' in a row-major scan == larger value, then smaller flat index).  RESIDENT: the plane sits in
// shared memory (each input byte leaves HBM once); otherwise the same code reads the plane through L1/L2.
// The RoI's integer geometry is derived once per (RoI, plane), not once per output element.
// ---------------------------------------------------------------------------
// one element of the resident plane from a shared-space address, widened to the accumulator type
template <typename T> __device__ __forceinline__ typename Acc<T>::type lds_acc(uint32_t addr);
template <> __device__ __forceinline__ float lds_acc<float>(uint32_t addr) { return lds_f32(addr); }
template <> __device__ __forceinline__ float lds_acc<__half>(uint32_t addr) {
  unsigned short u;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(u) : "r"(addr));
  return __half2float(__ushort_as_half(u));
}
template <> __device__ __forceinline__ double lds_acc<double>(uint32_t addr) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
  return v;
}

__device__ __forceinline__ float acc_max(float a, float b) { return fmaxf(a, b); }     // NaN operands are dropped, as `v > best` drops them
__device__ __forceinline__ double acc_max(double a, double b) { return fmax(a, b); }

// One lane's share of one bin window on the resident plane: rows [hs, he), NC columns at byte offsets off[0..NC) from the row
// address (entries past the lane's own count repeat its last column: re-reading cannot change a maximum).  The inner loop is
// LDS + FMNMX per element; the arg-max is kept at ROW granularity (first row whose maximum beats the best so far), the column
// is recovered afterwards by re-reading that single row left to right - the reference's "first maximum in row-major order".
template <typename T, int NC>
__device__ __forceinline__ void pool_scan(uint32_t row_a, uint32_t row_step, const uint32_t (&off)[8], int hs, int he,
                                          typename Acc<T>::type neg_max, typename Acc<T>::type& best, uint32_t& best_row_a) {
  using A = typename Acc<T>::type;
  for (int h = hs; h < he; ++h, row_a += row_step) {
    A rm = lds_acc<T>(row_a + off[0]);
#pragma unroll
    for (int t = 1; t < NC; ++t) rm = acc_max(rm, lds_acc<T>(row_a + off[t]));
    if (rm > best) { best = rm; best_row_a = row_a; }
  }
  (void)neg_max;
}

template <typename T, bool RESIDENT>
__global__ void __launch_bounds__(RESIDENT ? 1024 : 256, RESIDENT ? 1 : 4)
roi_pool_plane_kernel(const T* __restrict__ input, const T* __restrict__ rois, T* __restrict__ output,
                      int32_t* __restrict__ argmax, int B, int C, int H, int W, int K, int PH, int PW,
                      typename Acc<T>::type scale) {
  using A = typename Acc<T>::type;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* plane_s = reinterpret_cast<T*>(smem_raw);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, NW = blockDim.x >> 5;
  // lane -> (bin column, sub-lane): Q = largest power of two with PW * Q <= 32 (1 when PW >= 17)
  int qshift = 0;
  while ((PW << (qshift + 1)) <= 32) ++qshift;
  const int Q = 1 << qshift, bins_per_pass = 32 >> qshift;
  const int pw_l = lane >> qshift, q = lane & (Q - 1);
  const A neg_max = (A)-3.402823466e+38F;   // -FLT_MAX for every dtype, as the reference initialises it

  for (PlaneSpans sp(B, C, K); sp.more(); sp.advance()) {
    const int pl = sp.pl, r0 = sp.r0, r1 = sp.r1;
    const int b = pl / C, c = pl - b * C;
    const T* __restrict__ plane = input + (int64_t)pl * H * W;
    if (RESIDENT) {
      __syncthreads();                       // previous plane no longer read
      stage_plane_flat<T>(plane_s, plane, H * W);
      __syncthreads();
      plane = plane_s;
    }
    for (int n = r0 + warp; n < r1; n += NW) {
      const PoolGeom<A> g = pool_geometry<T, A, A>(rois + (int64_t)n * 5, scale, PH, PW, 1);
      if (g.batch != b) continue;
      T* __restrict__ outp = output + ((int64_t)n * C + c) * PH * PW;
      int32_t* __restrict__ argp = argmax + ((int64_t)n * C + c) * PH * PW;
      for (int pw0 = 0; pw0 < PW; pw0 += bins_per_pass) {
        const int pw = pw0 + pw_l;
        const bool act = pw < PW;
        int ws = 0, we = 0;
        if (act) bin_window<T>(pw, g.bw, g.rsw, W, ws, we);
        // columns this lane scans in every window row: ws + q, ws + q + Q, ...; the warp loops to the widest lane's count
        const int ncol = act && we > ws + q ? (we - ws - q + Q - 1) >> qshift : 0;
        const int ncol_max = __reduce_max_sync(0xffffffffu, ncol);
        // byte offsets of this lane's columns inside a window row, relative to column col0; a lane with no column of its own
        // reads column 0 of the plane row range (valid memory) and is ignored afterwards
        const int col0 = ncol > 0 ? ws + q : 0;
        uint32_t off[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) off[t] = (uint32_t)(min(t, max(ncol - 1, 0)) << qshift) * (uint32_t)sizeof(T);
        for (int ph = 0; ph < PH; ++ph) {
          int hs, he;
          bin_window<T>(ph, g.bh, g.rsh, H, hs, he);
          A best = neg_max;
          int idx = -1;
          if (RESIDENT) {
            constexpr uint32_t ESZ = (uint32_t)sizeof(T);
            const uint32_t plane_a = smem_u32(plane_s);
            const uint32_t row_a0 = plane_a + (uint32_t)(hs * W + col0) * ESZ, row_step = (uint32_t)W * ESZ;
            if (ncol_max <= 8) {
              uint32_t best_row_a = 0xffffffffu;
              switch (ncol_max) {          // warp-uniform
                case 1: pool_scan<T, 1>(row_a0, row_step, off, hs, he, neg_max, best, best_row_a); break;
                case 2: pool_scan<T, 2>(row_a0, row_step, off, hs, he, neg_max, best, best_row_a); break;
                case 3: pool_scan<T, 3>(row_a0, row_step, off, hs, he, neg_max, best, best_row_a); break;
                case 4: pool_scan<T, 4>(row_a0, row_step, off, hs, he, neg_max, best, best_row_a); break;
                case 5: pool_scan<T, 5>(row_a0, row_step, off, hs, he, neg_max, best, best_row_a); break;
                case 6: pool_scan<T, 6>(row_a0, row_step, off, hs, he, neg_max, best, best_row_a); break;
                case 7: pool_scan<T, 7>(row_a0, row_step, off, hs, he, neg_max, best, best_row_a); break;
                case 8: pool_scan<T, 8>(row_a0, row_step, off, hs, he, neg_max, best, best_row_a); break;
                default: break;
              }
              if (ncol > 0 && best_row_a != 0xffffffffu) {
                // column of the first maximum inside the winning row; the VALUE is re-read there (keeps the sign of a zero)
                uint32_t a = best_row_a + off[0];
                for (int t = 0; t < ncol; ++t, a += (uint32_t)Q * ESZ) {
                  const A v = lds_acc<T>(a);
                  if (v == best) { best = v; idx = (int)((a - plane_a) / ESZ); break; }
                }
              } else {
                best = neg_max;             // lanes without a column of their own only repeated a neighbour's reads
              }
            } else {                        // very wide bins: plain loop, a warp-uniform trip count with idle lanes
              uint32_t row_a = row_a0 + off[0], best_a = 0xffffffffu;
              for (int h = hs; h < he; ++h, row_a += row_step) {
                uint32_t a = row_a;
                for (int t = 0; t < ncol_max; ++t, a += (uint32_t)Q * ESZ) {
                  if (t < ncol) {
                    const A v = lds_acc<T>(a);
                    if (v > best) { best = v; best_a = a; }
                  }
                }
              }
              idx = best_a == 0xffffffffu ? -1 : (int)((best_a - plane_a) / ESZ);
            }
          } else {
            for (int h = hs; h < he; ++h) {
              const T* __restrict__ row = plane + h * W;
              for (int x = ws + q; x < we; x += Q) {
                const A v = to_acc(row[x]);
                if (v > best) { best = v; idx = h * W + x; }
              }
            }
          }
          for (int o = 1; o < Q; o <<= 1) {
            const A ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
            if (ov > best || (ov == best && (unsigned)oi < (unsigned)idx)) { best = ov; idx = oi; }
          }
          if (act && q == 0) {
            const bool empty = (he <= hs) || (we <= ws);
            outp[ph * PW + pw] = from_acc<T, A>(empty ? (A)0 : best);
            argp[ph * PW + pw] = idx;
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------
// ps_roi_align (reference semantics: csrc/ops/cuda/ps_roi_align_kernel.cu:68-140).  Position-sensitive pooling
// reads input channel c_in = (c_out * PH + ph) * PW + pw for bin (ph, pw) only, i.e. an input plane serves exactly
// ONE bin position of one output channel, for every RoI.  So the work is organised by input plane: a CTA holds
// plane (b, c_in) (RESIDENT: in shared memory, one pass over HBM) and its THREADS are the RoIs - each thread
// evaluates its RoI's single bin on that plane (gh x gw samples).  The bin arithmetic is the reference's, with
// uncontracted coordinates, so degenerate RoIs give the same inf / NaN.
// ---------------------------------------------------------------------------
template <typename T, bool RESIDENT>
__global__ void __launch_bounds__(RESIDENT ? 1024 : 256, RESIDENT ? 1 : 4)
ps_roi_align_plane_kernel(const T* __restrict__ input, const T* __restrict__ rois, T* __restrict__ output,
                          int32_t* __restrict__ mapping, int B, int C, int H, int W, int K, int PH, int PW, int Cout,
                          typename Acc<T>::type scale, int sampling_ratio) {
  using A = typename Acc<T>::type;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* plane_s = reinterpret_cast<T*>(smem_raw);
  for (PlaneSpans sp(B, C, K); sp.more(); sp.advance()) {
    const int pl = sp.pl, r0 = sp.r0, r1 = sp.r1;
    const int b = pl / C, c_in = pl - b * C;
    const int pw = c_in % PW, ph = (c_in / PW) % PH, co = c_in / (PW * PH);
    const T* __restrict__ plane = input + (int64_t)pl * H * W;
    if (RESIDENT) {
      __syncthreads();
      stage_plane_flat<T>(plane_s, plane, H * W);
      __syncthreads();
      plane = plane_s;
    }
    for (int n = r0 + (int)threadIdx.x; n < r1; n += (int)blockDim.x) {
      const RoiGeom<A> g = roi_geometry<T, A>(rois + (int64_t)n * 5, scale, PH, PW, sampling_ratio, true, true);
      if (g.batch != b) continue;
      const A count = (A)(g.gh * g.gw);
      A sum = 0;
      // sample_coord with the bin origin hoisted out of the sample loops (the reference's hstart / wstart): the same bits,
      // and recomputing it per sample spills the fp64 kernel
      const A hstart = add_rn(mul_rn((A)ph, g.bin_h), g.start_h);
      const A wstart = add_rn(mul_rn((A)pw, g.bin_w), g.start_w);
      for (int iy = 0; iy < g.gh; ++iy) {
        const AxisEnt<A> ey = axis_entry<A>(add_rn(hstart, div_rn(mul_rn((A)((float)iy + .5f), g.bin_h), (A)g.gh)), H);
        for (int ix = 0; ix < g.gw; ++ix) {
          const AxisEnt<A> ex = axis_entry<A>(add_rn(wstart, div_rn(mul_rn((A)((float)ix + .5f), g.bin_w), (A)g.gw)), W);
          sum = add_rn(sum, bilinear_blend<T, A>(plane, W, ey, ex));
        }
      }
      const int64_t o = (((int64_t)n * Cout + co) * PH + ph) * PW + pw;
      output[o] = from_acc<T, A>(div_rn(sum, count));
      mapping[o] = c_in;
    }
  }
}

// ---------------------------------------------------------------------------
// ps_roi_pool (reference semantics: csrc/ops/cuda/ps_roi_pool_kernel.cu:15-78).  Same organisation as ps_roi_align:
// input plane c_in serves bin (ph, pw) of output channel c_out for every RoI, so a CTA holds the plane and its threads
// are the RoIs; each averages its bin window (integer bounds, clipped to size - 1 as the reference's forward does).
// The window is summed in the reference's order (rows, then columns, one rounding per add).
// ---------------------------------------------------------------------------
template <typename T, bool RESIDENT>
__global__ void __launch_bounds__(RESIDENT ? 1024 : 256, RESIDENT ? 1 : 4)
ps_roi_pool_plane_kernel(const T* __restrict__ input, const T* __restrict__ rois, T* __restrict__ output,
                         int32_t* __restrict__ mapping, int B, int C, int H, int W, int K, int PH, int PW, int Cout,
                         typename Acc<T>::type scale) {
  using A = typename Acc<T>::type;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* plane_s = reinterpret_cast<T*>(smem_raw);
  for (PlaneSpans sp(B, C, K); sp.more(); sp.advance()) {
    const int pl = sp.pl, r0 = sp.r0, r1 = sp.r1;
    const int b = pl / C, c_in = pl - b * C;
    const int pw = c_in % PW, ph = (c_in / PW) % PH, co = c_in / (PW * PH);
    const T* __restrict__ plane = input + (int64_t)pl * H * W;
    if (RESIDENT) {
      __syncthreads();
      stage_plane_flat<T>(plane_s, plane, H * W);
      __syncthreads();
      plane = plane_s;
    }
    for (int n = r0 + (int)threadIdx.x; n < r1; n += (int)blockDim.x) {
      const PoolGeom<A> g = pool_geometry<T, A, float>(rois + (int64_t)n * 5, scale, PH, PW, 0);
      if (g.batch != b) continue;
      int hs, he, ws, we;
      bin_window<T>(ph, g.bh, g.rsh, H - 1, hs, he);
      bin_window<T>(pw, g.bw, g.rsw, W - 1, ws, we);
      const bool empty = (he <= hs) || (we <= ws);
      A sum = 0;
      for (int h = hs; h < he; ++h)
        for (int x = ws; x < we; ++x) sum = rnd<T>(add_rn(sum, (A)to_acc(plane[h * W + x])));
      const A area = rnd<T>((A)((he - hs) * (we - ws)));
      const int64_t o = (((int64_t)n * Cout + co) * PH + ph) * PW + pw;
      output[o] = from_acc<T, A>(empty ? (A)0 : rnd<T>(div_rn(sum, area)));
      mapping[o] = c_in;
    }
  }
}

template <typename T>
int launch_roi_align_generic(const void* input, const void* rois, void* output, int C, int H, int W, int K,
                             int PH, int PW, double scale, int sr, int aligned, cudaStream_t st) {
  const int ch_per_cta = C >= 64 ? 32 : (C >= 16 ? 16 : C);
  dim3 grid((unsigned)K, (unsigned)ceil_div(C, ch_per_cta));
  roi_align_generic_kernel<T><<<grid, 256, 0, st>>>((const T*)input, (const T*)rois, (T*)output, C, H, W, PH, PW,
                                                   (typename Acc<T>::type)scale, sr, aligned, ch_per_cta);
  return check_launch("roi_align_generic_kernel");
}

}  // namespace
}  // namespace vb200

using namespace vb200;

namespace {
// Path selection shared by the workspace query and the launcher.
//   0 generic, 1 plane-resident thread-per-bin (any pooled size, sampling_ratio 1..4),
//   2 plane-resident line-wise lanes (7x7 bins, sampling_ratio 2: the detection-head shape).
int roi_align_path(int dtype, const void* input, int batch, int channels, int height, int width, int num_rois,
                   int pooled_h, int pooled_w, int sampling_ratio) {
  if (dtype != VB200_F32) return 0;
  if (height < 2 || width < 2) return 0;
  const size_t plane_bytes = ((size_t)(height + 2) * plane_pitch(width) + 2) * 4;
  const bool fits = plane_bytes + 1024 <= (size_t)max_smem_optin();
  const bool sr_ok = sampling_ratio >= 1 && sampling_ratio <= 4;
  const bool align_ok = width % 4 == 0 && (input == nullptr || ((uintptr_t)input % 16) == 0);
  const bool bins_ok = pooled_h * pooled_w <= kPlaneMaxThreads;
  const bool plane_ok = fits && sr_ok && align_ok && bins_ok;
  const size_t line_bytes = line_plane_bytes(height, line_pitch(width)) + kLineStageBytes;
  const bool shape7 = pooled_h == 7 && pooled_w == 7 && sampling_ratio == 2;
  const bool line_ok = shape7 && line_bytes + 1024 <= (size_t)max_smem_optin();
  const int64_t pairs = (int64_t)batch * channels * num_rois;
  int path = pairs >= 4096 ? (line_ok ? 2 : plane_ok ? 1 : 0) : 0;
  const char* force = env_override(ENV_ROI_ALIGN_PATH);   // "generic" | "plane" | "line" (testing / profiling)
  if (force && force[0] == 'g') path = 0;
  if (force && force[0] == 'p') path = plane_ok ? 1 : 0;
  if (force && force[0] == 'l') path = line_ok ? 2 : 0;
  return path;
}
size_t roi_align_geo_bytes(int num_rois, int pooled_h, int pooled_w, int sampling_ratio) {
  return align256((size_t)num_rois * (pooled_h + pooled_w) * sampling_ratio * sizeof(PackedEnt));
}
size_t roi_align_ws_bytes(int path, int num_rois, int pooled_h, int pooled_w, int sampling_ratio) {
  if (path == 1) return roi_align_geo_bytes(num_rois, pooled_h, pooled_w, sampling_ratio) + (size_t)num_rois * 4;
  if (path == 2) return (size_t)num_rois * sizeof(LineTab);
  return 0;
}
}  // namespace

extern "C" size_t vb200_roi_align_workspace_bytes(int dtype, int batch, int channels, int height, int width,
                                                  int num_rois, int pooled_h, int pooled_w,
                                                  int sampling_ratio) {
  if (num_rois <= 0 || channels <= 0) return 0;
  // the larger of the two table-driven paths, so the answer does not depend on the environment override
  size_t a = 0;
  for (int path = 1; path <= 2; ++path) {
    const size_t b = roi_align_ws_bytes(path, num_rois, pooled_h, pooled_w, sampling_ratio);
    a = b > a ? b : a;
  }
  return roi_align_path(dtype, nullptr, batch, channels, height, width, num_rois, pooled_h, pooled_w, sampling_ratio) ? a : 0;
}

static int roi_align_forward_impl(const void* input, const void* rois, void* output, int dtype,
                                  int batch, int channels, int height, int width, int num_rois,
                                  int pooled_h, int pooled_w, double spatial_scale,
                                  int sampling_ratio, int aligned, void* workspace,
                                  size_t workspace_bytes, vb200_stream stream, const PeerDst& peers, bool* peers_done) {
  VB200_REQUIRE(batch >= 0 && channels >= 0 && height >= 0 && width >= 0 && num_rois >= 0, "roi_align: negative size");
  VB200_REQUIRE(pooled_h > 0 && pooled_w > 0, "roi_align: pooled size must be positive");
  if (num_rois == 0 || channels == 0) return 0;
  VB200_REQUIRE(input && rois && output, "roi_align: null pointer");
  VB200_REQUIRE((int64_t)num_rois * channels * pooled_h * pooled_w < (1ll << 31) &&
                (int64_t)batch * channels * height * width < (1ll << 31), "roi_align: tensor too large for 32-bit indexing");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == VB200_F32) {
    const size_t geo_pad = roi_align_geo_bytes(num_rois, pooled_h, pooled_w, sampling_ratio);
    int path = roi_align_path(dtype, input, batch, channels, height, width, num_rois, pooled_h, pooled_w, sampling_ratio);
    if (path && (workspace == nullptr || ((uintptr_t)workspace % 16) != 0 ||
                 workspace_bytes < roi_align_ws_bytes(path, num_rois, pooled_h, pooled_w, sampling_ratio)))
      path = 0;
    if (path == 2) {
      const int pitch = line_pitch(width);
      const size_t smem = line_plane_bytes(height, pitch) + kLineStageBytes;
      LineTab* tab = (LineTab*)workspace;
      LevelSet none = {};
      roi_align_line_geometry_kernel<7, 2, false><<<ceil_div(num_rois * 32, 256), 256, 0, st>>>(
          (const float*)rois, tab, num_rois, height, width, (float)spatial_scale, aligned, pitch, batch, none, nullptr,
          nullptr, nullptr);
      int rc = check_launch("roi_align_line_geometry_kernel");
      if (rc) return rc;
      const int64_t pairs = (int64_t)batch * channels * num_rois;
      const int grid = (int)(pairs < sm_count() ? pairs : sm_count());
      constexpr auto local = roi_align_line_kernel<7, 2, false, kLineLocal>;
      constexpr auto to_peers = roi_align_line_kernel<7, 2, false, kLinePeers>;
      constexpr auto multicast = roi_align_line_kernel<7, 2, false, kLineMulticast>;
      const auto kernel = peers.mc ? multicast : peers.n > 0 ? to_peers : local;
      VB200_CUDA_TRY(peers.mc ? ensure_dyn_smem<multicast>(smem) : peers.n > 0 ? ensure_dyn_smem<to_peers>(smem)
                                                                                : ensure_dyn_smem<local>(smem));
      if (peers_done) *peers_done = true;        // this kernel writes the peer destinations itself
      // programmatic dependent launch: the gather kernel zeroes its pads and stages its first plane while
      // the geometry kernel is still running, and waits (griddepcontrol.wait) before it reads the table
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kLineThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[0].val.programmaticStreamSerializationAllowed = 1;
      cfg.attrs = attr; cfg.numAttrs = 1;
      VB200_CUDA_TRY(cudaLaunchKernelEx(&cfg, kernel, (const float*)input, (const LineTab*)tab,
                                        (float*)output, batch, channels, height, width, num_rois, pitch, none,
                                        (const int*)nullptr, (const int*)nullptr, peers));
      return check_launch("roi_align_line_kernel");
    }
    const bool use_plane = path == 1;
    if (use_plane) {
      const int pitch = plane_pitch(width);
      const size_t plane_bytes = ((size_t)(height + 2) * pitch + 2) * 4;
      const int nbins = pooled_h * pooled_w;
      const int nthreads = nbins <= kPlaneMaxThreads ? (kPlaneMaxThreads / nbins) * nbins : 0;
      const int64_t pairs = (int64_t)batch * channels * num_rois;
      const int ent = (pooled_h + pooled_w) * sampling_ratio;
      PackedEnt* geo = (PackedEnt*)workspace;
      int32_t* rb = (int32_t*)((char*)workspace + geo_pad);
      const int nt = num_rois * ent;
      roi_align_geometry_kernel<<<ceil_div(nt, 256), 256, 0, st>>>((const float*)rois, geo, rb, num_rois, height,
                                                                   width, pooled_h, pooled_w, (float)spatial_scale,
                                                                   sampling_ratio, aligned, pitch);
      int rc = check_launch("roi_align_geometry_kernel");
      if (rc) return rc;
      const int grid = (int)(pairs < sm_count() ? pairs : sm_count());
      const size_t smem = plane_bytes + 128;
#define VB200_LAUNCH_PLANE(SR)                                                                                     \
  {                                                                                                                \
    VB200_CUDA_TRY(ensure_dyn_smem<roi_align_plane_kernel<SR>>(smem));                                                               \
    roi_align_plane_kernel<SR><<<grid, nthreads, smem, st>>>((const float*)input, geo, rb, (float*)output,         \
                                                             batch, channels, height, width, num_rois,            \
                                                             pooled_h, pooled_w, pitch);                          \
  }
      switch (sampling_ratio) {
        case 1: VB200_LAUNCH_PLANE(1) break;
        case 2: VB200_LAUNCH_PLANE(2) break;
        case 3: VB200_LAUNCH_PLANE(3) break;
        default: VB200_LAUNCH_PLANE(4) break;
      }
#undef VB200_LAUNCH_PLANE
      return check_launch("roi_align_plane_kernel");
    }
  }
  return dispatch_roi_dtype(dtype, "roi_align: unsupported dtype %d (float, double, half as the reference)", [&](auto t) {
    return launch_roi_align_generic<decltype(t)>(input, rois, output, channels, height, width, num_rois, pooled_h, pooled_w,
                                                 spatial_scale, sampling_ratio, aligned, st);
  });
}

extern "C" int vb200_roi_align_forward(const void* input, const void* rois, void* output, int dtype,
                                       int batch, int channels, int height, int width, int num_rois,
                                       int pooled_h, int pooled_w, double spatial_scale,
                                       int sampling_ratio, int aligned, void* workspace,
                                       size_t workspace_bytes, vb200_stream stream) {
  return roi_align_forward_impl(input, rois, output, dtype, batch, channels, height, width, num_rois, pooled_h, pooled_w, spatial_scale,
                                sampling_ratio, aligned, workspace, workspace_bytes, stream, PeerDst{}, nullptr);
}

// roi_align fused with the all-gather of its output: outputs[0] is the caller's slot of its gathered buffer, outputs[1..n) the
// same slot of the peers' buffers (peer-mapped), or - when `multicast_output` is not NULL - one NVSwitch multicast address of
// that slot that reaches every rank.  The line kernel stores every finished bin to all of them; configurations it does not
// cover are computed into outputs[0] and copied to the peers on the same stream.
extern "C" int vb200_roi_align_forward_gather(const void* input, const void* rois, void* const* outputs, int n_outputs,
                                              void* multicast_output, int dtype, int batch, int channels, int height, int width,
                                              int num_rois, int pooled_h, int pooled_w, double spatial_scale, int sampling_ratio,
                                              int aligned, void* workspace, size_t workspace_bytes, vb200_stream stream) {
  VB200_REQUIRE(outputs && n_outputs >= 1 && n_outputs <= 8, "roi_align_gather: 1..8 destinations");
  for (int d = 0; d < n_outputs; ++d) VB200_REQUIRE(outputs[d] != nullptr, "roi_align_gather: null destination");
  PeerDst pd = {};
  pd.mc = dtype == VB200_F32 ? (float*)multicast_output : nullptr;
  pd.n = pd.mc ? 0 : n_outputs - 1;
  for (int d = 0; d < pd.n; ++d) pd.dst[d] = (float*)outputs[d + 1];
  bool done = false;
  const int rc = roi_align_forward_impl(input, rois, outputs[0], dtype, batch, channels, height, width, num_rois, pooled_h, pooled_w,
                                        spatial_scale, sampling_ratio, aligned, workspace, workspace_bytes, stream, pd, &done);
  if (rc || done || n_outputs == 1 || num_rois == 0 || channels == 0) return rc;
  const size_t esize = dtype == VB200_F64 ? 8 : dtype == VB200_F32 ? 4 : 2;
  const size_t bytes = (size_t)num_rois * channels * pooled_h * pooled_w * esize;
  for (int d = 1; d < n_outputs; ++d)
    VB200_CUDA_TRY(cudaMemcpyAsync(outputs[d], outputs[0], bytes, cudaMemcpyDefault, (cudaStream_t)stream));
  return 0;
}

// ---- fused MultiScaleRoIAlign ------------------------------------------------------------------------------------
namespace {
struct MsWs { LineTab* tab; int* lvl_count; int* bucket; size_t total; };
MsWs carve_ms(void* base, int K, int num_levels) {
  Carver c(base);
  MsWs w;
  w.tab = c.take<LineTab>(K);
  w.lvl_count = c.take<int>(kMaxLevels);
  w.bucket = c.take<int>((size_t)num_levels * K);
  w.total = c.off;
  return w;
}
}  // namespace

extern "C" size_t vb200_multiscale_roi_align_workspace_bytes(int num_rois, int num_levels) {
  if (num_rois <= 0 || num_levels <= 0) return 0;
  return carve_ms(nullptr, num_rois, num_levels).total;
}

extern "C" int vb200_multiscale_roi_align_supported(int dtype, int num_levels, const int* heights, const int* widths, int pooled_h,
                                                    int pooled_w, int sampling_ratio) {
  if (dtype != VB200_F32 || num_levels < 1 || num_levels > kMaxLevels) return 0;
  if (pooled_h != 7 || pooled_w != 7 || sampling_ratio != 2) return 0;
  for (int l = 0; l < num_levels; ++l) {
    if (heights[l] < 2 || widths[l] < 2) return 0;
    if (line_plane_bytes(heights[l], line_pitch(widths[l])) + kLineStageBytes + 1024 > (size_t)max_smem_optin()) return 0;
  }
  return 1;
}

extern "C" int vb200_multiscale_roi_align_forward(const void* const* level_ptrs, const int* heights, const int* widths,
                                                  const double* scales, int num_levels, const void* rois, void* output,
                                                  int32_t* levels_out, int dtype, int batch, int channels, int num_rois,
                                                  int pooled_h, int pooled_w, int sampling_ratio, int k_min, int k_max,
                                                  double canonical_scale, double canonical_level, double eps, void* workspace,
                                                  size_t workspace_bytes, vb200_stream stream) {
  VB200_REQUIRE(vb200_multiscale_roi_align_supported(dtype, num_levels, heights, widths, pooled_h, pooled_w, sampling_ratio),
                "multiscale_roi_align: unsupported configuration (fp32, 7x7 bins, sampling_ratio 2, <= 8 levels, planes that fit shared memory)");
  if (num_rois == 0 || channels == 0 || batch == 0) return 0;
  VB200_REQUIRE(level_ptrs && rois && output && levels_out, "multiscale_roi_align: null pointer");
  const MsWs ws = carve_ms(workspace, num_rois, num_levels);
  VB200_REQUIRE(workspace && ((uintptr_t)workspace % 16) == 0 && workspace_bytes >= ws.total, "multiscale_roi_align: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  LevelSet L = {};
  L.num_levels = num_levels;
  L.k_min = k_min; L.k_max = k_max;
  L.inv_s0 = 1.0f / (float)canonical_scale; L.lvl0 = (float)canonical_level; L.eps = (float)eps;
  size_t smem = 0;
  for (int l = 0; l < num_levels; ++l) {
    VB200_REQUIRE(level_ptrs[l] != nullptr, "multiscale_roi_align: null level pointer");
    VB200_REQUIRE((int64_t)batch * channels * heights[l] * widths[l] < (1ll << 31), "multiscale_roi_align: level too large for 32-bit indexing");
    L.lv[l].base = (const float*)level_ptrs[l];
    L.lv[l].H = heights[l]; L.lv[l].W = widths[l]; L.lv[l].pitch = line_pitch(widths[l]);
    L.lv[l].scale = (float)scales[l];
    const size_t bts = line_plane_bytes(heights[l], L.lv[l].pitch);
    smem = bts > smem ? bts : smem;
  }
  smem += kLineStageBytes;
  VB200_REQUIRE((int64_t)num_rois * channels * 49 < (1ll << 31), "multiscale_roi_align: output too large for 32-bit indexing");
  VB200_CUDA_TRY(cudaMemsetAsync(ws.lvl_count, 0, kMaxLevels * sizeof(int), st));
  roi_align_line_geometry_kernel<7, 2, true><<<ceil_div(num_rois * 32, 256), 256, 0, st>>>(
      (const float*)rois, ws.tab, num_rois, 0, 0, 0.f, 0, 0, batch, L, ws.lvl_count, ws.bucket, levels_out);
  int rc = check_launch("roi_align_line_geometry_kernel");
  if (rc) return rc;
  const int64_t pairs = (int64_t)batch * channels * num_rois;
  const int grid = (int)(pairs < sm_count() ? pairs : sm_count());
  VB200_CUDA_TRY(ensure_dyn_smem<roi_align_line_kernel<7, 2, true, kLineLocal>>(smem));
  roi_align_line_kernel<7, 2, true, kLineLocal><<<grid, kLineThreads, smem, st>>>(nullptr, ws.tab, (float*)output, batch, channels, 0, 0, num_rois, 0,
                                                                     L, ws.lvl_count, ws.bucket, PeerDst{});
  return check_launch("roi_align_line_kernel");
}

// Plane residency pays when the RoIs of a plane touch more bytes than the plane has; tiny problems read through L2.
template <typename T>
static bool plane_resident_ok(int H, int W, int64_t bytes_touched_per_plane) {
  const size_t plane_bytes = (size_t)H * W * sizeof(T);
  return plane_bytes + 1024 <= (size_t)max_smem_optin() && bytes_touched_per_plane >= (int64_t)plane_bytes;
}

template <typename T>
static int launch_roi_pool(const void* input, const void* rois, void* output, int32_t* argmax, int B, int C, int H, int W,
                           int K, int PH, int PW, double scale, cudaStream_t st) {
  using A = typename Acc<T>::type;
  const int64_t pairs = (int64_t)B * C * K;
  if (pairs == 0) return 0;
  // a RoI reads its whole window; count a conservative 16 x 16 window per RoI for the residency decision
  const bool resident = plane_resident_ok<T>(H, W, (int64_t)K * 256 * (int64_t)sizeof(T) / (B > 1 ? B : 1));
  if (resident) {
    const size_t smem = (size_t)H * W * sizeof(T) + 16;
    const int grid = (int)(pairs < sm_count() ? pairs : sm_count());
    VB200_CUDA_TRY(ensure_dyn_smem<roi_pool_plane_kernel<T, true>>(smem));
    roi_pool_plane_kernel<T, true><<<grid, 1024, smem, st>>>((const T*)input, (const T*)rois, (T*)output, argmax, B, C, H, W, K,
                                                            PH, PW, (A)scale);
  } else {
    const int64_t want = ceil_div64(pairs, 8);          // 8 warps per CTA, one (RoI, plane) pair per warp
    const int grid = (int)(want < (int64_t)sm_count() * 8 ? want : (int64_t)sm_count() * 8);
    roi_pool_plane_kernel<T, false><<<grid, 256, 0, st>>>((const T*)input, (const T*)rois, (T*)output, argmax, B, C, H, W, K, PH,
                                                         PW, (A)scale);
  }
  return check_launch("roi_pool_plane_kernel");
}

extern "C" int vb200_roi_pool_forward(const void* input, const void* rois, void* output, int32_t* argmax,
                                      int dtype, int batch, int channels, int height, int width, int num_rois,
                                      int pooled_h, int pooled_w, double spatial_scale, vb200_stream stream) {
  VB200_REQUIRE(pooled_h > 0 && pooled_w > 0, "roi_pool: pooled size must be positive");
  if (num_rois == 0 || channels == 0) return 0;
  VB200_REQUIRE(input && rois && output && argmax, "roi_pool: null pointer");
  VB200_REQUIRE((int64_t)batch * channels * height * width < (1ll << 31), "roi_pool: input too large for 32-bit indexing");
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_roi_dtype(dtype, "roi_pool: unsupported dtype %d", [&](auto t) {
    return launch_roi_pool<decltype(t)>(input, rois, output, argmax, batch, channels, height, width, num_rois, pooled_h, pooled_w, spatial_scale, st);
  });
}

template <typename T>
static int launch_ps_roi_align(const void* input, const void* rois, void* output, int32_t* mapping, int B, int C, int H, int W,
                               int K, int PH, int PW, double scale, int sr, cudaStream_t st) {
  using A = typename Acc<T>::type;
  const int Cout = C / (PH * PW);
  const int64_t pairs = (int64_t)B * C * K;
  if (pairs == 0 || Cout == 0) return 0;
  const int grid_s = sr > 0 ? sr : 2;
  // a RoI touches gh * gw * 4 sectors of 32 bytes on its plane
  const bool resident = plane_resident_ok<T>(H, W, (int64_t)K * grid_s * grid_s * 4 * 32 / (B > 1 ? B : 1));
  if (resident) {
    const size_t smem = (size_t)H * W * sizeof(T) + 16;
    const int grid = (int)(pairs < sm_count() ? pairs : sm_count());
    VB200_CUDA_TRY(ensure_dyn_smem<ps_roi_align_plane_kernel<T, true>>(smem));
    ps_roi_align_plane_kernel<T, true><<<grid, 1024, smem, st>>>((const T*)input, (const T*)rois, (T*)output, mapping, B, C, H, W,
                                                                K, PH, PW, Cout, (A)scale, sr);
  } else {
    const int64_t want = ceil_div64(pairs, 256);
    const int grid = (int)(want < (int64_t)sm_count() * 8 ? want : (int64_t)sm_count() * 8);
    ps_roi_align_plane_kernel<T, false><<<grid, 256, 0, st>>>((const T*)input, (const T*)rois, (T*)output, mapping, B, C, H, W, K,
                                                             PH, PW, Cout, (A)scale, sr);
  }
  return check_launch("ps_roi_align_plane_kernel");
}

extern "C" int vb200_ps_roi_align_forward(const void* input, const void* rois, void* output,
                                          int32_t* channel_mapping, int dtype, int batch, int channels,
                                          int height, int width, int num_rois, int pooled_h, int pooled_w,
                                          double spatial_scale, int sampling_ratio, vb200_stream stream) {
  VB200_REQUIRE(pooled_h > 0 && pooled_w > 0, "ps_roi_align: pooled size must be positive");
  VB200_REQUIRE(channels % (pooled_h * pooled_w) == 0,
                "input channels must be a multiple of pooling height * pooling width");
  if (num_rois == 0 || channels == 0) return 0;
  VB200_REQUIRE(input && rois && output && channel_mapping, "ps_roi_align: null pointer");
  VB200_REQUIRE((int64_t)batch * channels * height * width < (1ll << 31), "ps_roi_align: input too large for 32-bit indexing");
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_roi_dtype(dtype, "ps_roi_align: unsupported dtype %d", [&](auto t) {
    return launch_ps_roi_align<decltype(t)>(input, rois, output, channel_mapping, batch, channels, height, width, num_rois, pooled_h, pooled_w, spatial_scale, sampling_ratio, st);
  });
}

template <typename T>
static int launch_ps_roi_pool(const void* input, const void* rois, void* output, int32_t* mapping, int B, int C, int H, int W, int K,
                              int PH, int PW, double scale, cudaStream_t st) {
  using A = typename Acc<T>::type;
  const int Cout = C / (PH * PW);
  const int64_t pairs = (int64_t)B * C * K;
  if (pairs == 0 || Cout == 0) return 0;
  const bool resident = plane_resident_ok<T>(H, W, (int64_t)K * 64 * (int64_t)sizeof(T) / (B > 1 ? B : 1));
  if (resident) {
    const size_t smem = (size_t)H * W * sizeof(T) + 16;
    const int grid = (int)(pairs < sm_count() ? pairs : sm_count());
    VB200_CUDA_TRY(ensure_dyn_smem<ps_roi_pool_plane_kernel<T, true>>(smem));
    ps_roi_pool_plane_kernel<T, true><<<grid, 1024, smem, st>>>((const T*)input, (const T*)rois, (T*)output, mapping, B, C, H, W, K, PH,
                                                               PW, Cout, (A)scale);
  } else {
    const int64_t want = ceil_div64(pairs, 256);
    const int grid = (int)(want < (int64_t)sm_count() * 8 ? want : (int64_t)sm_count() * 8);
    ps_roi_pool_plane_kernel<T, false><<<grid, 256, 0, st>>>((const T*)input, (const T*)rois, (T*)output, mapping, B, C, H, W, K, PH, PW,
                                                            Cout, (A)scale);
  }
  return check_launch("ps_roi_pool_plane_kernel");
}

extern "C" int vb200_ps_roi_pool_forward(const void* input, const void* rois, void* output, int32_t* channel_mapping, int dtype,
                                         int batch, int channels, int height, int width, int num_rois, int pooled_h, int pooled_w,
                                         double spatial_scale, vb200_stream stream) {
  VB200_REQUIRE(pooled_h > 0 && pooled_w > 0, "ps_roi_pool: pooled size must be positive");
  VB200_REQUIRE(channels % (pooled_h * pooled_w) == 0, "input channels must be a multiple of pooling height * pooling width");
  if (num_rois == 0 || channels == 0) return 0;
  VB200_REQUIRE(input && rois && output && channel_mapping, "ps_roi_pool: null pointer");
  VB200_REQUIRE((int64_t)batch * channels * height * width < (1ll << 31), "ps_roi_pool: input too large for 32-bit indexing");
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_roi_dtype(dtype, "ps_roi_pool: unsupported dtype %d", [&](auto t) {
    return launch_ps_roi_pool<decltype(t)>(input, rois, output, channel_mapping, batch, channels, height, width, num_rois, pooled_h, pooled_w, spatial_scale, st);
  });
}
