// deform_conv2d_tc.cu — tensor-core (Hopper wgmma) path for deform_conv2d.
//
// Reference: csrc/ops/cuda/deform_conv2d_kernel.cu:136-209 (deformable_im2col writes a
// [C_in*kh*kw, pixels] buffer to HBM) + :1234-1239 (cuBLAS addmm) + transpose/copy/bias passes.
//
// Here the op is ONE implicit GEMM whose gathered operand never touches HBM:
//     D[pixel, cout] = sum_k A[pixel, k] * Wt[cout, k],   k = (channel slab, tap, channel in slab)
//   * a CTA owns M = 128 output pixels x N = BN output channels; two consumer warpgroups each own 64 pixel
//     rows and their fp32 accumulator fragment (registers), and issue wgmma.mma_async m64nBNk16 on them;
//   * A tiles are SYNTHESISED by the consumer warps themselves: per (pixel, tap) the 4 bilinear corner
//     offsets and weights (x modulation mask) come from a per-CTA table built once; channels are the
//     fastest axis of a channels-last staging copy of the input, so every corner read is a 128-bit vector
//     load; the blend is rounded to the operand format and stored into the swizzled K-major shared-memory
//     tile the wgmma descriptor expects.  The gather of step q+1 overlaps the wgmma of step q;
//   * B (weights) tiles are pre-packed once per call into the exact swizzled shared-memory image, so a
//     stage is filled by one 1-D bulk async copy (TMA engine) completing on an mbarrier, issued by a
//     dedicated copy warp;
//   * epilogue: accumulators + bias, rounded, transposed through shared memory and written as 16-byte
//     runs of each output channel (NCHW).
#include "async_copy.cuh"
#include <type_traits>

#include "common.cuh"
#include "dcn_geometry.cuh"

namespace vb200 {


namespace {

constexpr int TC_BM = 128;
constexpr int WG_CONSUMERS = 256;                   // two warpgroups x 64 pixel rows
constexpr int WG_THREADS = WG_CONSUMERS + 128;       // + the weight-copy warpgroup (one thread issues the copies)
// registers are allotted per warpgroup: the copy warpgroup gives its share to the consumers (128 x 40 + 256 x 232 <= 64 K)
constexpr int WG_REGS_COPY = 40, WG_REGS_CONSUMER = 232;
// 16-byte chunk c of tile row r is stored at chunk c ^ swz(r): 128-byte rows (KB = 64, SWIZZLE_128B) or
// 64-byte rows (KB = 32, SWIZZLE_64B).
template <int KB> __host__ __device__ constexpr int tc_swz(int r) { return KB == 64 ? (r & 7) : ((r >> 1) & 3); }

// ---- pre-pass 1: NCHW -> NHWC (16-bit elements) -------------------------------------------
// 64 channels x 64 pixels per CTA; 32-bit global accesses on both sides (2 pixels in, 2 channels out),
// 128-byte rows per warp access.  Requires C % 64 == 0 and HW % 2 == 0 (else the scalar kernel below).
template <typename T>
__global__ void __launch_bounds__(256)
nchw_to_nhwc64_kernel(const T* __restrict__ in, T* __restrict__ out, int C, int HW) {
  __shared__ __align__(4) unsigned short tile[64][66];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 64, p0 = blockIdx.x * 64;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned short* __restrict__ src = reinterpret_cast<const unsigned short*>(in) + (int64_t)b * C * HW;
  unsigned short* __restrict__ dst = reinterpret_cast<unsigned short*>(out) + (int64_t)b * C * HW;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = warp + i * 8, p = p0 + 2 * lane;
    uint32_t v = 0u;
    if (p < HW) v = __ldg(reinterpret_cast<const uint32_t*>(src + (int64_t)(c0 + c) * HW + p));
    *reinterpret_cast<uint32_t*>(&tile[c][2 * lane]) = v;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int pl = warp + i * 8, p = p0 + pl;
    if (p < HW) {
      const uint32_t v = (uint32_t)tile[2 * lane][pl] | ((uint32_t)tile[2 * lane + 1][pl] << 16);
      *reinterpret_cast<uint32_t*>(dst + (int64_t)p * C + c0 + 2 * lane) = v;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
nchw_to_nhwc_kernel(const T* __restrict__ in, T* __restrict__ out, int C, int HW) {
  __shared__ T tile[32][33];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8
  const T* __restrict__ src = in + (int64_t)b * C * HW;
  T* __restrict__ dst = out + (int64_t)b * C * HW;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + i * 8, p = p0 + tx;
    if (c < C && p < HW) tile[ty + i * 8][tx] = src[(int64_t)c * HW + p];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int p = p0 + ty + i * 8, c = c0 + tx;
    if (c < C && p < HW) dst[(int64_t)p * C + c] = tile[tx][ty + i * 8];
  }
}

// ---- pre-pass 2: weights [Cout][Cin][KK] -> swizzled K-major tiles ---------------------------
// K order: (64-channel slab, tap, half) -> stage q = (cslab*KK + tap) * (64/KB) + half; tile (nt, q) holds
// BN rows x KB k as the exact shared-memory image: byte = r*(2*KB) + ((kc/8) ^ swz(r))*16 + (kc%8)*2.
template <typename T, int KB>
__global__ void __launch_bounds__(256)
pack_weights_kernel(const T* __restrict__ w, T* __restrict__ packed, int Cout, int Cin, int KK, int BN) {
  const int64_t total = (int64_t)Cout * Cin * KK;
  constexpr int SPLIT = 64 / KB;
  const int n_q = (Cin / 64) * KK * SPLIT;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int tap = (int)(e % KK);
    const int ci = (int)((e / KK) % Cin);
    const int co = (int)(e / KK / Cin);
    const int nt = co / BN, r = co % BN;
    const int cslab = ci / 64, kc64 = ci % 64;
    const int half = kc64 / KB, kc = kc64 % KB;
    const int q = (cslab * KK + tap) * SPLIT + half;
    const int64_t tile_base = ((int64_t)nt * n_q + q) * BN * KB;
    const int off_bytes = r * (2 * KB) + (((kc >> 3) ^ tc_swz<KB>(r)) << 4) + ((kc & 7) << 1);
    packed[tile_base + (off_bytes >> 1)] = w[e];
  }
}

// ---- wgmma wrappers ---------------------------------------------------------------------------
// K-major swizzled shared-memory matrix descriptor (sm_90 GMMA): start>>4 [0,14) | LBO>>4 [16,30) (unused for
// swizzled K-major: 1) | SBO>>4 [32,46) = bytes between 8-row groups (8 * row bytes) | layout [62,64):
// 1 = SWIZZLE_128B, 2 = SWIZZLE_64B.  The 16-element K steps inside a row advance the start address by 32 bytes.
template <int ROW_BYTES>
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr) {
  constexpr uint64_t sbo = (uint64_t)(8 * ROW_BYTES) >> 4;
  constexpr uint64_t layout = ROW_BYTES == 128 ? 1ull : 2ull;
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | (sbo << 32) | (layout << 62);
}
template <int N> __device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator registers across the asynchronous MMAs
template <int R> __device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] += A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory, fp32 accumulator fragment:
// d[4j + 2h + e] = (row 16 * warp + lane / 4 + 8h, column 8j + 2 (lane % 4) + e) of the warpgroup's 64 rows.
// FMT: 1 = bf16, 0 = fp16.
template <int N> struct Wgmma;
template <> struct Wgmma<64> {
  template <int FMT> static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db) {
    if constexpr (FMT == 1)
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                   : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                   : "l"(da), "l"(db));
    else
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                   : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                   : "l"(da), "l"(db));
  }
};
// bf16 m64n64k16 with a run-time scale-d: D = A B^T when scale_d == 0 (the accumulator's old value is ignored), else D += A B^T
__device__ __forceinline__ void wgmma64_bf16_sd(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(da), "l"(db), "r"(scale_d));
}
template <> struct Wgmma<128> {
  template <int FMT> static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db) {
    if constexpr (FMT == 1)
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                   : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                   : "l"(da), "l"(db));
    else
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                   : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                   : "l"(da), "l"(db));
  }
};
template <> struct Wgmma<256> {
  template <int FMT> static __device__ __forceinline__ void mma(float (&d)[128], uint64_t da, uint64_t db) {
    if constexpr (FMT == 1)
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
                   : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
                   : "l"(da), "l"(db));
    else
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
                   : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
                   : "l"(da), "l"(db));
  }
};

template <typename T> struct Elem;
template <> struct Elem<__nv_bfloat16> {
  static constexpr uint32_t kFmt = 1;
  static __device__ __forceinline__ float2 up(uint32_t u) { return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u)); }
  static __device__ __forceinline__ uint32_t pk(float a, float b) { __nv_bfloat162 v = __floats2bfloat162_rn(a, b); return *reinterpret_cast<uint32_t*>(&v); }
};
template <> struct Elem<__half> {
  static constexpr uint32_t kFmt = 0;
  static __device__ __forceinline__ uint32_t dup(float w) { __half2 v = __float2half2_rn(w); return *reinterpret_cast<uint32_t*>(&v); }
  static __device__ __forceinline__ uint32_t mul2(uint32_t w, uint32_t a) {
    __half2 r = __hmul2(*reinterpret_cast<__half2*>(&w), *reinterpret_cast<__half2*>(&a)); return *reinterpret_cast<uint32_t*>(&r); }
  static __device__ __forceinline__ uint32_t fma2p(uint32_t w, uint32_t a, uint32_t c) {
    __half2 r = __hfma2(*reinterpret_cast<__half2*>(&w), *reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&c));
    return *reinterpret_cast<uint32_t*>(&r); }
  static __device__ __forceinline__ float2 up(uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); }
  static __device__ __forceinline__ uint32_t pk(float a, float b) { __half2 v = __floats2half2_rn(a, b); return *reinterpret_cast<uint32_t*>(&v); }
};

// Writes the finished [BN channels][128 pixels] tile (shared memory, row pitch LD elements) to NCHW `out` and to the
// peer slots of the fused all-gather: 16-byte runs along the pixels of each channel where the tile is whole and aligned.
template <typename T, int BN>
__device__ __forceinline__ void store_tile(const T* tile, int LD, T* __restrict__ out, const DcnParams& p, int b, int nt, int pix0,
                                           int tid) {
  constexpr int EPC = 16 / (int)sizeof(T);               // elements per 16-byte chunk
  constexpr int CPR = TC_BM / EPC;                       // chunks per channel row of the tile
  const int HWo = p.out_h * p.out_w;
  bool vec = pix0 + TC_BM <= HWo && (HWo % EPC) == 0 && (reinterpret_cast<uintptr_t>(out) % 16) == 0;
  for (int d = 0; d < p.n_peer; ++d) vec = vec && (reinterpret_cast<uintptr_t>(p.peer_out[d]) % 16) == 0;
  for (int idx = tid; idx < BN * CPR; idx += WG_CONSUMERS) {
    const int ch = idx / CPR, seg = idx - ch * CPR;
    const T* src = tile + ch * LD + seg * EPC;
    const int64_t e0 = ((int64_t)b * p.c_out + nt * BN + ch) * HWo + pix0 + seg * EPC;
    if (vec) {
      const uint4 v = *reinterpret_cast<const uint4*>(src);
      *reinterpret_cast<uint4*>(out + e0) = v;
      for (int d = 0; d < p.n_peer; ++d) *reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.peer_out[d]) + e0) = v;
    } else {
#pragma unroll
      for (int e = 0; e < EPC; ++e) {
        if (pix0 + seg * EPC + e < HWo) {
          out[e0 + e] = src[e];
          for (int d = 0; d < p.n_peer; ++d) reinterpret_cast<T*>(p.peer_out[d])[e0 + e] = src[e];
        }
      }
    }
  }
}

// 16-bit storage types.  BN = output channels per CTA (128 or 256: one m64nBNk16 accumulator per warpgroup), K depth 64
// per stage (128-byte rows, SWIZZLE_128B), STAGES x (A 16 KB + B BN x 128 B).
template <typename T, int BN, int STAGES>
__global__ void __launch_bounds__(WG_THREADS, 1)
deform_conv2d_tc_kernel(const T* __restrict__ nhwc, const T* __restrict__ wpacked, const T* __restrict__ offset,
                        const T* __restrict__ mask, const T* __restrict__ bias, T* __restrict__ out, DcnParams p) {
  constexpr int ROW_BYTES = 128;
  constexpr int A_BYTES = TC_BM * ROW_BYTES;
  constexpr int B_BYTES = BN * ROW_BYTES;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // the A rows of a stage are rewritten once every warp of the warpgroup has waited for the MMAs of three steps back
  static_assert(STAGES >= 3, "A-tile reuse distance");
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* stages = smem;
  uint64_t* fullB = reinterpret_cast<uint64_t*>(stages + STAGES * STAGE_BYTES);
  uint64_t* empty = fullB + STAGES;
  DcnTabEnt* tab = reinterpret_cast<DcnTabEnt*>(stages + ((STAGES * STAGE_BYTES + 2 * STAGES * 8 + 31) & ~31));

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int KK = p.kh * p.kw;
  const int HWo = p.out_h * p.out_w, HWi = p.in_h * p.in_w;
  const int tiles_per_img = ceil_div(HWo, TC_BM);
  const int b = blockIdx.x / tiles_per_img;
  const int pix0 = (blockIdx.x % tiles_per_img) * TC_BM;
  const int nt = blockIdx.y;
  const int c_per_off = p.c_in / p.offset_groups;
  const int slabs_per_og = (c_per_off / 64) * KK;      // 64-channel steps per offset group
  const int n_q = (p.c_in / 64) * KK;                  // pipeline stages consumed per tile

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&fullB[s], 1); mbar_init(&empty[s], WG_CONSUMERS / 32); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= WG_CONSUMERS / 32) {
    // ================= weight tiles: one bulk copy per stage =================
    regs_dec<WG_REGS_COPY>();
    if (warp == WG_CONSUMERS / 32 && lane == 0) {
      const unsigned char* wsrc = reinterpret_cast<const unsigned char*>(wpacked) + (int64_t)nt * n_q * B_BYTES;
      for (int q = 0; q < n_q; ++q) {
        const int st = q % STAGES;
        mbar_wait(&empty[st], ((uint32_t)(q / STAGES) & 1u) ^ 1u);
        mbar_expect_tx(&fullB[st], (uint32_t)B_BYTES);
        bulk_g2s(stages + st * STAGE_BYTES + A_BYTES, wsrc + (int64_t)q * B_BYTES, (uint32_t)B_BYTES, &fullB[st]);
      }
    }
    return;
  }

  // ================= consumer warpgroups: gather A, issue the MMAs =================
  regs_inc<WG_REGS_CONSUMER>();
  const int wg = warp >> 2;
  // lane = (pixel sub-index pq, 16-byte chunk c): one warp load instruction reads four complete 128-byte lines
  // (4 pixels x 64 channels)
  const int cchunk = lane & 7, pq = lane >> 3;
  const int prow0 = warp * 16 + pq;                     // + 4 * i, i = 0..3; warpgroup wg owns rows [64 wg, 64 wg + 64)
  const T* __restrict__ in_b = nhwc + (int64_t)b * HWi * p.c_in;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  int q = 0;
  for (int og = 0; og < p.offset_groups; ++og) {
    asm volatile("bar.sync 1, %0;" ::"n"(WG_CONSUMERS));     // previous table no longer read
    const T* __restrict__ off_b = offset + ((int64_t)b * p.offset_groups + og) * 2 * KK * HWo;
    const T* __restrict__ msk_b = p.use_mask ? mask + ((int64_t)b * p.offset_groups + og) * KK * HWo : nullptr;
    fill_sample_table<TC_BM>(tab, off_b, msk_b, p, 0, KK, pix0, p.c_in * (int)sizeof(T), tid, WG_CONSUMERS);
    asm volatile("bar.sync 1, %0;" ::"n"(WG_CONSUMERS));
    // channel slab outer, tap inner (L1 reuse across taps)
    for (int sl = 0; sl < slabs_per_og; ++sl, ++q) {
      const int cs_local = sl / KK, tap = sl - cs_local * KK;
      // corner offsets are 32-bit BYTE offsets (image < 2^30 elements): uniform 64-bit base + 32-bit offset
      const char* __restrict__ in_c = reinterpret_cast<const char*>(in_b + og * c_per_off + cs_local * 64);
      const uint32_t lane_off = (uint32_t)cchunk * 16u;
      uint4 v[4][4];                                       // [pixel][corner]
      float4 wq[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {                        // all 16 loads in flight before the blend
        const DcnTabEnt* se = tab + tap * TC_BM + prow0 + 4 * i;
        const uint4 o = *reinterpret_cast<const uint4*>(se->o);
        wq[i] = *reinterpret_cast<const float4*>(se->w);
        v[i][0] = __ldg(reinterpret_cast<const uint4*>(in_c + (o.x + lane_off)));
        v[i][1] = __ldg(reinterpret_cast<const uint4*>(in_c + (o.y + lane_off)));
        v[i][2] = __ldg(reinterpret_cast<const uint4*>(in_c + (o.z + lane_off)));
        v[i][3] = __ldg(reinterpret_cast<const uint4*>(in_c + (o.w + lane_off)));
      }
      const int st = q % STAGES;
      unsigned char* a_tile = stages + st * STAGE_BYTES;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float wv[4] = {wq[i].x, wq[i].y, wq[i].z, wq[i].w};
        uint4 o;
        if constexpr (std::is_same<T, __half>::value) {
          // fp16: blend in the storage format (HFMA2): 16 instructions per 8 channels instead of 52 (unpack + FFMA + pack).
          // Every step rounds to 16 bits - the A operand is rounded to that format anyway; the whole op stays inside its 1e-2
          // bound.  bf16 keeps the fp32 blend: packed in bf16 the blend exceeds that bound (DESIGN §4.5).
          const uint32_t w0 = Elem<T>::dup(wv[0]), w1 = Elem<T>::dup(wv[1]), w2_ = Elem<T>::dup(wv[2]), w3 = Elem<T>::dup(wv[3]);
          o.x = Elem<T>::fma2p(w3, v[i][3].x, Elem<T>::fma2p(w2_, v[i][2].x, Elem<T>::fma2p(w1, v[i][1].x, Elem<T>::mul2(w0, v[i][0].x))));
          o.y = Elem<T>::fma2p(w3, v[i][3].y, Elem<T>::fma2p(w2_, v[i][2].y, Elem<T>::fma2p(w1, v[i][1].y, Elem<T>::mul2(w0, v[i][0].y))));
          o.z = Elem<T>::fma2p(w3, v[i][3].z, Elem<T>::fma2p(w2_, v[i][2].z, Elem<T>::fma2p(w1, v[i][1].z, Elem<T>::mul2(w0, v[i][0].z))));
          o.w = Elem<T>::fma2p(w3, v[i][3].w, Elem<T>::fma2p(w2_, v[i][2].w, Elem<T>::fma2p(w1, v[i][1].w, Elem<T>::mul2(w0, v[i][0].w))));
        } else {
          unsigned long long acc2[4] = {0ull, 0ull, 0ull, 0ull};   // 8 channels as 4 fp32 pairs
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const uint32_t u[4] = {v[i][c].x, v[i][c].y, v[i][c].z, v[i][c].w};
            const unsigned long long w2 = pack2(wv[c], wv[c]);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 f = Elem<T>::up(u[k]);
              acc2[k] = fma2(w2, pack2(f.x, f.y), acc2[k]);
            }
          }
          o.x = Elem<T>::pk(lo32(acc2[0]), hi32(acc2[0])); o.y = Elem<T>::pk(lo32(acc2[1]), hi32(acc2[1]));
          o.z = Elem<T>::pk(lo32(acc2[2]), hi32(acc2[2])); o.w = Elem<T>::pk(lo32(acc2[3]), hi32(acc2[3]));
        }
        const int prow = prow0 + 4 * i;
        *reinterpret_cast<uint4*>(a_tile + prow * ROW_BYTES + ((cchunk ^ tc_swz<64>(prow)) << 4)) = o;
      }
      fence_proxy_async();                  // generic-proxy stores -> visible to the tensor core (async proxy)
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");     // the warpgroup's 64 rows are complete
      mbar_wait(&fullB[st], (uint32_t)(q / STAGES) & 1u);
      const uint32_t a_addr = smem_u32(a_tile) + (uint32_t)(wg * 64 * ROW_BYTES);
      const uint32_t b_addr = smem_u32(a_tile) + A_BYTES;
      wg_fence_acc(acc);
      wg_fence();
#pragma unroll
      for (int k = 0; k < 64 / 16; ++k)
        Wgmma<BN>::template mma<Elem<T>::kFmt>(acc, wg_desc<ROW_BYTES>(a_addr + k * 32), wg_desc<ROW_BYTES>(b_addr + k * 32));
      wg_commit();
      wg_wait<1>();                         // the MMAs of step q-1 are done: its stage may be refilled
      wg_fence_acc(acc);
      if (lane == 0 && q > 0) mbar_arrive(&empty[(q - 1) % STAGES]);
    }
  }
  wg_wait<0>();
  wg_fence_acc(acc);

  // ================= epilogue: registers -> transposed tile in shared memory -> NCHW =================
  asm volatile("bar.sync 1, %0;" ::"n"(WG_CONSUMERS) : "memory");     // every MMA has read its last stage
  constexpr int LD = TC_BM + 8;                         // padded pixel rows (16-byte aligned)
  static_assert(BN * LD * (int)sizeof(T) <= STAGES * STAGE_BYTES, "epilogue tile must fit the pipeline stages");
  T* tile = reinterpret_cast<T*>(stages);
  const int row_base = warp * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = 8 * j + 2 * (lane & 3) + e;
      const float bv = bias ? to_acc(bias[nt * BN + col]) : 0.f;
      tile[col * LD + row_base] = from_acc<T, float>(acc[4 * j + e] + bv);
      tile[col * LD + row_base + 8] = from_acc<T, float>(acc[4 * j + 2 + e] + bv);
    }
  }
  asm volatile("bar.sync 1, %0;" ::"n"(WG_CONSUMERS) : "memory");
  store_tile<T, BN>(tile, LD, out, p, b, nt, pix0, tid);
}


// =================================================================================================
// fp32 inputs on the tensor core: three-way bf16 split (bf16x3).
// A float v is v1 + v2 + v3 with v1 = bf16(v), v2 = bf16(v - v1), v3 = bf16(v - v1 - v2) (8 + 8 + 8 mantissa bits); the
// product a*b is a1b1 + (a1b2 + a2b1) + (a2b2 + a1b3 + a3b1) + O(2^-24): SIX bf16 MMAs per K step reproduce the fp32
// product to about 2^-24 relative - inside the 1e-5 budget of the fp32 rows with the accumulation below - at 6x the
// bf16 tensor time, still several times faster than a SIMT fp32 implicit GEMM (or the reference's im2col + SGEMM).  Same structure as
// deform_conv2d_tc_kernel: M = 128 pixels, N = BN couts, K step 32 channels (SWIZZLE_64B); a stage holds A1 A2 A3
// (8 KB each) and B1 B2 B3 (BN x 64 B each); the gather reads a channels-last fp32 staging copy (one 128-byte line =
// 32 channels per pixel corner), blends in fp32 and writes the three splits.
// ACCUMULATION: the tensor core adds into its fp32 accumulator with truncation (about one ulp of the accumulator per MMA
// instruction, a bias that grows linearly with the number of MMAs into one accumulator).  So (1) the five correction
// terms go to their OWN accumulator (its magnitude is 2^-8 of the result, so its truncation is invisible), (2) the
// a1 b1 terms alternate over TWO accumulators by K step and (3) after every T3_FOLD of its own K steps an accumulator is
// added, round-to-nearest, into a register total, so none takes more than 16 truncating MMAs.  The fold reads an
// accumulator whose MMAs are complete while the MMAs of the next step (into the other one) are in flight, so the
// pipeline does not drain; the accumulator's next MMA then overwrites it (scale-d 0) - zeroing the registers instead
// would serialise the wgmma pipeline.  Without (3) (three rotating accumulators) the error grew with depth past the 1e-5
// bound: 2.2e-5 of 1 + |ref| at K = 10240 on post-ReLU-like activations.  The epilogue adds the total, the two and the
// corrections with round-to-nearest.
// BN = 64: 2 + 1 accumulators + the total x 32 registers per thread.
// =================================================================================================
constexpr int T3_KB = 32, T3_STAGES = 4, T3_MAIN = 2, T3_FOLD = 8;
constexpr int T3_ROW = 2 * T3_KB;                 // 64-byte tile rows
constexpr int T3_A = TC_BM * T3_ROW;              // 8 KB per A split

__device__ __forceinline__ void split3(float v, __nv_bfloat16& a, __nv_bfloat16& b, __nv_bfloat16& c) {
  a = __float2bfloat16_rn(v);
  const float r1 = v - __bfloat162float(a);      // exact: the residual has at most 16 significant bits
  b = __float2bfloat16_rn(r1);
  c = __float2bfloat16_rn(r1 - __bfloat162float(b));
}

template <int R>
__device__ __forceinline__ void fold_acc(float (&total)[R], const float (&a)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) total[i] = __fadd_rn(total[i], a[i]);
}

// weights [Cout][Cin][KK] fp32 -> per (n tile, stage q = cslab32 * KK + tap): B1 | B2 | B3 swizzled tiles of BN x 32
__global__ void __launch_bounds__(256)
pack_weights3_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ packed, int Cout, int Cin, int KK, int BN) {
  const int64_t total = (int64_t)Cout * Cin * KK;
  const int n_q = (Cin / T3_KB) * KK;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int tap = (int)(e % KK);
    const int ci = (int)((e / KK) % Cin);
    const int co = (int)(e / KK / Cin);
    const int nt = co / BN, r = co % BN;
    const int cslab = ci / T3_KB, kc = ci % T3_KB;
    const int q = cslab * KK + tap;
    const int64_t stage_base = ((int64_t)nt * n_q + q) * 3 * BN * T3_KB;            // elements
    const int off = (r * T3_ROW + (((kc >> 3) ^ tc_swz<T3_KB>(r)) << 4) + ((kc & 7) << 1)) >> 1;
    __nv_bfloat16 b1, b2, b3;
    split3(w[e], b1, b2, b3);
    packed[stage_base + off] = b1;
    packed[stage_base + (int64_t)BN * T3_KB + off] = b2;
    packed[stage_base + (int64_t)2 * BN * T3_KB + off] = b3;
  }
}

template <int BN>
__global__ void __launch_bounds__(WG_THREADS, 1)
deform_conv2d_tc3_kernel(const float* __restrict__ nhwc, const __nv_bfloat16* __restrict__ wpacked, const float* __restrict__ offset,
                         const float* __restrict__ mask, const float* __restrict__ bias, float* __restrict__ out, DcnParams p) {
  constexpr int B_BYTES = BN * T3_ROW;                    // one B split
  constexpr int STAGE_BYTES = 3 * T3_A + 3 * B_BYTES;
  static_assert(T3_STAGES >= 3, "A-tile reuse distance");
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* stages = smem;
  uint64_t* fullB = reinterpret_cast<uint64_t*>(stages + T3_STAGES * STAGE_BYTES);
  uint64_t* empty = fullB + T3_STAGES;
  DcnTabEnt* tab = reinterpret_cast<DcnTabEnt*>(stages + ((T3_STAGES * STAGE_BYTES + 2 * T3_STAGES * 8 + 31) & ~31));

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int KK = p.kh * p.kw;
  const int HWo = p.out_h * p.out_w, HWi = p.in_h * p.in_w;
  const int tiles_per_img = ceil_div(HWo, TC_BM);
  const int b = blockIdx.x / tiles_per_img;
  const int pix0 = (blockIdx.x % tiles_per_img) * TC_BM;
  const int nt = blockIdx.y;
  const int c_per_off = p.c_in / p.offset_groups;
  const int slabs_per_og = (c_per_off / T3_KB) * KK;      // 32-channel steps per offset group
  const int n_q = (p.c_in / T3_KB) * KK;                  // stages consumed per tile

  if (tid == 0) {
    for (int s = 0; s < T3_STAGES; ++s) { mbar_init(&fullB[s], 1); mbar_init(&empty[s], WG_CONSUMERS / 32); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= WG_CONSUMERS / 32) {
    regs_dec<WG_REGS_COPY>();
    if (warp == WG_CONSUMERS / 32 && lane == 0) {
      const unsigned char* wsrc = reinterpret_cast<const unsigned char*>(wpacked) + (int64_t)nt * n_q * 3 * B_BYTES;
      for (int q = 0; q < n_q; ++q) {
        const int st = q % T3_STAGES;
        mbar_wait(&empty[st], ((uint32_t)(q / T3_STAGES) & 1u) ^ 1u);
        mbar_expect_tx(&fullB[st], (uint32_t)(3 * B_BYTES));
        bulk_g2s(stages + st * STAGE_BYTES + 3 * T3_A, wsrc + (int64_t)q * 3 * B_BYTES, (uint32_t)(3 * B_BYTES), &fullB[st]);
      }
    }
    return;
  }

  regs_inc<WG_REGS_CONSUMER>();
  const int wg = warp >> 2;
  const int cchunk = lane & 7, pq = lane >> 3;             // lane -> (pixel sub-index, 4-channel chunk of the 32-channel line)
  const int prow0 = warp * 16 + pq;
  const float* __restrict__ in_b = nhwc + (int64_t)b * HWi * p.c_in;
  float acc0[BN / 2], acc1[BN / 2], accs[BN / 2];      // main accumulators (q mod 2) + corrections
  float total[BN / 2];                                                // folded main accumulators (round-to-nearest)
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; accs[i] = 0.f; total[i] = 0.f; }
  int q = 0;
  for (int og = 0; og < p.offset_groups; ++og) {
    asm volatile("bar.sync 1, %0;" ::"n"(WG_CONSUMERS));
    const float* __restrict__ off_b = offset + ((int64_t)b * p.offset_groups + og) * 2 * KK * HWo;
    const float* __restrict__ msk_b = p.use_mask ? mask + ((int64_t)b * p.offset_groups + og) * KK * HWo : nullptr;
    fill_sample_table<TC_BM>(tab, off_b, msk_b, p, 0, KK, pix0, p.c_in * (int)sizeof(float), tid, WG_CONSUMERS);
    asm volatile("bar.sync 1, %0;" ::"n"(WG_CONSUMERS));
    for (int sl = 0; sl < slabs_per_og; ++sl, ++q) {
      const int cs_local = sl / KK, tap = sl - cs_local * KK;
      const char* __restrict__ in_c = reinterpret_cast<const char*>(in_b + og * c_per_off + cs_local * T3_KB);
      const uint32_t lane_off = (uint32_t)cchunk * 16u;
      float4 v[4][4];
      float4 wq[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const DcnTabEnt* se = tab + tap * TC_BM + prow0 + 4 * i;
        const uint4 o = *reinterpret_cast<const uint4*>(se->o);
        wq[i] = *reinterpret_cast<const float4*>(se->w);
        v[i][0] = __ldg(reinterpret_cast<const float4*>(in_c + (o.x + lane_off)));
        v[i][1] = __ldg(reinterpret_cast<const float4*>(in_c + (o.y + lane_off)));
        v[i][2] = __ldg(reinterpret_cast<const float4*>(in_c + (o.z + lane_off)));
        v[i][3] = __ldg(reinterpret_cast<const float4*>(in_c + (o.w + lane_off)));
      }
      const int st = q % T3_STAGES;
      unsigned char* a_tile = stages + st * STAGE_BYTES;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        // fp32 blend in the reference's tap order (w1 v1 + w2 v2 + w3 v3 + w4 v4, deform_conv2d_kernel.cu:128-133)
        float r[4];
        r[0] = wq[i].x * v[i][0].x + wq[i].y * v[i][1].x + wq[i].z * v[i][2].x + wq[i].w * v[i][3].x;
        r[1] = wq[i].x * v[i][0].y + wq[i].y * v[i][1].y + wq[i].z * v[i][2].y + wq[i].w * v[i][3].y;
        r[2] = wq[i].x * v[i][0].z + wq[i].y * v[i][1].z + wq[i].z * v[i][2].z + wq[i].w * v[i][3].z;
        r[3] = wq[i].x * v[i][0].w + wq[i].y * v[i][1].w + wq[i].z * v[i][2].w + wq[i].w * v[i][3].w;
        __nv_bfloat16 s1[4], s2[4], s3[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) split3(r[k], s1[k], s2[k], s3[k]);
        const int prow = prow0 + 4 * i;
        // this lane's 4 channels are half of a 16-byte chunk: chunk (cchunk >> 1), byte half (cchunk & 1)
        const int boff = prow * T3_ROW + ((((cchunk >> 1) ^ tc_swz<T3_KB>(prow)) << 4) | ((cchunk & 1) << 3));
        *reinterpret_cast<uint2*>(a_tile + boff) = *reinterpret_cast<const uint2*>(s1);
        *reinterpret_cast<uint2*>(a_tile + T3_A + boff) = *reinterpret_cast<const uint2*>(s2);
        *reinterpret_cast<uint2*>(a_tile + 2 * T3_A + boff) = *reinterpret_cast<const uint2*>(s3);
      }
      fence_proxy_async();
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
      mbar_wait(&fullB[st], (uint32_t)(q / T3_STAGES) & 1u);
      const uint32_t a_addr = smem_u32(a_tile) + (uint32_t)(wg * 64 * T3_ROW);
      const uint32_t b_addr = smem_u32(a_tile) + 3 * T3_A;
      wg_fence_acc(acc0); wg_fence_acc(acc1); wg_fence_acc(accs); wg_fence_acc(total);
      wg_fence();
      // correction terms (a3b1, a1b3, a2b2, a2b1, a1b2) -> their own accumulator
      constexpr int ia[5] = {2, 0, 1, 1, 0}, ib[5] = {0, 2, 1, 0, 1};
#pragma unroll
      for (int t = 0; t < 5; ++t) {
#pragma unroll
        for (int k = 0; k < T3_KB / 16; ++k)
          Wgmma<BN>::template mma<1>(accs, wg_desc<T3_ROW>(a_addr + ia[t] * T3_A + k * 32), wg_desc<T3_ROW>(b_addr + ib[t] * B_BYTES + k * 32));
      }
      // a1 b1 -> main accumulator q mod 2, restarted (scale-d 0) when it was folded into the total after its last step
      const int m = q % T3_MAIN;
      const int keep = (q >= T3_MAIN && ((q - T3_MAIN) / T3_MAIN) % T3_FOLD == T3_FOLD - 1) ? 0 : 1;
      static_assert(BN == 64, "the main-accumulator MMAs are written for m64n64k16");
#pragma unroll
      for (int k = 0; k < T3_KB / 16; ++k) {
        const uint64_t da = wg_desc<T3_ROW>(a_addr + k * 32), db = wg_desc<T3_ROW>(b_addr + k * 32);
        const int sd = k == 0 ? keep : 1;
        if (m == 0) wgmma64_bf16_sd(acc0, da, db, sd);
        else wgmma64_bf16_sd(acc1, da, db, sd);
      }
      wg_commit();
      wg_wait<1>();
      wg_fence_acc(acc0); wg_fence_acc(acc1); wg_fence_acc(accs); wg_fence_acc(total);
      if (lane == 0 && q > 0) mbar_arrive(&empty[(q - 1) % T3_STAGES]);
      // step q-1 is complete: fold its main accumulator once that accumulator has taken T3_FOLD steps, if a later step
      // (q+1) restarts it; otherwise the epilogue adds it
      if (q > 0 && q + 1 < n_q && ((q - 1) / T3_MAIN) % T3_FOLD == T3_FOLD - 1) {
        if ((q - 1) % T3_MAIN == 0) fold_acc(total, acc0);
        else fold_acc(total, acc1);
      }
    }
  }
  wg_wait<0>();
  wg_fence_acc(acc0); wg_fence_acc(acc1); wg_fence_acc(accs); wg_fence_acc(total);

  // ================= epilogue: registers -> transposed tile in shared memory -> NCHW fp32 =================
  asm volatile("bar.sync 1, %0;" ::"n"(WG_CONSUMERS) : "memory");
  constexpr int LD = TC_BM + 4;
  static_assert(BN * LD * 4 <= T3_STAGES * STAGE_BYTES, "epilogue tile must fit the pipeline stages");
  float* tile = reinterpret_cast<float*>(stages);
  const int row_base = warp * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 4 * j + 2 * h + e, col = 8 * j + 2 * (lane & 3) + e;
        const float main = total[i] + (acc1[i] + acc0[i]);
        tile[col * LD + row_base + 8 * h] = (main + accs[i]) + (bias ? bias[nt * BN + col] : 0.f);
      }
    }
  }
  asm volatile("bar.sync 1, %0;" ::"n"(WG_CONSUMERS) : "memory");
  store_tile<float, BN>(tile, LD, out, p, b, nt, pix0, tid);
}

size_t tc3_smem_bytes(int BN, int KK) {
  return (size_t)T3_STAGES * (3 * T3_A + 3 * BN * T3_ROW) + 64 + (size_t)KK * TC_BM * sizeof(DcnTabEnt) + 1024;
}
constexpr int T3_BN = 64;
bool tc3_eligible(int dtype, const DcnParams& p) {
  if (dtype != VB200_F32 || p.groups != 1) return false;
  if (p.c_in % p.offset_groups != 0 || (p.c_in / p.offset_groups) % T3_KB != 0) return false;
  if (p.c_out % 128 != 0 || tc3_smem_bytes(T3_BN, p.kh * p.kw) > (size_t)max_smem_optin()) return false;
  if ((int64_t)p.in_h * p.in_w * p.c_in * 4 >= (1ll << 31)) return false;      // 32-bit byte offsets into one image
  const char* env = env_override(ENV_DCN_PATH);
  if (env && env[0] == 's') return false;
  return true;
}

// BN = 256: 3 stages x 48 KB; BN = 128: 4 stages x 32 KB (plus the [KK][128] sampling table).
constexpr int tc_stages(int BN) { return BN == 256 ? 3 : 4; }
size_t tc_smem_bytes(int BN, int KK) {
  return (size_t)tc_stages(BN) * (TC_BM + BN) * 128 + 64 + (size_t)KK * TC_BM * sizeof(DcnTabEnt) + 1024;
}
int tc_pick_bn(const DcnParams& p) {
  const int KK = p.kh * p.kw;
  for (const int bn : {256, 128})
    if (p.c_out % bn == 0 && tc_smem_bytes(bn, KK) <= (size_t)max_smem_optin()) return bn;
  return 0;
}

bool tc_eligible(int dtype, const DcnParams& p) {
  if (dtype != VB200_BF16 && dtype != VB200_F16) return false;
  if (p.groups != 1) return false;
  if (p.c_in % p.offset_groups != 0 || (p.c_in / p.offset_groups) % 64 != 0) return false;
  if (p.c_out % 128 != 0) return false;
  if (tc_pick_bn(p) == 0) return false;
  if ((int64_t)p.in_h * p.in_w * p.c_in >= (1ll << 30)) return false;      // 32-bit byte offsets into one image
  const char* env = env_override(ENV_DCN_PATH);
  if (env && env[0] == 's') return false;
  return true;
}

template <typename T>
int pack_tc_weights(const void* weight, T* wpacked, const DcnParams& p, cudaStream_t st) {
  pack_weights_kernel<T, 64><<<sm_count() * 4, 256, 0, st>>>((const T*)weight, wpacked, p.c_out, p.c_in, p.kh * p.kw, tc_pick_bn(p));
  return check_launch("pack_weights_kernel");
}

template <typename T>
int launch_tc(const void* input, const void* weight, const void* offset, const void* mask, const void* bias, void* out,
              const DcnParams& p_in, void* workspace, size_t workspace_bytes, cudaStream_t st, const DcnHints& hints) {
  DcnParams p = p_in;
  const int KK = p.kh * p.kw, HWi = p.in_h * p.in_w, HWo = p.out_h * p.out_w;
  const size_t nhwc_bytes = hints.input_is_nhwc ? 0 : align256((size_t)p.batch * HWi * p.c_in * sizeof(T));
  const size_t w_bytes = hints.packed_weight ? 0 : align256((size_t)p.c_out * p.c_in * KK * sizeof(T));
  if (nhwc_bytes + w_bytes > 0 && (workspace == nullptr || workspace_bytes < nhwc_bytes + w_bytes || ((uintptr_t)workspace % 256) != 0))
    return 0;       // no usable workspace: the SIMT kernel serves the call (a C-ABI caller may pass none)
  T* nhwc = hints.input_is_nhwc ? (T*)const_cast<void*>(input) : (T*)workspace;
  T* wpacked = hints.packed_weight ? (T*)const_cast<void*>(hints.packed_weight) : (T*)((char*)workspace + nhwc_bytes);
  if (hints.input_is_nhwc) {
    if (((uintptr_t)input % 16) != 0) { set_error("deform_conv2d: channels-last input must be 16-byte aligned"); return VB200_EINVAL; }
  } else if (HWi % 2 == 0 && p.c_in % 64 == 0 && ((uintptr_t)input % 4) == 0) {
    dim3 tg((unsigned)ceil_div(HWi, 64), (unsigned)(p.c_in / 64), (unsigned)p.batch);
    nchw_to_nhwc64_kernel<T><<<tg, 256, 0, st>>>((const T*)input, nhwc, p.c_in, HWi);
  } else {
    dim3 tg((unsigned)ceil_div(HWi, 32), (unsigned)ceil_div(p.c_in, 32), (unsigned)p.batch);
    nchw_to_nhwc_kernel<T><<<tg, 256, 0, st>>>((const T*)input, nhwc, p.c_in, HWi);
  }
  int rc = hints.input_is_nhwc ? 0 : check_launch("nchw_to_nhwc_kernel");
  if (rc) return rc;
  if (!hints.packed_weight) {
    rc = pack_tc_weights<T>(weight, wpacked, p, st);
    if (rc) return rc;
  }
  const int BN = tc_pick_bn(p);
  dim3 grid((unsigned)(p.batch * ceil_div(HWo, TC_BM)), (unsigned)(p.c_out / BN));
  const size_t smem = tc_smem_bytes(BN, KK);
  p.n_peer = hints.peer_out ? hints.n_peer : 0;
  for (int d = 0; d < p.n_peer; ++d) p.peer_out[d] = hints.peer_out[d];
  if (hints.peers_done) *hints.peers_done = true;
#define VB200_TC_LAUNCH(BN_)                                                                                              \
  {                                                                                                                       \
    VB200_CUDA_TRY(ensure_dyn_smem<deform_conv2d_tc_kernel<T, BN_, tc_stages(BN_)>>(smem));                               \
    deform_conv2d_tc_kernel<T, BN_, tc_stages(BN_)><<<grid, WG_THREADS, smem, st>>>(                                      \
        nhwc, wpacked, (const T*)offset, (const T*)mask, (const T*)bias, (T*)out, p);                                     \
  }
  if (BN == 256) VB200_TC_LAUNCH(256) else VB200_TC_LAUNCH(128)
#undef VB200_TC_LAUNCH
  rc = check_launch("deform_conv2d_tc_kernel");
  return rc ? rc : 1;
}

}  // namespace

int launch_tc3(const void* input, const void* weight, const void* offset, const void* mask, const void* bias, void* out,
               const DcnParams& p_in, void* workspace, size_t workspace_bytes, cudaStream_t st, const DcnHints& hints) {
  DcnParams p = p_in;
  p.n_peer = 0;                                           // the caller copies to the peer destinations
  const int KK = p.kh * p.kw, HWi = p.in_h * p.in_w, HWo = p.out_h * p.out_w;
  const size_t nhwc_bytes = hints.input_is_nhwc ? 0 : align256((size_t)p.batch * HWi * p.c_in * 4);
  const size_t w_bytes = hints.packed_weight ? 0 : align256((size_t)p.c_out * p.c_in * KK * 3 * 2);
  if (nhwc_bytes + w_bytes > 0 && (workspace == nullptr || workspace_bytes < nhwc_bytes + w_bytes || ((uintptr_t)workspace % 256) != 0))
    return 0;   // SIMT kernel serves the call
  float* nhwc = hints.input_is_nhwc ? (float*)const_cast<void*>(input) : (float*)workspace;
  __nv_bfloat16* wpacked = hints.packed_weight ? (__nv_bfloat16*)const_cast<void*>(hints.packed_weight) : (__nv_bfloat16*)((char*)workspace + nhwc_bytes);
  int rc = 0;
  if (!hints.input_is_nhwc) {
    dim3 tg((unsigned)ceil_div(HWi, 32), (unsigned)ceil_div(p.c_in, 32), (unsigned)p.batch);
    nchw_to_nhwc_kernel<float><<<tg, 256, 0, st>>>((const float*)input, nhwc, p.c_in, HWi);
    rc = check_launch("nchw_to_nhwc_kernel");
    if (rc) return rc;
  } else if (((uintptr_t)input % 16) != 0) { set_error("deform_conv2d: channels-last input must be 16-byte aligned"); return VB200_EINVAL; }
  if (!hints.packed_weight) {
    pack_weights3_kernel<<<sm_count() * 4, 256, 0, st>>>((const float*)weight, wpacked, p.c_out, p.c_in, KK, T3_BN);
    rc = check_launch("pack_weights3_kernel");
    if (rc) return rc;
  }
  dim3 grid((unsigned)(p.batch * ceil_div(HWo, TC_BM)), (unsigned)(p.c_out / T3_BN));
  const size_t smem = tc3_smem_bytes(T3_BN, KK);
  VB200_CUDA_TRY(ensure_dyn_smem<deform_conv2d_tc3_kernel<T3_BN>>(smem));
  deform_conv2d_tc3_kernel<T3_BN><<<grid, WG_THREADS, smem, st>>>(nhwc, wpacked, (const float*)offset, (const float*)mask,
                                                                  (const float*)bias, (float*)out, p);
  rc = check_launch("deform_conv2d_tc3_kernel");
  return rc ? rc : 1;
}

size_t deform_conv2d_tc_workspace(int dtype, const DcnParams& p) {
  if (tc3_eligible(dtype, p))
    return align256((size_t)p.batch * p.in_h * p.in_w * p.c_in * 4) + align256((size_t)p.c_out * p.c_in * p.kh * p.kw * 6);
  if (!tc_eligible(dtype, p)) return 0;
  const size_t nhwc = align256((size_t)p.batch * p.in_h * p.in_w * p.c_in * 2);
  const size_t w = align256((size_t)p.c_out * p.c_in * p.kh * p.kw * 2);
  return nhwc + w;
}

int deform_conv2d_tc_try(const void* input, const void* weight, const void* offset, const void* mask, const void* bias,
                         void* out, int dtype, const DcnParams& p, void* workspace, size_t workspace_bytes, cudaStream_t st,
                         const DcnHints& hints) {
  if (tc3_eligible(dtype, p)) return launch_tc3(input, weight, offset, mask, bias, out, p, workspace, workspace_bytes, st, hints);
  if (!tc_eligible(dtype, p)) return 0;
  if (dtype == VB200_BF16)
    return launch_tc<__nv_bfloat16>(input, weight, offset, mask, bias, out, p, workspace, workspace_bytes, st, hints);
  return launch_tc<__half>(input, weight, offset, mask, bias, out, p, workspace, workspace_bytes, st, hints);
}

// Packed-weight image for the tensor-core path of this shape (0: the shape does not take that path).
size_t deform_conv2d_tc_packed_bytes(int dtype, const DcnParams& p) {
  if (tc3_eligible(dtype, p)) return align256((size_t)p.c_out * p.c_in * p.kh * p.kw * 6);
  if (tc_eligible(dtype, p)) return align256((size_t)p.c_out * p.c_in * p.kh * p.kw * 2);
  return 0;
}
int deform_conv2d_tc_pack(const void* weight, void* packed, int dtype, const DcnParams& p, cudaStream_t st) {
  if (tc3_eligible(dtype, p)) {
    pack_weights3_kernel<<<sm_count() * 4, 256, 0, st>>>((const float*)weight, (__nv_bfloat16*)packed, p.c_out, p.c_in, p.kh * p.kw, T3_BN);
    return check_launch("pack_weights3_kernel");
  }
  if (dtype == VB200_BF16) return pack_tc_weights<__nv_bfloat16>(weight, (__nv_bfloat16*)packed, p, st);
  return pack_tc_weights<__half>(weight, (__half*)packed, p, st);
}

}  // namespace vb200
