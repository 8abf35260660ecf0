// deform_conv2d.cu — deformable convolution forward (DCNv1/v2), sm_90a.
//
// Reference: csrc/ops/cuda/deform_conv2d_kernel.cu:97-209 (bilinear + deformable_im2col),
// :1035-1255 (host: materialised `columns` buffer + per-group cuBLAS addmm + transpose/copy/bias);
// CPU twin csrc/ops/cpu/deform_conv2d_kernel.cpp:95-209,921-1151.
//
// Design (not a port): the im2col matrix is never written to HBM.  The op is an
// implicit GEMM  out[oc, pix] = sum_k W[oc, k] * col[k, pix],  k = (ci, tap):
//   * SIMT kernel (this file; fp32 / fp16 / bf16 storage, fp32 accumulate): a CTA owns
//     a 128(oc) x 64(pix) output tile of one image.  Per offset group it builds a
//     sampling table in shared memory ONCE (per chunk of taps for kernels whose table
//     exceeds shared memory, KK > 106) — for each (tap, pixel): 4 clamped corner
//     offsets + 4 bilinear weights (zeroed out of bounds, pre-multiplied by the
//     modulation mask) — and reuses it for every input channel of that group, so a
//     col element costs 4 loads + 4 FMAs.  K is walked in slabs of 16; A (weights) and
//     B (sampled columns) slabs live in shared memory, each thread accumulates an 8x4
//     register tile.  Bias is fused into the epilogue; output is written once, NCHW.
//   * wgmma kernel (deform_conv2d_tc.cu): same decomposition with the B slab written
//     as a swizzled bf16 K-major tile and the contraction on the Hopper tensor cores.
#include <type_traits>

#include "common.cuh"
#include "dcn_geometry.cuh"

namespace vb200 {


namespace {

constexpr int BM = 128, BN = 64, BK = 16, DCN_THREADS = 256;
constexpr int BMP = BM + 4;   // padded A-slab row (bank spread for the transposing store)

template <typename T>
__global__ void __launch_bounds__(DCN_THREADS)
deform_conv2d_simt_kernel(const T* __restrict__ input, const T* __restrict__ weight, const T* __restrict__ offset,
                          const T* __restrict__ mask, const T* __restrict__ bias, T* __restrict__ out, DcnParams p, int tab_taps) {
  extern __shared__ __align__(16) unsigned char dsm[];
  const int KK = p.kh * p.kw;
  DcnTabEnt* tab = reinterpret_cast<DcnTabEnt*>(dsm);                 // [tab_taps][BN]
  float* As = reinterpret_cast<float*>(tab + (size_t)tab_taps * BN);  // [BK][BM]
  float* Bs = As + BK * BMP;                                          // [BK][BN]

  const int tid = threadIdx.x;
  const int HWo = p.out_h * p.out_w;
  const int pix0 = blockIdx.x * BN;
  const int cout_g = p.c_out / p.groups, cin_g = p.c_in / p.groups;
  const int m_tiles = ceil_div(cout_g, BM);
  const int g = blockIdx.y / m_tiles;
  const int oc0 = (blockIdx.y % m_tiles) * BM;          // within group
  const int b = blockIdx.z;
  const int c_per_off = p.c_in / p.offset_groups;
  const int Kg = cin_g * KK;                            // weight row length for this group

  const int tm = tid / 16, tn = tid % 16;               // 16 x 16 threads; micro-tile 8 (m) x 4 (n)
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const T* __restrict__ in_b = input + (int64_t)b * p.c_in * p.in_h * p.in_w;
  const int ci_lo = g * cin_g, ci_hi = ci_lo + cin_g;   // channels of this weight group
  const int og_lo = ci_lo / c_per_off, og_hi = (ci_hi - 1) / c_per_off;

  for (int og = og_lo; og <= og_hi; ++og) {
    const T* __restrict__ off_b = offset + ((int64_t)b * p.offset_groups + og) * 2 * KK * HWo;
    const T* __restrict__ msk_b = p.use_mask ? mask + ((int64_t)b * p.offset_groups + og) * KK * HWo : nullptr;
    const int c_start = max(ci_lo, og * c_per_off), c_end = min(ci_hi, (og + 1) * c_per_off);
    // taps [t0, t0 + nt) per table; one chunk (t0 = 0, nt = KK) unless the whole table exceeds shared memory.  Within a chunk
    // the contraction index kl = (channel - c_start) * nt + (tap - t0), so with one chunk k = k_start + kl, the weight row order.
    for (int t0 = 0; t0 < KK; t0 += tab_taps) {
      const int nt = min(tab_taps, KK - t0);
      // ---- sampling table for (offset group og, taps [t0, t0 + nt), this pixel tile) ----
      __syncthreads();
      fill_sample_table<BN>(tab, off_b, msk_b, p, t0, nt, pix0, 1, tid, DCN_THREADS);
      __syncthreads();

      const int cil0 = c_start - ci_lo, nk = (c_end - c_start) * nt;
      for (int k0 = 0; k0 < nk; k0 += BK) {
        // A slab: As[kk][m] = W[g*cout_g + oc0 + m][cil * KK + tap]
        for (int e = tid; e < BK * BM; e += DCN_THREADS) {
          const int m = e / BK, kk = e - m * BK;
          const int kl = k0 + kk, oc = oc0 + m;
          float v = 0.f;
          if (kl < nk && oc < cout_g) {
            const int cl = kl / nt, tap = t0 + (kl - cl * nt);
            v = to_acc(weight[((int64_t)(g * cout_g + oc)) * Kg + (cil0 + cl) * KK + tap]);
          }
          As[kk * BMP + m] = v;
        }
        // B slab: Bs[kk][px] = sum_q w_q * in[ci][o_q]
        for (int e = tid; e < BK * BN; e += DCN_THREADS) {
          const int kk = e / BN, px = e - kk * BN;
          const int kl = k0 + kk;
          float v = 0.f;
          if (kl < nk) {
            const int cl = kl / nt, tl = kl - cl * nt;
            const T* __restrict__ pl = in_b + (int64_t)(c_start + cl) * p.in_h * p.in_w;
            const DcnTabEnt se = tab[tl * BN + px];
            v = se.w[0] * to_acc(pl[se.o[0]]);
            v = fmaf(se.w[1], to_acc(pl[se.o[1]]), v);
            v = fmaf(se.w[2], to_acc(pl[se.o[2]]), v);
            v = fmaf(se.w[3], to_acc(pl[se.o[3]]), v);
          }
          Bs[kk * BN + px] = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
          float a[8], bb[4];
          const float4 a0 = *reinterpret_cast<const float4*>(As + kk * BMP + tm * 8);
          const float4 a1 = *reinterpret_cast<const float4*>(As + kk * BMP + tm * 8 + 4);
          const float4 b0 = *reinterpret_cast<const float4*>(Bs + kk * BN + tn * 4);
          a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
          bb[0] = b0.x; bb[1] = b0.y; bb[2] = b0.z; bb[3] = b0.w;
#pragma unroll
          for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        __syncthreads();
      }
    }
  }
  // ---- epilogue: + bias, NCHW store ----
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int oc = oc0 + tm * 8 + i;
    if (oc >= cout_g) continue;
    const int ocg = g * cout_g + oc;
    const float bv = bias ? to_acc(bias[ocg]) : 0.f;
    T* __restrict__ o = out + ((int64_t)b * p.c_out + ocg) * HWo;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int pix = pix0 + tn * 4 + j;
      if (pix < HWo) o[pix] = from_acc<T, float>(acc[i][j] + bv);
    }
  }
}

template <typename T>
int launch_simt(const void* input, const void* weight, const void* offset, const void* mask, const void* bias, void* out,
                const DcnParams& p, cudaStream_t st) {
  const int KK = p.kh * p.kw;
  // the sampling table holds every tap when it fits (up to 106 taps with H100's 227 KB opt-in), else as many taps as fit
  const size_t slabs = (size_t)(BK * BMP + BK * BN) * 4;
  const size_t optin = (size_t)max_smem_optin();
  const size_t fit = optin > 1024 + slabs ? (optin - 1024 - slabs) / (BN * sizeof(DcnTabEnt)) : 0;
  if (fit == 0) {       // not even one tap of the table fits (the chunk loop would not advance)
    set_error("deform_conv2d: %zu bytes of opt-in shared memory hold no tap of the sampling table", optin);
    return VB200_EUNSUPPORTED;
  }
  const int tab_taps = (size_t)KK < fit ? KK : (int)fit;
  const size_t smem = (size_t)tab_taps * BN * sizeof(DcnTabEnt) + slabs;
  if (smem > 48 * 1024)
    VB200_CUDA_TRY(ensure_dyn_smem<deform_conv2d_simt_kernel<T>>(smem));
  const int cout_g = p.c_out / p.groups;
  dim3 grid((unsigned)ceil_div(p.out_h * p.out_w, BN), (unsigned)(p.groups * ceil_div(cout_g, BM)), (unsigned)p.batch);
  deform_conv2d_simt_kernel<T><<<grid, DCN_THREADS, smem, st>>>((const T*)input, (const T*)weight, (const T*)offset,
                                                               (const T*)mask, (const T*)bias, (T*)out, p, tab_taps);
  return check_launch("deform_conv2d_simt_kernel");
}

// ---- float64 (the reference dispatches FLOATING_TYPES_AND_HALF; its gradcheck tests run in double) --------------------
// One thread per output element, double accumulation, bilinear_interpolate exactly as deform_conv2d_kernel.cu:97-134.
// A correctness path for tests, not a performance path.
__global__ void __launch_bounds__(256)
deform_conv2d_f64_kernel(const double* __restrict__ in, const double* __restrict__ w, const double* __restrict__ off,
                         const double* __restrict__ mask, const double* __restrict__ bias, double* __restrict__ out, DcnParams p) {
  const int HWo = p.out_h * p.out_w, HWi = p.in_h * p.in_w, KK = p.kh * p.kw;
  const int64_t total = (int64_t)p.batch * p.c_out * HWo;
  const int cin_g = p.c_in / p.groups, cout_g = p.c_out / p.groups, c_per_off = p.c_in / p.offset_groups;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int pix = (int)(idx % HWo);
    const int co = (int)((idx / HWo) % p.c_out);
    const int b = (int)(idx / HWo / p.c_out);
    const int g = co / cout_g;
    double sum = 0;
    for (int ci = 0; ci < cin_g; ++ci) {
      const int c = g * cin_g + ci, og = c / c_per_off;
      const double* __restrict__ plane = in + ((int64_t)b * p.c_in + c) * HWi;
      const int64_t ob = ((int64_t)b * p.offset_groups + og) * 2 * KK;
      for (int tap = 0; tap < KK; ++tap) {
        double y, x, m;
        sample_position<double>(off + ob * HWo, mask + ob / 2 * HWo, p, tap, pix, y, x, m);
        const Sample<double> s = make_sample<double, true>(y, x, p.in_h, p.in_w);
        double val = 0;
        if (s.inside) {
          double wt[4], v[4];
          corner_weights(s, wt);
          corner_values(plane, s, v);
          val = blend(wt, v);
        }
        sum += w[((int64_t)co * cin_g + ci) * KK + tap] * (m * val);
      }
    }
    out[idx] = sum + (bias ? bias[co] : 0.0);
  }
}

}  // namespace

// deform_conv2d_tc.cu: returns 1 if handled, 0 if not applicable, other = error
int deform_conv2d_tc_try(const void* input, const void* weight, const void* offset, const void* mask, const void* bias,
                         void* out, int dtype, const DcnParams& p, void* workspace, size_t workspace_bytes, cudaStream_t st,
                         const DcnHints& hints);
size_t deform_conv2d_tc_workspace(int dtype, const DcnParams& p);
size_t deform_conv2d_tc_packed_bytes(int dtype, const DcnParams& p);
int deform_conv2d_tc_pack(const void* weight, void* packed, int dtype, const DcnParams& p, cudaStream_t st);

}  // namespace vb200

using namespace vb200;

// The workspace and packed-weight queries take no stride, padding or dilation: what they size depends on the channel and kernel
// sizes alone, so they fill only those and check nothing.
extern "C" size_t vb200_deform_conv2d_workspace_bytes(int dtype, int batch, int c_in, int in_h, int in_w, int c_out,
                                                      int kh, int kw, int out_h, int out_w, int groups,
                                                      int offset_groups) {
  return deform_conv2d_tc_workspace(dtype, DcnParams{batch, c_in, in_h, in_w, c_out, kh, kw, 0, 0, 0, 0, 0, 0, groups, offset_groups,
                                                     0, out_h, out_w});
}

extern "C" size_t vb200_deform_conv2d_packed_weight_bytes(int dtype, int c_in, int c_out, int kh, int kw, int groups, int offset_groups) {
  return deform_conv2d_tc_packed_bytes(dtype, DcnParams{1, c_in, 8, 8, c_out, kh, kw, 0, 0, 0, 0, 0, 0, groups, offset_groups});
}

extern "C" int vb200_deform_conv2d_pack_weight(const void* weight, void* packed, int dtype, int c_in, int c_out, int kh, int kw, int groups,
                                               int offset_groups, vb200_stream stream) {
  const DcnParams p{1, c_in, 8, 8, c_out, kh, kw, 0, 0, 0, 0, 0, 0, groups, offset_groups};
  VB200_REQUIRE(weight && packed, "deform_conv2d_pack_weight: null pointer");
  VB200_REQUIRE(deform_conv2d_tc_packed_bytes(dtype, p) > 0, "deform_conv2d_pack_weight: this shape does not take the tensor-core path");
  return deform_conv2d_tc_pack(weight, packed, dtype, p, (cudaStream_t)stream);
}

static int dcn_forward_impl(const void* input, const void* weight, const void* offset, const void* mask, const void* bias, void* out,
                            int dtype, const DcnParams& p, void* workspace, size_t workspace_bytes, vb200_stream stream,
                            const DcnHints& hints) {
  if (p.batch == 0 || p.c_out == 0) return 0;
  VB200_REQUIRE(input && weight && offset && out && (!p.use_mask || mask), "deform_conv2d: null pointer");
  VB200_REQUIRE((int64_t)p.c_in * p.in_h * p.in_w < (1ll << 31) && p.batch <= 65535, "deform_conv2d: tensor too large");
  cudaStream_t st = (cudaStream_t)stream;
  const char* force = env_override(ENV_DCN_PATH);   // "simt" forces the SIMT kernel
  if (!(force && force[0] == 's')) {
    const int rc = deform_conv2d_tc_try(input, weight, offset, mask, bias, out, dtype, p, workspace, workspace_bytes, st, hints);
    if (rc != 0) return rc == 1 ? 0 : rc;
  }
  VB200_REQUIRE(!hints.input_is_nhwc, "deform_conv2d: a channels-last input is only accepted by the tensor-core path (this shape / dtype takes the SIMT kernel)");
  return dispatch_dcn_dtype(dtype, "deform_conv2d: unsupported dtype %d", [&](auto t) {
    using T = decltype(t);
    if constexpr (std::is_same<T, double>::value) {
      const int64_t total = (int64_t)p.batch * p.c_out * p.out_h * p.out_w;
      const int grid = (int)(ceil_div64(total, 256) < (int64_t)sm_count() * 16 ? ceil_div64(total, 256) : (int64_t)sm_count() * 16);
      deform_conv2d_f64_kernel<<<grid, 256, 0, st>>>((const double*)input, (const double*)weight, (const double*)offset,
                                                    (const double*)mask, (const double*)bias, (double*)out, p);
      return check_launch("deform_conv2d_f64_kernel");
    } else {
      return launch_simt<T>(input, weight, offset, mask, bias, out, p, st);
    }
  });
}

// outs[0] is the output (the caller's slot of its own gathered buffer when fused with an all-gather), outs[1..n) the same slot
// of the peers' buffers (peer-mapped).  The wgmma kernel's epilogue stores each element to all of them; shapes that take another
// kernel are computed into outs[0] and copied to the peers on the same stream.
extern "C" int vb200_deform_conv2d_forward(const void* input, const void* weight, const void* packed_weight, int input_is_nhwc,
                                           const void* offset, const void* mask, const void* bias, void* const* outs, int n_outs,
                                           int dtype, int batch, int c_in, int in_h, int in_w, int c_out, int kh, int kw, int stride_h,
                                           int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int groups, int offset_groups,
                                           int use_mask, void* workspace, size_t workspace_bytes, vb200_stream stream) {
  VB200_REQUIRE(outs && n_outs >= 1 && n_outs <= 8, "deform_conv2d_forward: 1..8 destinations");
  for (int d = 0; d < n_outs; ++d) VB200_REQUIRE(outs[d] != nullptr, "deform_conv2d_forward: null destination");
  DcnParams p;
  int rc = dcn_params(p, batch, c_in, in_h, in_w, c_out, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, groups, offset_groups,
                      use_mask);
  if (rc) return rc;
  bool done = false;
  rc = dcn_forward_impl(input, weight, offset, mask, bias, outs[0], dtype, p, workspace, workspace_bytes, stream,
                        DcnHints{packed_weight, input_is_nhwc, outs + 1, n_outs - 1, &done});
  if (rc || done || n_outs == 1 || batch == 0 || c_out == 0) return rc;
  const size_t esize = dtype == VB200_F64 ? 8 : dtype == VB200_F32 ? 4 : 2;
  const size_t bytes = (size_t)batch * c_out * p.out_h * p.out_w * esize;
  for (int d = 1; d < n_outs; ++d) VB200_CUDA_TRY(cudaMemcpyAsync(outs[d], outs[0], bytes, cudaMemcpyDefault, (cudaStream_t)stream));
  return 0;
}
