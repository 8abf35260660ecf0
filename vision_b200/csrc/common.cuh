// common.cuh — shared helpers for the sm_90a kernels behind include/vision_b200.h.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/vision_b200.h"

namespace vb200 {

// ---- error plumbing -------------------------------------------------------
char* last_error_buf();
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launch_count;

inline int check_launch(const char* what) {
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

#define VB200_CUDA_TRY(...)                                                         \
  do {                                                                              \
    cudaError_t _e = (__VA_ARGS__);                                                 \
    if (_e != cudaSuccess) {                                                        \
      vb200::set_error("%s failed: %s", #__VA_ARGS__, cudaGetErrorString(_e));      \
      return (int)_e;                                                               \
    }                                                                               \
  } while (0)

#define VB200_REQUIRE(cond, ...)                                                    \
  do {                                                                              \
    if (!(cond)) {                                                                  \
      vb200::set_error(__VA_ARGS__);                                                \
      return VB200_EINVAL;                                                          \
    }                                                                               \
  } while (0)

// device attribute cache (per current device)
int sm_count();
int max_smem_optin();

// VB200_* path overrides (testing / profiling): read from the environment ONCE when the library first needs them
// (no getenv on the per-call path); vb200_reload_env() re-reads them.  nullptr when unset.
enum EnvKey { ENV_ROI_ALIGN_PATH, ENV_NMS_PATH, ENV_BNMS_PATH, ENV_RESIZE_PATH, ENV_DCN_PATH, ENV_ROI_BWD_PATH, ENV_BNMS_GRAPH,
              ENV_COUNT };
const char* env_override(EnvKey k);
int env_generation();     // bumped by every (re)load of the overrides: caches keyed on it forget their entries

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device) instead of on every launch: remembers the
// largest size already granted.
template <auto kernel>
inline cudaError_t ensure_dyn_smem(size_t bytes) {
  static size_t granted[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (bytes <= granted[dev]) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) granted[dev] = bytes;
  return e;
}

// ---- dtype traits -----------------------------------------------------------
template <typename T> struct Acc { using type = float; };
template <> struct Acc<double> { using type = double; };

template <typename T> __device__ __forceinline__ typename Acc<T>::type to_acc(T v) { return (typename Acc<T>::type)v; }
template <> __device__ __forceinline__ float to_acc<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_acc<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_acc<uint8_t>(uint8_t v) { return (float)v; }

template <typename T, typename A> __device__ __forceinline__ T from_acc(A v) { return (T)v; }
template <> __device__ __forceinline__ __half from_acc<__half, float>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_acc<__nv_bfloat16, float>(float v) { return __float2bfloat16_rn(v); }

// Round-to-nearest single ops that the compiler may not contract into FMAs:
// used wherever the reference's x86 CPU arithmetic (no contraction) must be
// reproduced bit-for-bit (sample coordinates, NMS IoU).
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

// fp32 pairs carried in one 64-bit value; fma2 is two round-to-nearest FMAs, one per element
__device__ __forceinline__ unsigned long long pack2(float x, float y) {
  return (unsigned long long)__float_as_uint(x) | ((unsigned long long)__float_as_uint(y) << 32);
}
__device__ __forceinline__ float lo32(unsigned long long v) { return __uint_as_float((uint32_t)v); }
__device__ __forceinline__ float hi32(unsigned long long v) { return __uint_as_float((uint32_t)(v >> 32)); }
__device__ __forceinline__ unsigned long long fma2(unsigned long long a, unsigned long long b, unsigned long long c) {
  return pack2(__fmaf_rn(lo32(a), lo32(b), lo32(c)), __fmaf_rn(hi32(a), hi32(b), hi32(c)));
}

// torch.maximum / torch.minimum: a NaN in either operand is the result
template <typename A> __device__ __forceinline__ A nan_max(A a, A b) { return a != a ? a : b != b ? b : (a > b ? a : b); }
template <typename A> __device__ __forceinline__ A nan_min(A a, A b) { return a != a ? a : b != b ? b : (a < b ? a : b); }

__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// atomicAdd of an accumulator-type value into a T element, rounded to T first.
template <typename T> __device__ __forceinline__ void atomic_add(T* p, typename Acc<T>::type v) { atomicAdd(p, (T)v); }
template <> __device__ __forceinline__ void atomic_add<__half>(__half* p, float v) { atomicAdd(p, __float2half_rn(v)); }
template <> __device__ __forceinline__ void atomic_add<__nv_bfloat16>(__nv_bfloat16* p, float v) {
  atomicAdd(p, __float2bfloat16_rn(v));
}

// ---- workspaces ---------------------------------------------------------------
inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// Carves a workspace into 256-byte aligned arrays; with base == nullptr only sizes are accumulated.
struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* b) : base((char*)b) {}
  template <typename T> T* take(size_t count) {
    T* p = base ? (T*)(base + off) : nullptr;
    off += align256(count * sizeof(T));
    return p;
  }
};

}  // namespace vb200
