// Shared helpers for the sm_90a kernels behind include/dpvo_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <algorithm>
#include <cstdlib>

#include "../../include/dpvo_b200.h"

namespace dpvo {

// ---- error plumbing -------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;

inline int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return DPVO_OK;
  set_error("%s: %s", what, cudaGetErrorString(e));
  return DPVO_ERR_CUDA;
}

// Call after every kernel launch: counts the launch and surfaces launch-configuration errors.
#define DPVO_LAUNCH_CHECK(name)                                           \
  do {                                                                    \
    ::dpvo::g_launches.fetch_add(1, std::memory_order_relaxed);           \
    cudaError_t _e = cudaPeekAtLastError();                               \
    if (_e != cudaSuccess) {                                              \
      cudaGetLastError();                                                 \
      return ::dpvo::check_cuda(_e, name);                                \
    }                                                                     \
  } while (0)

#define DPVO_REQUIRE(cond, ...)                                           \
  do {                                                                    \
    if (!(cond)) {                                                        \
      ::dpvo::set_error(__VA_ARGS__);                                     \
      return DPVO_ERR_INVALID;                                            \
    }                                                                     \
  } while (0)

inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 132;
  }
  return n;
}

inline size_t dtype_size(int dtype) {
  switch (dtype) {
    case DPVO_F16: case DPVO_BF16: return 2;
    case DPVO_F32: return 4;
    case DPVO_F64: return 8;
  }
  return 0;
}

// ---- scalar conversion ------------------------------------------------------------------
template <typename T> struct acc_of { using type = float; };
template <> struct acc_of<double> { using type = double; };

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f32<double>(double v) { return (float)v; }

template <typename A, typename T> __device__ __forceinline__ A to_acc(T v) { return (A)to_f32<T>(v); }
template <> __device__ __forceinline__ double to_acc<double, double>(double v) { return v; }

template <typename T, typename A> __device__ __forceinline__ T from_acc(A v);
template <> __device__ __forceinline__ float from_acc<float, float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_acc<__half, float>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_acc<__nv_bfloat16, float>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ double from_acc<double, double>(double v) { return v; }
template <> __device__ __forceinline__ double from_acc<double, float>(float v) { return (double)v; }
template <> __device__ __forceinline__ float from_acc<float, double>(double v) { return (float)v; }

// floor of a coordinate as an int that is safe for address arithmetic: non-finite or huge
// coordinates map far outside any image, so every tap is out of bounds (== 0), which is what
// static_cast<int>(floor(x)) gives in the reference for such values in practice.
__device__ __forceinline__ int safe_floor_int(float v) {
  if (!(fabsf(v) < 1.0e8f)) return -(1 << 28);
  return (int)floorf(v);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int warp_min_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int warp_max_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace dpvo
