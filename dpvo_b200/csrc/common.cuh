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
#include <utility>

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

#define DPVO_REQUIRE(cond, ...)                                           \
  do {                                                                    \
    if (!(cond)) {                                                        \
      ::dpvo::set_error(__VA_ARGS__);                                     \
      return DPVO_ERR_INVALID;                                            \
    }                                                                     \
  } while (0)

// SM count of the current device, asked once per device (132 when it cannot be asked)
inline int sm_count() {
  constexpr int kDevices = 64;
  static std::atomic<int> cached[kDevices];                          // 0 = not asked yet
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev < kDevices && (n = cached[dev].load(std::memory_order_relaxed)) > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 132;
  if (dev < kDevices) cached[dev].store(n, std::memory_order_relaxed);
  return n;
}

// Lets `kernel` take `smem` bytes of dynamic shared memory on the current device.  Above the 48 KiB default this is needed
// before a launch, and before an occupancy query that is to count such CTAs.  The limit is a per-device attribute, so it
// is set on every call.
template <typename K> int allow_smem(const char* name, K* kernel, size_t smem) {
  if (smem <= 48 * 1024) return DPVO_OK;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) return DPVO_OK;
  cudaGetLastError();
  set_error("%s: cudaFuncSetAttribute: %s", name, cudaGetErrorString(e));
  return DPVO_ERR_CUDA;
}

// Launches `kernel` on stream `st` and counts it in dpvo_launch_count().  ATTR, when given, is a launch attribute switched
// on for this launch (cudaLaunchAttributeCooperative: a grid whose CTAs synchronise).  A failed launch returns its own
// error as "<name>: <error>" and leaves no pending error behind.
template <cudaLaunchAttributeID ATTR = cudaLaunchAttributeIgnore, typename... P, typename... A>
int launch(const char* name, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  if (int rc = allow_smem(name, kernel, smem)) return rc;
  cudaLaunchAttribute attr;
  attr.id = ATTR;
  attr.val.cooperative = 1;
  cudaLaunchConfig_t cfg;
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cfg.attrs = &attr; cfg.numAttrs = ATTR == cudaLaunchAttributeIgnore ? 0 : 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return check_cuda(e, name);
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return DPVO_OK;
}

inline size_t dtype_size(int dtype) {
  switch (dtype) {
    case DPVO_F16: case DPVO_BF16: return 2;
    case DPVO_F32: return 4;
    case DPVO_F64: return 8;
  }
  return 0;
}

// every array of a workspace starts on a 256-byte boundary: round-up of sizes and of the workspace pointer
inline int64_t align256(int64_t v) { return (v + 255) & ~(int64_t)255; }
inline char* align256(void* p) { return (char*)(((uintptr_t)p + 255) & ~(uintptr_t)255); }

// Carves a workspace into consecutive arrays, each rounded up to `align` bytes.  On a null base it only measures, so
// one layout function gives both a workspace's size (bytes()) and, on the real base, its arrays: the two cannot differ.
struct WsLayout {
  char* base; int64_t align, used = 0;
  explicit WsLayout(void* b = nullptr, int64_t a = 256) : base((char*)b), align(a) {}
  template <typename T> T* take(int64_t count) {
    T* p = base ? reinterpret_cast<T*>(base + used) : nullptr;
    used += (count * (int64_t)sizeof(T) + align - 1) / align * align;
    return p;
  }
  int64_t bytes() const { return used; }
};

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
