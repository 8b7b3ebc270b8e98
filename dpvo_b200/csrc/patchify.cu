// altcorr.patchify: (2R+2)^2 x C window gather around integer-floored coordinates and its
// transpose.  Replaces dpvo/altcorr/correlation_kernel.cu:16-80, 288-333.
//
// Forward writes every output element (zeros outside the map), so no separate memset pass is
// needed (the reference allocates with torch::zeros and then overwrites the in-bounds part).
// Thread mapping: one thread per output element with the window column fastest, so the
// [B,M,C,D,D] store is fully coalesced and an NCHW read touches D contiguous elements.
#include "common.cuh"

namespace dpvo {

template <typename T>
__global__ void patchify_fwd_kernel(const T* __restrict__ net, int64_t sb, int64_t sc, int64_t sy, int64_t sx,
                                    const float* __restrict__ coords, T* __restrict__ patches,
                                    int M, int C, int H, int W, int R, int64_t total) {
  const int D = 2 * R + 2;
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < total; n += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = n;
    const int jj = (int)(r % D); r /= D;
    const int ii = (int)(r % D); r /= D;
    const int c = (int)(r % C); r /= C;
    const int m = (int)(r % M); r /= M;
    const int b = (int)r;
    const float x = coords[((int64_t)b * M + m) * 2 + 0];
    const float y = coords[((int64_t)b * M + m) * 2 + 1];
    const int i = safe_floor_int(y) + (ii - R);
    const int j = safe_floor_int(x) + (jj - R);
    T v = from_acc<T, typename acc_of<T>::type>(0);
    if (i >= 0 && i < H && j >= 0 && j < W) v = net[b * sb + c * sc + (int64_t)i * sy + (int64_t)j * sx];
    patches[n] = v;
  }
}

template <typename T> __device__ __forceinline__ void atomic_add_t(T* p, T v) { atomicAdd(p, v); }

template <typename T>
__global__ void patchify_bwd_kernel(const T* __restrict__ grad, const float* __restrict__ coords,
                                    T* __restrict__ net_grad, int M, int C, int H, int W, int R, int64_t total) {
  const int D = 2 * R + 2;
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < total; n += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = n;
    const int jj = (int)(r % D); r /= D;
    const int ii = (int)(r % D); r /= D;
    const int c = (int)(r % C); r /= C;
    const int m = (int)(r % M); r /= M;
    const int b = (int)r;
    const float x = coords[((int64_t)b * M + m) * 2 + 0];
    const float y = coords[((int64_t)b * M + m) * 2 + 1];
    const int i = safe_floor_int(y) + (ii - R);
    const int j = safe_floor_int(x) + (jj - R);
    if (i >= 0 && i < H && j >= 0 && j < W)
      atomic_add_t(&net_grad[(((int64_t)b * C + c) * H + i) * W + j], grad[n]);
  }
}

template <typename T>
static int patchify_fwd_launch(const void* net, const int64_t* s, const float* coords, void* patches,
                               int B, int M, int C, int H, int W, int R, cudaStream_t st) {
  const int D = 2 * R + 2;
  const int64_t total = (int64_t)B * M * C * D * D;
  if (total == 0) return DPVO_OK;
  const int threads = 256;
  const int64_t blocks = std::min<int64_t>((total + threads - 1) / threads, (int64_t)sm_count() * 16);
  return launch("patchify_fwd_kernel", patchify_fwd_kernel<T>, (unsigned)blocks, threads, 0, st,
                reinterpret_cast<const T*>(net), s[0], s[1], s[2], s[3], coords, reinterpret_cast<T*>(patches), M, C, H, W, R, total);
}

template <typename T>
static int patchify_bwd_launch(const void* grad, const float* coords, void* net_grad,
                               int B, int M, int C, int H, int W, int R, cudaStream_t st) {
  const int D = 2 * R + 2;
  const int64_t total = (int64_t)B * M * C * D * D;
  if (total == 0) return DPVO_OK;
  const int threads = 256;
  const int64_t blocks = std::min<int64_t>((total + threads - 1) / threads, (int64_t)sm_count() * 16);
  return launch("patchify_bwd_kernel", patchify_bwd_kernel<T>, (unsigned)blocks, threads, 0, st,
                reinterpret_cast<const T*>(grad), coords, reinterpret_cast<T*>(net_grad), M, C, H, W, R, total);
}

}  // namespace dpvo

using namespace dpvo;

extern "C" int dpvo_patchify_forward(const void* net, const int64_t* net_strides, const float* coords,
                                     void* patches, int dtype, int B, int M, int C, int H, int W,
                                     int radius, void* stream) {
  DPVO_REQUIRE(B >= 0 && M >= 0 && C >= 0 && H > 0 && W > 0 && radius >= 0, "patchify_forward: bad sizes");
  if ((int64_t)B * M * C == 0) return DPVO_OK;
  DPVO_REQUIRE(net && net_strides && coords && patches, "patchify_forward: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case DPVO_F16: return patchify_fwd_launch<__half>(net, net_strides, coords, patches, B, M, C, H, W, radius, st);
    case DPVO_BF16: return patchify_fwd_launch<__nv_bfloat16>(net, net_strides, coords, patches, B, M, C, H, W, radius, st);
    case DPVO_F32: return patchify_fwd_launch<float>(net, net_strides, coords, patches, B, M, C, H, W, radius, st);
    case DPVO_F64: return patchify_fwd_launch<double>(net, net_strides, coords, patches, B, M, C, H, W, radius, st);
  }
  set_error("patchify_forward: unknown dtype %d", dtype);
  return DPVO_ERR_INVALID;
}

extern "C" int dpvo_patchify_backward(const void* gradient, const float* coords, void* net_grad,
                                      int dtype, int B, int M, int C, int H, int W, int radius,
                                      void* stream) {
  DPVO_REQUIRE(B >= 0 && M >= 0 && C >= 0 && H > 0 && W > 0 && radius >= 0, "patchify_backward: bad sizes");
  if ((int64_t)B * M * C == 0) return DPVO_OK;
  DPVO_REQUIRE(gradient && coords && net_grad, "patchify_backward: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case DPVO_F16: return patchify_bwd_launch<__half>(gradient, coords, net_grad, B, M, C, H, W, radius, st);
    case DPVO_BF16: return patchify_bwd_launch<__nv_bfloat16>(gradient, coords, net_grad, B, M, C, H, W, radius, st);
    case DPVO_F32: return patchify_bwd_launch<float>(gradient, coords, net_grad, B, M, C, H, W, radius, st);
    case DPVO_F64: return patchify_bwd_launch<double>(gradient, coords, net_grad, B, M, C, H, W, radius, st);
  }
  set_error("patchify_backward: unknown dtype %d", dtype);
  return DPVO_ERR_INVALID;
}
