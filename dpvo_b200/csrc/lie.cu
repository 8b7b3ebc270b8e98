// lietorch_backends for sm_90a: SO3, RxSO3, SE3, Sim3, float and double, forward + backward.
// Replaces dpvo/lietorch/src/lietorch_gpu.cu:20-601 (Eigen template kernels) with register math
// from lie.cuh.  One group element per thread, grid-stride, outputs fully written (the reference
// allocates with torch::zeros and overwrites; the unused last gradient component stays 0).
// SO3 / SE3 (the groups on the DPVO hot path) have hand-specialised operators (lie_ops.cuh); RxSO3 / Sim3 (loop closure
// only, SURVEY 8(f)) run the generic small-matrix operators of lie_scaled.cuh.
#include "common.cuh"
#include "lie_ops.cuh"
#include "lie_scaled.cuh"

namespace dpvo {
using namespace lie;

template <int G> struct GroupDims;
template <> struct GroupDims<DPVO_SO3> { static constexpr int N = 4, K = 3; };
template <> struct GroupDims<DPVO_SE3> { static constexpr int N = 7, K = 6; };

template <int G, typename S, int OP>
__global__ void __launch_bounds__(256) lie_kernel(const LieArgs A) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += (int64_t)gridDim.x * blockDim.x) {
    if constexpr (G == DPVO_SE3) se3_op<S, OP>(A, i);
    else so3_op<S, OP>(A, i);
  }
}

// RxSO3 / Sim3: the generic operators (op codes of lie_scaled.cuh follow the enum of lie_ops.cuh)
template <int G, typename S, int OP>
__global__ void __launch_bounds__(128) lie_scaled_kernel(const LieArgs A) {
  static_assert((int)OP_JINV == (int)SOP_JINV && (int)OP_ACT4_B == (int)SOP_ACT4_B, "operator codes must match");
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += (int64_t)gridDim.x * blockDim.x) {
    if constexpr (G == DPVO_SIM3)
      scaled_group_op<Sim3g<S>, S>(OP, (const S*)A.in0, (const S*)A.in1, (const S*)A.in2, (S*)A.out0, (S*)A.out1, (long long)i);
    else
      scaled_group_op<RxSO3g<S>, S>(OP, (const S*)A.in0, (const S*)A.in1, (const S*)A.in2, (S*)A.out0, (S*)A.out1, (long long)i);
  }
}

template <int OP>
static int lie_launch(int group, int dtype, const LieArgs& A, cudaStream_t st, const char* name) {
  if (A.n < 0) { set_error("%s: negative batch", name); return DPVO_ERR_INVALID; }
  if (A.n == 0) return DPVO_OK;
  if (!A.in0 || !A.out0) { set_error("%s: null pointer", name); return DPVO_ERR_INVALID; }
  if (group != DPVO_SE3 && group != DPVO_SO3 && group != DPVO_RXSO3 && group != DPVO_SIM3) {
    set_error("%s: unknown group id %d (SO3 = 1, RxSO3 = 2, SE3 = 3, Sim3 = 4)", name, group);
    return DPVO_ERR_INVALID;
  }
  if (dtype != DPVO_F32 && dtype != DPVO_F64) {
    set_error("%s: dtype %d not supported (f32/f64)", name, dtype);
    return DPVO_ERR_UNSUPPORTED;
  }
  const bool f32 = dtype == DPVO_F32;
  if (group == DPVO_RXSO3 || group == DPVO_SIM3) {
    const unsigned sb = (unsigned)std::min<int64_t>((A.n + 127) / 128, (int64_t)sm_count() * 8);
    const auto kern = group == DPVO_SIM3 ? (f32 ? lie_scaled_kernel<DPVO_SIM3, float, OP> : lie_scaled_kernel<DPVO_SIM3, double, OP>)
                                         : (f32 ? lie_scaled_kernel<DPVO_RXSO3, float, OP> : lie_scaled_kernel<DPVO_RXSO3, double, OP>);
    return launch(name, kern, sb, 128, 0, st, A);
  }
  const int threads = 256;
  const unsigned blocks = (unsigned)std::min<int64_t>((A.n + threads - 1) / threads, (int64_t)sm_count() * 8);
  const auto kern = group == DPVO_SE3 ? (f32 ? lie_kernel<DPVO_SE3, float, OP> : lie_kernel<DPVO_SE3, double, OP>)
                                      : (f32 ? lie_kernel<DPVO_SO3, float, OP> : lie_kernel<DPVO_SO3, double, OP>);
  return launch(name, kern, blocks, threads, 0, st, A);
}

}  // namespace dpvo

using namespace dpvo;

#define LIE_ARGS(i0, i1, i2, o0, o1, n) LieArgs{(i0), (i1), (i2), (o0), (o1), (n)}

extern "C" {
int dpvo_lie_exp(int g, int dt, const void* a, void* X, int64_t n, void* s) {
  return lie_launch<OP_EXP>(g, dt, LIE_ARGS(a, nullptr, nullptr, X, nullptr, n), (cudaStream_t)s, "lie_exp");
}
int dpvo_lie_exp_backward(int g, int dt, const void* grad, const void* a, void* da, int64_t n, void* s) {
  return lie_launch<OP_EXP_B>(g, dt, LIE_ARGS(grad, a, nullptr, da, nullptr, n), (cudaStream_t)s, "lie_exp_backward");
}
int dpvo_lie_log(int g, int dt, const void* X, void* a, int64_t n, void* s) {
  return lie_launch<OP_LOG>(g, dt, LIE_ARGS(X, nullptr, nullptr, a, nullptr, n), (cudaStream_t)s, "lie_log");
}
int dpvo_lie_log_backward(int g, int dt, const void* grad, const void* X, void* dX, int64_t n, void* s) {
  return lie_launch<OP_LOG_B>(g, dt, LIE_ARGS(grad, X, nullptr, dX, nullptr, n), (cudaStream_t)s, "lie_log_backward");
}
int dpvo_lie_inv(int g, int dt, const void* X, void* Y, int64_t n, void* s) {
  return lie_launch<OP_INV>(g, dt, LIE_ARGS(X, nullptr, nullptr, Y, nullptr, n), (cudaStream_t)s, "lie_inv");
}
int dpvo_lie_inv_backward(int g, int dt, const void* grad, const void* X, void* dX, int64_t n, void* s) {
  return lie_launch<OP_INV_B>(g, dt, LIE_ARGS(grad, X, nullptr, dX, nullptr, n), (cudaStream_t)s, "lie_inv_backward");
}
int dpvo_lie_mul(int g, int dt, const void* X, const void* Y, void* Z, int64_t n, void* s) {
  return lie_launch<OP_MUL>(g, dt, LIE_ARGS(X, Y, nullptr, Z, nullptr, n), (cudaStream_t)s, "lie_mul");
}
int dpvo_lie_mul_backward(int g, int dt, const void* grad, const void* X, const void* Y, void* dX, void* dY, int64_t n, void* s) {
  return lie_launch<OP_MUL_B>(g, dt, LIE_ARGS(grad, X, Y, dX, dY, n), (cudaStream_t)s, "lie_mul_backward");
}
int dpvo_lie_adj(int g, int dt, const void* X, const void* a, void* b, int64_t n, void* s) {
  return lie_launch<OP_ADJ>(g, dt, LIE_ARGS(X, a, nullptr, b, nullptr, n), (cudaStream_t)s, "lie_adj");
}
int dpvo_lie_adj_backward(int g, int dt, const void* grad, const void* X, const void* a, void* dX, void* da, int64_t n, void* s) {
  return lie_launch<OP_ADJ_B>(g, dt, LIE_ARGS(grad, X, a, dX, da, n), (cudaStream_t)s, "lie_adj_backward");
}
int dpvo_lie_adjT(int g, int dt, const void* X, const void* a, void* b, int64_t n, void* s) {
  return lie_launch<OP_ADJT>(g, dt, LIE_ARGS(X, a, nullptr, b, nullptr, n), (cudaStream_t)s, "lie_adjT");
}
int dpvo_lie_adjT_backward(int g, int dt, const void* grad, const void* X, const void* a, void* dX, void* da, int64_t n, void* s) {
  return lie_launch<OP_ADJT_B>(g, dt, LIE_ARGS(grad, X, a, dX, da, n), (cudaStream_t)s, "lie_adjT_backward");
}
int dpvo_lie_act(int g, int dt, const void* X, const void* p, void* q, int64_t n, void* s) {
  return lie_launch<OP_ACT>(g, dt, LIE_ARGS(X, p, nullptr, q, nullptr, n), (cudaStream_t)s, "lie_act");
}
int dpvo_lie_act_backward(int g, int dt, const void* grad, const void* X, const void* p, void* dX, void* dp, int64_t n, void* s) {
  return lie_launch<OP_ACT_B>(g, dt, LIE_ARGS(grad, X, p, dX, dp, n), (cudaStream_t)s, "lie_act_backward");
}
int dpvo_lie_act4(int g, int dt, const void* X, const void* p, void* q, int64_t n, void* s) {
  return lie_launch<OP_ACT4>(g, dt, LIE_ARGS(X, p, nullptr, q, nullptr, n), (cudaStream_t)s, "lie_act4");
}
int dpvo_lie_act4_backward(int g, int dt, const void* grad, const void* X, const void* p, void* dX, void* dp, int64_t n, void* s) {
  return lie_launch<OP_ACT4_B>(g, dt, LIE_ARGS(grad, X, p, dX, dp, n), (cudaStream_t)s, "lie_act4_backward");
}
int dpvo_lie_as_matrix(int g, int dt, const void* X, void* T, int64_t n, void* s) {
  return lie_launch<OP_MATRIX>(g, dt, LIE_ARGS(X, nullptr, nullptr, T, nullptr, n), (cudaStream_t)s, "lie_as_matrix");
}
int dpvo_lie_projector(int g, int dt, const void* X, void* Pm, int64_t n, void* s) {
  return lie_launch<OP_PROJ>(g, dt, LIE_ARGS(X, nullptr, nullptr, Pm, nullptr, n), (cudaStream_t)s, "lie_projector");
}
int dpvo_lie_jinv(int g, int dt, const void* X, const void* a, void* b, int64_t n, void* s) {
  return lie_launch<OP_JINV>(g, dt, LIE_ARGS(X, a, nullptr, b, nullptr, n), (cudaStream_t)s, "lie_jinv");
}
}
