// lietorch_backends for sm_90a: SO3, RxSO3, SE3, Sim3, float and double, forward + backward.
// Replaces dpvo/lietorch/src/lietorch_gpu.cu:20-601 (Eigen template kernels) with register math
// from lie.cuh.  One group element per thread, grid-stride, outputs fully written (the reference
// allocates with torch::zeros and overwrites; the unused last gradient component stays 0).
// SO3 / SE3 (the groups on the DPVO hot path) have hand-specialised operators below; RxSO3 / Sim3 (loop closure
// only, SURVEY 8(f)) run the generic small-matrix operators of lie_scaled.cuh.
#include "common.cuh"
#include "lie.cuh"
#include "lie_scaled.cuh"

namespace dpvo {
using namespace lie;

template <int G> struct GroupDims;
template <> struct GroupDims<DPVO_SO3> { static constexpr int N = 4, K = 3; };
template <> struct GroupDims<DPVO_SE3> { static constexpr int N = 7, K = 6; };

template <typename S> __device__ __forceinline__ V3<S> ld3(const S* p) { return v3<S>(p[0], p[1], p[2]); }
template <typename S> __device__ __forceinline__ void st3(S* p, V3<S> v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }
template <typename S> __device__ __forceinline__ Tan6<S> ld6(const S* p) { Tan6<S> a; a.tau = ld3(p); a.phi = ld3(p + 3); return a; }
template <typename S> __device__ __forceinline__ void st6(S* p, const Tan6<S>& a) { st3(p, a.tau); st3(p + 3, a.phi); }
template <typename S> __device__ __forceinline__ void stq(S* p, const Quat<S>& q) { p[0] = q.x; p[1] = q.y; p[2] = q.z; p[3] = q.w; }
template <typename S> __device__ __forceinline__ Tan6<S> neg6(const Tan6<S>& a) { Tan6<S> r; r.tau = -a.tau; r.phi = -a.phi; return r; }

enum Op {
  OP_EXP, OP_EXP_B, OP_LOG, OP_LOG_B, OP_INV, OP_INV_B, OP_MUL, OP_MUL_B, OP_ADJ, OP_ADJ_B,
  OP_ADJT, OP_ADJT_B, OP_ACT, OP_ACT_B, OP_ACT4, OP_ACT4_B, OP_MATRIX, OP_PROJ, OP_JINV
};

// pointer bundle: in0..in2 inputs, out0..out1 outputs (meaning depends on the op)
struct LieArgs { const void* in0; const void* in1; const void* in2; void* out0; void* out1; int64_t n; };

// ---------------------------------------------------------------------------- SE3 ---
template <typename S, int OP>
__device__ __forceinline__ void se3_op(const LieArgs& A, int64_t i) {
  constexpr int N = 7, K = 6;
  const S* i0 = (const S*)A.in0; const S* i1 = (const S*)A.in1; const S* i2 = (const S*)A.in2;
  S* o0 = (S*)A.out0; S* o1 = (S*)A.out1;
  if constexpr (OP == OP_EXP) {                       // in0 a[K] -> out0 X[N]      lietorch_gpu.cu:20-30
    se3_store(se3_exp(ld6(i0 + i * K)), o0 + i * N);
  } else if constexpr (OP == OP_EXP_B) {              // in0 grad[N], in1 a[K] -> out0 da[K]   :32-44
    st6(o0 + i * K, row_times_left_jacobian(ld6(i0 + i * N), ld6(i1 + i * K)));
  } else if constexpr (OP == OP_LOG) {                // in0 X -> out0 a           :46-56
    st6(o0 + i * K, se3_log(se3_load(i0 + i * N)));
  } else if constexpr (OP == OP_LOG_B) {              // in0 grad[K], in1 X -> out0 dX[N]      :58-70
    const Tan6<S> a = se3_log(se3_load(i1 + i * N));
    st6(o0 + i * N, row_times_left_jacobian_inverse(ld6(i0 + i * K), a));
    o0[i * N + 6] = S(0);
  } else if constexpr (OP == OP_INV) {                // :72-82
    se3_store(se3_inv(se3_load(i0 + i * N)), o0 + i * N);
  } else if constexpr (OP == OP_INV_B) {              // in0 grad[N], in1 X -> dX = -dY Adj(Y)   :85-97
    const SE3<S> Y = se3_inv(se3_load(i1 + i * N));
    st6(o0 + i * N, neg6(se3_adjT(Y, ld6(i0 + i * N))));
    o0[i * N + 6] = S(0);
  } else if constexpr (OP == OP_MUL) {                // in0 X, in1 Y -> Z         :100-110
    se3_store(se3_mul(se3_load(i0 + i * N), se3_load(i1 + i * N)), o0 + i * N);
  } else if constexpr (OP == OP_MUL_B) {              // in0 grad, in1 X, (in2 Y) -> dX, dY   :112-125
    const Tan6<S> dZ = ld6(i0 + i * N);
    st6(o0 + i * N, dZ); o0[i * N + 6] = S(0);
    st6(o1 + i * N, se3_adjT(se3_load(i1 + i * N), dZ)); o1[i * N + 6] = S(0);
  } else if constexpr (OP == OP_ADJ) {                // in0 X, in1 a -> b        :127-138
    st6(o0 + i * K, se3_adj(se3_load(i0 + i * N), ld6(i1 + i * K)));
  } else if constexpr (OP == OP_ADJ_B) {              // in0 grad[K], in1 X, in2 a -> dX[N], da[K]   :140-158
    const SE3<S> X = se3_load(i1 + i * N);
    const Tan6<S> db = ld6(i0 + i * K);
    const Tan6<S> b = se3_adj(X, ld6(i2 + i * K));
    st6(o1 + i * K, se3_adjT(X, db));
    st6(o0 + i * N, neg6(row_times_adj(db, b))); o0[i * N + 6] = S(0);
  } else if constexpr (OP == OP_ADJT) {               // :161-172
    st6(o0 + i * K, se3_adjT(se3_load(i0 + i * N), ld6(i1 + i * K)));
  } else if constexpr (OP == OP_ADJT_B) {             // :174-188
    const SE3<S> X = se3_load(i1 + i * N);
    const Tan6<S> Xdb = se3_adj(X, ld6(i0 + i * K));
    st6(o1 + i * K, Xdb);
    st6(o0 + i * N, neg6(row_times_adj(ld6(i2 + i * K), Xdb))); o0[i * N + 6] = S(0);
  } else if constexpr (OP == OP_ACT) {                // in0 X, in1 p[3] -> q[3]     :190-202
    const SE3<S> X = se3_load(i0 + i * N);
    st3(o0 + i * 3, q_rot(X.q, ld3(i1 + i * 3)) + X.t);
  } else if constexpr (OP == OP_ACT_B) {              // in0 grad[3], in1 X, in2 p -> dX[N], dp[3]  :204-221
    const SE3<S> X = se3_load(i1 + i * N);
    const V3<S> dq = ld3(i0 + i * 3);
    const V3<S> q = q_rot(X.q, ld3(i2 + i * 3)) + X.t;
    st3(o1 + i * 3, rowmul(dq, q_matrix(X.q)));
    Tan6<S> dX; dX.tau = dq; dX.phi = cross(q, dq);
    st6(o0 + i * N, dX); o0[i * N + 6] = S(0);
  } else if constexpr (OP == OP_ACT4) {               // :224-236
    const SE3<S> X = se3_load(i0 + i * N);
    const S w = i1[i * 4 + 3];
    st3(o0 + i * 4, q_rot(X.q, ld3(i1 + i * 4)) + w * X.t);
    o0[i * 4 + 3] = w;
  } else if constexpr (OP == OP_ACT4_B) {             // :238-256
    const SE3<S> X = se3_load(i1 + i * N);
    const V3<S> dq = ld3(i0 + i * 4);
    const S dq4 = i0[i * 4 + 3], w = i2[i * 4 + 3];
    const V3<S> q = q_rot(X.q, ld3(i2 + i * 4)) + w * X.t;
    st3(o1 + i * 4, rowmul(dq, q_matrix(X.q)));
    o1[i * 4 + 3] = dot(dq, X.t) + dq4;
    Tan6<S> dX; dX.tau = w * dq; dX.phi = cross(q, dq);
    st6(o0 + i * N, dX); o0[i * N + 6] = S(0);
  } else if constexpr (OP == OP_MATRIX) {             // row-major 4x4   :258-269
    const SE3<S> X = se3_load(i0 + i * N);
    const M3<S> R = q_matrix(X.q);
    S* T = o0 + i * 16;
    for (int r = 0; r < 3; ++r) { T[r * 4 + 0] = R.m[r][0]; T[r * 4 + 1] = R.m[r][1]; T[r * 4 + 2] = R.m[r][2]; }
    T[3] = X.t.x; T[7] = X.t.y; T[11] = X.t.z;
    T[12] = S(0); T[13] = S(0); T[14] = S(0); T[15] = S(1);
  } else if constexpr (OP == OP_PROJ) {               // se3.h:116-122, row-major 7x7   :271-280
    const SE3<S> X = se3_load(i0 + i * N);
    S* Pm = o0 + i * 49;
    for (int k = 0; k < 49; ++k) Pm[k] = S(0);
    const M3<S> H = hat(-X.t);
    for (int r = 0; r < 3; ++r) {
      Pm[r * 7 + r] = S(1);
      for (int c = 0; c < 3; ++c) Pm[r * 7 + 3 + c] = H.m[r][c];
    }
    S J[4][4];
    so3_projector(X.q, J);
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) Pm[(3 + r) * 7 + 3 + c] = J[r][c];
  } else if constexpr (OP == OP_JINV) {               // :282-294
    const Tan6<S> a = se3_log(se3_load(i0 + i * N));
    st6(o0 + i * K, left_jacobian_inverse_times(a, ld6(i1 + i * K)));
  }
}

// ---------------------------------------------------------------------------- SO3 ---
template <typename S, int OP>
__device__ __forceinline__ void so3_op(const LieArgs& A, int64_t i) {
  constexpr int N = 4, K = 3;
  const S* i0 = (const S*)A.in0; const S* i1 = (const S*)A.in1; const S* i2 = (const S*)A.in2;
  S* o0 = (S*)A.out0; S* o1 = (S*)A.out1;
  if constexpr (OP == OP_EXP) {
    stq(o0 + i * N, so3_exp(ld3(i0 + i * K)));
  } else if constexpr (OP == OP_EXP_B) {
    st3(o0 + i * K, rowmul(ld3(i0 + i * N), so3_left_jacobian(ld3(i1 + i * K))));
  } else if constexpr (OP == OP_LOG) {
    st3(o0 + i * K, so3_log(q_load(i0 + i * N)));
  } else if constexpr (OP == OP_LOG_B) {
    const V3<S> a = so3_log(q_load(i1 + i * N));
    st3(o0 + i * N, rowmul(ld3(i0 + i * K), so3_left_jacobian_inverse(a))); o0[i * N + 3] = S(0);
  } else if constexpr (OP == OP_INV) {
    stq(o0 + i * N, q_inv(q_load(i0 + i * N)));
  } else if constexpr (OP == OP_INV_B) {
    const Quat<S> Y = q_inv(q_load(i1 + i * N));
    st3(o0 + i * N, -rowmul(ld3(i0 + i * N), q_matrix(Y))); o0[i * N + 3] = S(0);
  } else if constexpr (OP == OP_MUL) {
    stq(o0 + i * N, q_mul(q_load(i0 + i * N), q_load(i1 + i * N)));
  } else if constexpr (OP == OP_MUL_B) {
    const V3<S> dZ = ld3(i0 + i * N);
    st3(o0 + i * N, dZ); o0[i * N + 3] = S(0);
    st3(o1 + i * N, rowmul(dZ, q_matrix(q_load(i1 + i * N)))); o1[i * N + 3] = S(0);
  } else if constexpr (OP == OP_ADJ) {
    st3(o0 + i * K, q_matrix(q_load(i0 + i * N)) * ld3(i1 + i * K));
  } else if constexpr (OP == OP_ADJ_B) {
    const M3<S> R = q_matrix(q_load(i1 + i * N));
    const V3<S> db = ld3(i0 + i * K), b = R * ld3(i2 + i * K);
    st3(o1 + i * K, rowmul(db, R));
    st3(o0 + i * N, -cross(db, b)); o0[i * N + 3] = S(0);
  } else if constexpr (OP == OP_ADJT) {
    st3(o0 + i * K, rowmul(ld3(i1 + i * K), q_matrix(q_load(i0 + i * N))));
  } else if constexpr (OP == OP_ADJT_B) {
    const M3<S> R = q_matrix(q_load(i1 + i * N));
    const V3<S> Rdb = R * ld3(i0 + i * K);
    st3(o1 + i * K, Rdb);
    st3(o0 + i * N, -cross(ld3(i2 + i * K), Rdb)); o0[i * N + 3] = S(0);
  } else if constexpr (OP == OP_ACT) {
    st3(o0 + i * 3, q_rot(q_load(i0 + i * N), ld3(i1 + i * 3)));
  } else if constexpr (OP == OP_ACT_B) {
    const Quat<S> X = q_load(i1 + i * N);
    const V3<S> dq = ld3(i0 + i * 3), q = q_rot(X, ld3(i2 + i * 3));
    st3(o1 + i * 3, rowmul(dq, q_matrix(X)));
    st3(o0 + i * N, cross(q, dq)); o0[i * N + 3] = S(0);
  } else if constexpr (OP == OP_ACT4) {
    st3(o0 + i * 4, q_rot(q_load(i0 + i * N), ld3(i1 + i * 4)));
    o0[i * 4 + 3] = i1[i * 4 + 3];
  } else if constexpr (OP == OP_ACT4_B) {
    const Quat<S> X = q_load(i1 + i * N);
    const V3<S> dq = ld3(i0 + i * 4), q = q_rot(X, ld3(i2 + i * 4));
    st3(o1 + i * 4, rowmul(dq, q_matrix(X)));
    o1[i * 4 + 3] = i0[i * 4 + 3];
    st3(o0 + i * N, cross(q, dq)); o0[i * N + 3] = S(0);
  } else if constexpr (OP == OP_MATRIX) {
    const M3<S> R = q_matrix(q_load(i0 + i * N));
    S* T = o0 + i * 16;
    for (int k = 0; k < 16; ++k) T[k] = S(0);
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) T[r * 4 + c] = R.m[r][c];
    T[15] = S(1);
  } else if constexpr (OP == OP_PROJ) {
    S J[4][4];
    so3_projector(q_load(i0 + i * N), J);
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) o0[i * 16 + r * 4 + c] = J[r][c];
  } else if constexpr (OP == OP_JINV) {
    const V3<S> a = so3_log(q_load(i0 + i * N));
    st3(o0 + i * K, so3_left_jacobian_inverse(a) * ld3(i1 + i * K));
  }
}

template <int G, typename S, int OP>
__global__ void __launch_bounds__(256) lie_kernel(const LieArgs A) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += (int64_t)gridDim.x * blockDim.x) {
    if constexpr (G == DPVO_SE3) se3_op<S, OP>(A, i);
    else so3_op<S, OP>(A, i);
  }
}

// RxSO3 / Sim3: the generic operators (op codes of lie_scaled.cuh follow the enum above)
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
  const int threads = 256;
  const unsigned blocks = (unsigned)std::min<int64_t>((A.n + threads - 1) / threads, (int64_t)sm_count() * 8);
  if (group == DPVO_RXSO3 || group == DPVO_SIM3) {
    const unsigned sb = (unsigned)std::min<int64_t>((A.n + 127) / 128, (int64_t)sm_count() * 8);
    if (group == DPVO_SIM3) {
      if (dtype == DPVO_F32) lie_scaled_kernel<DPVO_SIM3, float, OP><<<sb, 128, 0, st>>>(A);
      else lie_scaled_kernel<DPVO_SIM3, double, OP><<<sb, 128, 0, st>>>(A);
    } else {
      if (dtype == DPVO_F32) lie_scaled_kernel<DPVO_RXSO3, float, OP><<<sb, 128, 0, st>>>(A);
      else lie_scaled_kernel<DPVO_RXSO3, double, OP><<<sb, 128, 0, st>>>(A);
    }
  } else if (group == DPVO_SE3) {
    if (dtype == DPVO_F32) lie_kernel<DPVO_SE3, float, OP><<<blocks, threads, 0, st>>>(A);
    else lie_kernel<DPVO_SE3, double, OP><<<blocks, threads, 0, st>>>(A);
  } else {
    if (dtype == DPVO_F32) lie_kernel<DPVO_SO3, float, OP><<<blocks, threads, 0, st>>>(A);
    else lie_kernel<DPVO_SO3, double, OP><<<blocks, threads, 0, st>>>(A);
  }
  DPVO_LAUNCH_CHECK(name);
  return DPVO_OK;
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
