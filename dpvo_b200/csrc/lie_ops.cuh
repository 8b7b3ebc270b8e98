// The SO3 / SE3 operators of lietorch_backends, one group element per call: so3_op / se3_op run operator OP on element
// i of the batch arrays in LieArgs.  __host__ __device__, so tools/lie_host_check.cu runs on the host the very code the
// kernels of lie.cu run on the device.
#pragma once
#include <stdint.h>
#include "lie.cuh"

namespace dpvo {
using namespace lie;

template <typename S> LIE_HD V3<S> ld3(const S* p) { return v3<S>(p[0], p[1], p[2]); }
template <typename S> LIE_HD void st3(S* p, V3<S> v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }
template <typename S> LIE_HD Tan6<S> ld6(const S* p) { Tan6<S> a; a.tau = ld3(p); a.phi = ld3(p + 3); return a; }
template <typename S> LIE_HD void st6(S* p, const Tan6<S>& a) { st3(p, a.tau); st3(p + 3, a.phi); }
template <typename S> LIE_HD void stq(S* p, const Quat<S>& q) { p[0] = q.x; p[1] = q.y; p[2] = q.z; p[3] = q.w; }
template <typename S> LIE_HD Tan6<S> neg6(const Tan6<S>& a) { Tan6<S> r; r.tau = -a.tau; r.phi = -a.phi; return r; }

enum Op {
  OP_EXP, OP_EXP_B, OP_LOG, OP_LOG_B, OP_INV, OP_INV_B, OP_MUL, OP_MUL_B, OP_ADJ, OP_ADJ_B,
  OP_ADJT, OP_ADJT_B, OP_ACT, OP_ACT_B, OP_ACT4, OP_ACT4_B, OP_MATRIX, OP_PROJ, OP_JINV
};

// pointer bundle: in0..in2 inputs, out0..out1 outputs (meaning depends on the op)
struct LieArgs { const void* in0; const void* in1; const void* in2; void* out0; void* out1; int64_t n; };

// ---------------------------------------------------------------------------- SE3 ---
template <typename S, int OP>
LIE_HD void se3_op(const LieArgs& A, int64_t i) {
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
LIE_HD void so3_op(const LieArgs& A, int64_t i) {
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

}  // namespace dpvo
