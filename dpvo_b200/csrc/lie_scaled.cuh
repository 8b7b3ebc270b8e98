// RxSO3 and Sim3 (group ids 2, 4 of lietorch_backends, dispatch.h:12-32) in registers, float / double.
// Semantics follow dpvo/lietorch/include/rxso3.h:11-324 and sim3.h:12-217:
//   * layouts RxSO3 [qx qy qz qw s], tangent [phi, sigma]; Sim3 [tx ty tz qx qy qz qw s], tangent [tau, phi, sigma]
//   * the quaternion is normalised on every load, the scale is taken as stored
//   * W(phi, sigma) as in rxso3.h:189-234, evaluated without its cancellation at small angles and scales (see
//     rxso3_calcW); Sim3::Log uses a general inverse of W (sim3.h:151-158); Sim3's left Jacobian is the series the
//     reference evaluates, i.e. truncated after the Xi^4/120 term (the 1/720 line is dead code behind a semicolon, sim3.h:169-180)
// These two groups are not on the DPVO hot path (loop closure only), so the operators are written once, generically,
// over small dense matrices: every backward operator of lietorch_gpu.cu:32-294 is a row vector times the group's
// left Jacobian / adjoint / action Jacobian.  Everything is __host__ __device__: tests/test_lie_scaled_host_cpu.py
// runs the very same functions on the host against the oracle.
#pragma once
#include "lie.cuh"

namespace dpvo {
namespace lie {

// ---- tiny dense helpers (K <= 7) -----------------------------------------------------------------
template <typename S, int R, int C> struct Mat { S m[R][C]; };

template <typename S, int R, int C> LIE_HD Mat<S, R, C> mat_zero() {
  Mat<S, R, C> A;
  for (int i = 0; i < R; ++i) for (int j = 0; j < C; ++j) A.m[i][j] = S(0);
  return A;
}
template <typename S, int K> LIE_HD Mat<S, K, K> mat_identity() {
  Mat<S, K, K> A = mat_zero<S, K, K>();
  for (int i = 0; i < K; ++i) A.m[i][i] = S(1);
  return A;
}
template <typename S, int R, int Q, int C> LIE_HD Mat<S, R, C> matmul(const Mat<S, R, Q>& a, const Mat<S, Q, C>& b) {
  Mat<S, R, C> r;
  for (int i = 0; i < R; ++i)
    for (int j = 0; j < C; ++j) {
      S s = S(0);
      for (int k = 0; k < Q; ++k) s += a.m[i][k] * b.m[k][j];
      r.m[i][j] = s;
    }
  return r;
}
template <typename S, int R, int C> LIE_HD void set_block(Mat<S, R, C>& A, int r0, int c0, const M3<S>& B) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) A.m[r0 + i][c0 + j] = B.m[i][j];
}
// y = A x ; y = x^T A
template <typename S, int R, int C> LIE_HD void mat_vec(const Mat<S, R, C>& A, const S* x, S* y) {
  for (int i = 0; i < R; ++i) { S s = S(0); for (int j = 0; j < C; ++j) s += A.m[i][j] * x[j]; y[i] = s; }
}
template <typename S, int R, int C> LIE_HD void row_mat(const S* x, const Mat<S, R, C>& A, S* y) {
  for (int j = 0; j < C; ++j) { S s = S(0); for (int i = 0; i < R; ++i) s += x[i] * A.m[i][j]; y[j] = s; }
}
template <typename S> LIE_HD M3<S> m3_inverse(const M3<S>& a) {
  const S c00 = a.m[1][1] * a.m[2][2] - a.m[1][2] * a.m[2][1];
  const S c01 = a.m[1][2] * a.m[2][0] - a.m[1][0] * a.m[2][2];
  const S c02 = a.m[1][0] * a.m[2][1] - a.m[1][1] * a.m[2][0];
  const S det = a.m[0][0] * c00 + a.m[0][1] * c01 + a.m[0][2] * c02;
  const S id = S(1) / det;
  M3<S> r;
  r.m[0][0] = c00 * id; r.m[0][1] = (a.m[0][2] * a.m[2][1] - a.m[0][1] * a.m[2][2]) * id; r.m[0][2] = (a.m[0][1] * a.m[1][2] - a.m[0][2] * a.m[1][1]) * id;
  r.m[1][0] = c01 * id; r.m[1][1] = (a.m[0][0] * a.m[2][2] - a.m[0][2] * a.m[2][0]) * id; r.m[1][2] = (a.m[0][2] * a.m[1][0] - a.m[0][0] * a.m[1][2]) * id;
  r.m[2][0] = c02 * id; r.m[2][1] = (a.m[0][1] * a.m[2][0] - a.m[0][0] * a.m[2][1]) * id; r.m[2][2] = (a.m[0][0] * a.m[1][1] - a.m[0][1] * a.m[1][0]) * id;
  return r;
}

// W(phi, sigma) = A hat(phi) + B hat(phi)^2 + C I = sum_k (hat(phi) + sigma I)^k / (k+1)!      rxso3.h:189-234
// The reference's closed forms cancel as sigma and theta go to 0 (e.g. C = (e^sigma - 1) / sigma lost ulp / sigma, 1e-3
// relative in float at sigma = 1e-5) and switched to their limits only below 1e-6.  Here, with z = sigma + i theta:
//   * |z| < 1: the double series A = sum b_k / (k+1)!, B = sum c_k / (k+1)!, C = sum sigma^k / (k+1)!, where
//     z^k = a_k + i theta b_k and c_k = (sigma^k - a_k) / theta^2 follow a_{k+1} = sigma a_k - theta^2 b_k,
//     b_{k+1} = a_k + sigma b_k, c_{k+1} = sigma c_k + b_k -- polynomials, no division, no cancellation.  WSeriesTerms<S>
//     terms make the first dropped one (< k^2 / (2 (k+1)!)) smaller than half an ulp of S at |z| = 1;
//   * |z| >= 1: C = expm1(sigma) / sigma (1 at sigma = 0) and the closed forms, which have no cancellation there, except
//     that B loses ~ulp / theta^2 as theta -> 0 at |sigma| >= 1 -- harmless for W, where B multiplies hat(phi)^2 of norm
//     theta^2 -- and, below theta = sqrt(ulp) (WSeriesTerms<S>::theta_limit), the theta -> 0 limits, whose truncation is below an ulp.
template <typename S> struct WSeriesTerms;
template <> struct WSeriesTerms<float> { static constexpr int n = 13; static constexpr double theta_limit = 2.5e-4; };
template <> struct WSeriesTerms<double> { static constexpr int n = 20; static constexpr double theta_limit = 1e-8; };

template <typename S> LIE_HD M3<S> rxso3_calcW(V3<S> phi, S sigma) {
  const S t2 = dot(phi, phi), th = sqrt(t2);
  const M3<S> Phi = hat(phi), Phi2 = Phi * Phi;
  S A, B, C;
  if (sigma * sigma + t2 < S(1)) {
    S a = S(1), b = S(0), c = S(0), sk = S(1), f = S(1);     // k = 0; f = 1 / (k+1)!
    A = S(0); B = S(0); C = S(0);
#pragma unroll 1
    for (int k = 0; k < WSeriesTerms<S>::n; ++k) {
      C += sk * f; A += b * f; B += c * f;
      const S an = sigma * a - t2 * b, bn = a + sigma * b, cn = sigma * c + b;
      a = an; b = bn; c = cn; sk *= sigma; f /= S(k + 2);
    }
  } else {
    const S sc = exp(sigma);
    C = (sigma == S(0)) ? S(1) : expm1(sigma) / sigma;
    if (th < S(WSeriesTerms<S>::theta_limit)) {                // |sigma| >= 1 here
      const S s2 = sigma * sigma;
      A = ((sigma - S(1)) * sc + S(1)) / s2;
      B = (sc * S(0.5) * s2 + sc - S(1) - sigma * sc) / (s2 * sigma);
    } else {
      const S a = sc * sin(th), b = sc * cos(th), c = t2 + sigma * sigma;
      A = (a * sigma + (S(1) - b) * th) / (th * c);
      B = (C - ((b - S(1)) * sigma + a * th) / c) / t2;
    }
  }
  return A * Phi + B * Phi2 + C * m3_identity<S>();
}

// ================================================================================== RxSO3
template <typename S> struct RxSO3g {
  static constexpr int N = 5, K = 4;
  Quat<S> q; S s;

  static LIE_HD RxSO3g load(const S* d) { RxSO3g X; X.q = q_load(d); X.s = d[4]; return X; }
  LIE_HD void store(S* d) const { d[0] = q.x; d[1] = q.y; d[2] = q.z; d[3] = q.w; d[4] = s; }
  static LIE_HD RxSO3g exp_(const S* a) { RxSO3g X; X.q = so3_exp(v3<S>(a[0], a[1], a[2])); X.s = exp(a[3]); return X; }
  LIE_HD void log_(S* a) const { const V3<S> p = so3_log(q); a[0] = p.x; a[1] = p.y; a[2] = p.z; a[3] = log(s); }
  LIE_HD RxSO3g inv() const { RxSO3g Y; Y.q = q_inv(q); Y.s = S(1) / s; return Y; }
  LIE_HD RxSO3g mul(const RxSO3g& o) const { RxSO3g Z; Z.q = q_mul(q, o.q); Z.s = s * o.s; return Z; }
  LIE_HD V3<S> act(V3<S> p) const { return s * q_rot(q, p); }
  LIE_HD void act4(const S* p, S* o) const { const V3<S> r = act(v3<S>(p[0], p[1], p[2])); o[0] = r.x; o[1] = r.y; o[2] = r.z; o[3] = p[3]; }
  LIE_HD Mat<S, 4, 4> Adj() const {                              // rxso3.h:68-72
    Mat<S, 4, 4> A = mat_identity<S, 4>();
    set_block(A, 0, 0, q_matrix(q));
    return A;
  }
  static LIE_HD Mat<S, 4, 4> adj_small(const S* a) {             // rxso3.h:122-131
    Mat<S, 4, 4> A = mat_zero<S, 4, 4>();
    set_block(A, 0, 0, hat(v3<S>(a[0], a[1], a[2])));
    return A;
  }
  static LIE_HD Mat<S, 4, 4> left_jacobian(const S* a) {         // rxso3.h:293-298
    Mat<S, 4, 4> J = mat_identity<S, 4>();
    set_block(J, 0, 0, so3_left_jacobian(v3<S>(a[0], a[1], a[2])));
    return J;
  }
  static LIE_HD Mat<S, 4, 4> left_jacobian_inverse(const S* a) { // rxso3.h:300-305
    Mat<S, 4, 4> J = mat_identity<S, 4>();
    set_block(J, 0, 0, so3_left_jacobian_inverse(v3<S>(a[0], a[1], a[2])));
    return J;
  }
  LIE_HD Mat<S, 4, 4> matrix() const {                           // 4x4: s R in the rotation block
    Mat<S, 4, 4> T = mat_identity<S, 4>();
    set_block(T, 0, 0, s * q_matrix(q));
    return T;
  }
  LIE_HD Mat<S, 5, 5> projector() const {                        // rxso3.h:85-100
    Mat<S, 5, 5> P = mat_zero<S, 5, 5>();
    S J[4][4];
    so3_projector(q, J);
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 3; ++j) P.m[i][j] = J[i][j];
    P.m[4][3] = s;
    return P;
  }
  static LIE_HD Mat<S, 3, 4> act_jacobian(V3<S> p) {             // rxso3.h:307-311: [hat(-p) | p]
    Mat<S, 3, 4> J;
    const M3<S> H = hat(-p);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) J.m[i][j] = H.m[i][j];
    J.m[0][3] = p.x; J.m[1][3] = p.y; J.m[2][3] = p.z;
    return J;
  }
  static LIE_HD Mat<S, 4, 4> act4_jacobian(const S* p) {         // rxso3.h:313-318
    Mat<S, 4, 4> J = mat_zero<S, 4, 4>();
    set_block(J, 0, 0, hat(v3<S>(-p[0], -p[1], -p[2])));
    J.m[0][3] = p[0]; J.m[1][3] = p[1]; J.m[2][3] = p[2];
    return J;
  }
};

// =================================================================================== Sim3
template <typename S> struct Sim3g {
  static constexpr int N = 8, K = 7;
  V3<S> t; RxSO3g<S> R;

  static LIE_HD Sim3g load(const S* d) { Sim3g X; X.t = v3<S>(d[0], d[1], d[2]); X.R = RxSO3g<S>::load(d + 3); return X; }
  LIE_HD void store(S* d) const { d[0] = t.x; d[1] = t.y; d[2] = t.z; R.store(d + 3); }
  static LIE_HD Sim3g exp_(const S* a) {                         // sim3.h:160-167
    Sim3g X;
    X.R = RxSO3g<S>::exp_(a + 3);
    X.t = rxso3_calcW(v3<S>(a[3], a[4], a[5]), a[6]) * v3<S>(a[0], a[1], a[2]);
    return X;
  }
  LIE_HD void log_(S* a) const {                                 // sim3.h:151-158
    R.log_(a + 3);
    const V3<S> tau = m3_inverse(rxso3_calcW(v3<S>(a[3], a[4], a[5]), a[6])) * t;
    a[0] = tau.x; a[1] = tau.y; a[2] = tau.z;
  }
  LIE_HD Sim3g inv() const { Sim3g Y; Y.R = R.inv(); Y.t = -Y.R.act(t); return Y; }
  LIE_HD Sim3g mul(const Sim3g& o) const { Sim3g Z; Z.R = R.mul(o.R); Z.t = t + R.act(o.t); return Z; }
  LIE_HD V3<S> act(V3<S> p) const { return R.act(p) + t; }
  LIE_HD void act4(const S* p, S* o) const {
    const V3<S> r = R.act(v3<S>(p[0], p[1], p[2])) + p[3] * t;
    o[0] = r.x; o[1] = r.y; o[2] = r.z; o[3] = p[3];
  }
  LIE_HD Mat<S, 7, 7> Adj() const {                              // sim3.h:98-110
    Mat<S, 7, 7> A = mat_identity<S, 7>();
    const M3<S> Rm = q_matrix(R.q);
    set_block(A, 0, 0, R.s * Rm);
    set_block(A, 0, 3, hat(t) * Rm);
    A.m[0][6] = -t.x; A.m[1][6] = -t.y; A.m[2][6] = -t.z;
    set_block(A, 3, 3, Rm);
    return A;
  }
  static LIE_HD Mat<S, 7, 7> adj_small(const S* a) {             // sim3.h:133-149
    Mat<S, 7, 7> A = mat_zero<S, 7, 7>();
    const V3<S> tau = v3<S>(a[0], a[1], a[2]), phi = v3<S>(a[3], a[4], a[5]);
    const M3<S> Phi = hat(phi);
    set_block(A, 0, 0, Phi + a[6] * m3_identity<S>());
    set_block(A, 0, 3, hat(tau));
    A.m[0][6] = -tau.x; A.m[1][6] = -tau.y; A.m[2][6] = -tau.z;
    set_block(A, 3, 3, Phi);
    return A;
  }
  static LIE_HD Mat<S, 7, 7> left_jacobian(const S* a) {         // sim3.h:169-180 (series as evaluated, see the header)
    const Mat<S, 7, 7> Xi = adj_small(a), Xi2 = matmul(Xi, Xi), Xi3 = matmul(Xi, Xi2), Xi4 = matmul(Xi2, Xi2);
    Mat<S, 7, 7> J = mat_identity<S, 7>();
    for (int i = 0; i < 7; ++i)
      for (int j = 0; j < 7; ++j)
        J.m[i][j] += S(1.0 / 2.0) * Xi.m[i][j] + S(1.0 / 6.0) * Xi2.m[i][j] + S(1.0 / 24.0) * Xi3.m[i][j] + S(1.0 / 120.0) * Xi4.m[i][j];
    return J;
  }
  static LIE_HD Mat<S, 7, 7> left_jacobian_inverse(const S* a) { // sim3.h:182-191
    const Mat<S, 7, 7> Xi = adj_small(a), Xi2 = matmul(Xi, Xi), Xi4 = matmul(Xi2, Xi2);
    Mat<S, 7, 7> J = mat_identity<S, 7>();
    for (int i = 0; i < 7; ++i)
      for (int j = 0; j < 7; ++j) J.m[i][j] += S(-1.0 / 2.0) * Xi.m[i][j] + S(1.0 / 12.0) * Xi2.m[i][j] - S(1.0 / 720.0) * Xi4.m[i][j];
    return J;
  }
  LIE_HD Mat<S, 4, 4> matrix() const {
    Mat<S, 4, 4> T = R.matrix();
    T.m[0][3] = t.x; T.m[1][3] = t.y; T.m[2][3] = t.z;
    return T;
  }
  LIE_HD Mat<S, 8, 8> projector() const {                        // sim3.h:88-96
    Mat<S, 8, 8> P = mat_zero<S, 8, 8>();
    const M3<S> H = hat(-t);
    for (int i = 0; i < 3; ++i) {
      P.m[i][i] = S(1);
      for (int j = 0; j < 3; ++j) P.m[i][3 + j] = H.m[i][j];
    }
    P.m[0][6] = t.x; P.m[1][6] = t.y; P.m[2][6] = t.z;
    const Mat<S, 5, 5> Q = R.projector();
    for (int i = 0; i < 5; ++i) for (int j = 0; j < 5; ++j) P.m[3 + i][3 + j] = Q.m[i][j];
    return P;
  }
  static LIE_HD Mat<S, 3, 7> act_jacobian(V3<S> p) {             // sim3.h:193-199: [I | hat(-p) | p]
    Mat<S, 3, 7> J = mat_zero<S, 3, 7>();
    const M3<S> H = hat(-p);
    for (int i = 0; i < 3; ++i) { J.m[i][i] = S(1); for (int j = 0; j < 3; ++j) J.m[i][3 + j] = H.m[i][j]; }
    J.m[0][6] = p.x; J.m[1][6] = p.y; J.m[2][6] = p.z;
    return J;
  }
  static LIE_HD Mat<S, 4, 7> act4_jacobian(const S* p) {         // sim3.h:201-207
    Mat<S, 4, 7> J = mat_zero<S, 4, 7>();
    const M3<S> H = hat(v3<S>(-p[0], -p[1], -p[2]));
    for (int i = 0; i < 3; ++i) { J.m[i][i] = p[3]; for (int j = 0; j < 3; ++j) J.m[i][3 + j] = H.m[i][j]; }
    J.m[0][6] = p[0]; J.m[1][6] = p[1]; J.m[2][6] = p[2];
    return J;
  }
};

// ---- the 19 operators of lietorch_backends, written once over a group G --------------------------
// Op codes as in lie.cu.  Pointers are the bases of the batch arrays, i the element; gradients w.r.t. group
// elements have the embedding width N with components K..N-1 set to zero (lietorch_gpu.cu:41-42).
enum ScaledOp {
  SOP_EXP, SOP_EXP_B, SOP_LOG, SOP_LOG_B, SOP_INV, SOP_INV_B, SOP_MUL, SOP_MUL_B, SOP_ADJ, SOP_ADJ_B,
  SOP_ADJT, SOP_ADJT_B, SOP_ACT, SOP_ACT_B, SOP_ACT4, SOP_ACT4_B, SOP_MATRIX, SOP_PROJ, SOP_JINV
};

template <typename S, int N, int K> LIE_HD void store_padded(S* d, const S* v) {
  for (int k = 0; k < K; ++k) d[k] = v[k];
  for (int k = K; k < N; ++k) d[k] = S(0);
}

template <typename G, typename S>
LIE_HD void scaled_group_op(int op, const S* i0, const S* i1, const S* i2, S* o0, S* o1, long long i) {
  constexpr int N = G::N, K = G::K;
  S tmp[K], tmp2[K];
  switch (op) {
    case SOP_EXP: G::exp_(i0 + i * K).store(o0 + i * N); break;
    case SOP_EXP_B: {                                       // da = grad[:K] J_l(a)
      row_mat(i0 + i * N, G::left_jacobian(i1 + i * K), o0 + i * K);
    } break;
    case SOP_LOG: G::load(i0 + i * N).log_(o0 + i * K); break;
    case SOP_LOG_B: {                                       // dX = grad J_l^-1(log X)
      G::load(i1 + i * N).log_(tmp);
      row_mat(i0 + i * K, G::left_jacobian_inverse(tmp), tmp2);
      store_padded<S, N, K>(o0 + i * N, tmp2);
    } break;
    case SOP_INV: G::load(i0 + i * N).inv().store(o0 + i * N); break;
    case SOP_INV_B: {                                       // dX = -grad[:K] Adj(X^-1)
      row_mat(i0 + i * N, G::load(i1 + i * N).inv().Adj(), tmp);
      for (int k = 0; k < K; ++k) tmp[k] = -tmp[k];
      store_padded<S, N, K>(o0 + i * N, tmp);
    } break;
    case SOP_MUL: G::load(i0 + i * N).mul(G::load(i1 + i * N)).store(o0 + i * N); break;
    case SOP_MUL_B: {                                       // dX = dZ, dY = dZ Adj(X)
      store_padded<S, N, K>(o0 + i * N, i0 + i * N);
      row_mat(i0 + i * N, G::load(i1 + i * N).Adj(), tmp);
      store_padded<S, N, K>(o1 + i * N, tmp);
    } break;
    case SOP_ADJ: mat_vec(G::load(i0 + i * N).Adj(), i1 + i * K, o0 + i * K); break;
    case SOP_ADJ_B: {                                       // b = Adj(X) a; dX = -grad adj(b); da = grad Adj(X)
      const auto A = G::load(i1 + i * N).Adj();
      mat_vec(A, i2 + i * K, tmp);
      row_mat(i0 + i * K, G::adj_small(tmp), tmp2);
      for (int k = 0; k < K; ++k) tmp2[k] = -tmp2[k];
      store_padded<S, N, K>(o0 + i * N, tmp2);
      row_mat(i0 + i * K, A, o1 + i * K);
    } break;
    case SOP_ADJT: row_mat(i1 + i * K, G::load(i0 + i * N).Adj(), o0 + i * K); break;
    case SOP_ADJT_B: {                                      // Xdb = Adj(X) grad; dX = -a adj(Xdb); da = Xdb
      mat_vec(G::load(i1 + i * N).Adj(), i0 + i * K, tmp);
      row_mat(i2 + i * K, G::adj_small(tmp), tmp2);
      for (int k = 0; k < K; ++k) tmp2[k] = -tmp2[k];
      store_padded<S, N, K>(o0 + i * N, tmp2);
      for (int k = 0; k < K; ++k) o1[i * K + k] = tmp[k];
    } break;
    case SOP_ACT: {
      const V3<S> q = G::load(i0 + i * N).act(v3<S>(i1[i * 3], i1[i * 3 + 1], i1[i * 3 + 2]));
      o0[i * 3] = q.x; o0[i * 3 + 1] = q.y; o0[i * 3 + 2] = q.z;
    } break;
    case SOP_ACT_B: {                                       // dX = grad J_act(q), dp = grad T[:3,:3]
      const G X = G::load(i1 + i * N);
      const V3<S> q = X.act(v3<S>(i2[i * 3], i2[i * 3 + 1], i2[i * 3 + 2]));
      row_mat(i0 + i * 3, G::act_jacobian(q), tmp);
      store_padded<S, N, K>(o0 + i * N, tmp);
      const Mat<S, 4, 4> T = X.matrix();
      for (int j = 0; j < 3; ++j) o1[i * 3 + j] = i0[i * 3] * T.m[0][j] + i0[i * 3 + 1] * T.m[1][j] + i0[i * 3 + 2] * T.m[2][j];
    } break;
    case SOP_ACT4: G::load(i0 + i * N).act4(i1 + i * 4, o0 + i * 4); break;
    case SOP_ACT4_B: {                                      // dX = grad J_act4(q), dp = grad T
      const G X = G::load(i1 + i * N);
      S q[4];
      X.act4(i2 + i * 4, q);
      row_mat(i0 + i * 4, G::act4_jacobian(q), tmp);
      store_padded<S, N, K>(o0 + i * N, tmp);
      row_mat(i0 + i * 4, X.matrix(), o1 + i * 4);
    } break;
    case SOP_MATRIX: {
      const Mat<S, 4, 4> T = G::load(i0 + i * N).matrix();
      for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) o0[i * 16 + r * 4 + c] = T.m[r][c];
    } break;
    case SOP_PROJ: {
      const auto P = G::load(i0 + i * N).projector();
      for (int r = 0; r < N; ++r) for (int c = 0; c < N; ++c) o0[i * N * N + r * N + c] = P.m[r][c];
    } break;
    case SOP_JINV: {                                        // b = J_l^-1(log X) a
      G::load(i0 + i * N).log_(tmp);
      mat_vec(G::left_jacobian_inverse(tmp), i1 + i * K, o0 + i * K);
    } break;
    default: break;
  }
}

}  // namespace lie
}  // namespace dpvo
