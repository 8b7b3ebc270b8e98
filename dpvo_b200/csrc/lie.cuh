// Eigen-free SO3 / SE3 math in registers, templated on the scalar (float / double).
// Semantics follow dpvo/lietorch/include/so3.h:31-220 and se3.h:36-217:
//   * element layout SO3 [qx qy qz qw], SE3 [tx ty tz qx qy qz qw]
//   * quaternions are normalised whenever a group element is constructed (so3.h:31-37)
//   * so3_exp / so3_log switch to their series at theta < EPS = 1e-6 (common.h:7); their closed forms sin(t/2)/t and
//     atan(n/w)/n do not cancel, so the switch only keeps 0/0 away and serves float and double alike
//   * the Jacobian coefficients do cancel at small angles, and are evaluated differently from the reference; see
//     "Jacobian coefficients" below
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace dpvo {
namespace lie {

#define LIE_HD __host__ __device__ __forceinline__
constexpr double kEps = 1e-6;
constexpr double kPi = 3.14159265358979323846;

template <typename S> struct V3 { S x, y, z; };
template <typename S> struct M3 { S m[3][3]; };
template <typename S> struct Quat { S x, y, z, w; };

template <typename S> LIE_HD V3<S> v3(S x, S y, S z) { V3<S> r; r.x = x; r.y = y; r.z = z; return r; }
template <typename S> LIE_HD V3<S> operator+(V3<S> a, V3<S> b) { return v3<S>(a.x + b.x, a.y + b.y, a.z + b.z); }
template <typename S> LIE_HD V3<S> operator-(V3<S> a, V3<S> b) { return v3<S>(a.x - b.x, a.y - b.y, a.z - b.z); }
template <typename S> LIE_HD V3<S> operator-(V3<S> a) { return v3<S>(-a.x, -a.y, -a.z); }
template <typename S> LIE_HD V3<S> operator*(S s, V3<S> a) { return v3<S>(s * a.x, s * a.y, s * a.z); }
template <typename S> LIE_HD V3<S> cross(V3<S> a, V3<S> b) {
  return v3<S>(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
template <typename S> LIE_HD S dot(V3<S> a, V3<S> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

template <typename S> LIE_HD M3<S> m3_identity() {
  M3<S> r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = (i == j) ? S(1) : S(0);
  return r;
}
template <typename S> LIE_HD M3<S> m3_zero() {
  M3<S> r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = S(0);
  return r;
}
// so3.h:109-117
template <typename S> LIE_HD M3<S> hat(V3<S> p) {
  M3<S> r;
  r.m[0][0] = S(0); r.m[0][1] = -p.z; r.m[0][2] = p.y;
  r.m[1][0] = p.z;  r.m[1][1] = S(0); r.m[1][2] = -p.x;
  r.m[2][0] = -p.y; r.m[2][1] = p.x;  r.m[2][2] = S(0);
  return r;
}
template <typename S> LIE_HD M3<S> operator*(const M3<S>& a, const M3<S>& b) {
  M3<S> r;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
  return r;
}
template <typename S> LIE_HD M3<S> operator+(const M3<S>& a, const M3<S>& b) {
  M3<S> r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = a.m[i][j] + b.m[i][j];
  return r;
}
template <typename S> LIE_HD M3<S> operator-(const M3<S>& a, const M3<S>& b) {
  M3<S> r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = a.m[i][j] - b.m[i][j];
  return r;
}
template <typename S> LIE_HD M3<S> operator*(S s, const M3<S>& a) {
  M3<S> r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = s * a.m[i][j];
  return r;
}
template <typename S> LIE_HD V3<S> operator*(const M3<S>& a, V3<S> v) {
  return v3<S>(a.m[0][0] * v.x + a.m[0][1] * v.y + a.m[0][2] * v.z,
               a.m[1][0] * v.x + a.m[1][1] * v.y + a.m[1][2] * v.z,
               a.m[2][0] * v.x + a.m[2][1] * v.y + a.m[2][2] * v.z);
}
// row vector times matrix
template <typename S> LIE_HD V3<S> rowmul(V3<S> v, const M3<S>& a) {
  return v3<S>(v.x * a.m[0][0] + v.y * a.m[1][0] + v.z * a.m[2][0],
               v.x * a.m[0][1] + v.y * a.m[1][1] + v.z * a.m[2][1],
               v.x * a.m[0][2] + v.y * a.m[1][2] + v.z * a.m[2][2]);
}

// ---- SO3 ------------------------------------------------------------------------------
template <typename S> LIE_HD Quat<S> q_normalized(S x, S y, S z, S w) {
  const S n = sqrt(x * x + y * y + z * z + w * w);
  Quat<S> q; q.x = x / n; q.y = y / n; q.z = z / n; q.w = w / n;
  return q;
}
template <typename S> LIE_HD Quat<S> q_load(const S* d) { return q_normalized<S>(d[0], d[1], d[2], d[3]); }
template <typename S> LIE_HD V3<S> q_vec(const Quat<S>& q) { return v3<S>(q.x, q.y, q.z); }
// so3.h:43-45
template <typename S> LIE_HD Quat<S> q_inv(const Quat<S>& q) { return q_normalized<S>(-q.x, -q.y, -q.z, q.w); }
// so3.h:51-53 (Hamilton product, then normalise)
template <typename S> LIE_HD Quat<S> q_mul(const Quat<S>& a, const Quat<S>& b) {
  return q_normalized<S>(a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
                         a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
                         a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x,
                         a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z);
}
// so3.h:55-60
template <typename S> LIE_HD V3<S> q_rot(const Quat<S>& q, V3<S> p) {
  V3<S> uv = cross(q_vec(q), p);
  uv = uv + uv;
  return p + q.w * uv + cross(q_vec(q), uv);
}
template <typename S> LIE_HD M3<S> q_matrix(const Quat<S>& q) {
  const S tx = S(2) * q.x, ty = S(2) * q.y, tz = S(2) * q.z;
  const S twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const S txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const S tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  M3<S> r;
  r.m[0][0] = S(1) - (tyy + tzz); r.m[0][1] = txy - twz;          r.m[0][2] = txz + twy;
  r.m[1][0] = txy + twz;          r.m[1][1] = S(1) - (txx + tzz); r.m[1][2] = tyz - twx;
  r.m[2][0] = txz - twy;          r.m[2][1] = tyz + twx;          r.m[2][2] = S(1) - (txx + tyy);
  return r;
}
// so3.h:123-157
template <typename S> LIE_HD V3<S> so3_log(const Quat<S>& q) {
  const S sn = q.x * q.x + q.y * q.y + q.z * q.z;
  const S w = q.w;
  S f;
  if ((double)sn < kEps * kEps) {
    f = S(2) / w - S(2.0 / 3.0) * sn / (w * w * w);
  } else {
    const S n = sqrt(sn);
    if (fabs((double)w) < kEps) f = (w > S(0)) ? S(kPi) / n : -S(kPi) / n;
    else f = S(2) * atan(n / w) / n;
  }
  return f * q_vec(q);
}
// so3.h:159-176
template <typename S> LIE_HD Quat<S> so3_exp(V3<S> phi) {
  const S t2 = dot(phi, phi);
  const S th = sqrt(t2);
  S im, re;
  if ((double)th < kEps) {
    const S t4 = t2 * t2;
    im = S(0.5) - S(1.0 / 48.0) * t2 + S(1.0 / 3840.0) * t4;
    re = S(1) - S(1.0 / 8.0) * t2 + S(1.0 / 384.0) * t4;
  } else {
    im = sin(S(0.5) * th) / th;
    re = cos(S(0.5) * th);
  }
  return q_normalized<S>(im * phi.x, im * phi.y, im * phi.z, re);
}
// ---- Jacobian coefficients ---------------------------------------------------------------------------------------
// lietorch's closed forms, e.g. (t - sin t) / t^3, lose about ulp / t^2 relative to the coefficient as t -> 0 (ulp / t^4
// for the Q coefficients), and switched to two-term series only below t = 1e-6 for both float and double: at t = 1e-4 the
// float J and Q were wrong in the 4th digit, the double ones in the 10th.  Here every coefficient is within a few ulp of
// S over the whole range:
//   * (1 - cos t) / t^2 = 2 (sin(t/2) / t)^2 everywhere -- no cancellation; sin(t/2) / t is so3_exp's coefficient;
//   * (t - sin t) / t^3, (t^2/2 - (1 - cos t)) / t^4 and lietorch's J^-1 coefficient (1 - t cos(t/2) / (2 sin(t/2))) / t^2
//     by their Taylor series below t = 1, where the closed forms above lose at most ~24 ulp;
//   * Q's third coefficient (2t - 3 sin t + t cos t) / (2 t^5) by its series below t = 2, where its closed form, written
//     (3 c_B - c_A) / (2 t^2) over the two J coefficients, loses at most ~15 ulp.
// The switches depend on the cancellation, not on S; the number of terms is per type (SeriesTerms), each series cut
// where its first dropped term is below half an ulp of S at the switch.
template <typename S> struct SeriesTerms;
template <> struct SeriesTerms<float> { static constexpr int sin3 = 5, cos4 = 4, jinv = 5, q3 = 6; };
template <> struct SeriesTerms<double> { static constexpr int sin3 = 8, cos4 = 8, jinv = 10, q3 = 10; };

// sum_k c[k] x^k over the first n coefficients, Horner
template <int n, typename S, int M> LIE_HD S series(const double (&c)[M], S x) {
  static_assert(n <= M, "not enough coefficients");
  S p = S(c[n - 1]);
#pragma unroll
  for (int k = n - 2; k >= 0; --k) p = p * x + S(c[k]);
  return p;
}
// sin(t/2) / t, as in so3_exp
template <typename S> LIE_HD S sinc_half(S th, S t2) {
  return (th < S(kEps)) ? S(0.5) - S(1.0 / 48.0) * t2 + S(1.0 / 3840.0) * t2 * t2 : sin(S(0.5) * th) / th;
}
// (1 - cos t) / t^2
template <typename S> LIE_HD S coef_cos2(S th, S t2) { const S h = sinc_half(th, t2); return S(2) * h * h; }
// (t - sin t) / t^3 = sum_k (-1)^k t^2k / (2k+3)!
template <typename S> LIE_HD S coef_sin3(S th, S t2) {
  constexpr double c[] = {0.16666666666666666, -0.008333333333333333, 0.0001984126984126984, -2.7557319223985893e-06,
                          2.505210838544172e-08, -1.6059043836821613e-10, 7.647163731819816e-13, -2.8114572543455206e-15};
  return (th < S(1)) ? series<SeriesTerms<S>::sin3>(c, t2) : (th - sin(th)) / (t2 * th);
}
// (t^2/2 - (1 - cos t)) / t^4 = sum_k (-1)^k t^2k / (2k+4)!
template <typename S> LIE_HD S coef_cos4(S th, S t2) {
  constexpr double c[] = {0.041666666666666664, -0.001388888888888889, 2.48015873015873e-05, -2.755731922398589e-07,
                          2.08767569878681e-09, -1.1470745597729725e-11, 4.779477332387385e-14, -1.5619206968586225e-16};
  return (th < S(1)) ? series<SeriesTerms<S>::cos4>(c, t2) : (S(0.5) - coef_cos2(th, t2)) / t2;
}
// (1 - t cos(t/2) / (2 sin(t/2))) / t^2 = sum_{n>=1} |B_2n| t^(2n-2) / (2n)!
template <typename S> LIE_HD S coef_jinv(S th, S t2) {
  constexpr double c[] = {0.08333333333333333, 0.001388888888888889, 3.306878306878307e-05, 8.267195767195768e-07,
                          2.08767569878681e-08, 5.284190138687493e-10, 1.3382536530684679e-11, 3.3896802963225827e-13,
                          8.586062056277845e-15, 2.174868698558062e-16};
  if (th < S(1)) return series<SeriesTerms<S>::jinv>(c, t2);
  const S ht = S(0.5) * th;
  return (S(1) - th * cos(ht) / (S(2) * sin(ht))) / t2;
}
// (2t - 3 sin t + t cos t) / (2 t^5) = sum_k (-1)^k (k+1) t^2k / (2k+5)!
template <typename S> LIE_HD S coef_q3(S th, S t2) {
  constexpr double c[] = {0.008333333333333333, -0.0003968253968253968, 8.267195767195768e-06, -1.0020843354176688e-07,
                          8.029521918410807e-10, -4.58829823909189e-12, 1.9680200780418645e-14, -6.576508197299464e-17,
                          1.7615646957052136e-19, -3.868170170630684e-22};
  return (th < S(2)) ? series<SeriesTerms<S>::q3>(c, t2) : (S(3) * coef_sin3(th, t2) - coef_cos2(th, t2)) / (S(2) * t2);
}

// so3.h:178-197
template <typename S> LIE_HD M3<S> so3_left_jacobian(V3<S> phi) {
  const M3<S> Phi = hat(phi), Phi2 = Phi * Phi;
  const S t2 = dot(phi, phi), th = sqrt(t2);
  return m3_identity<S>() + coef_cos2(th, t2) * Phi + coef_sin3(th, t2) * Phi2;
}
// so3.h:199-215
template <typename S> LIE_HD M3<S> so3_left_jacobian_inverse(V3<S> phi) {
  const M3<S> Phi = hat(phi), Phi2 = Phi * Phi;
  const S t2 = dot(phi, phi), th = sqrt(t2);
  return m3_identity<S>() + S(-0.5) * Phi + coef_jinv(th, t2) * Phi2;
}
// so3.h:83-93: 4x4 orthogonal projector, row major
template <typename S> LIE_HD void so3_projector(const Quat<S>& q, S (&J)[4][4]) {
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) J[i][j] = S(0);
  const M3<S> H = hat(-q_vec(q));
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) J[i][j] = S(0.5) * (((i == j) ? q.w : S(0)) + H.m[i][j]);
  J[3][0] = S(0.5) * (-q.x); J[3][1] = S(0.5) * (-q.y); J[3][2] = S(0.5) * (-q.z);
}

// ---- SE3 ------------------------------------------------------------------------------
template <typename S> struct SE3 { V3<S> t; Quat<S> q; };
template <typename S> struct Tan6 { V3<S> tau, phi; };

template <typename S> LIE_HD SE3<S> se3_load(const S* d) {
  SE3<S> X; X.t = v3<S>(d[0], d[1], d[2]); X.q = q_load<S>(d + 3); return X;
}
template <typename S> LIE_HD void se3_store(const SE3<S>& X, S* d) {
  d[0] = X.t.x; d[1] = X.t.y; d[2] = X.t.z; d[3] = X.q.x; d[4] = X.q.y; d[5] = X.q.z; d[6] = X.q.w;
}
// se3.h:36-38
template <typename S> LIE_HD SE3<S> se3_inv(const SE3<S>& X) {
  SE3<S> Y; Y.q = q_inv(X.q); Y.t = -(q_rot(Y.q, X.t)); return Y;
}
// se3.h:45-47
template <typename S> LIE_HD SE3<S> se3_mul(const SE3<S>& A, const SE3<S>& B) {
  SE3<S> Z; Z.q = q_mul(A.q, B.q); Z.t = A.t + q_rot(A.q, B.t); return Z;
}
// se3.h:58-67  Adj(X) a
template <typename S> LIE_HD Tan6<S> se3_adj(const SE3<S>& X, const Tan6<S>& a) {
  const M3<S> R = q_matrix(X.q);
  const V3<S> Rphi = R * a.phi;
  Tan6<S> b; b.tau = R * a.tau + cross(X.t, Rphi); b.phi = Rphi; return b;
}
// se3.h:84-86  Adj(X)^T a   (== row vector a times Adj(X))
template <typename S> LIE_HD Tan6<S> se3_adjT(const SE3<S>& X, const Tan6<S>& a) {
  const M3<S> R = q_matrix(X.q);
  Tan6<S> b;
  b.tau = rowmul(a.tau, R);
  b.phi = rowmul(cross(a.tau, X.t) + a.phi, R);   // (tx R)^T a1 + R^T a2 = R^T (a1 x t + a2)
  return b;
}
// row vector g times adj(b), adj(b) = [[Phi, Tau],[0, Phi]] (se3.h:101-114)
template <typename S> LIE_HD Tan6<S> row_times_adj(const Tan6<S>& g, const Tan6<S>& b) {
  Tan6<S> r;
  r.tau = cross(g.tau, b.phi);
  r.phi = cross(g.tau, b.tau) + cross(g.phi, b.phi);
  return r;
}
// se3.h:147-176
template <typename S> LIE_HD M3<S> se3_calcQ(const Tan6<S>& a) {
  const M3<S> Tau = hat(a.tau), Phi = hat(a.phi);
  const S t2 = dot(a.phi, a.phi), th = sqrt(t2);
  const S c1 = coef_sin3(th, t2), c2 = coef_cos4(th, t2), c3 = coef_q3(th, t2);
  const M3<S> PT = Phi * Tau, TP = Tau * Phi, PTP = PT * Phi;
  return S(0.5) * Tau + c1 * (PT + TP + PTP) + c2 * (Phi * PT + TP * Phi - S(3) * PTP) +
         c3 * (PTP * Phi + Phi * PTP);
}
// se3.h:124-142
template <typename S> LIE_HD Tan6<S> se3_log(const SE3<S>& X) {
  Tan6<S> a; a.phi = so3_log(X.q); a.tau = so3_left_jacobian_inverse(a.phi) * X.t; return a;
}
template <typename S> LIE_HD SE3<S> se3_exp(const Tan6<S>& a) {
  SE3<S> X; X.q = so3_exp(a.phi); X.t = so3_left_jacobian(a.phi) * a.tau; return X;
}
// row vector g times left_jacobian(a) = [[J, Q],[0, J]]  (se3.h:178-189)
template <typename S> LIE_HD Tan6<S> row_times_left_jacobian(const Tan6<S>& g, const Tan6<S>& a) {
  const M3<S> J = so3_left_jacobian(a.phi), Q = se3_calcQ(a);
  Tan6<S> r; r.tau = rowmul(g.tau, J); r.phi = rowmul(g.tau, Q) + rowmul(g.phi, J); return r;
}
// left_jacobian_inverse(a) = [[Ji, -Ji Q Ji],[0, Ji]]  (se3.h:191-205)
template <typename S> LIE_HD Tan6<S> row_times_left_jacobian_inverse(const Tan6<S>& g, const Tan6<S>& a) {
  const M3<S> Ji = so3_left_jacobian_inverse(a.phi), Q = se3_calcQ(a);
  const M3<S> B = Ji * Q * Ji;
  Tan6<S> r; r.tau = rowmul(g.tau, Ji); r.phi = rowmul(g.phi, Ji) - rowmul(g.tau, B); return r;
}
template <typename S> LIE_HD Tan6<S> left_jacobian_inverse_times(const Tan6<S>& a, const Tan6<S>& v) {
  const M3<S> Ji = so3_left_jacobian_inverse(a.phi), Q = se3_calcQ(a);
  Tan6<S> r; r.phi = Ji * v.phi; r.tau = Ji * v.tau - Ji * (Q * r.phi); return r;
}

}  // namespace lie
}  // namespace dpvo
