// Flow magnitude of one patch pixel (dpvo/projective_ops.py:flow_mag, beta = 0.5), shared by the loop-candidate scores
// (loop.cu, the centre pixel) and the keyframe motion test (keyframe.cu, all 9 pixels).
#pragma once
#include "lie.cuh"

namespace dpvo {

// flow of pixel `pix` (0..8, row-major in the 3x3 patch) of patch k from frame i to frame j:
// 0.5 |full - origin| + 0.5 |translation only - origin|, valid when the fully transformed point has Z > 0.2
// (projective_ops.py:111, 120-130).  The origin is the pixel reprojected into its own frame through Pi Pi^-1, with
// frame i's intrinsics, as flow_mag's coords0 is.
__device__ __forceinline__ float patch_flow(const float* __restrict__ poses, const float* __restrict__ patches,
                                            const float* __restrict__ intr, int64_t i, int64_t j, int64_t k, int pix,
                                            bool& valid) {
  using namespace lie;
  const float* pk = patches + k * 27;
  const float x = pk[pix], y = pk[9 + pix], d = pk[18 + pix];
  const float fxi = intr[4 * i], fyi = intr[4 * i + 1], cxi = intr[4 * i + 2], cyi = intr[4 * i + 3];
  const float fxj = intr[4 * j], fyj = intr[4 * j + 1], cxj = intr[4 * j + 2], cyj = intr[4 * j + 3];
  const V3<float> p = v3<float>((x - cxi) / fxi, (y - cyi) / fyi, 1.f);
  const SE3<float> Pi = se3_load(poses + 7 * i), Pj = se3_load(poses + 7 * j);
  const SE3<float> Pii = se3_inv(Pi);
  // origin: the patch reprojected into its own frame
  const SE3<float> Gii = se3_mul(Pi, Pii);
  const V3<float> X0 = q_rot(Gii.q, p) + d * Gii.t;
  const float d0 = 1.f / fmaxf(X0.z, 0.1f);
  const float u0 = fxi * (d0 * X0.x) + cxi, v0 = fyi * (d0 * X0.y) + cyi;
  const SE3<float> Gij = se3_mul(Pj, Pii);
  const V3<float> X1 = q_rot(Gij.q, p) + d * Gij.t;
  const float d1 = 1.f / fmaxf(X1.z, 0.1f);
  const float u1 = fxj * (d1 * X1.x) + cxj, v1 = fyj * (d1 * X1.y) + cyj;
  const V3<float> X2 = p + d * Gij.t;
  const float d2 = 1.f / fmaxf(X2.z, 0.1f);
  const float u2 = fxj * (d2 * X2.x) + cxj, v2 = fyj * (d2 * X2.y) + cyj;
  valid = X1.z > 0.2f;
  const float f1 = sqrtf((u1 - u0) * (u1 - u0) + (v1 - v0) * (v1 - v0));
  const float f2 = sqrtf((u2 - u0) * (u2 - u0) + (v2 - v0) * (v2 - v0));
  return 0.5f * f1 + 0.5f * f2;
}

}  // namespace dpvo
