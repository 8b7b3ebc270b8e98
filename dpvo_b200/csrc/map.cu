// The map of DPVO.update (dpvo/dpvo.py:358-360): the world point of every patch centre of frames [0, n),
//   points = pops.point_cloud(SE3(poses), patches[:, :m], intrinsics, ix[:m])[..., 1, 1, :3] / [..., 1, 1, 3:]
// for B >= 1 streams of F frame slots each in one launch: grid (patch blocks, B), one thread per patch.
// The arithmetic is point_cloud's, operation for operation:
//   (xn, yn, 1, d) = ((x - cx) / fx, (y - cy) / fy, 1, d)    iproj, one rounding per torch op
//   Y = se3_inv(pose), stored and loaded again               SE3.inv() is a kernel of its own: its output is fp32
//                                                            memory that the act4 kernel loads (and renormalises)
//   P = act4(Y, (xn, yn, 1, d))                              lie_ops.cuh's OP_ACT4, the lietorch kernels' operator
//   point = P.xyz / P.w
#include "common.cuh"
#include "lie_ops.cuh"

namespace dpvo {

constexpr int MAP_THREADS = 128;
constexpr int MAP_MAX_STREAMS = 64;

// pops.point_cloud's two lietorch operators, each the very operator body of the lietorch kernels (lie_ops.cuh's se3_op)
// in a function of its own: SE3.inv() and act4 are separate kernels there, whose operands are memory, so nothing may be
// folded or contracted across them here either
__device__ __noinline__ void se3_inv_op(const float* X, float* Y) { se3_op<float, OP_INV>(LieArgs{X, nullptr, nullptr, Y, nullptr, 1}, 0); }
__device__ __noinline__ void se3_act4_op(const float* X, const float* p, float* q) {
  se3_op<float, OP_ACT4>(LieArgs{X, p, nullptr, q, nullptr, 1}, 0);
}

struct MapParams {
  const float* poses;              // [B F, 7]
  const float* patches;            // [B F M, 3, 3, 3]
  const float* intr;               // [B F, 4]
  float* points;                   // [B F M, 3]
  int64_t F;
  int M;
  int64_t n[MAP_MAX_STREAMS];      // frames of each stream
};

__global__ void __launch_bounds__(MAP_THREADS) point_cloud_kernel(const __grid_constant__ MapParams p) {
  using namespace lie;
  const int b = blockIdx.y;
  const int64_t k = (int64_t)blockIdx.x * MAP_THREADS + threadIdx.x;
  if (k >= p.n[b] * p.M) return;
  const int64_t f = (int64_t)b * p.F + k / p.M;                       // the patch's frame, global
  const int64_t row = (int64_t)b * p.F * p.M + k;
  const float* q = p.patches + row * 27;
  const float* K = p.intr + f * 4;
  const float x = q[4], y = q[9 + 4], d = q[18 + 4];                  // channels x, y, d of the centre pixel [1][1]
  const float X[4] = {__fdiv_rn(__fsub_rn(x, K[2]), K[0]), __fdiv_rn(__fsub_rn(y, K[3]), K[1]), 1.0f, d};
  float Y[7], P[4];
  se3_inv_op(p.poses + f * 7, Y);
  se3_act4_op(Y, X, P);
  float* out = p.points + row * 3;
  out[0] = __fdiv_rn(P[0], P[3]);
  out[1] = __fdiv_rn(P[1], P[3]);
  out[2] = __fdiv_rn(P[2], P[3]);
}

}  // namespace dpvo

using namespace dpvo;

extern "C" int dpvo_point_cloud(const float* poses, const float* patches, const float* intrinsics, int64_t F, int M, int B,
                                const int64_t* n, float* points, void* stream) {
  DPVO_REQUIRE(B >= 1 && B <= MAP_MAX_STREAMS, "point_cloud: B=%d streams, 1 to %d supported", B, MAP_MAX_STREAMS);
  DPVO_REQUIRE(F >= 1 && M >= 1, "point_cloud: bad sizes (frames=%lld, M=%d)", (long long)F, M);
  DPVO_REQUIRE(poses && patches && intrinsics && n && points, "point_cloud: null pointer");
  MapParams p{};
  p.poses = poses; p.patches = patches; p.intr = intrinsics; p.points = points; p.F = F; p.M = M;
  int64_t most = 0;
  for (int b = 0; b < B; ++b) {
    DPVO_REQUIRE(n[b] >= 0 && n[b] <= F, "point_cloud: stream %d has n=%lld frames, outside [0, %lld]", b, (long long)n[b],
                 (long long)F);
    p.n[b] = n[b];
    most = std::max(most, n[b] * M);
  }
  if (most == 0) return DPVO_OK;
  return launch("point_cloud_kernel", point_cloud_kernel, dim3((unsigned)((most + MAP_THREADS - 1) / MAP_THREADS), (unsigned)B), MAP_THREADS, 0,
                (cudaStream_t)stream, p);
}
