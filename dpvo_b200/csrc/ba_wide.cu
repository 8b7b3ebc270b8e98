// fastba, wide windows: Gauss-Newton bundle adjustment when the number of free poses exceeds what the on-chip
// cluster solver of ba.cu holds (N = t1 - t0 > 32) or when the caller asks for the block-sparse form
// (cuda_ba.forward(..., eff_impl=True): the global BA of loop closure, dpvo/dpvo.py:312-326).
//
// Replaces dpvo/fastba/block_e.cu:38-299 (EfficentE: host-built index tables, E_lookup, three atomic kernels per
// product) and the eff_impl branch of ba_cuda.cu:495-563.  Same normal equations, different organisation:
//
//   the pose/depth coupling E is block sparse by construction -- patch k of frame i couples only to frame i and to
//   the frames j it is observed in -- so the Schur complement  S = B - E diag(Q) E^T  splits into one small dense
//   product PER SOURCE FRAME:  with A_i = [E_self ; E_j1 ; E_j2 ; ...] (6(n_i+1) rows, one column per patch of
//   frame i),  E diag(Q) E^T = sum_i A_i diag(Q_i) A_i^T.
//
//   ba_wide_frame_kernel<SYSTEM>   one CTA per source frame.  Its edges are contiguous in the (i, j)-sorted pair
//       grouping the update operator already builds.  Warps walk the pairs: edges are linearised (ba_edge.cuh), the
//       6x6 pose blocks and gradients of a pair are reduced with warp shuffles and added to S / y, the coupling
//       rows go to shared memory (A_i never exists in global memory, no index tables, no host loop).  Then
//       Q_i = 1/(C_i + lambda), and the CTA forms A_i diag(Q_i) A_i^T and A_i (Q_i u_i) from shared memory and
//       subtracts them from S / y (one atomic per matrix entry and frame instead of one per entry, frame AND patch).
//   [dense Cholesky of the 6N x 6N system: library call in the caller, exactly as the reference does]
//   ba_wide_frame_kernel<UPDATE>   same walk (the state has not moved yet), now dZ_i = Q_i (u_i - A_i^T dX) and the
//       depth retraction of the frame's patches (clamps of ba_cuda.cu:218-221).
//   ba_wide_pose_kernel            left retraction of the free poses.
// Float atomics into S make the last bits run-to-run dependent, as in the reference (ba_cuda.cu:339-373).
#include "common.cuh"
#include "ba_edge.cuh"

namespace dpvo {

constexpr int BW_THREADS = 256;
constexpr int BW_WARPS = BW_THREADS / 32;
constexpr int BW_REC = 90;

struct BaWideArgs {
  float* poses; float* patches; const float* intrinsics;
  const float* target; const float* weight; const float* lmbda;
  const int64_t* ii; const int64_t* jj; const int64_t* kk;
  int64_t E; int P; int PPF; int t0; int N;
  const int32_t* p_order; const int32_t* p_start; const int64_t* p_key_i; const int64_t* p_key_j; const int32_t* p_n;
  float* S; float* y;          // [6N, 6N], [6N]
  const float* dX;             // [6N] (update pass)
  int max_blocks;              // coupling blocks (self + observers) that fit the shared-memory budget
  int* status;                 // device flag: 1 = a frame has more observers than max_blocks, 2 = patch id outside its frame's slot range
};

__device__ __forceinline__ int lower_bound_i64(const int64_t* a, int n, int64_t v) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < v) lo = mid + 1; else hi = mid; }
  return lo;
}

template <bool SYSTEM>
__global__ void __launch_bounds__(BW_THREADS)
ba_wide_frame_kernel(const BaWideArgs a) {
  extern __shared__ float bw_smem[];
  const int frame = blockIdx.x;
  const int Gp = *a.p_n;
  const int lo = lower_bound_i64(a.p_key_i, Gp, (int64_t)frame), hi = lower_bound_i64(a.p_key_i, Gp, (int64_t)frame + 1);
  const int np = hi - lo;
  if (np == 0) return;
  if (np + 1 > a.max_blocks) { if (threadIdx.x == 0) atomicMax(a.status, 1); return; }
  const int PPF = a.PPF, nb = np + 1;
  // shared: A[nb][PPF][6] (block 0 = the frame itself), C[PPF], u[PPF], cnt[PPF] (edges seen), blk_pose[nb]
  float* A = bw_smem;
  float* Cs = A + (size_t)nb * PPF * 6;
  float* us = Cs + PPF;
  float* qs = us + PPF;
  int* cnt = reinterpret_cast<int*>(qs + PPF);
  int* blk_pose = cnt + PPF;
  for (int i = threadIdx.x; i < nb * PPF * 6; i += BW_THREADS) A[i] = 0.0f;
  for (int i = threadIdx.x; i < PPF; i += BW_THREADS) { Cs[i] = 0.0f; us[i] = 0.0f; cnt[i] = 0; }
  const int self_pose = frame - a.t0;
  if (threadIdx.x == 0) blk_pose[0] = (self_pose >= 0 && self_pose < a.N) ? self_pose : -1;
  for (int b = threadIdx.x; b < np; b += BW_THREADS) {
    const int jp = (int)(a.p_key_j[lo + b] - a.t0);
    blk_pose[1 + b] = (jp >= 0 && jp < a.N) ? jp : -1;
  }
  __syncthreads();

  const EdgeCam K = {a.intrinsics[0], a.intrinsics[1], a.intrinsics[2], a.intrinsics[3]};
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int N6 = 6 * a.N;
  // ---- pass over the pairs of this frame: one warp per pair
  for (int b = warp; b < np; b += BW_WARPS) {
    const int p = lo + b;
    const int gs = a.p_start[p], ge = a.p_start[p + 1];
    float acc[BW_REC];
    if (SYSTEM) {
#pragma unroll
      for (int k = 0; k < BW_REC; ++k) acc[k] = 0.0f;
    }
    for (int idx = gs + lane; idx < ge; idx += 32) {
      const int64_t e = a.p_order[idx];
      const int64_t kx = a.kk[e];
      const int64_t slot64 = kx - (int64_t)frame * PPF;
      if (slot64 < 0 || slot64 >= PPF) { atomicMax(a.status, 2); continue; }
      const int s = (int)slot64;
      EdgeLin L;
      linearize_edge_at(a.poses, a.patches, a.P, a.target, a.weight, e, a.ii[e], a.jj[e], kx, K, L);
      float c = 0.f, u = 0.f, Ei[6] = {0, 0, 0, 0, 0, 0}, Ej[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float wz = L.w[r] * L.Jz[r];
        c += wz * L.Jz[r];
        u += wz * L.r[r];
#pragma unroll
        for (int k = 0; k < 6; ++k) { Ei[k] -= wz * L.Ji[r][k]; Ej[k] += wz * L.Jj[r][k]; }
        if (SYSTEM) {
          const float w = L.w[r];
          int o = 0;
#pragma unroll
          for (int x = 0; x < 6; ++x)
#pragma unroll
            for (int yy = x; yy < 6; ++yy) acc[o++] += w * L.Ji[r][x] * L.Ji[r][yy];
#pragma unroll
          for (int x = 0; x < 6; ++x)
#pragma unroll
            for (int yy = 0; yy < 6; ++yy) acc[o++] += -w * L.Ji[r][x] * L.Jj[r][yy];
#pragma unroll
          for (int x = 0; x < 6; ++x)
#pragma unroll
            for (int yy = x; yy < 6; ++yy) acc[o++] += w * L.Jj[r][x] * L.Jj[r][yy];
#pragma unroll
          for (int x = 0; x < 6; ++x) acc[o++] += -w * L.r[r] * L.Ji[r][x];
#pragma unroll
          for (int x = 0; x < 6; ++x) acc[o++] += w * L.r[r] * L.Jj[r][x];
        }
      }
      atomicAdd(&Cs[s], c);
      atomicAdd(&us[s], u);
      atomicAdd(&cnt[s], 1);
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        atomicAdd(&A[(size_t)s * 6 + k], Ei[k]);                              // block 0: the source frame
        atomicAdd(&A[((size_t)(1 + b) * PPF + s) * 6 + k], Ej[k]);            // block 1 + b: the observing frame
      }
    }
    if (SYSTEM) {
      // pose blocks of the pair (i, j): reduced over the warp, added to B (inside S) and to the gradient
      const int pi = blk_pose[0], pj = blk_pose[1 + b];
      int o = 0;
#pragma unroll
      for (int x = 0; x < 6; ++x)
#pragma unroll
        for (int yy = x; yy < 6; ++yy, ++o) {
          const float v = warp_sum(acc[o]);
          if (lane == 0 && pi >= 0) {
            atomicAdd(&a.S[(size_t)(6 * pi + x) * N6 + 6 * pi + yy], v);
            if (yy != x) atomicAdd(&a.S[(size_t)(6 * pi + yy) * N6 + 6 * pi + x], v);
          }
        }
#pragma unroll
      for (int x = 0; x < 6; ++x)
#pragma unroll
        for (int yy = 0; yy < 6; ++yy, ++o) {
          const float v = warp_sum(acc[o]);
          if (lane == 0 && pi >= 0 && pj >= 0) {
            atomicAdd(&a.S[(size_t)(6 * pi + x) * N6 + 6 * pj + yy], v);
            atomicAdd(&a.S[(size_t)(6 * pj + yy) * N6 + 6 * pi + x], v);
          }
        }
#pragma unroll
      for (int x = 0; x < 6; ++x)
#pragma unroll
        for (int yy = x; yy < 6; ++yy, ++o) {
          const float v = warp_sum(acc[o]);
          if (lane == 0 && pj >= 0) {
            atomicAdd(&a.S[(size_t)(6 * pj + x) * N6 + 6 * pj + yy], v);
            if (yy != x) atomicAdd(&a.S[(size_t)(6 * pj + yy) * N6 + 6 * pj + x], v);
          }
        }
#pragma unroll
      for (int x = 0; x < 6; ++x, ++o) { const float v = warp_sum(acc[o]); if (lane == 0 && pi >= 0) atomicAdd(&a.y[6 * pi + x], v); }
#pragma unroll
      for (int x = 0; x < 6; ++x, ++o) { const float v = warp_sum(acc[o]); if (lane == 0 && pj >= 0) atomicAdd(&a.y[6 * pj + x], v); }
    }
  }
  __syncthreads();
  const float lm = a.lmbda[0];
  for (int s = threadIdx.x; s < PPF; s += BW_THREADS) qs[s] = 1.0f / (Cs[s] + lm);
  __syncthreads();

  if (SYSTEM) {
    // ---- S -= A diag(Q) A^T,  y -= A (Q u): every thread owns entries (block a, row ka) x (block b, row kb)
    const int R = nb * 6;
    for (int ent = threadIdx.x; ent < R * R; ent += BW_THREADS) {
      const int ra = ent / R, rb = ent - ra * R;
      const int ba = ra / 6, ka = ra - ba * 6, bb = rb / 6, kb = rb - bb * 6;
      const int pa = blk_pose[ba], pb = blk_pose[bb];
      if (pa < 0 || pb < 0) continue;
      const float* Aa = A + (size_t)ba * PPF * 6 + ka;
      const float* Ab = A + (size_t)bb * PPF * 6 + kb;
      float g = 0.0f;
      for (int s = 0; s < PPF; ++s) g += qs[s] * Aa[s * 6] * Ab[s * 6];
      if (g != 0.0f) atomicAdd(&a.S[(size_t)(6 * pa + ka) * N6 + 6 * pb + kb], -g);
    }
    for (int ra = threadIdx.x; ra < R; ra += BW_THREADS) {
      const int ba = ra / 6, ka = ra - ba * 6;
      const int pa = blk_pose[ba];
      if (pa < 0) continue;
      const float* Aa = A + (size_t)ba * PPF * 6 + ka;
      float g = 0.0f;
      for (int s = 0; s < PPF; ++s) g += qs[s] * us[s] * Aa[s * 6];
      if (g != 0.0f) atomicAdd(&a.y[6 * pa + ka], -g);
    }
  } else {
    // ---- dZ = Q (u - A^T dX), depth retraction of this frame's patches (ba_cuda.cu:208-229)
    const int PP = a.P * a.P;
    for (int s = threadIdx.x; s < PPF; s += BW_THREADS) {
      if (cnt[s] == 0) continue;
      float dot = 0.0f;
      for (int b = 0; b < nb; ++b) {
        const int pb = blk_pose[b];
        if (pb < 0) continue;
        const float* Ab = A + ((size_t)b * PPF + s) * 6;
#pragma unroll
        for (int k = 0; k < 6; ++k) dot += Ab[k] * a.dX[6 * pb + k];
      }
      const float dz = qs[s] * (us[s] - dot);
      float* pk = a.patches + ((int64_t)frame * PPF + s) * 3 * PP + 2 * PP;
      float d = pk[0] + dz;
      d = (d > 20.0f) ? 1.0f : d;
      d = fmaxf(d, 1e-4f);
      for (int i = 0; i < PP; ++i) pk[i] = d;
    }
  }
}

// S += I o (1e-4 S + 1)   (ba_cuda.cu:546, 560)
__global__ void ba_wide_damp_kernel(float* S, int N6) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N6) { float& d = S[(size_t)i * N6 + i]; d += 1e-4f * d + 1.0f; }
}

__global__ void ba_wide_pose_kernel(float* poses, const float* dX, int t0, int N) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n < N) retract_pose(poses + (int64_t)(t0 + n) * 7, dX + 6 * n);
}

static size_t bw_smem_bytes(int blocks, int PPF) { return ((size_t)blocks * PPF * 6 + 3 * PPF) * 4 + ((size_t)PPF + blocks) * 4 + 64; }

}  // namespace dpvo

using namespace dpvo;

static int bw_fill(BaWideArgs& a, float* poses, float* patches, const float* intrinsics, const float* target, const float* weight,
                   const float* lmbda, const int64_t* ii, const int64_t* jj, const int64_t* kk, int64_t E, int P, int PPF, int t0, int t1,
                   const int32_t* p_order, const int32_t* p_start, const int64_t* p_key_i, const int64_t* p_key_j, const int32_t* p_n,
                   int* status) {
  a.poses = poses; a.patches = patches; a.intrinsics = intrinsics; a.target = target; a.weight = weight; a.lmbda = lmbda;
  a.ii = ii; a.jj = jj; a.kk = kk; a.E = E; a.P = P; a.PPF = PPF; a.t0 = t0; a.N = t1 - t0;
  a.p_order = p_order; a.p_start = p_start; a.p_key_i = p_key_i; a.p_key_j = p_key_j; a.p_n = p_n;
  a.S = nullptr; a.y = nullptr; a.dX = nullptr; a.status = status;
  // coupling blocks that fit: leave room below the 227 KB opt-in limit
  const size_t budget = 200 * 1024;
  int blocks = 2;
  while (bw_smem_bytes(blocks + 1, PPF) <= budget) ++blocks;
  a.max_blocks = blocks;
  return DPVO_OK;
}

// Assemble S = B - E Q E^T + damping and y = v - E Q u for poses [t0, t1).  `status` is a device int the caller zeroes and
// may read back after the stream has drained (non-zero: the graph does not fit this path's assumptions).
extern "C" int dpvo_ba_wide_system(float* poses, float* patches, const float* intrinsics, const float* target, const float* weight,
                                   const float* lmbda, const int64_t* ii, const int64_t* jj, const int64_t* kk, int64_t E, int P, int PPF,
                                   int t0, int t1, const int32_t* p_order, const int32_t* p_start, const int64_t* p_key_i,
                                   const int64_t* p_key_j, const int32_t* p_n, float* S, float* y, int* status, void* stream) {
  DPVO_REQUIRE(E >= 0 && P > 0 && PPF > 0 && t1 > t0 && t0 >= 0, "ba_wide_system: bad sizes");
  DPVO_REQUIRE(poses && patches && intrinsics && target && weight && lmbda && ii && jj && kk && p_order && p_start && p_key_i &&
               p_key_j && p_n && S && y && status, "ba_wide_system: null pointer");
  DPVO_REQUIRE(PPF <= 1024, "ba_wide_system: patches per frame %d > 1024", PPF);
  cudaStream_t st = (cudaStream_t)stream;
  BaWideArgs a;
  bw_fill(a, poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, E, P, PPF, t0, t1, p_order, p_start, p_key_i, p_key_j, p_n, status);
  a.S = S; a.y = y;
  const int N6 = 6 * a.N;
  int rc = check_cuda(cudaMemsetAsync(S, 0, (size_t)N6 * N6 * 4, st), "ba_wide_system: memset");
  if (rc) return rc;
  rc = check_cuda(cudaMemsetAsync(y, 0, (size_t)N6 * 4, st), "ba_wide_system: memset");
  if (rc) return rc;
  if (E > 0) {     // source frames are 0 .. t1-1
    rc = launch("ba_wide_frame_kernel<system>", ba_wide_frame_kernel<true>, (unsigned)t1, BW_THREADS, bw_smem_bytes(a.max_blocks, PPF), st, a);
    if (rc) return rc;
  }
  return launch("ba_wide_damp_kernel", ba_wide_damp_kernel, (N6 + 127) / 128, 128, 0, st, S, N6);
}

// Apply a solved pose step dX [6 (t1 - t0)]: depth back-substitution + retraction, then pose retraction.
extern "C" int dpvo_ba_wide_update(float* poses, float* patches, const float* intrinsics, const float* target, const float* weight,
                                   const float* lmbda, const int64_t* ii, const int64_t* jj, const int64_t* kk, int64_t E, int P, int PPF,
                                   int t0, int t1, const int32_t* p_order, const int32_t* p_start, const int64_t* p_key_i,
                                   const int64_t* p_key_j, const int32_t* p_n, const float* dX, int* status, void* stream) {
  DPVO_REQUIRE(E >= 0 && P > 0 && PPF > 0 && t1 > t0 && t0 >= 0, "ba_wide_update: bad sizes");
  DPVO_REQUIRE(poses && patches && intrinsics && target && weight && lmbda && ii && jj && kk && p_order && p_start && p_key_i &&
               p_key_j && p_n && dX && status, "ba_wide_update: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  BaWideArgs a;
  bw_fill(a, poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, E, P, PPF, t0, t1, p_order, p_start, p_key_i, p_key_j, p_n, status);
  a.dX = dX;
  if (E > 0) {
    const int rc = launch("ba_wide_frame_kernel<update>", ba_wide_frame_kernel<false>, (unsigned)t1, BW_THREADS, bw_smem_bytes(a.max_blocks, PPF), st, a);
    if (rc) return rc;
  }
  return launch("ba_wide_pose_kernel", ba_wide_pose_kernel, (a.N + 63) / 64, 64, 0, st, poses, dX, t0, a.N);
}

// ---- cuda_ba.solve_system: pose-graph normal equations (ba.cpp:120-167) ---------------------------------------------
namespace dpvo {
// one thread per (residual, row a of the 14-column stacked Jacobian [J_i | J_j], column c): adds
// sum_k J[k][a] J[k][c] to A and, for c == 0, -sum_k J[k][a] res[k] to b
__global__ void posegraph_kernel(const float* __restrict__ Ji, const float* __restrict__ Jj, const int64_t* __restrict__ ii,
                                 const int64_t* __restrict__ jj, const float* __restrict__ res, int64_t r, int64_t n,
                                 double* __restrict__ A, double* __restrict__ b) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= r * 196) return;
  const int64_t x = t / 196;
  const int ac = (int)(t - x * 196), a = ac / 14, c = ac - a * 14;
  const float* Ja = (a < 7 ? Ji : Jj) + x * 49 + (a % 7);
  const float* Jc = (c < 7 ? Ji : Jj) + x * 49 + (c % 7);
  const int64_t row = (a < 7 ? ii[x] : jj[x]) * 7 + (a % 7);
  const int64_t col = (c < 7 ? ii[x] : jj[x]) * 7 + (c % 7);
  double acc = 0.0, g = 0.0;
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    acc += (double)Ja[k * 7] * (double)Jc[k * 7];
    g += (double)Ja[k * 7] * (double)res[x * 7 + k];
  }
  atomicAdd(&A[row * (n * 7) + col], acc);
  if (c == 0) atomicAdd(&b[row], -g);
}
__global__ void posegraph_damp_kernel(double* A, int64_t n7, double ep, double lm) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n7) { double& d = A[i * n7 + i]; d += d * lm + ep; }
}
}  // namespace dpvo

extern "C" int dpvo_posegraph_system(const float* J_i, const float* J_j, const int64_t* ii, const int64_t* jj, const float* res,
                                     int64_t r, int64_t n, double ep, double lm, double* A, double* b, void* stream) {
  DPVO_REQUIRE(r >= 0 && n > 0, "posegraph_system: bad sizes");
  DPVO_REQUIRE(A && b && (r == 0 || (J_i && J_j && ii && jj && res)), "posegraph_system: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n7 = n * 7;
  int rc = check_cuda(cudaMemsetAsync(A, 0, (size_t)n7 * n7 * 8, st), "posegraph_system: memset");
  if (rc) return rc;
  rc = check_cuda(cudaMemsetAsync(b, 0, (size_t)n7 * 8, st), "posegraph_system: memset");
  if (rc) return rc;
  if (r > 0) {
    const int64_t total = r * 196;
    rc = launch("posegraph_kernel", posegraph_kernel, (unsigned)((total + 255) / 256), 256, 0, st, J_i, J_j, ii, jj, res, r, n, A, b);
    if (rc) return rc;
  }
  return launch("posegraph_damp_kernel", posegraph_damp_kernel, (unsigned)((n7 + 127) / 128), 128, 0, st, A, n7, ep, lm);
}
