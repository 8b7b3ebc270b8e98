// fastba: in-place Gauss-Newton bundle adjustment over the patch graph, sm_90a.
//
// Replaces dpvo/fastba/ba_cuda.cu:232-376 (per-edge kernel with ~340 global float atomics per
// edge), the ~30 ATen launches per iteration around it (:484-563, dense E, matmuls, cuSOLVER
// potrf/potrs on a 60x60 system) and the retraction kernels (:178-229) with TWO launches per
// Gauss-Newton iteration and no float atomics:
//
//   ba_reduce_kernel  one warp per work item, warp-shuffle reductions only
//       * pair items  (edges sharing (i,j), from the ij grouping): sum of the 6x6 pose blocks
//                     JiJi^T, JiJj^T, JjJj^T and the pose gradients -> one 90-float record
//       * patch items (edges sharing a patch, from the kk grouping): C_k, u_k and the dense row
//                     E_k (6N) of the pose/depth coupling -> global
//   ba_solve_kernel   one 8-CTA thread-block cluster
//       * each CTA forms its share of the Schur products  sum_k Q_k E_k E_k^T, sum_k Q_k u_k E_k
//       * partials are reduced over distributed shared memory in a fixed order
//       * CTA 0 assembles B from the pair records, applies the damping, Cholesky-factors and
//         solves the 6N x 6N system in shared memory, retracts the poses
//       * all CTAs back-substitute the depth updates and retract the patches
//   batched (ba_reduce_batched_kernel, ba_solve_batched_kernel): B streams' independent windows in the same two
//       launches, each stream on its slice of the shared groupings and scratch, one 8-CTA cluster per stream
// Results are bit-reproducible run to run (the reference's are not: unordered atomics).
#include "common.cuh"
#include "ba_edge.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace dpvo {

constexpr int BA_MAX_N = 32;          // free poses held on chip
constexpr int BA_REC = 90;            // floats per pair record
constexpr int BA_CLUSTER = 8;
constexpr int BA_SOLVE_THREADS = 512;

struct BaArgs {
  float* poses; float* patches; const float* intrinsics;
  const float* target; const float* weight; const float* lmbda;
  const int64_t* ii; const int64_t* jj; const int64_t* kk;
  int64_t E; int P; int t0; int N;     // N = t1 - t0 free poses
  // kk grouping (patches)
  const int32_t* k_order; const int32_t* k_start; const int64_t* k_key; const int32_t* k_n;
  // ij grouping (pose pairs)
  const int32_t* p_order; const int32_t* p_start; const int64_t* p_key_i; const int64_t* p_key_j;
  const int32_t* p_n;
  // scratch
  float* Ed;      // [M][6N]
  float* Qk;      // [M]   1/(C+lambda)
  float* uk;      // [M]
  float* rec;     // [Gp][90]
  float* dX;      // [6N]
  float* part;    // [n_part][6N(6N+3)/2] per-CTA partial reduced systems (fast path), NULL = the solve cluster forms S itself
  int n_part;
  long long* dbg; // optional phase timestamps of the solve kernel (cluster rank 0), NULL = off
};

// per-edge linearisation (own SE3 operators of lie.cuh, see ba_edge.cuh)
__device__ __forceinline__ void linearize_edge(const BaArgs& a, int64_t e, float fx, float fy, float cx, float cy, EdgeLin& L) {
  const EdgeCam K = {fx, fy, cx, cy};
  linearize_edge_at(a.poses, a.patches, a.P, a.target, a.weight, e, a.ii[e], a.jj[e], a.kk[e], K, L);
}

// ==========================================================================================
// kernel A: per-pair and per-patch reductions
// ==========================================================================================
constexpr int BA_RED_WARPS = 4;
constexpr int BA_FAST_WARPS = 16;     // fast path: warps per CTA, each with a private copy of the reduced system
constexpr int BA_FAST_MAX_N = 12;     // 16 packed copies (upper triangle + gradient, 6N(6N+3)/2 floats) fit in shared memory up to here
__host__ __device__ constexpr int ba_packed_entries(int N6) { return N6 * (N6 + 1) / 2 + N6; }
// packed upper triangle, row-major: entry (r, c), r <= c
__device__ __forceinline__ int ba_tri(int N6, int r, int c) { return r * N6 - (r * (r - 1)) / 2 + (c - r); }

// SYSTEM = false: pair records and patch rows go to global memory, the solve cluster forms the reduced system.
// SYSTEM = true (0 < N <= BA_FAST_MAX_N, the sliding-window case): every warp also applies its items to a private
// copy of the reduced pose system  S = B - E Q E^T,  y = v - E Q u  (upper triangle; row 6N = y) in shared memory --
// the Schur rank-1 update of a patch right after its row E_k is formed, the 6x6 pose blocks of a pair right after its
// record is summed -- so that this work runs on every SM instead of inside the 8-CTA solve cluster.  Items are dealt
// to warps statically, a warp applies its items in order, the copies of a CTA are added in warp order and the CTAs'
// partial systems are summed in CTA order by the solve kernel: still no float atomics, still bit-reproducible.
// A copy is stored packed (upper triangle row-major, then the gradient): 7.4 KB for 10 free poses.
// Entries [LO, HI) of the 90-float record of a pair: the lanes sum their edges in index order, one warp reduction per
// entry, lane (k mod 32) keeps entry k in mine[k / 32].  Every entry's sum is independent of the others, so the record
// comes out bit-identical whether it is formed in one pass or in two (which recomputes each edge's linearisation but
// holds only half of the accumulators in registers).
template <int LO, int HI>
__device__ __forceinline__ void ba_pair_record(const BaArgs& a, int gs, int ge, int lane, float fx, float fy, float cx, float cy,
                                               float (&mine)[3]) {
  float acc[HI - LO];
#pragma unroll
  for (int k = 0; k < HI - LO; ++k) acc[k] = 0.0f;
  for (int idx = gs + lane; idx < ge; idx += 32) {
    EdgeLin L;
    linearize_edge(a, a.p_order[idx], fx, fy, cx, cy, L);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float w = L.w[r];
      int o = 0;
#define BA_ACC(v) do { if (o >= LO && o < HI) acc[o - LO] += (v); ++o; } while (0)
#pragma unroll
      for (int x = 0; x < 6; ++x)
#pragma unroll
        for (int y = x; y < 6; ++y) BA_ACC(w * L.Ji[r][x] * L.Ji[r][y]);
#pragma unroll
      for (int x = 0; x < 6; ++x)
#pragma unroll
        for (int y = 0; y < 6; ++y) BA_ACC(-w * L.Ji[r][x] * L.Jj[r][y]);
#pragma unroll
      for (int x = 0; x < 6; ++x)
#pragma unroll
        for (int y = x; y < 6; ++y) BA_ACC(w * L.Jj[r][x] * L.Jj[r][y]);
#pragma unroll
      for (int x = 0; x < 6; ++x) BA_ACC(-w * L.r[r] * L.Ji[r][x]);
#pragma unroll
      for (int x = 0; x < 6; ++x) BA_ACC(w * L.r[r] * L.Jj[r][x]);
#undef BA_ACC
    }
  }
#pragma unroll
  for (int k = LO; k < HI; ++k) {
    const float s = warp_sum(acc[k - LO]);
    if ((k & 31) == lane) mine[k >> 5] = s;
  }
}

// Gk / Gp: the patch and pair groups this launch (batched: this stream) reduces; blockIdx.x deals the items.
// SPLIT_PAIRS: form the pair records in two passes (ba_pair_record) -- the batched fast path, which is held to 128
// registers by its 512-thread CTAs, then needs no local memory.
template <bool SYSTEM, bool SPLIT_PAIRS = false>
__device__ __forceinline__ void ba_reduce_body(const BaArgs& a, const int Gk, const int Gp) {
  constexpr int WARPS = SYSTEM ? BA_FAST_WARPS : BA_RED_WARPS;
  extern __shared__ __align__(16) float red_smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float* ek = red_smem + wib * (6 * BA_MAX_N);
  const int n_ent = ba_packed_entries(6 * a.N);
  float* recw = red_smem + WARPS * (6 * BA_MAX_N) + wib * 96;                         // SYSTEM: this warp's pair record
  float* Sw = red_smem + WARPS * (6 * BA_MAX_N + 96) + (size_t)wib * n_ent;           // SYSTEM: this warp's copy, [6N+1][6N]
  if constexpr (SYSTEM) {
    for (int i = lane; i < n_ent; i += 32) Sw[i] = 0.0f;
    __syncwarp();
  }
  const float fx = a.intrinsics[0], fy = a.intrinsics[1], cx = a.intrinsics[2], cy = a.intrinsics[3];
  const float lm = a.lmbda[0];
  const int N = a.N, N6 = 6 * a.N;
  const int nwarps = gridDim.x * WARPS;

  for (int item = blockIdx.x * WARPS + wib; item < Gk + Gp; item += nwarps) {
    if (item < Gk) {
      // ------------------------------------------------------------ patch item
      const int g = item;
      const int gs = a.k_start[g], ge = a.k_start[g + 1];
      for (int i = lane; i < N6; i += 32) ek[i] = 0.0f;
      __syncwarp();
      float Csum = 0.0f, usum = 0.0f;
      for (int base = gs; base < ge; base += 32) {
        const bool act = base + lane < ge;
        float c = 0.f, u = 0.f, Ei[6] = {0, 0, 0, 0, 0, 0}, Ej[6] = {0, 0, 0, 0, 0, 0};
        int ix = -1, jx = -1;
        if (act) {
          const int64_t e = a.k_order[base + lane];
          EdgeLin L;
          linearize_edge(a, e, fx, fy, cx, cy, L);
          ix = (int)(a.ii[e] - a.t0); jx = (int)(a.jj[e] - a.t0);
          if (ix < 0 || ix >= N) ix = -1;
          if (jx < 0 || jx >= N) jx = -1;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            c += L.w[r] * L.Jz[r] * L.Jz[r];
            u += L.w[r] * L.r[r] * L.Jz[r];
#pragma unroll
            for (int k = 0; k < 6; ++k) {
              Ei[k] += -L.w[r] * L.Jz[r] * L.Ji[r][k];
              Ej[k] += L.w[r] * L.Jz[r] * L.Jj[r][k];
            }
          }
        }
        Csum += warp_sum(c);
        usum += warp_sum(u);
        if (N > 0) {
          // source-pose block: all edges of a patch normally share ix -> one shuffle reduction
          const int ix0 = __shfl_sync(0xffffffffu, ix, 0);
          const bool same_i = __all_sync(0xffffffffu, !act || ix == ix0);
          const unsigned dup = __match_any_sync(0xffffffffu, act ? jx : -2 - lane);
          const bool uniq_j = __all_sync(0xffffffffu, !act || jx < 0 || __popc(dup) == 1);
          if (same_i) {
#pragma unroll
            for (int k = 0; k < 6; ++k) {
              const float s = warp_sum(Ei[k]);
              if (lane == 0 && ix0 >= 0) ek[6 * ix0 + k] += s;
            }
          }
          __syncwarp();
          if (uniq_j) {
            if (act && jx >= 0) {
#pragma unroll
              for (int k = 0; k < 6; ++k) ek[6 * jx + k] += Ej[k];
            }
          }
          __syncwarp();
          if (!same_i || !uniq_j) {
            // general graphs: ordered, lane-serial accumulation (still deterministic)
            for (int l = 0; l < 32; ++l) {
              if (lane == l && act) {
                if (!same_i && ix >= 0) for (int k = 0; k < 6; ++k) ek[6 * ix + k] += Ei[k];
                if (!uniq_j && jx >= 0) for (int k = 0; k < 6; ++k) ek[6 * jx + k] += Ej[k];
              }
              __syncwarp();
            }
          }
        }
      }
      __syncwarp();
      for (int i = lane; i < N6; i += 32) a.Ed[(int64_t)g * N6 + i] = ek[i];
      const float qk = 1.0f / (Csum + lm);
      if (lane == 0) { a.Qk[g] = qk; a.uk[g] = usum; }
      if constexpr (SYSTEM) {
        // S -= Q_k E_k E_k^T (upper triangle), y -= Q_k u_k E_k: lanes stride the columns of a row; rows are independent
        // read-modify-writes of disjoint addresses, unrolled so that their shared-memory latencies overlap.  A patch that
        // touches no free pose (all of a long video but its last window) has a zero row and nothing to add.
        __syncwarp();
        bool nz = false;
        for (int c = lane; c < N6; c += 32) nz |= ek[c] != 0.0f;
        if (__any_sync(0xffffffffu, nz)) {
        int base = 0;
#pragma unroll 4
        for (int r = 0; r < N6; ++r) {
          const float er = qk * ek[r];
          float* srow = Sw + base - r;                          // srow[c] = entry (r, c)
          for (int c = r + lane; c < N6; c += 32) srow[c] -= er * ek[c];
          base += N6 - r;
        }
        for (int c = lane; c < N6; c += 32) Sw[base + c] -= qk * usum * ek[c];
        }
      }
      __syncwarp();
    } else {
      // ------------------------------------------------------------ pair item
      const int p = item - Gk;
      const int gs = a.p_start[p], ge = a.p_start[p + 1];
      float mine[3] = {0.f, 0.f, 0.f};
      if constexpr (SPLIT_PAIRS) {
        ba_pair_record<0, BA_REC / 2>(a, gs, ge, lane, fx, fy, cx, cy, mine);
        ba_pair_record<BA_REC / 2, BA_REC>(a, gs, ge, lane, fx, fy, cx, cy, mine);
      } else {                                          // one pass: the single-window launches
        float acc[BA_REC];
#pragma unroll
        for (int k = 0; k < BA_REC; ++k) acc[k] = 0.0f;
        for (int idx = gs + lane; idx < ge; idx += 32) {
          EdgeLin L;
          linearize_edge(a, a.p_order[idx], fx, fy, cx, cy, L);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const float w = L.w[r];
            int o = 0;
#pragma unroll
            for (int x = 0; x < 6; ++x)
#pragma unroll
              for (int y = x; y < 6; ++y) acc[o++] += w * L.Ji[r][x] * L.Ji[r][y];
#pragma unroll
            for (int x = 0; x < 6; ++x)
#pragma unroll
              for (int y = 0; y < 6; ++y) acc[o++] += -w * L.Ji[r][x] * L.Jj[r][y];
#pragma unroll
            for (int x = 0; x < 6; ++x)
#pragma unroll
              for (int y = x; y < 6; ++y) acc[o++] += w * L.Jj[r][x] * L.Jj[r][y];
#pragma unroll
            for (int x = 0; x < 6; ++x) acc[o++] += -w * L.r[r] * L.Ji[r][x];
#pragma unroll
            for (int x = 0; x < 6; ++x) acc[o++] += w * L.r[r] * L.Jj[r][x];
          }
        }
#pragma unroll
        for (int k = 0; k < BA_REC; ++k) {
          const float s = warp_sum(acc[k]);
          if ((k & 31) == lane) mine[k >> 5] = s;
        }
      }
      if constexpr (!SYSTEM) {
        float* rp = a.rec + (int64_t)p * BA_REC;
        rp[lane] = mine[0];
        rp[32 + lane] = mine[1];
        if (64 + lane < BA_REC) rp[64 + lane] = mine[2];
      } else {
        // the record goes straight into this warp's system: every entry of S is owned by one (virtual) thread id of
        // the 63 below for the whole record, as in the solve kernel's assembly (diagonal blocks: id (x,y) serves the
        // source- and the target-pose block; off-diagonal blocks are stored for the ordered pose pair)
        recw[lane] = mine[0];
        recw[32 + lane] = mine[1];
        if (64 + lane < BA_REC) recw[64 + lane] = mine[2];
        __syncwarp();
        const long long fi = a.p_key_i[p] - a.t0, fj = a.p_key_j[p] - a.t0;
        const int bi = (fi >= 0 && fi < N) ? (int)fi : -1, bj = (fj >= 0 && fj < N) ? (int)fj : -1;
        for (int id = lane; id < 63; id += 32) {
          const float* rc = recw;
          if (id < 21) {
            int x = 0, rem = id;
            while (rem >= 6 - x) { rem -= 6 - x; ++x; }
            const int y = x + rem;
            if (bi >= 0) {
              float v = rc[id];
              if (bi == bj) v += rc[57 + id] + rc[21 + x * 6 + y] + rc[21 + y * 6 + x];   // self edge i -> i
              Sw[ba_tri(N6, 6 * bi + x, 6 * bi + y)] += v;
            }
            if (bj >= 0 && bi != bj) Sw[ba_tri(N6, 6 * bj + x, 6 * bj + y)] += rc[57 + id];
          } else if (id < 57) {
            const int e = id - 21, x = e / 6, y = e - 6 * x;
            if (bi >= 0 && bj >= 0 && bi != bj) {
              if (bi < bj) Sw[ba_tri(N6, 6 * bi + x, 6 * bj + y)] += rc[21 + x * 6 + y];
              else Sw[ba_tri(N6, 6 * bj + x, 6 * bi + y)] += rc[21 + y * 6 + x];
            }
          } else {
            const int c = id - 57;
            if (bi >= 0) Sw[N6 * (N6 + 1) / 2 + 6 * bi + c] += rc[78 + c] + ((bi == bj) ? rc[84 + c] : 0.0f);
            if (bj >= 0 && bi != bj) Sw[N6 * (N6 + 1) / 2 + 6 * bj + c] += rc[84 + c];
          }
        }
        __syncwarp();
      }
    }
  }
  if constexpr (SYSTEM) {
    // the CTA's partial system: copies added in warp order, one entry per thread
    __syncthreads();
    const float* S0 = red_smem + WARPS * (6 * BA_MAX_N + 96);
    float* out = a.part + (int64_t)blockIdx.x * n_ent;
    for (int i = threadIdx.x; i < n_ent; i += WARPS * 32) {
      float v = S0[i];
#pragma unroll
      for (int w = 1; w < WARPS; ++w) v += S0[(size_t)w * n_ent + i];
      out[i] = v;
    }
  }
}

template <bool SYSTEM>
__global__ void __launch_bounds__((SYSTEM ? BA_FAST_WARPS : BA_RED_WARPS) * 32)
ba_reduce_kernel(const BaArgs a) {
  ba_reduce_body<SYSTEM>(a, *a.k_n, (a.N > 0) ? *a.p_n : 0);
}

// ==========================================================================================
// kernel B: Schur complement, solve, retraction -- one thread-block cluster
// ==========================================================================================
constexpr int BA_LD = 6 * BA_MAX_N + 1;       // leading dimension (odd: conflict-free columns); row N6 = rhs
constexpr int BA_REC_CHUNK = 64;              // pair records staged per round
constexpr int BA_ELD = 6 * BA_MAX_N + 4;      // row pitch of the staged E rows [E_k | u_k | 0..]: a multiple of 4, rows load as float4
constexpr int BA_ECH = 32;                    // patches per Schur chunk

struct SolveSmem {
  float S[BA_LD][BA_LD];                      // upper triangle while accumulating, lower triangle for the factor
  float dx[6 * BA_MAX_N];
  float inv_diag[6 * BA_MAX_N];               // 1 / L_kk, kept by the factorisation for the back substitution
  union alignas(16) {
    float Et[2][BA_ECH][BA_ELD];              // double-buffered tiles of augmented E rows (Schur phase)
    float recs[BA_REC_CHUNK][BA_REC];         // pair records (assembly phase)
  };
  int rec_i[BA_REC_CHUNK], rec_j[BA_REC_CHUNK];
};

// One thread-block cluster per Gauss-Newton iteration:
//   1. every CTA: - sum_k Q_k E_k E_k^T (2x2 register micro-tiles) and - sum_k Q_k u_k E_k over its
//      slice of the patches, then + the 6x6 pose blocks of its share of the (i,j) pair records
//   2. CTA 0 sums the 8 partial systems over distributed shared memory in rank order
//   3. CTA 0: damping, blocked (6x6) right-looking Cholesky of the rhs-augmented matrix -- the forward
//      substitution falls out of the factorisation -- and a one-warp back substitution
//   4. every CTA: depth updates dZ = Q (u - E^T dX) for its patches (one warp per patch, coalesced),
//      patch retraction; CTA 0: SE3 retraction of the free poses
__device__ __forceinline__ void ba_solve_body(const BaArgs& a, const int Gk, const int Gp) {
  extern __shared__ __align__(16) unsigned char solve_smem_raw[];
  SolveSmem& sm = *reinterpret_cast<SolveSmem*>(solve_smem_raw);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = a.N, N6 = 6 * N;
  const int P = a.P;
  const int per = (Gk + BA_CLUSTER - 1) / BA_CLUSTER;
  const int m0 = min(Gk, rank * per), m1 = min(Gk, m0 + per);
#define BA_STAMP(i) do { if (a.dbg && rank == 0 && tid == 0) a.dbg[i] = clock64(); } while (0)
  BA_STAMP(0);

  if (N > 0 && a.part) {
    // ---- 1 (fast path). The reduced system arrives as per-CTA partial sums from ba_reduce_kernel<true>: the cluster
    // adds them in CTA order, one entry per thread, 32 loads in flight, and deposits the sums in CTA 0's shared memory.
    SolveSmem* root = cluster.map_shared_rank(&sm, 0);
    const int n_ent = ba_packed_entries(N6), n_tri = N6 * (N6 + 1) / 2;
    // two adjacent lanes per entry: the even lane adds the first half of the partial systems, the odd lane the second half
    // (both in CTA order), one shuffle joins them -- half the dependent-load rounds of one thread per entry
    const int half_parts = (a.n_part + 1) / 2;
    const int limit = ((2 * n_ent + 31) / 32) * 32;               // warp-uniform loop bound (the shuffle needs every lane)
    for (int idx = rank * BA_SOLVE_THREADS + tid; idx < limit; idx += BA_CLUSTER * BA_SOLVE_THREADS) {
      const int e = idx >> 1, hf = idx & 1;
      const bool valid = e < n_ent;
      const int cb = hf ? half_parts : 0, ce = hf ? a.n_part : half_parts;
      float s = 0.0f;
      if (valid) {
        for (int c0 = cb; c0 < ce; c0 += 32) {
          float v[32];
#pragma unroll
          for (int u = 0; u < 32; ++u) v[u] = (c0 + u < ce) ? __ldcg(a.part + (int64_t)(c0 + u) * n_ent + e) : 0.0f;
#pragma unroll
          for (int u = 0; u < 32; ++u) s += v[u];
        }
      }
      const float other = __shfl_xor_sync(0xffffffffu, s, 1);
      if (valid && hf == 0) {
        int row = N6, col = e - n_tri;                              // gradient entries follow the packed triangle
        if (e < n_tri) {
          int rem = e;
          row = 0;
          while (rem >= N6 - row) { rem -= N6 - row; ++row; }
          col = row + rem;
        }
        root->S[row][col] = s + other;
      }
    }
    BA_STAMP(1);
  } else if (N > 0) {
    for (int o = tid; o < (N6 + 1) * N6; o += BA_SOLVE_THREADS) sm.S[o / N6][o % N6] = 0.0f;
    __syncthreads();
    // ---- 1a. Schur products over this CTA's patches.  Rows are staged as sqrt(Q_k) [E_k | u_k | 0..]: the gradient
    // term - sum_k Q_k u_k E_k becomes one more column of the same register-tiled product.  4x4 tiles (two 16-byte
    // shared loads per 16 FMAs -- with 2x2 tiles the phase was bound by shared-memory bandwidth), the rows of a
    // chunk split over up to three thread groups per tile, and the next chunk in flight in registers meanwhile.
    // Warp w stages rows w and w+16 of a chunk, lanes stride the columns: no integer division in the loop.
    const int NA = (N6 + 4) & ~3, H = NA / 4, n_tiles4 = H * (H + 1) / 2;
    const int n_chunks = (m1 - m0 + BA_ECH - 1) / BA_ECH;
    constexpr int NWARP = BA_SOLVE_THREADS / 32;
    constexpr int RPW = BA_ECH / NWARP;                                  // rows per warp and chunk
    constexpr int CPL = (BA_ELD + 31) / 32;                              // columns per lane
    static_assert(BA_ECH % NWARP == 0, "chunk rows divide over the warps");
    float pre[RPW][CPL], preq[RPW];
    auto fetch_chunk = [&](int ch) {                         // loads only: nothing here waits for them
      const int mbase = m0 + ch * BA_ECH;
#pragma unroll
      for (int rr = 0; rr < RPW; ++rr) {
        const int g = mbase + warp + rr * NWARP;
        const bool on = g < m1;
        preq[rr] = on ? a.Qk[g] : 0.f;                                    // rows past the slice add nothing
#pragma unroll
        for (int u = 0; u < CPL; ++u) {
          const int c = lane + 32 * u;
          float v = 0.f;
          if (on && c < N6) v = a.Ed[(int64_t)g * N6 + c];
          else if (on && c == N6) v = a.uk[g];
          pre[rr][u] = v;
        }
      }
    };
    auto store_chunk = [&](int buf) {
#pragma unroll
      for (int rr = 0; rr < RPW; ++rr) {
        const float sq = sqrtf(preq[rr]);
#pragma unroll
        for (int u = 0; u < CPL; ++u) {
          const int c = lane + 32 * u;
          if (c < NA) sm.Et[buf][warp + rr * NWARP][c] = sq * pre[rr][u];
        }
      }
    };
    // work item of a thread: tile (r4 <= c4) and k-split, constant over the chunks, so the 4x4 accumulator stays
    // in registers for the whole slice and S is touched once at the end (rounds > 1 only beyond 20 free poses;
    // the slice is then staged once per round)
    const int ksplit = max(1, min(3, BA_SOLVE_THREADS / n_tiles4));
    const int rounds = (n_tiles4 * ksplit + BA_SOLVE_THREADS - 1) / BA_SOLVE_THREADS;
    const int kper = (BA_ECH + ksplit - 1) / ksplit;
    for (int rd = 0; rd < rounds; ++rd) {
      const int item = tid + rd * BA_SOLVE_THREADS;
      const int sp = item / n_tiles4, mt = item - sp * n_tiles4;
      const bool live = sp < ksplit;
      int r4 = 0, c4 = 0;
      if (live) {
        int rem = mt;
        while (rem >= H - r4) { rem -= H - r4; ++r4; }
        c4 = r4 + rem;
      }
      const int kb = sp * kper, ke = live ? min(BA_ECH, kb + kper) : kb;
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      if (rd == 0) BA_STAMP(11);
      if (n_chunks > 0) { fetch_chunk(0); store_chunk(0); }
      __syncthreads();
      if (rd == 0) BA_STAMP(12);
      for (int ch = 0; ch < n_chunks; ++ch) {
        const int buf = ch & 1;
        if (ch + 1 < n_chunks) fetch_chunk(ch + 1);
        if (ch == 1) BA_STAMP(13);
#pragma unroll 4
        for (int k = kb; k < ke; ++k) {
          const float4 e = *reinterpret_cast<const float4*>(&sm.Et[buf][k][4 * r4]);
          const float4 f = *reinterpret_cast<const float4*>(&sm.Et[buf][k][4 * c4]);
          const float ev[4] = {e.x, e.y, e.z, e.w}, fv[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] += ev[i] * fv[j];
        }
        if (ch == 1) BA_STAMP(14);
        if (ch + 1 < n_chunks) store_chunk(buf ^ 1);
        __syncthreads();
        if (ch == 1) BA_STAMP(15);
      }
      // the k-splits of a tile add into S one after the other (fixed order)
      for (int ph = 0; ph < ksplit; ++ph) {
        if (live && sp == ph) {
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int row = 4 * r4 + i, col = 4 * c4 + j;
              if (col < N6) { if (row <= col) sm.S[row][col] -= acc[i][j]; }
              else if (col == N6 && row < N6) sm.S[N6][row] -= acc[i][j];     // augmented column = gradient row
            }
        }
        __syncthreads();
      }
    }
    BA_STAMP(1);
    // ---- 1b. pose blocks from this CTA's share of the pair records (pairs rank, rank+8, ...)
    const int n_mine = (Gp > rank) ? (Gp - rank + BA_CLUSTER - 1) / BA_CLUSTER : 0;
    for (int c0 = 0; c0 < n_mine; c0 += BA_REC_CHUNK) {
      const int cn = min(BA_REC_CHUNK, n_mine - c0);
      for (int i = tid; i < cn * BA_REC; i += BA_SOLVE_THREADS) {
        const int r = i / BA_REC, e = i - r * BA_REC;
        sm.recs[r][e] = a.rec[(int64_t)(rank + (int64_t)(c0 + r) * BA_CLUSTER) * BA_REC + e];
      }
      if (tid < cn) {
        const int p = rank + (c0 + tid) * BA_CLUSTER;
        long long fi = a.p_key_i[p] - a.t0, fj = a.p_key_j[p] - a.t0;
        sm.rec_i[tid] = (fi >= 0 && fi < N) ? (int)fi : -1;
        sm.rec_j[tid] = (fj >= 0 && fj < N) ? (int)fj : -1;
      }
      __syncthreads();
      if (tid < 63) {
        // Every entry of S is owned by ONE thread for all records (diagonal blocks: thread (x,y) serves both the
        // source-pose and the target-pose block; off-diagonal blocks are stored for the ordered pose pair, the
        // thread takes the transposed element when the record runs the other way), so records need no barrier
        // between them and are applied in index order by each owner.
        int x = 0, y = 0;
        if (tid < 21) { int rem = tid; while (rem >= 6 - x) { rem -= 6 - x; ++x; } y = x + rem; }
        else if (tid < 57) { const int e = tid - 21; x = e / 6; y = e - 6 * x; }
        for (int r = 0; r < cn; ++r) {
          const int bi = sm.rec_i[r], bj = sm.rec_j[r];
          const float* rc = sm.recs[r];
          if (tid < 21) {                                    // upper triangles of J_i J_i^T -> (i,i) and J_j J_j^T -> (j,j)
            if (bi >= 0) {
              float v = rc[tid];
              if (bi == bj) v += rc[57 + tid] + rc[21 + x * 6 + y] + rc[21 + y * 6 + x];   // self edge i -> i
              sm.S[6 * bi + x][6 * bi + y] += v;
            }
            if (bj >= 0 && bi != bj) sm.S[6 * bj + x][6 * bj + y] += rc[57 + tid];
          } else if (tid < 57) {                             // -J_i J_j^T -> block (min, max)
            if (bi >= 0 && bj >= 0 && bi != bj) {
              if (bi < bj) sm.S[6 * bi + x][6 * bj + y] += rc[21 + x * 6 + y];
              else sm.S[6 * bj + x][6 * bi + y] += rc[21 + y * 6 + x];
            }
          } else {                                           // gradient of pose i and pose j
            const int c = tid - 57;
            if (bi >= 0) sm.S[N6][6 * bi + c] += rc[78 + c] + ((bi == bj) ? rc[84 + c] : 0.0f);
            if (bj >= 0 && bi != bj) sm.S[N6][6 * bj + c] += rc[84 + c];
          }
        }
      }
      __syncthreads();
    }
  }
  BA_STAMP(2);
  cluster.sync();
  BA_STAMP(3);

  if (N > 0 && rank == 0) {
    // ---- 2. fixed-order reduction over distributed shared memory; mirror into the lower triangle
    for (int o = tid; o < (N6 + 1) * N6; o += BA_SOLVE_THREADS) {
      const int row = o / N6, col = o - row * N6;
      if (row < N6 && row > col) continue;
      float s = sm.S[row][col];
      if (!a.part) for (int r = 1; r < BA_CLUSTER; ++r) s += cluster.map_shared_rank(&sm, r)->S[row][col];
      if (row == col) s += 1e-4f * s + 1.0f;            // S += I * (1e-4 * S + 1)   ba_cuda.cu:560
      sm.S[row][col] = s;
      if (row < N6) sm.S[col][row] = s;
    }
  }
  BA_STAMP(4);
  cluster.sync();   // peers may now reuse their shared memory
  BA_STAMP(5);

  if (N > 0 && rank == 0) {
    // ---- 3. blocked Cholesky of [S; y^T] (lower storage, row N6 = rhs): 6-column panels.
    // Per panel: (a) one thread factors the 6x6 diagonal block and inverts the factor entirely in registers (the
    // shared-memory version spent > 3000 cycles per panel in dependent loads); (b) the rows below become
    // A_ik L_kk^-T, 21 independent FMAs per row, no divisions; (c) the trailing update runs on a (16 x 32) thread
    // grid -- a warp shares row i (broadcast loads), lanes stride j <= i -- with no integer division.
    float* linv = &sm.Et[0][0][0];                         // 21 entries of L_kk^-1 (row-major lower), free E-tile area
    for (int kb = 0; kb < N; ++kb) {
      const int k0 = 6 * kb;
      if (tid == 0) {
        float A[6][6], Li[6][6];
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
          for (int c = 0; c <= r; ++c) A[r][c] = sm.S[k0 + r][k0 + c];
#pragma unroll
        for (int c = 0; c < 6; ++c) {
          float d = A[c][c];
#pragma unroll
          for (int l = 0; l < c; ++l) d -= A[c][l] * A[c][l];
          d = sqrtf(d);
          const float id = 1.0f / d;
          A[c][c] = d;
          Li[c][c] = id;
#pragma unroll
          for (int r = c + 1; r < 6; ++r) {
            float v = A[r][c];
#pragma unroll
            for (int l = 0; l < c; ++l) v -= A[r][l] * A[c][l];
            A[r][c] = v * id;
          }
        }
        // inverse of the lower-triangular factor, column by column
#pragma unroll
        for (int c = 0; c < 6; ++c)
#pragma unroll
          for (int r = c + 1; r < 6; ++r) {
            float v = 0.f;
#pragma unroll
            for (int l = c; l < r; ++l) v -= A[r][l] * Li[l][c];
            Li[r][c] = v * Li[r][r];
          }
#pragma unroll
        for (int r = 0; r < 6; ++r) {
          sm.inv_diag[k0 + r] = Li[r][r];
#pragma unroll
          for (int c = 0; c <= r; ++c) { sm.S[k0 + r][k0 + c] = A[r][c]; linv[r * (r + 1) / 2 + c] = Li[r][c]; }
        }
      }
      __syncthreads();
      for (int i = k0 + 6 + tid; i <= N6; i += BA_SOLVE_THREADS) {     // panel: rows below (+ rhs row)
        float av[6], v[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) av[c] = sm.S[i][k0 + c];
#pragma unroll
        for (int c = 0; c < 6; ++c) {                                  // (A L^-T)[c] = sum_{l <= c} A[l] Linv[c][l]
          float t = 0.f;
#pragma unroll
          for (int l = 0; l <= c; ++l) t += av[l] * linv[c * (c + 1) / 2 + l];
          v[c] = t;
        }
#pragma unroll
        for (int c = 0; c < 6; ++c) sm.S[i][k0 + c] = v[c];
      }
      __syncthreads();
      for (int i = k0 + 6 + warp; i <= N6; i += BA_SOLVE_THREADS / 32) {   // trailing rows (i = N6: the rhs row)
        float li[6];
#pragma unroll
        for (int l = 0; l < 6; ++l) li[l] = sm.S[i][k0 + l];
        const int jend = min(i, N6 - 1);
        for (int j = k0 + 6 + lane; j <= jend; j += 32) {
          float t = 0.0f;
#pragma unroll
          for (int l = 0; l < 6; ++l) t += li[l] * sm.S[j][k0 + l];
          sm.S[i][j] -= t;
        }
      }
      __syncthreads();
    }
    BA_STAMP(6);
    // row N6 now holds z = L^-1 y; back substitution L^T x = z with one warp, z kept in registers
    // (lane l owns entries l, l+32, ...): per step one row of L from shared memory, one shuffle, no stores
    if (tid < 32) {
      constexpr int ZR = (6 * BA_MAX_N + 31) / 32;
      float z[ZR];
#pragma unroll
      for (int u = 0; u < ZR; ++u) z[u] = (lane + 32 * u < N6) ? sm.S[N6][lane + 32 * u] : 0.0f;
#pragma unroll
      for (int uk = ZR - 1; uk >= 0; --uk) {                // segment of 32 unknowns whose z lives in z[uk]
        if (32 * uk >= N6) continue;
        for (int kk = min(31, N6 - 1 - 32 * uk); kk >= 0; --kk) {
          const int k = 32 * uk + kk;
          // (1/d) z_k instead of z_k / d: the factor is stored with its reciprocal diagonal
          const float xk = __shfl_sync(0xffffffffu, z[uk], kk) * sm.inv_diag[k];
          if (lane == kk) sm.dx[k] = xk;
#pragma unroll
          for (int u = 0; u < ZR; ++u) {
            if (u <= uk) {
              const int i = lane + 32 * u;
              if (i < k) z[u] -= sm.S[k][i] * xk;
            }
          }
        }
      }
    }
    __syncthreads();
    for (int i = tid; i < N6; i += BA_SOLVE_THREADS) a.dX[i] = sm.dx[i];
  }
  BA_STAMP(7);
  cluster.sync();
  BA_STAMP(8);

  // ---- 4. depth back-substitution dZ = Q (u - E^T dX) and patch retraction (ba_cuda.cu:209-229)
  float* dxs = &sm.Et[0][0][0];      // per-CTA copy of dX (N6 <= 192 floats) in the free E-tile area
  if (N > 0) {
    const SolveSmem* root = cluster.map_shared_rank(&sm, 0);
    for (int i = tid; i < N6; i += BA_SOLVE_THREADS) dxs[i] = root->dx[i];
  }
  __syncthreads();
  {
    // Scalars of a patch (key, Q, u, current depth) are fetched one THREAD per patch -- two dependent global
    // latencies for the whole slice instead of per patch --, the dot products E_k . dX one WARP per patch with the
    // rows of eight patches in flight, the new depth is written back thread per patch.
    constexpr int NW = BA_SOLVE_THREADS / 32;
    constexpr int DB = 8;
    constexpr int ER = (6 * BA_MAX_N + 31) / 32;
    float* sc_q = dxs + 6 * BA_MAX_N;                      // [BA_SOLVE_THREADS] each, in the free E-tile area
    float* sc_u = sc_q + BA_SOLVE_THREADS;
    float* sc_dot = sc_u + BA_SOLVE_THREADS;
    for (int base = m0; base < m1; base += BA_SOLVE_THREADS) {
      const int cnt = min(BA_SOLVE_THREADS, m1 - base);
      float* pd = nullptr;
      float d0 = 0.f;
      if (tid < cnt) {
        const int g = base + tid;
        sc_q[tid] = a.Qk[g];
        sc_u[tid] = a.uk[g];
        pd = a.patches + (a.k_key[g] * 3 + 2) * P * P;
        d0 = pd[0];
      }
      for (int q0 = warp; q0 < cnt; q0 += NW * DB) {
        float er[DB][ER];
#pragma unroll
        for (int b = 0; b < DB; ++b) {
          const int q = q0 + b * NW;
#pragma unroll
          for (int u = 0; u < ER; ++u) {
            const int k = lane + 32 * u;
            er[b][u] = (q < cnt && k < N6) ? a.Ed[(int64_t)(base + q) * N6 + k] : 0.0f;
          }
        }
#pragma unroll
        for (int b = 0; b < DB; ++b) {
          const int q = q0 + b * NW;
          float dot = 0.0f;
#pragma unroll
          for (int u = 0; u < ER; ++u) {
            const int k = lane + 32 * u;
            if (k < N6) dot += er[b][u] * dxs[k];
          }
          dot = warp_sum(dot);
          if (lane == 0 && q < cnt) sc_dot[q] = dot;
        }
      }
      __syncthreads();
      if (tid < cnt) {
        const float dz = sc_q[tid] * (sc_u[tid] - sc_dot[tid]);
        float d = d0 + dz;
        d = (d > 20.0f) ? 1.0f : d;
        d = fmaxf(d, 1e-4f);
        for (int i = 0; i < P * P; ++i) pd[i] = d;
      }
      __syncthreads();
    }
  }
  BA_STAMP(9);
  // ---- 5. pose retraction (ba_cuda.cu:178-206), after every CTA is done reading dx
  cluster.sync();
  BA_STAMP(10);
  if (N > 0 && rank == 0 && tid < N) {
    retract_pose(a.poses + (int64_t)(a.t0 + tid) * 7, sm.dx + 6 * tid);
  }
#undef BA_STAMP
}

__global__ void __cluster_dims__(BA_CLUSTER, 1, 1) __launch_bounds__(BA_SOLVE_THREADS, 1)
ba_solve_kernel(const BaArgs a) {
  ba_solve_body(a, *a.k_n, (a.N > 0) ? *a.p_n : 0);
}

// ==========================================================================================
// batched: B independent sliding windows in one reduce and one solve launch
// ==========================================================================================
// Stream b owns frames [b F, (b+1) F) and patches [b F M, (b+1) F M).  The groupings are built over the concatenated
// edge list; their keys ascend, so the patch groups and the pair groups of stream b form one contiguous range each.
// ba_stream_bounds_kernel finds the ranges on the device: bounds[b] = first patch group of stream b (bounds[B] = the
// number of patch groups), bounds[B + 1 + b] likewise for the pair groups.  No edge joins two streams (the host layer
// rejects such edge lists), so a stream's groups hold only its own edges and every stream is the single-window
// problem on a slice of the groupings and of the scratch.
constexpr int BA_MAX_STREAMS = 64;

struct BaBatch {
  int B;
  int64_t F, FM;                       // frames and patches per stream
  int t0[BA_MAX_STREAMS];              // global index of the first free pose
  int N[BA_MAX_STREAMS];               // free poses; 0 = the stream is left untouched
  const int32_t* bounds;               // [2 (B + 1)], written by ba_stream_bounds_kernel
  int64_t ed_pitch;                    // floats per patch-group row of Ed: 6 max_b N_b
  int64_t part_stride;                 // floats of partial systems per stream (fast path)
};

// bounds[b] = the first group whose key belongs to stream >= b.  Each entry is written by exactly one thread: the one
// at the group where the stream index of the sorted keys steps past b.
__global__ void __launch_bounds__(256)
ba_stream_bounds_kernel(const int64_t* __restrict__ k_key, const int32_t* __restrict__ k_n, const int64_t* __restrict__ p_key_i,
                        const int32_t* __restrict__ p_n, int64_t FM, int64_t F, int B, int32_t* __restrict__ bounds) {
  const int Gk = *k_n, Gp = p_n ? *p_n : 0;
  auto stream_of = [&](int64_t key, int64_t per) { const int64_t s = key / per; return (int)(s < 0 ? 0 : (s > B ? B : s)); };
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t <= Gk + 1 + Gp; t += gridDim.x * blockDim.x) {
    const bool pair = t > Gk;
    const int g = pair ? t - Gk - 1 : t, G = pair ? Gp : Gk;
    const int64_t* key = pair ? p_key_i : k_key;
    const int64_t per = pair ? F : FM;
    int32_t* out = bounds + (pair ? B + 1 : 0);
    const int s_prev = (g == 0) ? -1 : stream_of(key[g - 1], per);
    const int s_cur = (g == G) ? B : stream_of(key[g], per);
    for (int b = s_prev + 1; b <= s_cur; ++b) out[b] = g;
  }
}

// the single-window arguments of stream b: its group ranges, its window, its camera and its slices of the scratch
__device__ __forceinline__ BaArgs ba_stream_args(const BaArgs& a, const BaBatch& bb, int b, int& Gk, int& Gp) {
  const int k0 = bb.bounds[b], p0 = bb.bounds[bb.B + 1 + b];
  Gk = bb.bounds[b + 1] - k0;
  Gp = bb.bounds[bb.B + 2 + b] - p0;
  BaArgs s = a;
  s.t0 = bb.t0[b]; s.N = bb.N[b];
  s.intrinsics = a.intrinsics + (int64_t)b * bb.F * 4;
  s.k_start = a.k_start + k0; s.k_key = a.k_key + k0;
  s.p_start = a.p_start + p0; s.p_key_i = a.p_key_i + p0; s.p_key_j = a.p_key_j + p0;
  s.Ed = a.Ed + (int64_t)k0 * bb.ed_pitch;
  s.Qk = a.Qk + k0; s.uk = a.uk + k0;
  s.rec = a.rec + (int64_t)p0 * BA_REC;
  s.dX = a.dX + (int64_t)b * 6 * BA_MAX_N;
  s.part = a.part ? a.part + (int64_t)b * bb.part_stride : nullptr;
  s.dbg = nullptr;
  return s;
}

// grid (partitions per stream, B): blockIdx.y is the stream, blockIdx.x deals that stream's items as the single-window
// launch deals them, so each stream's partial sums are those of a launch on that stream alone
template <bool SYSTEM>
__global__ void __launch_bounds__((SYSTEM ? BA_FAST_WARPS : BA_RED_WARPS) * 32)
ba_reduce_batched_kernel(const BaArgs a, const BaBatch bb) {
  int Gk, Gp;
  const BaArgs s = ba_stream_args(a, bb, blockIdx.y, Gk, Gp);
  if (s.N == 0 || Gk == 0) return;                   // an empty window or a stream without edges: nothing to do
  ba_reduce_body<SYSTEM, SYSTEM>(s, Gk, Gp);
}

// B clusters of 8 CTAs: cluster c solves stream c
__global__ void __cluster_dims__(BA_CLUSTER, 1, 1) __launch_bounds__(BA_SOLVE_THREADS, 1)
ba_solve_batched_kernel(const BaArgs a, const BaBatch bb) {
  int Gk, Gp;
  const BaArgs s = ba_stream_args(a, bb, blockIdx.x / BA_CLUSTER, Gk, Gp);
  if (s.N == 0 || Gk == 0) return;                   // uniform over the cluster: no CTA waits at a cluster barrier alone
  ba_solve_body(s, Gk, Gp);
}

// ==========================================================================================
// reprojection (cuda_ba.reproject, ba_cuda.cu:379-429; pops.transform, projective_ops.py:53-68)
// ==========================================================================================
template <bool CLAMP>
__global__ void reproject_kernel(const float* __restrict__ poses, const float* __restrict__ patches,
                                 const float* __restrict__ intrinsics, const int64_t* __restrict__ ii,
                                 const int64_t* __restrict__ jj, const int64_t* __restrict__ kk,
                                 float* __restrict__ coords, int64_t E, int P) {
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < E; n += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ix = ii[n], jx = jj[n], kx = kk[n];
    const float* Ki = CLAMP ? intrinsics + ix * 4 : intrinsics;
    const float* Kj = CLAMP ? intrinsics + jx * 4 : intrinsics;
    // the lietorch path (pops.transform) loads group elements normalised (so3.h:35-37); cuda_ba.reproject does not
    const lie::SE3<float> G = edge_relative_pose(poses, ix, jx, CLAMP);
    const float* pk = patches + kx * 3 * P * P;
    float* out = coords + n * 2 * P * P;
    for (int i = 0; i < P * P; ++i) {
      const lie::V3<float> p = lie::v3<float>((pk[i] - Ki[2]) / Ki[0], (pk[P * P + i] - Ki[3]) / Ki[1], 1.0f);
      const lie::V3<float> Pj = lie::q_rot(G.q, p) + pk[2 * P * P + i] * G.t;
      const float Xj[3] = {Pj.x, Pj.y, Pj.z};
      if (CLAMP) {
        const float d = 1.0f / fmaxf(Xj[2], 0.1f);
        out[i] = Kj[0] * (d * Xj[0]) + Kj[2];
        out[P * P + i] = Kj[1] * (d * Xj[1]) + Kj[3];
      } else {
        out[i] = Kj[0] * (Xj[0] / Xj[2]) + Kj[2];
        out[P * P + i] = Kj[1] * (Xj[1] / Xj[2]) + Kj[3];
      }
    }
  }
}

}  // namespace dpvo

using namespace dpvo;

// ---- workspaces and kernel arguments ---------------------------------------------------------
namespace {
// an edge grouping as dpvo_group_edges leaves it; key_j is the target frame of the pair grouping, NULL for the patches
struct BaGroups { const int32_t* order; const int32_t* start; const int64_t* key_i; const int64_t* key_j; const int32_t* n; };

// scratch of the reduce and solve kernels: Ed rows of 6 max(N, 1) floats, one dX per stream
struct BaScratch { float *Ed, *Qk, *uk, *rec, *dX; };
BaScratch ba_scratch_layout(int64_t E, int N, int streams, WsLayout& L) {
  BaScratch s;
  s.Ed = L.take<float>(E * 6 * std::max(N, 1)); s.Qk = L.take<float>(E); s.uk = L.take<float>(E);
  s.rec = L.take<float>(E * BA_REC); s.dX = L.take<float>((int64_t)streams * 6 * BA_MAX_N);
  return s;
}

// dpvo_ba_forward: the outputs of its two groupings (key_j: pairs only), the scratch, the two groupings' workspaces
struct BaGrouping {
  int32_t *order, *of, *start, *n; int64_t *key_i, *key_j;
  BaGroups groups() const { return {order, start, key_i, key_j, n}; }
};
struct BaForwardWs { BaGrouping k, p; BaScratch s; void *gws_k, *gws_p; };
BaForwardWs ba_forward_layout(int64_t E, int N, WsLayout& L) {
  BaForwardWs w;
  for (BaGrouping* g : {&w.k, &w.p}) {
    g->order = L.take<int32_t>(E); g->of = L.take<int32_t>(E); g->start = L.take<int32_t>(E + 1);
    g->key_i = L.take<int64_t>(E); g->key_j = g == &w.p ? L.take<int64_t>(E) : nullptr; g->n = L.take<int32_t>(1);
  }
  w.s = ba_scratch_layout(E, N, 1, L);
  w.gws_k = L.take<char>(dpvo_group_workspace_bytes(E)); w.gws_p = L.take<char>(dpvo_group_workspace_bytes(E));
  return w;
}

// batched: the stream bounds, then the scratch with Ed rows of 6 max_b N_b floats and one dX per stream, then
// (every N_b <= BA_FAST_MAX_N) B x sm_count partial reduced systems
int64_t ba_batched_part_floats(int max_free_poses) {
  return (max_free_poses > 0 && max_free_poses <= BA_FAST_MAX_N) ? (int64_t)sm_count() * ba_packed_entries(6 * max_free_poses) : 0;
}
struct BaBatchedWs { int32_t* bounds; BaScratch s; float* part; };
BaBatchedWs ba_batched_layout(int64_t E, int B, int max_free_poses, WsLayout& L) {
  BaBatchedWs w;
  w.bounds = L.take<int32_t>(2 * (int64_t)(B + 1)); w.s = ba_scratch_layout(E, max_free_poses, B, L);
  w.part = L.take<float>((int64_t)B * ba_batched_part_floats(max_free_poses));
  return w;
}

BaArgs ba_args(float* poses, float* patches, const float* intrinsics, const float* target, const float* weight,
               const float* lmbda, const int64_t* ii, const int64_t* jj, const int64_t* kk, int64_t E, int P, int t0, int N,
               const BaGroups& k, const BaGroups& p, const BaScratch& s) {
  BaArgs a;
  a.poses = poses; a.patches = patches; a.intrinsics = intrinsics; a.target = target; a.weight = weight;
  a.lmbda = lmbda; a.ii = ii; a.jj = jj; a.kk = kk; a.E = E; a.P = P; a.t0 = t0; a.N = N;
  a.k_order = k.order; a.k_start = k.start; a.k_key = k.key_i; a.k_n = k.n;
  a.p_order = p.order; a.p_start = p.start; a.p_key_i = p.key_i; a.p_key_j = p.key_j; a.p_n = p.n;
  a.Ed = s.Ed; a.Qk = s.Qk; a.uk = s.uk; a.rec = s.rec; a.dX = s.dX;
  a.part = nullptr; a.n_part = 0; a.dbg = nullptr;
  return a;
}

// fast-path reduce, windows of up to N free poses: per warp an E row, a pair record and a packed reduced system
size_t ba_fast_smem(int N) { return (size_t)BA_FAST_WARPS * (6 * BA_MAX_N + 96 + (size_t)ba_packed_entries(6 * N)) * sizeof(float); }
}  // namespace

extern "C" int64_t dpvo_ba_workspace_bytes(int64_t E, int n_free_poses) {
  if (E < 0) E = 0;
  WsLayout L;
  ba_forward_layout(E, n_free_poses, L);
  return L.bytes() + 256;
}

static int ba_run(BaArgs& a, int iterations, cudaStream_t st) {
#ifdef DPVO_B200_PERF_EXPERIMENTS
  static long long* dbg = nullptr;
  const bool timing = getenv("DPVO_B200_BA_TIMING") != nullptr;
  if (timing && !dbg) cudaMalloc(&dbg, 16 * sizeof(long long));
  a.dbg = timing ? dbg : nullptr;
#else
  const bool timing = false;
  a.dbg = nullptr;
#endif
  const int red_blocks = sm_count() * 4;
  // sliding-window sizes: the reduced system is assembled by the reduce kernel (one partial per CTA, stored where the
  // pair records of the general path would go -- the fast path does not materialise them)
  a.part = nullptr; a.n_part = 0;
  if (a.N > 0 && a.N <= BA_FAST_MAX_N && (int64_t)sm_count() * ba_packed_entries(6 * a.N) <= a.E * (int64_t)BA_REC) {
    a.part = a.rec;
    a.n_part = sm_count();
  }
  const bool fast = a.part != nullptr;
  for (int it = 0; it < iterations; ++it) {
    int rc = fast ? launch("ba_reduce_kernel", ba_reduce_kernel<true>, a.n_part, BA_FAST_WARPS * 32, ba_fast_smem(a.N), st, a)
                  : launch("ba_reduce_kernel", ba_reduce_kernel<false>, red_blocks, BA_RED_WARPS * 32, BA_RED_WARPS * 6 * BA_MAX_N * sizeof(float), st, a);
    if (!rc) rc = launch("ba_solve_kernel", ba_solve_kernel, BA_CLUSTER, BA_SOLVE_THREADS, sizeof(SolveSmem), st, a);
    if (rc) return rc;
  }
#ifdef DPVO_B200_PERF_EXPERIMENTS
  if (timing) {
    long long h[16];
    cudaStreamSynchronize(st);
    cudaMemcpy(h, dbg, sizeof(h), cudaMemcpyDeviceToHost);
    const char* names[10] = {"schur", "pair blocks", "cluster.sync", "dsmem reduce", "cluster.sync", "cholesky", "back-subst", "cluster.sync", "depth update", "cluster.sync"};
    fprintf(stderr, "[ba_solve phases, SM cycles]");
    for (int i = 0; i < 10; ++i) fprintf(stderr, " %s=%lld", names[i], h[i + 1] - h[i]);
    fprintf(stderr, " total=%lld | schur detail: setup %lld, first chunk staged %lld, chunk 1: multiply %lld, stage next + barrier %lld\n", h[10] - h[0],
            h[11] - h[0], h[12] - h[11], h[14] - h[13], h[15] - h[14]);
  }
#else
  (void)timing;
#endif
  return DPVO_OK;
}

extern "C" int64_t dpvo_ba_grouped_workspace_bytes(int64_t E, int n_free_poses) {
  if (E < 0) E = 0;
  WsLayout L;
  ba_scratch_layout(E, n_free_poses, 1, L);
  return L.bytes() + 512;
}

extern "C" int dpvo_ba_forward_grouped(float* poses, float* patches, const float* intrinsics,
                                       const float* target, const float* weight, const float* lmbda,
                                       const int64_t* ii, const int64_t* jj, const int64_t* kk,
                                       int64_t E, int P, int t0, int t1, int iterations,
                                       const int32_t* k_order, const int32_t* k_start, const int64_t* k_key, const int32_t* k_n,
                                       const int32_t* p_order, const int32_t* p_start, const int64_t* p_key_i,
                                       const int64_t* p_key_j, const int32_t* p_n,
                                       void* workspace, int64_t workspace_bytes, void* stream) {
  DPVO_REQUIRE(E >= 0 && P > 0 && iterations >= 0 && t1 >= t0, "ba_forward_grouped: bad sizes");
  if (E == 0 || iterations == 0) return DPVO_OK;
  DPVO_REQUIRE(poses && patches && intrinsics && target && weight && lmbda && ii && jj && kk && workspace && k_order &&
               k_start && k_key && k_n, "ba_forward_grouped: null pointer");
  const int N = t1 - t0;
  DPVO_REQUIRE(N == 0 || (p_order && p_start && p_key_i && p_key_j && p_n), "ba_forward_grouped: pair grouping missing");
  if (N > BA_MAX_N) { set_error("ba_forward_grouped: %d free poses > %d", N, BA_MAX_N); return DPVO_ERR_UNSUPPORTED; }
  if (workspace_bytes < dpvo_ba_grouped_workspace_bytes(E, N)) { set_error("ba_forward_grouped: workspace too small"); return DPVO_ERR_WORKSPACE; }
  WsLayout L(align256(workspace));
  const BaScratch s = ba_scratch_layout(E, N, 1, L);
  BaArgs a = ba_args(poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, E, P, t0, N,
                     {k_order, k_start, k_key, nullptr, k_n}, {p_order, p_start, p_key_i, p_key_j, p_n}, s);
  return ba_run(a, iterations, (cudaStream_t)stream);
}

extern "C" int64_t dpvo_ba_batched_workspace_bytes(int64_t E, int B, int max_free_poses) {
  if (E < 0) E = 0;
  if (B < 1) B = 1;
  WsLayout L;
  ba_batched_layout(E, B, max_free_poses, L);
  return L.bytes() + 256;
}

extern "C" int dpvo_ba_forward_batched(float* poses, float* patches, const float* intrinsics,
                                       const float* target, const float* weight, const float* lmbda,
                                       const int64_t* ii, const int64_t* jj, const int64_t* kk,
                                       int64_t E, int P, int B, int frames_per_stream, int patches_per_frame,
                                       const int* t0, const int* t1, int iterations,
                                       const int32_t* k_order, const int32_t* k_start, const int64_t* k_key, const int32_t* k_n,
                                       const int32_t* p_order, const int32_t* p_start, const int64_t* p_key_i,
                                       const int64_t* p_key_j, const int32_t* p_n,
                                       void* workspace, int64_t workspace_bytes, void* stream) {
  DPVO_REQUIRE(E >= 0 && P > 0 && iterations >= 0 && B >= 1 && frames_per_stream > 0 && patches_per_frame > 0,
               "ba_forward_batched: bad sizes");
  DPVO_REQUIRE(t0 && t1, "ba_forward_batched: null window arrays");
  if (B > BA_MAX_STREAMS) { set_error("ba_forward_batched: %d streams > %d", B, BA_MAX_STREAMS); return DPVO_ERR_UNSUPPORTED; }
  BaBatch bb;
  bb.B = B; bb.F = frames_per_stream; bb.FM = (int64_t)frames_per_stream * patches_per_frame;
  int max_n = 0;
  for (int b = 0; b < B; ++b) {
    const int n = t1[b] - t0[b];
    DPVO_REQUIRE(n >= 0 && (n == 0 || (t0[b] >= (int64_t)b * frames_per_stream && t1[b] <= (int64_t)(b + 1) * frames_per_stream)),
                 "ba_forward_batched: window [%d, %d) of stream %d is not inside its frames [%lld, %lld)", t0[b], t1[b], b,
                 (long long)b * frames_per_stream, (long long)(b + 1) * frames_per_stream);
    if (n > BA_MAX_N) { set_error("ba_forward_batched: stream %d has %d free poses > %d", b, n, BA_MAX_N); return DPVO_ERR_UNSUPPORTED; }
    bb.t0[b] = t0[b]; bb.N[b] = n;
    max_n = std::max(max_n, n);
  }
  if (E == 0 || iterations == 0 || max_n == 0) return DPVO_OK;
  DPVO_REQUIRE(poses && patches && intrinsics && target && weight && lmbda && ii && jj && kk && workspace && k_order &&
               k_start && k_key && k_n && p_order && p_start && p_key_i && p_key_j && p_n, "ba_forward_batched: null pointer");
  if (workspace_bytes < dpvo_ba_batched_workspace_bytes(E, B, max_n)) { set_error("ba_forward_batched: workspace too small"); return DPVO_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  WsLayout L(align256(workspace));
  const BaBatchedWs w = ba_batched_layout(E, B, max_n, L);
  BaArgs a = ba_args(poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, E, P, 0, max_n,
                     {k_order, k_start, k_key, nullptr, k_n}, {p_order, p_start, p_key_i, p_key_j, p_n}, w.s);
  // the fast path applies to the whole batch when every window fits it, the general path otherwise
  const bool fast = max_n <= BA_FAST_MAX_N;
  a.part = fast ? w.part : nullptr;
  a.n_part = fast ? sm_count() : 0;
  bb.part_stride = ba_batched_part_floats(max_n);
  bb.ed_pitch = 6 * (int64_t)max_n;
  bb.bounds = w.bounds;
  {
    const int64_t items = E + 2;                 // at most Gk + 1 + Gp + 1 <= E + 2
    const unsigned grid = (unsigned)std::min<int64_t>((items + 255) / 256, (int64_t)sm_count() * 4);
    const int rc = launch("ba_stream_bounds_kernel", ba_stream_bounds_kernel, grid, 256, 0, st, k_key, k_n, p_key_i, p_n, bb.FM, bb.F, B, w.bounds);
    if (rc) return rc;
  }
  for (int it = 0; it < iterations; ++it) {
    // shared memory sized for the widest window of the batch
    int rc = fast ? launch("ba_reduce_batched_kernel", ba_reduce_batched_kernel<true>, dim3(a.n_part, B), BA_FAST_WARPS * 32, ba_fast_smem(max_n), st, a, bb)
                  : launch("ba_reduce_batched_kernel", ba_reduce_batched_kernel<false>, dim3(sm_count() * 4, B), BA_RED_WARPS * 32,
                           BA_RED_WARPS * 6 * BA_MAX_N * sizeof(float), st, a, bb);
    if (!rc) rc = launch("ba_solve_batched_kernel", ba_solve_batched_kernel, BA_CLUSTER * B, BA_SOLVE_THREADS, sizeof(SolveSmem), st, a, bb);
    if (rc) return rc;
  }
  return DPVO_OK;
}

extern "C" int dpvo_ba_forward(float* poses, float* patches, const float* intrinsics,
                               const float* target, const float* weight, const float* lmbda,
                               const int64_t* ii, const int64_t* jj, const int64_t* kk,
                               int64_t E, int64_t n_poses, int64_t n_patches, int P,
                               int t0, int t1, int iterations,
                               void* workspace, int64_t workspace_bytes, void* stream) {
  DPVO_REQUIRE(E >= 0 && P > 0 && iterations >= 0 && t1 >= t0, "ba_forward: bad sizes");
  if (E == 0 || iterations == 0) return DPVO_OK;
  DPVO_REQUIRE(poses && patches && intrinsics && target && weight && lmbda && ii && jj && kk && workspace,
               "ba_forward: null pointer");
  (void)n_poses; (void)n_patches;
  const int N = t1 - t0;
  if (N > BA_MAX_N) {
    set_error("ba_forward: %d free poses > %d supported by the on-chip solver (use the block-sparse path)", N, BA_MAX_N);
    return DPVO_ERR_UNSUPPORTED;
  }
  if (workspace_bytes < dpvo_ba_workspace_bytes(E, N)) {
    set_error("ba_forward: workspace %lld B < required %lld B", (long long)workspace_bytes,
              (long long)dpvo_ba_workspace_bytes(E, N));
    return DPVO_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  WsLayout L(align256(workspace));
  const BaForwardWs w = ba_forward_layout(E, N, L);
  const int64_t gb = dpvo_group_workspace_bytes(E);
  int rc = dpvo_group_edges(kk, nullptr, nullptr, E, w.k.order, w.k.of, w.k.start, w.k.key_i, nullptr, w.k.n, w.gws_k, gb, st);
  if (rc) return rc;
  if (N > 0) {
    rc = dpvo_group_edges(ii, jj, nullptr, E, w.p.order, w.p.of, w.p.start, w.p.key_i, w.p.key_j, w.p.n, w.gws_p, gb, st);
    if (rc) return rc;
  }
  // from here on the path of dpvo_ba_forward_grouped
  BaArgs a = ba_args(poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, E, P, t0, N, w.k.groups(), w.p.groups(), w.s);
  return ba_run(a, iterations, st);
}

extern "C" int dpvo_reproject(const float* poses, const float* patches, const float* intrinsics,
                              const int64_t* ii, const int64_t* jj, const int64_t* kk,
                              float* coords, int64_t E, int P, int clamp_depth, void* stream) {
  DPVO_REQUIRE(E >= 0 && P > 0, "reproject: bad sizes");
  if (E == 0) return DPVO_OK;
  DPVO_REQUIRE(poses && patches && intrinsics && ii && jj && kk && coords, "reproject: null pointer");
  const int threads = 128;
  const unsigned blocks = (unsigned)std::min<int64_t>((E + threads - 1) / threads, (int64_t)sm_count() * 16);
  return launch("reproject_kernel", clamp_depth ? reproject_kernel<true> : reproject_kernel<false>, blocks, threads, 0, (cudaStream_t)stream, poses,
                patches, intrinsics, ii, jj, kk, coords, E, P);
}
