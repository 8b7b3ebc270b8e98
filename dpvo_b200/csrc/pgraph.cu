// Device-resident patch-graph bookkeeping on fixed-capacity edge arrays.
//
// The reference keeps the edge lists (ii, jj, kk) and the per-edge recurrent state as tensors whose LENGTH changes every
// frame: torch.cat in append_factors (dpvo/dpvo.py:215-222), boolean-mask indexing in remove_factors (:224-238, one
// device->host sync per mask), index shifting in keyframe (:282-286).  A captured CUDA graph of update() cannot follow
// that.  Here the arrays have a fixed capacity and every slot is either an ACTIVE edge or a PARKED one:
//   * a parked slot holds the dummy edge (ii = jj = dummy_frame, kk = dummy_patch): a reserved frame / patch that no
//     real edge refers to, so parked edges form their own patch group and their own (i, j) pair in every grouping of
//     the update operator and never mix with real rows; the caller zeroes their confidence weights before bundle
//     adjustment (active is the mask), and the dummy frame lies outside every optimisation window
//   * removal parks slots in place (nothing moves, the recurrent state of the other edges stays where it is)
//   * append fills the parked slots in index order and zeroes the state rows of the new edges (dpvo.py:220-221)
// Everything is decided from device-resident scalars (frame counter, keyframe index, enable flag), so the calls are
// CUDA-graph capturable and need no host synchronisation.  The number of active edges is tracked with integer atomics.
#include "common.cuh"

namespace dpvo {

constexpr int PG_THREADS = 1024;

// rule 0 (dpvo.py:300,306): park the active edges whose patch belongs to a frame older than *frame - param
// rule 1 (dpvo.py:282-286): park the edges that touch frame k = *frame, then renumber the frames / patches above k
__global__ void __launch_bounds__(256)
pgraph_remove_kernel(int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, int64_t cap, int rule, const int64_t* frame,
                     int64_t param, const int32_t* enable, int64_t dummy_frame, int64_t dummy_patch, int M, int32_t* n_active) {
  if (enable && *enable == 0) return;
  const int64_t f = *frame;
  int removed = 0;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < cap; e += (int64_t)gridDim.x * blockDim.x) {
    if (!active[e]) continue;
    int64_t i = ii[e], j = jj[e], k = kk[e];
    bool drop;
    if (rule == 0) drop = (k / M) < f - param;
    else drop = (i == f) || (j == f);
    if (drop) {
      ii[e] = dummy_frame; jj[e] = dummy_frame; kk[e] = dummy_patch; active[e] = 0;
      ++removed;
    } else if (rule == 1) {
      if (i > f) { kk[e] = k - M; ii[e] = i - 1; }
      if (j > f) jj[e] = j - 1;
    }
  }
  // one integer atomic per warp
  for (int o = 16; o > 0; o >>= 1) removed += __shfl_xor_sync(0xffffffffu, removed, o);
  if ((threadIdx.x & 31) == 0 && removed) atomicSub(n_active, removed);
}

// New edges go to the parked slots in index order.  One CTA: every thread owns a contiguous range of slots, counts its
// parked ones, a block scan gives the rank of its first parked slot, then it walks its range again and places edges.
__global__ void __launch_bounds__(PG_THREADS)
pgraph_append_kernel(int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, int64_t cap, const int64_t* new_ii, const int64_t* new_jj,
                     const int64_t* new_kk, int64_t n_new, const int32_t* enable, int32_t* slot_of_new, int32_t* n_active, int32_t* overflow) {
  __shared__ int warp_tot[PG_THREADS / 32 + 1];
  const bool on = !(enable && *enable == 0);
  const int64_t per = (cap + PG_THREADS - 1) / PG_THREADS;
  const int64_t s0 = min(cap, (int64_t)threadIdx.x * per), s1 = min(cap, s0 + per);
  int cnt = 0;
  if (on) for (int64_t e = s0; e < s1; ++e) cnt += active[e] ? 0 : 1;
  // exclusive scan over the block
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int i = 0; i < PG_THREADS / 32; ++i) { const int t = warp_tot[i]; warp_tot[i] = run; run += t; }
    warp_tot[PG_THREADS / 32] = run;
  }
  __syncthreads();
  int rank = warp_tot[w] + inc - cnt;
  const int total_free = warp_tot[PG_THREADS / 32];
  if (on) {
    for (int64_t e = s0; e < s1 && rank < n_new; ++e) {
      if (active[e]) continue;
      ii[e] = new_ii[rank]; jj[e] = new_jj[rank]; kk[e] = new_kk[rank]; active[e] = 1;
      if (slot_of_new) slot_of_new[rank] = (int32_t)e;
      ++rank;
    }
  }
  if (threadIdx.x == 0) {
    if (on) {
      const int placed = n_new < (int64_t)total_free ? (int)n_new : total_free;
      atomicAdd(n_active, placed);
      if (placed < n_new && overflow) *overflow = 1;          // capacity exhausted: the surplus edges are dropped and reported
    }
  }
  // edges that found no slot (overflow) or a disabled call: mark their slot as absent
  if (slot_of_new) for (int64_t r = threadIdx.x; r < n_new; r += PG_THREADS) if (!on || r >= total_free) slot_of_new[r] = -1;
}

// zero the fp32 state rows ([cap, 384] row-major) of freshly appended edges: 96 16-byte chunks per row
__global__ void __launch_bounds__(256)
pgraph_zero_rows_kernel(float* state, const int32_t* slot_of_new, int64_t n_new) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_new * 96; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / 96;
    const int c = (int)(t - r * 96);
    const int e = slot_of_new[r];
    if (e < 0) continue;
    *reinterpret_cast<float4*>(state + (int64_t)e * 384 + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// the edges DPVO adds for frame n - 1 (dpvo.py:362-375 __edges_forw / __edges_back with n >= r, the steady state):
//   forward : patches of frames [n - r, n - 1) -> frame n - 1           M (r - 1) edges
//   backward: patches of frame  n - 1          -> frames [n - r, n)     M r       edges
// written as (ii = source frame, jj = target frame, kk = patch), n read from the device
__global__ void __launch_bounds__(256)
pgraph_new_edges_kernel(const int64_t* n_dev, int M, int r, int64_t* ii, int64_t* jj, int64_t* kk) {
  const int64_t n = *n_dev;
  const int64_t nf = (int64_t)M * (r - 1), nb = (int64_t)M * r;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nf + nb; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t k, j;
    if (t < nf) { k = M * (n - r) + t; j = n - 1; }                           // meshgrid(patches, [n-1]), patch-major
    else { const int64_t u = t - nf; k = M * (n - 1) + u / r; j = (n - r) + u % r; }   // meshgrid(patches of n-1, frames), patch-major
    kk[t] = k; jj[t] = j; ii[t] = k / M;
  }
}

}  // namespace dpvo

using namespace dpvo;

extern "C" int dpvo_pgraph_remove(int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, int64_t cap, int rule,
                                  const int64_t* frame, int64_t param, const int32_t* enable, int64_t dummy_frame,
                                  int64_t dummy_patch, int M, int32_t* n_active, void* stream) {
  DPVO_REQUIRE(cap >= 0 && M > 0 && (rule == 0 || rule == 1), "pgraph_remove: bad arguments");
  if (cap == 0) return DPVO_OK;
  DPVO_REQUIRE(ii && jj && kk && active && frame && n_active, "pgraph_remove: null pointer");
  const unsigned grid = (unsigned)std::min<int64_t>((cap + 255) / 256, (int64_t)sm_count() * 4);
  return launch("pgraph_remove_kernel", pgraph_remove_kernel, grid, 256, 0, (cudaStream_t)stream, ii, jj, kk, active, cap, rule, frame, param,
                enable, dummy_frame, dummy_patch, M, n_active);
}

extern "C" int dpvo_pgraph_append(int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, int64_t cap, const int64_t* new_ii,
                                  const int64_t* new_jj, const int64_t* new_kk, int64_t n_new, const int32_t* enable,
                                  float* state, int32_t* slot_of_new, int32_t* n_active, int32_t* overflow, void* stream) {
  DPVO_REQUIRE(cap >= 0 && n_new >= 0, "pgraph_append: bad sizes");
  if (n_new == 0) return DPVO_OK;
  DPVO_REQUIRE(ii && jj && kk && active && new_ii && new_jj && new_kk && n_active, "pgraph_append: null pointer");
  DPVO_REQUIRE(!state || slot_of_new, "pgraph_append: zeroing the state rows needs the slot_of_new scratch");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = launch("pgraph_append_kernel", pgraph_append_kernel, 1, PG_THREADS, 0, st, ii, jj, kk, active, cap, new_ii, new_jj, new_kk, n_new,
                  enable, slot_of_new, n_active, overflow);
  if (rc || !state) return rc;
  const unsigned grid = (unsigned)std::min<int64_t>((n_new * 96 + 255) / 256, (int64_t)sm_count() * 8);
  return launch("pgraph_zero_rows_kernel", pgraph_zero_rows_kernel, grid, 256, 0, st, state, slot_of_new, n_new);
}

extern "C" int dpvo_pgraph_new_edges(const int64_t* n_dev, int M, int r, int64_t* ii, int64_t* jj, int64_t* kk, void* stream) {
  DPVO_REQUIRE(M > 0 && r > 1 && n_dev && ii && jj && kk, "pgraph_new_edges: bad arguments");
  const int64_t total = (int64_t)M * (2 * r - 1);
  const unsigned grid = (unsigned)((total + 255) / 256);
  return launch("pgraph_new_edges_kernel", pgraph_new_edges_kernel, grid, 256, 0, (cudaStream_t)stream, n_dev, M, r, ii, jj, kk);
}
