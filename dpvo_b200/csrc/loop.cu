// Proximity loop closure on the device (the DPV-SLAM back end of dpvo/patchgraph.py:56-91 and dpvo/dpvo.py:223-326):
//   * dpvo_loop_scores   the mean flow magnitude of every (old source frame i, recent target frame j) candidate pair
//                        (PatchGraph.edges_loop, the pops.flow_mag half of it)
//   * dpvo_loop_select   the greedy selection of reduce_edges (loop_closure/optim_utils.py:23-61) and the emission of the
//                        M edges of each accepted pair into the loop region of the edge store
//   * dpvo_pgraph_remove_store  the removal rule of keyframe() with the loop exception (dpvo.py:300-310); the removed
//                        edges go to an inactive store instead of being forgotten (remove_factors(store=True), :223-238)
//   * dpvo_loop_flags    what the host needs to decide the next update (any loop edge active, any long-range edge,
//                        the minimum active source frame), in one small record
//   * dpvo_loop_normalize  PatchGraph.normalize (patchgraph.py:84-91) before the global bundle adjustment
// The frame counter is a device scalar in every call but normalize (the global bundle adjustment around it is eager),
// and the grids are sized for the largest candidate range, so a frame's proposal, removal and flags can be captured.
#include "common.cuh"
#include "flow.cuh"

namespace dpvo {

constexpr int LOOP_THREADS = 1024;
constexpr int LOOP_MIN_GAP = 30;              // j - i < 30 is never a loop pair (optim_utils.py:44)
constexpr int LOOP_MAX_KEYS = 16384;          // candidate slots one selection CTA sorts in shared memory

struct LoopRange {
  int64_t n, l, i0, ni, j0;
};

// candidate pairs (dpvo/patchgraph.py:58-68): targets j in [n - freq, n - kf_index), sources i in [max(l - age, 0), l),
// l = n - removal; slot (jr, ir) = (j - j0, i - i0) of a fixed [J, age] layout keeps the flatmeshgrid order (j-major)
__device__ __forceinline__ LoopRange loop_range(int64_t n, int removal, int age, int freq) {
  LoopRange r;
  r.n = n; r.l = n - removal;
  r.i0 = r.l - age > 0 ? r.l - age : 0;
  r.ni = r.l > 0 ? r.l - r.i0 : 0;
  r.j0 = n - freq;
  return r;
}

// a proposal runs when n - last_global_ba >= GLOBAL_OPT_FREQ (dpvo.py:449-450)
__device__ __forceinline__ bool loop_due(int64_t n, const int64_t* last_ba, int freq) {
  return n - *last_ba >= freq;
}

// flow of the centre pixel of patch k from frame i to frame j (flow.cuh)
__device__ __forceinline__ float centre_flow(const float* __restrict__ poses, const float* __restrict__ patches,
                                             const float* __restrict__ intr, int64_t i, int64_t j, int64_t k, bool& valid) {
  return patch_flow(poses, patches, intr, i, j, k, 4, valid);
}

// one warp per candidate slot; lane l sums patches l, l + 32, ... in order, then a fixed butterfly: two launches give
// identical bits.  Slots outside the current range (or every slot, when no proposal is due) get +inf.
__global__ void __launch_bounds__(256)
loop_scores_kernel(const float* __restrict__ poses, const float* __restrict__ patches, const float* __restrict__ intr,
                   const int64_t* n_dev, const int64_t* last_ba, int M, int removal, int age, int freq, int J, float* scores) {
  const int64_t slot = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (slot >= (int64_t)J * age) return;
  const int jr = (int)(slot / age), ir = (int)(slot - (int64_t)jr * age);
  const LoopRange r = loop_range(*n_dev, removal, age, freq);
  const int64_t i = r.i0 + ir, j = r.j0 + jr;
  float score = INFINITY;
  if (loop_due(r.n, last_ba, freq) && ir < r.ni && j >= 0) {
    float sum = 0.f;
    int cnt = 0;
    for (int m = lane; m < M; m += 32) {
      bool ok;
      const float f = centre_flow(poses, patches, intr, i, j, i * M + m, ok);
      if (ok) { sum += f; ++cnt; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sum += __shfl_xor_sync(0xffffffffu, sum, o);
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((float)cnt > 0.75f * (float)M) score = sum / (float)cnt;
  }
  if (lane == 0) scores[slot] = score;
}

// reduce_edges (optim_utils.py:23-61) in one CTA: keep the slots with score < thresh, sort them by (score, slot) --
// the slot order is the candidate order, so ties resolve as a stable sort would -- then walk them in order: skip
// j - i < 30 and suppressed pairs, accept the rest and suppress (i +- 1, j), stop at max_pairs accepted.
__global__ void __launch_bounds__(LOOP_THREADS)
loop_select_kernel(const float* __restrict__ scores, const int64_t* n_dev, int64_t* last_ba, int removal, int age, int freq,
                   int J, int P2, float thresh, int max_pairs, int64_t* pairs, int32_t* n_pairs) {
  extern __shared__ unsigned long long keys[];                  // [P2] sort keys, then [J * age] suppression bytes
  uint8_t* sup = reinterpret_cast<uint8_t*>(keys + P2);
  __shared__ int nkeys;
  const LoopRange r = loop_range(*n_dev, removal, age, freq);
  if (!loop_due(r.n, last_ba, freq)) {                          // no proposal this frame: no pair, nothing emitted
    if (threadIdx.x == 0) *n_pairs = 0;
    return;
  }
  const int S = J * age;
  if (threadIdx.x == 0) nkeys = 0;
  __syncthreads();
  for (int s = threadIdx.x; s < S; s += LOOP_THREADS) {
    sup[s] = 0;
    const float v = scores[s];
    if (v < thresh && v < 1000.f) {                             // optim_utils.py:47: mag >= 1000 counts as inf
      const int at = atomicAdd(&nkeys, 1);                      // placement order is irrelevant: the sort fixes it
      keys[at] = ((unsigned long long)__float_as_uint(v) << 32) | (unsigned)s;   // v >= 0: bits order as values
    }
  }
  __syncthreads();
  const int nk = nkeys;
  int p2 = 1;
  while (p2 < nk) p2 <<= 1;
  for (int s = nk + threadIdx.x; s < p2; s += LOOP_THREADS) keys[s] = ~0ull;
  __syncthreads();
  // bitonic sort of p2 keys
  for (int k = 2; k <= p2; k <<= 1) {
    for (int jst = k >> 1; jst > 0; jst >>= 1) {
      for (int t = threadIdx.x; t < p2; t += LOOP_THREADS) {
        const int u = t ^ jst;
        if (u > t) {
          const unsigned long long a = keys[t], b = keys[u];
          const bool up = (t & k) == 0;
          if ((a > b) == up) { keys[t] = b; keys[u] = a; }
        }
      }
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) {
    int cnt = 0;
    for (int q = 0; q < nk && cnt < max_pairs; ++q) {
      const int s = (int)(keys[q] & 0xffffffffu);
      const int jr = s / age, ir = s - jr * age;
      const int64_t i = r.i0 + ir, j = r.j0 + jr;
      if (j - i < LOOP_MIN_GAP || sup[s]) continue;
      pairs[2 * cnt] = i; pairs[2 * cnt + 1] = j;
      ++cnt;
      sup[s] = 1;
      if (ir > 0) sup[s - 1] = 1;
      if (ir + 1 < age) sup[s + 1] = 1;
    }
    *n_pairs = cnt;
    if (cnt > 0) *last_ba = r.n;                                // dpvo.py:452-454
  }
}

// the M edges of accepted pair p go to loop-region slots p M + m: (ii, jj, kk) = (i, j, i M + m), state row zeroed
__global__ void __launch_bounds__(256)
loop_emit_kernel(const int64_t* pairs, const int32_t* n_pairs, int M, int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, int64_t region, float* state,
                 int32_t* n_active, int32_t* overflow) {
  const int64_t ne = (int64_t)(*n_pairs) * M;                   // this frame's count: 0 when no proposal ran
  int placed = 0, clash = 0;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < ne * 96; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = t / 96;
    const int c = (int)(t - e * 96);
    if (c == 0) {
      const int64_t p = e / M, m = e - p * M;
      const int64_t i = pairs[2 * p], j = pairs[2 * p + 1];
      clash += active[e] ? 1 : 0;
      placed += active[e] ? 0 : 1;
      ii[e] = i; jj[e] = j; kk[e] = i * M + m; active[e] = 1;
    }
    if (state) *reinterpret_cast<float4*>(state + e * 384 + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int o = 16; o > 0; o >>= 1) {
    placed += __shfl_xor_sync(0xffffffffu, placed, o);
    clash += __shfl_xor_sync(0xffffffffu, clash, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (placed) atomicAdd(n_active, placed);
    if (clash && overflow) *overflow = 1;                       // a loop edge was still active: it has been replaced
  }
}

// keyframe()'s removal with the loop exception (dpvo.py:300-310) that keeps what it removes (:223-238):
//   drop = kk / M < n - removal  &&  !((jj - ii) > 30 && jj > n - opt_window)
// One CTA, as pgraph_append: each thread owns a contiguous slot range, a block scan ranks the removed edges in slot
// order.  The store fills from its END downwards, one block of the removals of each call, so its used part
// [s_cap - count, s_cap) always ends where the active store begins and the two form one edge list.
__global__ void __launch_bounds__(LOOP_THREADS)
pgraph_remove_store_kernel(int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, const float* target, const float* weight,
                           int64_t cap, const int64_t* n_dev, int removal, int opt_window, const int32_t* enable,
                           int64_t dummy_frame, int64_t dummy_patch, int M, int32_t* n_active, int64_t* s_ii, int64_t* s_jj,
                           int64_t* s_kk, float* s_target, float* s_weight, int64_t s_cap, int32_t* s_count, int32_t* s_overflow) {
  __shared__ int warp_tot[LOOP_THREADS / 32 + 1];
  if (enable && *enable == 0) return;
  const int64_t n = *n_dev;
  const int64_t per = (cap + LOOP_THREADS - 1) / LOOP_THREADS;
  const int64_t e0 = min(cap, (int64_t)threadIdx.x * per), e1 = min(cap, e0 + per);
  auto drops = [&](int64_t e) {
    if (!active[e]) return false;
    const int64_t i = ii[e], j = jj[e];
    return kk[e] / M < n - removal && !((j - i) > LOOP_MIN_GAP && j > n - opt_window);
  };
  int cnt = 0;
  for (int64_t e = e0; e < e1; ++e) cnt += drops(e) ? 1 : 0;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int q = 0; q < LOOP_THREADS / 32; ++q) { const int t = warp_tot[q]; warp_tot[q] = run; run += t; }
    warp_tot[LOOP_THREADS / 32] = run;
  }
  __syncthreads();
  const int total = warp_tot[LOOP_THREADS / 32];
  const int64_t used = *s_count;
  const int64_t room = s_cap - used;
  const int64_t kept = total < room ? total : room;            // removals beyond the capacity are lost (and reported)
  const int64_t base = s_cap - used - kept;
  int64_t rank = warp_tot[w] + inc - cnt;
  for (int64_t e = e0; e < e1; ++e) {
    if (!drops(e)) continue;
    if (rank < kept) {
      const int64_t d = base + rank;
      s_ii[d] = ii[e]; s_jj[d] = jj[e]; s_kk[d] = kk[e];
      s_target[2 * d] = target[2 * e]; s_target[2 * d + 1] = target[2 * e + 1];
      s_weight[2 * d] = weight[2 * e]; s_weight[2 * d + 1] = weight[2 * e + 1];
    }
    ++rank;
    ii[e] = dummy_frame; jj[e] = dummy_frame; kk[e] = dummy_patch; active[e] = 0;
  }
  __syncthreads();                                              // every thread has read s_count
  if (threadIdx.x == 0) {
    if (total) atomicSub(n_active, total);
    *s_count = (int32_t)(used + kept);
    if (kept < total && s_overflow) *s_overflow = 1;
  }
}

// flags[0] = 1 + the offset of the last active edge in the loop region [normal, cap), 0 without one; flags[1] = 1 if an active edge has
// ii < n - removal - 1 (the global bundle adjustment condition, dpvo.py:348); flags[2] = min active ii (INT64_MAX
// without one); flags[3] = the inactive store's count (copied, so one read brings the host everything)
__global__ void __launch_bounds__(LOOP_THREADS)
loop_flags_kernel(const int64_t* ii, const uint8_t* active, int64_t cap, int64_t normal, int64_t n, int removal,
                  const int32_t* s_count, int64_t* flags) {
  __shared__ int64_t red[3][LOOP_THREADS / 32];
  int longr = 0;
  int64_t used = 0, mn = INT64_MAX;                             // used: 1 + the last active loop-region slot
  for (int64_t e = threadIdx.x; e < cap; e += LOOP_THREADS) {
    if (!active[e]) continue;
    const int64_t i = ii[e];
    if (e >= normal) used = e - normal + 1;                     // e ascends: the last one seen is this thread's largest
    longr |= i < n - removal - 1;
    mn = i < mn ? i : mn;
  }
  longr = __any_sync(0xffffffffu, longr);
  for (int o = 16; o > 0; o >>= 1) {
    const int64_t t = __shfl_xor_sync(0xffffffffu, mn, o);
    mn = t < mn ? t : mn;
    const int64_t u = __shfl_xor_sync(0xffffffffu, used, o);
    used = u > used ? u : used;
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[0][w] = used; red[1][w] = longr; red[2][w] = mn; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t a = 0, b = 0, c = INT64_MAX;
    for (int q = 0; q < LOOP_THREADS / 32; ++q) { a = red[0][q] > a ? red[0][q] : a; b |= red[1][q]; c = red[2][q] < c ? red[2][q] : c; }
    flags[0] = a; flags[1] = b; flags[2] = c; flags[3] = s_count ? *s_count : 0;
  }
}

// PatchGraph.normalize (patchgraph.py:84-91): s = mean of every depth value of patches[:n] (fp64, a fixed order:
// two launches give the same bits), depths /= s, translations *= s, the translations of the n_delta relative poses of
// a keyframe delta table (keyframe.cu) *= s, then every pose is rebased on pose 0
__global__ void __launch_bounds__(LOOP_THREADS)
loop_normalize_kernel(float* poses, float* patches, int64_t n, int M, int P, float* delta, int64_t n_delta) {
  __shared__ double red[LOOP_THREADS / 32];
  __shared__ float s_sh;
  __shared__ float p0[7];
  const int PP = P * P;
  const int64_t cnt = n * M * PP;
  double acc = 0.0;
  for (int64_t t = threadIdx.x; t < cnt; t += LOOP_THREADS) {
    const int64_t k = t / PP;
    acc += (double)patches[(k * 3 + 2) * PP + (t - k * PP)];
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int q = 0; q < LOOP_THREADS / 32; ++q) tot += red[q];
    s_sh = (float)(tot / (double)cnt);
    for (int c = 0; c < 7; ++c) p0[c] = poses[c] * (c < 3 ? s_sh : 1.f);
  }
  __syncthreads();
  const float s = s_sh;
  for (int64_t t = threadIdx.x; t < cnt; t += LOOP_THREADS) {
    const int64_t k = t / PP;
    patches[(k * 3 + 2) * PP + (t - k * PP)] /= s;
  }
  for (int64_t t = threadIdx.x; t < 3 * n_delta; t += LOOP_THREADS) delta[7 * (t / 3) + t % 3] *= s;   // dP.scale(s)
  using namespace lie;
  const SE3<float> P0inv = se3_inv(se3_load(p0));
  for (int64_t t = threadIdx.x; t < n; t += LOOP_THREADS) {
    float q[7];
    for (int c = 0; c < 7; ++c) q[c] = poses[7 * t + c] * (c < 3 ? s : 1.f);
    se3_store(se3_mul(se3_load(q), P0inv), poses + 7 * t);
  }
}

}  // namespace dpvo

using namespace dpvo;

namespace {
int loop_range_ok(int M, int removal, int max_age, int freq, int kf_index) {
  DPVO_REQUIRE(M > 0 && max_age > 0 && removal > 0 && kf_index >= 0 && freq > kf_index,
               "loop: bad range (M=%d, removal=%d, max_edge_age=%d, global_opt_freq=%d, keyframe_index=%d)", M, removal,
               max_age, freq, kf_index);
  const int64_t S = (int64_t)(freq - kf_index) * max_age;
  if (S > LOOP_MAX_KEYS) {
    set_error("loop: %lld candidate pairs per proposal ((global_opt_freq - keyframe_index) * max_edge_age); one selection holds %d",
              (long long)S, LOOP_MAX_KEYS);
    return DPVO_ERR_UNSUPPORTED;
  }
  return DPVO_OK;
}
}  // namespace

extern "C" int64_t dpvo_loop_candidates(int max_age, int freq, int kf_index) {
  if (max_age <= 0 || kf_index < 0 || freq <= kf_index) return 0;
  return (int64_t)(freq - kf_index) * max_age;
}

extern "C" int dpvo_loop_scores(const float* poses, const float* patches, const float* intrinsics, const int64_t* n_dev,
                                const int64_t* last_ba, int M, int removal, int max_age, int freq, int kf_index,
                                float* scores, void* stream) {
  const int rc = loop_range_ok(M, removal, max_age, freq, kf_index);
  if (rc != DPVO_OK) return rc;
  DPVO_REQUIRE(poses && patches && intrinsics && n_dev && last_ba && scores, "loop_scores: null pointer");
  const int J = freq - kf_index;
  const int64_t threads = (int64_t)J * max_age * 32;
  return launch("loop_scores_kernel", loop_scores_kernel, (unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream,
                poses, patches, intrinsics, n_dev, last_ba, M, removal, max_age, freq, J, scores);
}

extern "C" int dpvo_loop_select(const float* scores, const int64_t* n_dev, int64_t* last_ba, int M, int removal, int max_age,
                                int freq, int kf_index, float thresh, int max_pairs, int64_t* pairs, int32_t* n_pairs,
                                int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, int64_t region, float* state,
                                int32_t* n_active, int32_t* overflow, void* stream) {
  const int rc = loop_range_ok(M, removal, max_age, freq, kf_index);
  if (rc != DPVO_OK) return rc;
  DPVO_REQUIRE(max_pairs > 0, "loop_select: max_pairs=%d must be positive", max_pairs);
  DPVO_REQUIRE(region >= (int64_t)max_pairs * M, "loop_select: a loop region of %lld slots cannot hold %d pairs of %d edges",
               (long long)region, max_pairs, M);
  DPVO_REQUIRE(scores && n_dev && last_ba && pairs && n_pairs && ii && jj && kk && active && n_active,
               "loop_select: null pointer");
  const int J = freq - kf_index, S = J * max_age;
  int p2 = 1;
  while (p2 < S) p2 <<= 1;
  const size_t smem = (size_t)p2 * 8 + (size_t)S;
  cudaStream_t st = (cudaStream_t)stream;
  const int e = launch("loop_select_kernel", loop_select_kernel, 1, LOOP_THREADS, smem, st, scores, n_dev, last_ba, removal, max_age, freq, J, p2,
                       thresh, max_pairs, pairs, n_pairs);
  if (e != DPVO_OK) return e;
  const int64_t work = (int64_t)max_pairs * M * 96;
  const unsigned grid = (unsigned)std::min<int64_t>((work + 255) / 256, (int64_t)sm_count() * 8);
  return launch("loop_emit_kernel", loop_emit_kernel, grid, 256, 0, st, pairs, n_pairs, M, ii, jj, kk, active, region, state, n_active, overflow);
}

extern "C" int dpvo_pgraph_remove_store(int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, const float* target,
                                        const float* weight, int64_t cap, const int64_t* n_dev, int removal, int opt_window,
                                        const int32_t* enable, int64_t dummy_frame, int64_t dummy_patch, int M,
                                        int32_t* n_active, int64_t* s_ii, int64_t* s_jj, int64_t* s_kk, float* s_target,
                                        float* s_weight, int64_t s_cap, int32_t* s_count, int32_t* s_overflow, void* stream) {
  DPVO_REQUIRE(cap >= 0 && s_cap >= 0 && M > 0 && removal > 0 && opt_window > 0,
               "pgraph_remove_store: bad arguments (cap=%lld, store=%lld, M=%d, removal=%d, opt_window=%d)", (long long)cap,
               (long long)s_cap, M, removal, opt_window);
  DPVO_REQUIRE(s_cap <= INT32_MAX, "pgraph_remove_store: an inactive store of %lld slots exceeds the int32 count", (long long)s_cap);
  if (cap == 0) return DPVO_OK;
  DPVO_REQUIRE(ii && jj && kk && active && target && weight && n_dev && n_active && s_count, "pgraph_remove_store: null pointer");
  DPVO_REQUIRE(s_cap == 0 || (s_ii && s_jj && s_kk && s_target && s_weight), "pgraph_remove_store: null store pointer");
  return launch("pgraph_remove_store_kernel", pgraph_remove_store_kernel, 1, LOOP_THREADS, 0, (cudaStream_t)stream, ii, jj, kk, active, target,
                weight, cap, n_dev, removal, opt_window, enable, dummy_frame, dummy_patch, M, n_active, s_ii, s_jj, s_kk, s_target, s_weight,
                s_cap, s_count, s_overflow);
}

extern "C" int dpvo_loop_flags(const int64_t* ii, const uint8_t* active, int64_t cap, int64_t normal, int64_t n, int removal,
                               const int32_t* s_count, int64_t* flags, void* stream) {
  DPVO_REQUIRE(cap >= 0 && normal >= 0 && normal <= cap, "loop_flags: bad sizes (cap=%lld, normal=%lld)", (long long)cap,
               (long long)normal);
  DPVO_REQUIRE(flags && (cap == 0 || (ii && active)), "loop_flags: null pointer");
  return launch("loop_flags_kernel", loop_flags_kernel, 1, LOOP_THREADS, 0, (cudaStream_t)stream, ii, active, cap, normal, n, removal, s_count,
                flags);
}

extern "C" int dpvo_loop_normalize_deltas(float* poses, float* patches, int64_t n, int M, int P, float* delta, int64_t n_delta,
                                          void* stream) {
  DPVO_REQUIRE(n >= 0 && M > 0 && P > 0 && n_delta >= 0, "loop_normalize: bad sizes (n=%lld, M=%d, P=%d, deltas=%lld)", (long long)n, M,
               P, (long long)n_delta);
  if (n == 0) return DPVO_OK;
  DPVO_REQUIRE(poses && patches && (delta || n_delta == 0), "loop_normalize: null pointer");
  return launch("loop_normalize_kernel", loop_normalize_kernel, 1, LOOP_THREADS, 0, (cudaStream_t)stream, poses, patches, n, M, P, delta, n_delta);
}

extern "C" int dpvo_loop_normalize(float* poses, float* patches, int64_t n, int M, int P, void* stream) {
  return dpvo_loop_normalize_deltas(poses, patches, n, M, P, nullptr, 0, stream);
}
