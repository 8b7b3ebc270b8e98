// SoftAgg (blocks.py:31-43, net.py:87-88): the stacked f|g dense layer fused with its segment softmax (wgmma, sm_90a).
//
//   y[g, c] = sum_{i in g} softmax_g(G[i, c]) F[i, c]      F = fp16(X[order[i]] Wf^T + bf),  G = fp16(X[order[i]] Wg^T + bg)
//
// over the CSR of dpvo_group_edges (sorted positions i, group_start).  The [E, 2 dim] f|g output of the layer exists
// only to be reduced per group and channel, and the softmax is channel-wise, so a CTA that owns a channel slice
// finishes the reduction on chip: the layer's output never reaches global memory.
//
// softagg_fused_kernel: persistent, one CTA per SM, each CTA owns one 96-channel slice of the 384 channels for its
// whole life (CTA b: slice b % 4) and walks 64-row tiles of the sorted positions.
//   warps 8-11 producers    load the slice's 192 weight rows [Wf rows c..c+95 ; Wg rows c..c+95] once (6 k-blocks,
//                           144 KB, resident), then gather X[order[i]] rows with 16-byte cp.async into a 4-deep ring of
//                           64-row k-blocks in the SWIZZLE_128B K-major layout the descriptors expect
//   warps 0-7  consumers    two warpgroups taking alternate tiles of the CTA, so one warpgroup's reduction overlaps the
//                           other's MMAs.  wgmma.m64n192k16 puts f in acc[4 j ..] and g in acc[4 (j + 12) ..] for the same
//                           rows and channels of the same thread; the epilogue rounds f and g to fp16 where the separate
//                           layer rounds its output, stages the (f, g) pairs in shared memory, and 96 threads (one per
//                           channel) reduce each group segment of the tile over its rows in sorted order with
//                           softagg_reduce's arithmetic (half max, exp2f(g log2e - m log2e), fp32 sums, fp16 a / z).
//                           The segments come from the rows' group ids, prefetched during the MMAs.
// A group that lies inside one tile is written to y directly.  The first and the last segment of a tile may continue in
// the neighbouring tile: such a segment leaves its (max, sum of weights, weighted sum) per channel in a record
// [tile][first | last][3][dim], and softagg_combine_kernel merges the records of each crossing group in tile order and
// zeroes the padding rows of y.  No float atomics: every output element is written by one thread in a fixed order,
// so two launches give bit-identical results.
#include "common.cuh"
#include "tc.cuh"

namespace dpvo {

constexpr int SF_DIM = 384;                    // channels = K of the layer
constexpr int SF_CH = 96;                      // channels per CTA slice
constexpr int SF_SLICES = SF_DIM / SF_CH;
constexpr int SF_N = 2 * SF_CH;                // wgmma N: the slice's f and g columns
constexpr int SF_PAIRS = SF_CH / 2;            // channel pairs of a slice (staged (f, g) slots per row)
constexpr int SF_M = 64;                       // rows per tile (one warpgroup)
constexpr int SF_K = 64;                       // halves per k-block: 128 bytes, one swizzle atom
constexpr int SF_KB = SF_DIM / SF_K;
constexpr int SF_STAGES = 4;
// cp.async groups in flight per producer thread; a consumer returns the stage of k-block i - 1 only after it has issued
// the MMAs of k-block i, so LOOK must stay below ring depth - 1 (as in gemm.cu)
constexpr int SF_LOOK = SF_STAGES - 2;
constexpr int SF_CONS_THREADS = 256, SF_PROD_THREADS = 128, SF_THREADS = SF_CONS_THREADS + SF_PROD_THREADS;
constexpr int SF_A_BYTES = SF_M * 128, SF_B_BYTES = SF_N * 128;
constexpr int SF_REC = 3 * SF_DIM;             // floats per record: max, sum of weights, weighted sum
constexpr size_t SF_SMEM = (size_t)SF_KB * SF_B_BYTES + (size_t)SF_STAGES * SF_A_BYTES +
                           2 * SF_M * SF_PAIRS * sizeof(uint2) + 2 * SF_M * sizeof(int) + 3 * SF_STAGES * sizeof(uint64_t) + 1024;
static_assert(SF_SMEM <= 227 * 1024, "softagg_fused: shared memory");

__device__ __forceinline__ uint32_t h2_bits(__half2 v) { return *reinterpret_cast<uint32_t*>(&v); }
__device__ __forceinline__ __half2 bits_h2(uint32_t v) { return *reinterpret_cast<__half2*>(&v); }
// staged (f, g) pair of row r, channel pair p: the slot is XOR-swizzled by the row so that the fragment-layout writes
// (8 rows x 4 pairs per half warp) and the row-wise reads (48 pairs of one row) are both free of bank conflicts
__device__ __forceinline__ int sf_slot(int r, int p) { return r * SF_PAIRS + (p ^ ((r & 3) << 2)); }

__global__ void __launch_bounds__(SF_THREADS, 1)
softagg_fused_kernel(const __half* __restrict__ X, int64_t ldx, const int32_t* __restrict__ order,
                     const int32_t* __restrict__ group_of, const __half* __restrict__ W, const float* __restrict__ bias, __half* __restrict__ y,
                     float* __restrict__ rec, int E, int max_groups) {
  constexpr float LOG2E = 1.4426950408889634f;
  extern __shared__ unsigned char sf_smem_raw[];
  unsigned char* base = sf_smem_raw + ((1024u - (smem_u32(sf_smem_raw) & 1023u)) & 1023u);
  unsigned char* sB = base;                                        // resident weights, SF_KB k-blocks
  unsigned char* sA = sB + SF_KB * SF_B_BYTES;                      // operand ring
  uint2* sT = reinterpret_cast<uint2*>(sA + SF_STAGES * SF_A_BYTES); // [warpgroup][row][pair] staged (f, g)
  int* sGid = reinterpret_cast<int*>(sT + 2 * SF_M * SF_PAIRS);     // [warpgroup][row] group of the row
  // full[wg][stage]: each consumer warpgroup has its own full barriers.  A shared set would be ambiguous at the first
  // k-block of a tile, whose stage's previous fill belongs to the other warpgroup's tile and may be pending or already
  // followed by this fill: a parity wait cannot tell one phase behind from one phase ahead.  Per warpgroup, a stage's
  // barrier is never more than one phase ahead of its consumer.  The stage is released in fill order either way.
  uint64_t* full = reinterpret_cast<uint64_t*>(sGid + 2 * SF_M);
  uint64_t* empty = full + 2 * SF_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slice = blockIdx.x % SF_SLICES;
  const int tile0 = blockIdx.x / SF_SLICES, tstep = gridDim.x / SF_SLICES;
  const int n_tiles = (E + SF_M - 1) / SF_M;

  if (threadIdx.x == 0) {
    for (int s = 0; s < SF_STAGES; ++s) { mbar_init(&full[s], SF_PROD_THREADS); mbar_init(&full[SF_STAGES + s], SF_PROD_THREADS); mbar_init(&empty[s], 4); }
    mbar_init_fence();
  }
  __syncthreads();

  if (warp >= SF_CONS_THREADS / 32) {
    // =========================================================================== producers
    const int pt = threadIdx.x - SF_CONS_THREADS;
    // the slice's weights as the first cp.async group of every producer thread: a thread signals a k-block only after
    // its groups up to that k-block have landed, so every full barrier also publishes the weights
    const __half* wsl = W + (int64_t)slice * SF_N * SF_DIM;
    for (int c = pt; c < SF_KB * SF_N * 8; c += SF_PROD_THREADS) {
      const int kb = c / (SF_N * 8), row = (c >> 3) % SF_N, ch = c & 7;
      cp_async16(smem_u32(sB + kb * SF_B_BYTES + row * 128 + ((ch ^ (row & 7)) << 4)), wsl + (int64_t)row * SF_DIM + kb * SF_K + ch * 8, 16);
    }
    cp_async_commit();
    uint32_t it = 0;                          // k-block counter over all tiles of this CTA
    // k-block j belongs to the CTA's tile j / SF_KB, which the consumer warpgroup (j / SF_KB) % 2 takes
    auto arrive_full = [&](uint32_t j) { mbar_arrive(&full[((j / SF_KB) & 1) * SF_STAGES + j % SF_STAGES]); };
    int nsrc[4];                              // source rows of the next tile, fetched one tile ahead
    auto fetch_rows = [&](int tile) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int pos = tile * SF_M + ((pt + SF_PROD_THREADS * i) >> 3);
        nsrc[i] = (tile < n_tiles && pos < E) ? order[pos] : -1;
      }
    };
    fetch_rows(tile0);
    for (int tile = tile0; tile < n_tiles; tile += tstep) {
      const __half* arow[4]; uint32_t aoff[4], abytes[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = pt + SF_PROD_THREADS * i, row = c >> 3, ch = c & 7;
        const bool ok = nsrc[i] >= 0;
        arow[i] = X + (ok ? (int64_t)nsrc[i] : 0) * ldx + ch * 8;
        abytes[i] = ok ? 16u : 0u;
        aoff[i] = row * 128 + ((ch ^ (row & 7)) << 4);
      }
      fetch_rows(tile + tstep);
      for (int kb = 0; kb < SF_KB; ++kb, ++it) {
        const uint32_t s = it % SF_STAGES, ph = (it / SF_STAGES) & 1;
        mbar_wait(&empty[s], ph ^ 1);
        const uint32_t da = smem_u32(sA + s * SF_A_BYTES);
#pragma unroll
        for (int i = 0; i < 4; ++i) cp_async16(da + aoff[i], arow[i] + kb * SF_K, abytes[i]);
        cp_async_commit();
        if (it >= SF_LOOK) {
          cp_async_wait<SF_LOOK>();
          fence_proxy_async();
          arrive_full(it - SF_LOOK);
        }
      }
    }
    cp_async_wait<0>();
    fence_proxy_async();
    for (uint32_t j = (it >= SF_LOOK ? it - SF_LOOK : 0); j < it; ++j) arrive_full(j);
  } else {
    // =========================================================================== consumers: MMA + segment softmax
    const int wg = warp >> 2, wq = warp & 3, t = threadIdx.x & 127;
    uint2* tT = sT + wg * SF_M * SF_PAIRS;
    int* gid = sGid + wg * SF_M;
    const float* bsl = bias + slice * SF_N;
    uint64_t* wfull = full + wg * SF_STAGES;
    uint32_t phases = 0;                      // bit s: parity of this warpgroup's next fill of stage s
    float acc[96];
    auto release = [&](uint32_t s) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[s]); };
    uint32_t n = wg;                          // this tile's index among the CTA's tiles: its k-blocks are n * SF_KB ..
    for (int tile = tile0 + wg * tstep; tile < n_tiles; tile += 2 * tstep, n += 2) {
      const int m0 = tile * SF_M, nrows = min(SF_M, E - m0);
      // groups of the tile's rows and of the rows just before and after it, in flight during the MMAs
      const int my_gid = t < nrows ? group_of[order[m0 + t]] : -1;
      const int gid_before = m0 > 0 ? group_of[order[m0 - 1]] : -1;
      const int gid_after = m0 + SF_M < E ? group_of[order[m0 + SF_M]] : -1;
      uint32_t it = n * SF_KB, prev = 0;
      for (int kb = 0; kb < SF_KB; ++kb, ++it) {
        const uint32_t s = it % SF_STAGES;
        mbar_wait(&wfull[s], (phases >> s) & 1);
        phases ^= 1u << s;
        const uint64_t ad = wgmma_desc_sw128(smem_u32(sA + s * SF_A_BYTES));
        const uint64_t bd = wgmma_desc_sw128(smem_u32(sB + kb * SF_B_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < SF_K / 16; ++k) wgmma_m64n192k16(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (kb | k) != 0);
        wgmma_commit();
        if (kb > 0) { wgmma_wait<1>(); release(prev); }
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release(prev);

      named_bar_sync(1 + wg, 128);            // this warpgroup's previous reduction has finished reading tT / gid
      if (t < SF_M) gid[t] = my_gid;
      // fp16 f and g of rows r0, r0 + 8; channels 8 j + 2 (lane % 4) + {0, 1} of the slice = channel pair 4 j + lane % 4
      const int r0 = wq * 16 + (lane >> 2), q = lane & 3;
#pragma unroll
      for (int j = 0; j < SF_CH / 8; ++j) {
        const float2 bf = *reinterpret_cast<const float2*>(bsl + 8 * j + 2 * q);
        const float2 bg = *reinterpret_cast<const float2*>(bsl + SF_CH + 8 * j + 2 * q);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int r = r0 + 8 * rr;
          const __half2 f2 = __floats2half2_rn(acc[4 * j + 2 * rr] + bf.x, acc[4 * j + 2 * rr + 1] + bf.y);
          const __half2 g2 = __floats2half2_rn(acc[4 * (j + 12) + 2 * rr] + bg.x, acc[4 * (j + 12) + 2 * rr + 1] + bg.y);
          tT[sf_slot(r, 4 * j + q)] = make_uint2(h2_bits(f2), h2_bits(g2));
        }
      }
      named_bar_sync(1 + wg, 128);
      if (t < SF_CH) {                        // warps 0-2: one channel per thread
        // rows where a group segment starts, as a 64-bit mask that every lane builds from two ballots
        const int ga = gid[lane], gb = gid[lane + 32];
        const int pa = lane > 0 ? gid[lane - 1] : -2, pb = gid[lane + 31];
        const uint64_t starts = ((uint64_t)__ballot_sync(0xffffffffu, lane + 32 < nrows && gb != pb) << 32) |
                                __ballot_sync(0xffffffffu, lane < nrows && ga != pa);
        const int ch = slice * SF_CH + t, p = t >> 1, hi = t & 1;
        for (uint64_t mk = starts; mk;) {
          const int r = __ffsll((long long)mk) - 1;
          mk &= mk - 1;
          const int r1 = mk ? __ffsll((long long)mk) - 1 : nrows;
          const int g = gid[r];
          __half mx = __float2half_rn(-INFINITY);
#pragma unroll 4
          for (int i = r; i < r1; ++i) {
            const __half2 gv = bits_h2(tT[sf_slot(i, p)].y);
            mx = __hmax(mx, hi ? __high2half(gv) : __low2half(gv));
          }
          const float m = __half2float(mx), ml = m * LOG2E;
          float z = 0.f, a = 0.f;
#pragma unroll 4
          for (int i = r; i < r1; ++i) {
            const uint2 v = tT[sf_slot(i, p)];
            const __half2 fv = bits_h2(v.x), gv = bits_h2(v.y);
            const float w = exp2f((hi ? __high2float(gv) : __low2float(gv)) * LOG2E - ml);   // exp(g - max), <= 1
            z += w; a += w * (hi ? __high2float(fv) : __low2float(fv));
          }
          // a segment that continues before the tile's first row or after its last row is a partial result
          const bool open_lo = r == 0 && g == gid_before, open_hi = r1 == nrows && g == gid_after;
          if (open_lo || open_hi) {
#pragma unroll
            for (int slot = 0; slot < 2; ++slot) {
              if (!(slot ? open_hi : open_lo)) continue;
              float* R = rec + (int64_t)(2 * tile + slot) * SF_REC + ch;
              R[0] = m; R[SF_DIM] = z; R[2 * SF_DIM] = a;
            }
          } else if (g < max_groups) {
            y[(int64_t)g * SF_DIM + ch] = __float2half_rn(a / z);
          }
        }
      }
    }
  }
}

// One CTA per group (grid-stride), one thread per channel pair: merges the records of a group whose rows span more than
// one tile -- the last segment of its first tile, then the first segment of each following tile -- and writes zeros to
// the rows of y past the true group count, so that y is defined on all max_groups rows as softagg_reduce leaves it.
__global__ void __launch_bounds__(SF_DIM / 2)
softagg_combine_kernel(const int32_t* __restrict__ group_start, const int32_t* __restrict__ n_groups,
                       const float* __restrict__ rec, __half* __restrict__ y, int max_groups) {
  constexpr float LOG2E = 1.4426950408889634f;
  const int G = min(*n_groups, max_groups);
  const int ch = 2 * threadIdx.x;
  for (int g = blockIdx.x; g < max_groups; g += gridDim.x) {
    __half2* out = reinterpret_cast<__half2*>(y + (int64_t)g * SF_DIM + ch);
    if (g >= G) { *out = __float2half2_rn(0.f); continue; }
    const int s = group_start[g], e = group_start[g + 1];
    const int t0 = s / SF_M, t1 = (e - 1) / SF_M;
    if (e <= s || t0 == t1) continue;                      // written by softagg_fused_kernel
    float2 M = make_float2(-INFINITY, -INFINITY);
    for (int t = t0; t <= t1; ++t) {
      const float2 m = *reinterpret_cast<const float2*>(rec + (int64_t)(2 * t + (t == t0)) * SF_REC + ch);
      M.x = fmaxf(M.x, m.x); M.y = fmaxf(M.y, m.y);
    }
    const float ML0 = M.x * LOG2E, ML1 = M.y * LOG2E;
    float z0 = 0.f, z1 = 0.f, a0 = 0.f, a1 = 0.f;
    for (int t = t0; t <= t1; ++t) {
      const float* R = rec + (int64_t)(2 * t + (t == t0)) * SF_REC + ch;
      const float2 m = *reinterpret_cast<const float2*>(R), z = *reinterpret_cast<const float2*>(R + SF_DIM),
                   a = *reinterpret_cast<const float2*>(R + 2 * SF_DIM);
      const float c0 = exp2f(m.x * LOG2E - ML0), c1 = exp2f(m.y * LOG2E - ML1);
      z0 += c0 * z.x; a0 += c0 * a.x;
      z1 += c1 * z.y; a1 += c1 * a.y;
    }
    *out = __floats2half2_rn(a0 / z0, a1 / z1);
  }
}

}  // namespace dpvo

using namespace dpvo;

extern "C" int64_t dpvo_softagg_fused_workspace_bytes(int64_t E) {
  return (E < 0 ? 0 : (E + SF_M - 1) / SF_M) * 2 * SF_REC * (int64_t)sizeof(float);
}

extern "C" int dpvo_softagg_fused(const void* x16, int64_t ldx, const int32_t* order, const int32_t* group_of,
                                  const int32_t* group_start, const int32_t* n_groups, const void* w16, const float* bias,
                                  int64_t E, int64_t max_groups, void* y16, void* workspace, int64_t workspace_bytes,
                                  int dim, void* stream) {
  DPVO_REQUIRE(E >= 0 && E < (1ll << 31) && max_groups >= 0 && max_groups < (1ll << 31), "softagg_fused: bad sizes");
  DPVO_REQUIRE(dim == SF_DIM, "softagg_fused: dim=%d, the kernel is built for %d channels", dim, SF_DIM);
  if (max_groups == 0) return DPVO_OK;
  DPVO_REQUIRE(group_start && n_groups && y16 && (E == 0 || (x16 && order && group_of && w16 && bias && workspace)),
               "softagg_fused: null pointer");
  DPVO_REQUIRE(ldx >= dim && ldx % 8 == 0 && ((uintptr_t)x16 & 15) == 0 && ((uintptr_t)w16 & 15) == 0,
               "softagg_fused: X / W rows must be 16-byte aligned");
  DPVO_REQUIRE(((uintptr_t)bias & 7) == 0 && ((uintptr_t)y16 & 3) == 0 && ((uintptr_t)workspace & 7) == 0,
               "softagg_fused: bias, y or workspace misaligned");
  DPVO_REQUIRE(workspace_bytes >= dpvo_softagg_fused_workspace_bytes(E), "softagg_fused: workspace %lld B < required %lld B",
               (long long)workspace_bytes, (long long)dpvo_softagg_fused_workspace_bytes(E));
  cudaStream_t st = (cudaStream_t)stream;
  if (E > 0) {
    // a CTA keeps its channel slice: the grid is a multiple of the slice count
    const int64_t tiles = (E + SF_M - 1) / SF_M;
    const int64_t grid = std::max<int64_t>(SF_SLICES, std::min<int64_t>(tiles, sm_count() / SF_SLICES) * SF_SLICES);
    const int rc = launch("softagg_fused_kernel", softagg_fused_kernel, (unsigned)grid, SF_THREADS, SF_SMEM, st, (const __half*)x16, ldx, order,
                          group_of, (const __half*)w16, bias, (__half*)y16, (float*)workspace, (int)E, (int)max_groups);
    if (rc) return rc;
  }
  const unsigned grid = (unsigned)std::min<int64_t>(max_groups, (int64_t)sm_count() * 8);
  return launch("softagg_combine_kernel", softagg_combine_kernel, grid, SF_DIM / 2, 0, st, group_start, n_groups, (const float*)workspace,
                (__half*)y16, (int)max_groups);
}
