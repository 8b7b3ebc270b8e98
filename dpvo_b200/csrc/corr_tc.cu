// Patch <-> frame correlation on wgmma + TMA (sm_90a), level 0 of the pyramid.
//
// Per edge the nine 8x8 tap windows are covered by one (8+sx) x (8+sy) pixel box, sx/sy = spread of the nine anchors
// (2 at unit patch scale).  Boxes of up to 128 pixels (e.g. 11x11, 12x10) are handled here.  corr_bin.cu bins the
// edges first: it sends the rare more stretched edges to the list of the mma.sync kernel of corr.cu, runs level 1
// from one shared-memory region per bin, and leaves the other edges in bin order (target slot, then position), the
// order this kernel walks them in, so that the edges in flight on the GPU read neighbouring pixels of one frame.
// The box is a plain 4-D tile of the channels-last feature ring [slot][y][x][c]:
//   * ONE elected thread issues cp.async.bulk.tensor.4d loads (two 64-channel halves) with the
//     128-byte swizzle, picking the tensor map whose box matches the edge (one map per box shape, so no
//     byte is fetched that the edge does not need); pixels outside the map are zero-filled by the TMA unit,
//     which is exactly the reference's "out-of-bounds taps contribute 0" (correlation_kernel.cu:121-122)
//     -- no predicates, no per-lane address arithmetic
//   * the landed tile IS the canonical K-major SWIZZLE_128B operand: rows = box pixels, K = channels.
//     Two wgmma.m64n16k16 per k-step (rows 0-63 and 64-127 incl. padding, N=16 patch pixels incl. padding, K=16 x 8)
//     accumulate <box pixel, patch pixel> for all pairs in the registers of the warpgroup that owns the edge
//   * that warpgroup transposes the accumulator through shared memory and applies the bilinear blend + (x,y) ordering,
//     writing the level-0 half of each fp16 (level 0, level 1) pair
// Roles per CTA (persistent, one per SM): warps 0.. consumers (TC_NG warpgroups taking edges round-robin, each issuing
// its own MMAs), then TC_NP producer warps (alternate edges, coords prefetched two edges ahead); one shared-memory
// stage per warpgroup, refilled as soon as its MMAs have retired, keeps TMA, tensor pipe and the blends overlapped.
#include "common.cuh"
#include "tc.cuh"
#include <cstring>

namespace dpvo {

constexpr int TC_L0_SHAPES = 5;                // level-0 boxes: 8..12 per side (at most 128 pixels, see corr_bin.cu)
constexpr int TC_WIN0_BYTES = 128 * 128;       // one 64-channel half of a level-0 box (<= 128 rows x 128 B)
constexpr int TC_PAT_BYTES = 16 * 128;         // patch half: 16 rows (9 loaded) x 64 channels
constexpr int TC_PAT_TX = 9 * 128;
constexpr int TC_STAGE_BYTES = 2 * TC_WIN0_BYTES + 2 * TC_PAT_BYTES;
// one stage per consumer warpgroup: a stage is then always consumed by the same group, in order (with stages shared
// round-robin a group could wait on a stage two phases ahead of it, which a parity wait cannot tell apart)
constexpr int TC_STAGES = 2;
constexpr int TC_NG = 2;                       // consumer warpgroups
constexpr int TC_META = 16;                    // meta ring (> smem stages + consumer groups + 1)
constexpr int TC_NP = 2;                       // producer warps (alternate edges; must not exceed TC_STAGES, see the kernel)
constexpr int TC_THREADS = (4 * TC_NG + TC_NP) * 32;
static_assert(TC_NP <= TC_STAGES, "a producer may run at most one phase ahead of the stage it waits for");
static_assert(TC_STAGES == TC_NG, "each consumer warpgroup owns one stage");
constexpr int TC_RAWP = 129;                   // floats per patch pixel row of the transposed accumulator
constexpr int TC_RAW_FLOATS = (TC_NG * 9 * TC_RAWP + 3) & ~3;   // transpose tiles, rounded up so that the meta ring
                                                            // behind them stays 16-byte aligned
static_assert(TC_STAGE_BYTES % 1024 == 0, "stages must keep the 1024 B swizzle alignment");

struct TcMaps {
  CUtensorMap l0[TC_L0_SHAPES * TC_L0_SHAPES];   // [bw - 8][bh - 8]
  CUtensorMap pat;
};

struct TcArgs {
  const float* coords;       // [M, 2, 3, 3]
  const int64_t* ii; const int64_t* jj;
  __half* out; int64_t out_row;
  const int* order; const int* count;   // the edges to correlate, in bin order, and their number (device side)
};

struct __align__(16) TcMeta {   // what the producer hands to the consumers, per edge
  int bx, by, pitch, edge;      // box origin and width
};

struct TcBars {
  uint64_t full[TC_STAGES], empty[TC_STAGES];
};

// 64 registers: with those, one CTA of corr_fwd_l1_tiles (corr_bin.cu) fits beside this one on every SM
__global__ void __maxnreg__(64)
corr_fwd_tc(const __grid_constant__ TcMaps maps, const TcArgs a) {
  extern __shared__ unsigned char tc_smem_raw[];
  // 1024-byte alignment by pointer arithmetic on the shared array (keeps LDS/STS; an integer round trip gives generic LD/ST)
  unsigned char* base = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u);
  unsigned char* stages = base;                                        // [TC_STAGES][TC_STAGE_BYTES]
  float* raw = reinterpret_cast<float*>(base + TC_STAGES * TC_STAGE_BYTES);      // [TC_NG][9][TC_RAWP]
  TcMeta* meta = reinterpret_cast<TcMeta*>(raw + TC_RAW_FLOATS);
  TcBars* bars = reinterpret_cast<TcBars*>(meta + TC_META);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    // a stage is handed back by lane 0 of each of the four warps of the consuming warpgroup
    for (int s = 0; s < TC_STAGES; ++s) { mbar_init(&bars->full[s], 1); mbar_init(&bars->empty[s], 4); }
    mbar_init_fence();
  }
  __syncthreads();
  const int n = *a.count;

  if (warp >= 4 * TC_NG) {
    const int pw = warp - 4 * TC_NG;                 // producer index
    // ================================================================================ producers
    // TC_NP warps take edges alternately.  Parity waits stay unambiguous because a producer that has issued
    // edge i (stage free => MMA of edge i - STAGES retired) next waits for the stage of edge i + NP, whose
    // previous user is edge i + NP - STAGES <= i: at most one phase behind.
    // lanes 0..17 hold the 18 coordinates of an edge, lanes 18/19 its patch / frame slot; fetched two
    // edges ahead so that the dependent global loads never sit on the critical path of the TMA issue
    auto fetch = [&](int i, float& cv, int& iv) {
      cv = 0.f; iv = 0;
      if (i < n) {
        const int e = __ldg(a.order + i);
        if (lane < 18) cv = __ldg(a.coords + (int64_t)e * 18 + lane);
        else if (lane == 18) iv = (int)__ldg(a.ii + e);
        else if (lane == 19) iv = (int)__ldg(a.jj + e);
        else if (lane == 20) iv = e;
      }
    };
    float c0, c1, c2; int i0, i1, i2;
    const int G = gridDim.x * TC_NP;
    const int i_first = blockIdx.x + pw * gridDim.x;
    fetch(i_first, c0, i0);
    fetch(i_first + G, c1, i1);
    uint32_t it = pw;
    for (int i = i_first; i < n; i += G, it += TC_NP) {
      fetch(i + 2 * G, c2, i2);
      const uint32_t s = it % TC_STAGES, ph = (it / TC_STAGES) & 1;
      TcMeta& mt = meta[it % TC_META];
      const float xr = c0, yr = __shfl_down_sync(0xffffffffu, c0, 9);
      const int prow = __shfl_sync(0xffffffffu, i0, 18) * 9, slot = __shfl_sync(0xffffffffu, i0, 19);
      const int e = __shfl_sync(0xffffffffu, i0, 20);
      // box of the nine anchors: one warp-wide integer min / max each (lanes 0..8 hold the pixels); the per-pixel
      // weights are formed by the epilogue threads, off this warp's critical path.  corr_bin_count computed the same
      // box and admitted the edge only if it has 8..12 pixels per side and at most 128 in all.
      const int ax = safe_floor_int(xr) - 3, ay = safe_floor_int(yr) - 3;
      const bool px = lane < 9;
      const int bx = __reduce_min_sync(0xffffffffu, px ? ax : (1 << 28));
      const int by = __reduce_min_sync(0xffffffffu, px ? ay : (1 << 28));
      const int bw = min(__reduce_max_sync(0xffffffffu, px ? ax : -(1 << 28)) - bx, 64) + 8;
      const int bh = min(__reduce_max_sync(0xffffffffu, px ? ay : -(1 << 28)) - by, 64) + 8;
      if (lane == 0) *reinterpret_cast<int4*>(&mt) = make_int4(bx, by, bw, e);
      __syncwarp();
      mbar_wait(&bars->empty[s], ph ^ 1);
      if (lane == 0) {
        const uint32_t w0a = smem_u32(stages + (size_t)s * TC_STAGE_BYTES), pa = w0a + 2 * TC_WIN0_BYTES;
        mbar_arrive_expect_tx(&bars->full[s], 2 * 128 * bw * bh + 2 * TC_PAT_TX);
        // clamp wild origins so the coordinates stay in int32 range; such boxes are entirely out of bounds
        const int x0 = max(min(bx, 1 << 20), -(1 << 20)), y0 = max(min(by, 1 << 20), -(1 << 20));
        const CUtensorMap* m0 = &maps.l0[(bw - 8) * TC_L0_SHAPES + (bh - 8)];
        tma_load_4d(w0a, m0, 0, x0, y0, slot, &bars->full[s]);
        tma_load_4d(w0a + TC_WIN0_BYTES, m0, 64, x0, y0, slot, &bars->full[s]);
        tma_load_2d(pa, &maps.pat, 0, prow, &bars->full[s]);
        tma_load_2d(pa + TC_PAT_BYTES, &maps.pat, 64, prow, &bars->full[s]);
      }
      __syncwarp();
      c0 = c1; i0 = i1; c1 = c2; i1 = i2;
    }
  } else {
    // ================================================================================ consumers
    // TC_NG warpgroups take edges round-robin; a group issues the MMAs of its edge, owns one transpose tile and
    // hands the stage back as soon as its MMAs have retired.  Thread -> (patch pixel p, taps t0 + 14k): constant for the
    // kernel, so weights / base are read once per edge.
    const int eg = warp >> 2, wq = warp & 3;
    const int et = threadIdx.x & 127;
    // Thread -> (patch pixel p, tap row y, half of the tap columns): the 7 taps of a row share their bilinear corners
    // (tap x uses columns x, x+1 of rows y, y+1), so a thread that owns a run of taps reads each window value once --
    // 18 shared-memory loads per (p, y) instead of 28 when every tap was blended on its own.
    const int u = et % 63, hx = et / 63;             // hx = 0: tap columns 0..3, hx = 1: tap columns 4..6
    const int p = u % 9, yrow = u / 9;
    const int x0 = hx * 4, nx = 4 - hx;
    float* rw = raw + eg * (9 * TC_RAWP);
    uint32_t it = 0;
    for (int i = blockIdx.x; i < n; i += gridDim.x, ++it) {
      if ((int)(it % TC_NG) != eg) continue;
      const uint32_t s = it % TC_STAGES, ph = (it / TC_STAGES) & 1;
      const TcMeta& mt = meta[it % TC_META];
      // this thread's patch pixel: anchor and bilinear weights (independent of the box, so the loads and the
      // arithmetic overlap the wait for the stage)
      const int e = __ldg(a.order + i);
      const float x = __ldg(a.coords + (int64_t)e * 18 + p), y = __ldg(a.coords + (int64_t)e * 18 + 9 + p);
      const int ax = safe_floor_int(x) - 3, ay = safe_floor_int(y) - 3;
      const float fx = x - floorf(x), fy = y - floorf(y);
      const float4 w = make_float4((1.f - fx) * (1.f - fy), fx * (1.f - fy), (1.f - fx) * fy, fx * fy);
      mbar_wait(&bars->full[s], ph);
      const int4 box = *reinterpret_cast<const int4*>(&mt);             // bx by pitch edge
      float acc[2][8];                                // [rows 0-63 | 64-127][fragment]
      {
        const uint32_t wa = smem_u32(stages + (size_t)s * TC_STAGE_BYTES);
        const uint32_t pa = wa + 2 * TC_WIN0_BYTES;
        wgmma_fence();
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const uint64_t bd = wgmma_desc_sw128(pa + half * TC_PAT_BYTES);
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) {
            const uint64_t ad = wgmma_desc_sw128(wa + half * TC_WIN0_BYTES + rh * 64 * 128);
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_m64n16k16(acc[rh], ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), (half | k) != 0);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) wgmma_fence_regs(acc[rh]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->empty[s]);
      }
      // transpose: raw[p][r]   (rows past the box are padding); fragment i of row half rh: box pixel
      // r = 64 rh + 16 wq + lane / 4 + 8 ((i / 2) % 2), patch pixel 8 (i / 4) + 2 (lane % 4) + i % 2
#pragma unroll
      for (int rh = 0; rh < 2; ++rh)
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int r = rh * 64 + wq * 16 + (lane >> 2) + 8 * ((k >> 1) & 1);
          const int pp = 8 * (k >> 2) + 2 * (lane & 3) + (k & 1);
          if (pp < 9) rw[pp * TC_RAWP + r] = acc[rh][k];
        }
      named_bar_sync(1 + eg, 128);
      if (et < 126) {
        __half* orow = a.out + (int64_t)box.w * a.out_row;       // even halves: level 0 of each pair
        const int p0 = box.z;
        const float* r0 = rw + p * TC_RAWP + (ay - box.y + yrow) * p0 + (ax - box.x) + x0;
        float a0[5], b0[5];                          // rows y and y + 1, columns x0 .. x0 + nx
#pragma unroll
        for (int k = 0; k < 5; ++k) {
          if (k <= nx) { a0[k] = r0[k]; b0[k] = r0[p0 + k]; }
          else { a0[k] = b0[k] = 0.f; }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (k < nx) {
            const float o0 = w.x * a0[k] + w.y * a0[k + 1] + w.z * b0[k] + w.w * b0[k + 1];
            orow[2 * (((x0 + k) * 7 + yrow) * 9 + p)] = __float2half_rn(o0);   // tap (x, y) -> feature (x * 7 + y) * 9 + p
          }
        }
      }
      named_bar_sync(1 + eg, 128);   // tile free for this group's next edge
    }
  }

}

// corr.cu: the mma.sync kernel run over a device-side list of edges
int corr_launch_fallback_list(const void* fmap1, const int64_t* s1, const void* l0, const int64_t* s20, int H0, int W0,
                              const void* l1, const int64_t* s21, int H1, int W1, float div1, const float* coords,
                              const int64_t* ii, const int64_t* jj, void* out, int64_t out_row, int M,
                              const int* list, const int* count, cudaStream_t st);
// corr_bin.cu: the bins and the level-1 pass
int corr_bin_edges(const float* coords, const int64_t* jj, int M, int S2, int H1, int W1, float div1, void* workspace,
                   cudaStream_t st, int** list, int** count, int** order, int** ordered);
int corr_bin_level1(const void* fmap1, const void* l1, const int64_t* s21, int H1, int W1, int S2, float div1,
                    const float* coords, const int64_t* ii, void* out, int64_t out_row, int M, void* workspace,
                    cudaStream_t st);

// A second stream per device and host thread (with its fork / join events) on which the level-1 pass runs beside this
// kernel: level 0 is bound by the L2 -> SM feed, level 1 by its per-edge latency, and the shared memory of one CTA of
// each fits an SM together.  Created on first use, like the tensor-map cache; inside a stream capture the fork and
// join become graph edges.
struct TcSide {
  cudaStream_t s = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
};
static TcSide* tc_side() {
  static thread_local TcSide side[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  TcSide& t = side[dev];
  if (!t.s) {
    if (cudaStreamCreateWithFlags(&t.s, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&t.fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&t.join, cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError();
      t = TcSide();
      return nullptr;
    }
  }
  return &t;
}

size_t corr_tc_smem_bytes() {
  return (size_t)TC_STAGES * TC_STAGE_BYTES + TC_RAW_FLOATS * sizeof(float) + TC_META * sizeof(TcMeta) + sizeof(TcBars) + 1024;
}

// The tensor maps depend only on the ring buffers (pointer, strides, extents), which a VO front end allocates
// once: keep the last set per host thread and re-encode only when the buffers change.
struct TcMapKey {
  const void* p[2];
  int64_t s[4];
  int dims[4];
};
struct TcMapCache {
  bool valid = false;
  TcMapKey key;
  TcMaps maps;
};

static int tc_build_maps(TcMaps& m, const void* fmap1, int S1, const void* l0, const int64_t* s20, int H0, int W0, int S2) {
  memset(&m, 0, sizeof(m));
  for (int i = 0; i < TC_L0_SHAPES; ++i)
    for (int j = 0; j < TC_L0_SHAPES; ++j) {
      if ((8 + i) * (8 + j) > 128) continue;
      cuuint64_t dims[4] = {128, (cuuint64_t)W0, (cuuint64_t)H0, (cuuint64_t)S2};
      cuuint64_t strides[3] = {(cuuint64_t)s20[4] * 2, (cuuint64_t)s20[3] * 2, (cuuint64_t)s20[1] * 2};
      cuuint32_t box[4] = {64, (cuuint32_t)(8 + i), (cuuint32_t)(8 + j), 1};
      if (int rc = encode_tmap(&m.l0[i * TC_L0_SHAPES + j], "corr_tc", 4, l0, dims, strides, box)) return rc;
    }
  return encode_tmap_2d(&m.pat, "corr_tc", fmap1, (int64_t)S1 * 9, 128, 128, 9);
}

// Both levels of the correlation: binning and level 1 (corr_bin.cu), level 0 here, stretched edges on the mma.sync
// list kernel.  Returns DPVO_OK, or DPVO_ERR_UNSUPPORTED (before anything is launched) when the inputs do not have the
// layout these kernels need.
int corr_tc_forward(const void* fmap1, const int64_t* s1, int S1, const void* l0, const int64_t* s20, int H0, int W0,
                    const void* l1, const int64_t* s21, int H1, int W1, int S2, float div1, const float* coords,
                    const int64_t* ii, const int64_t* jj, void* out, int64_t out_row, int M, void* workspace,
                    cudaStream_t st) {
  // layout requirements: channels-last rings, patch features [slot][3][3][128] contiguous
  if (s20[2] != 1 || s21[2] != 1 || s1[2] != 1 || s1[4] != 128 || s1[3] != 384 || s1[1] != 1152) return DPVO_ERR_UNSUPPORTED;
  if (((uintptr_t)fmap1 & 15) || ((uintptr_t)l0 & 15) || ((uintptr_t)l1 & 15) || ((uintptr_t)out & 3)) return DPVO_ERR_UNSUPPORTED;
  for (int d = 1; d < 5; ++d) if (d != 2 && ((s20[d] % 8) || (s21[d] % 8))) return DPVO_ERR_UNSUPPORTED;
  static thread_local TcMapCache cache;
  TcMapKey key;
  memset(&key, 0, sizeof(key));
  key.p[0] = fmap1; key.p[1] = l0;
  key.s[0] = s20[1]; key.s[1] = s20[3]; key.s[2] = s20[4];
  key.dims[0] = S1; key.dims[1] = S2; key.dims[2] = H0; key.dims[3] = W0;
  if (!cache.valid || memcmp(&cache.key, &key, sizeof(key)) != 0) {
    cache.valid = false;
    if (tc_build_maps(cache.maps, fmap1, S1, l0, s20, H0, W0, S2)) return DPVO_ERR_UNSUPPORTED;
    cache.key = key;
    cache.valid = true;
  }
  const size_t smem = corr_tc_smem_bytes();
  // per-device function attribute: set on every call
  // the whole carveout as shared memory: a level-1 CTA can then join each SM while this kernel runs (an SM changes
  // its carveout only when idle)
  if (cudaFuncSetAttribute(corr_fwd_tc, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) != cudaSuccess) {
    cudaGetLastError();
    return DPVO_ERR_UNSUPPORTED;
  }
  TcSide* side = tc_side();
  if (!side) return DPVO_ERR_UNSUPPORTED;
  int *list, *count, *order, *ordered;
  int rc = corr_bin_edges(coords, jj, M, S2, H1, W1, div1, workspace, st, &list, &count, &order, &ordered);
  if (rc) return rc;
  rc = check_cuda(cudaEventRecord(side->fork, st), "corr_tc: fork");
  if (rc) return rc;
  TcArgs a;
  a.coords = coords; a.ii = ii; a.jj = jj; a.out = (__half*)out; a.out_row = out_row; a.order = order; a.count = ordered;
  const unsigned grid = (unsigned)std::min<int64_t>(M, sm_count());
  rc = launch("corr_fwd_tc", corr_fwd_tc, grid, TC_THREADS, smem, st, cache.maps, a);
  if (rc) return rc;
  // level 1 on the side stream, launched after level 0 so that the persistent level-0 CTAs are placed first
  rc = check_cuda(cudaStreamWaitEvent(side->s, side->fork, 0), "corr_tc: fork");
  if (!rc) rc = corr_bin_level1(fmap1, l1, s21, H1, W1, S2, div1, coords, ii, out, out_row, M, workspace, side->s);
  if (!rc) rc = check_cuda(cudaEventRecord(side->join, side->s), "corr_tc: join");
  if (!rc) rc = check_cuda(cudaStreamWaitEvent(st, side->join, 0), "corr_tc: join");
  if (rc) return rc;
  // edges whose reprojected patch is stretched beyond the boxes: both levels on the mma.sync path
  return corr_launch_fallback_list(fmap1, s1, l0, s20, H0, W0, l1, s21, H1, W1, div1, coords, ii, jj, out, out_row, M, list, count, st);
}

}  // namespace dpvo
