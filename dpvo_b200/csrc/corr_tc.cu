// Patch <-> frame correlation on wgmma + TMA (sm_90a), both pyramid levels in one launch.
//
// Per edge and level the nine 8x8 tap windows are covered by one (8+sx) x (8+sy) pixel box, sx/sy = spread of the
// nine anchors (2 at unit patch scale, 0..1 on the quarter-resolution level).  Boxes of up to 128 pixels on level 0
// (e.g. 11x11, 12x10) and up to 10x10 on level 1 are handled here; the rare more stretched edges are appended
// to a list and finished by the mma.sync kernel of corr.cu.  The box is a plain 4-D tile of the channels-last
// feature ring [slot][y][x][c]:
//   * ONE elected thread issues cp.async.bulk.tensor.4d loads (two 64-channel halves per level) with the
//     128-byte swizzle, picking the tensor map whose box matches the edge (one map per box shape, so no
//     byte is fetched that the edge does not need); pixels outside the map are zero-filled by the TMA unit,
//     which is exactly the reference's "out-of-bounds taps contribute 0" (correlation_kernel.cu:121-122)
//     -- no predicates, no per-lane address arithmetic
//   * the landed tile IS the canonical K-major SWIZZLE_128B operand: rows = box pixels, K = channels.
//     Two wgmma.m64n16k16 per k-step (rows 0-63 and 64-127 incl. padding, N=16 patch pixels incl. padding, K=16 x 8)
//     accumulate <box pixel, patch pixel> for all pairs in the registers of the warpgroup that owns the edge
//   * that warpgroup transposes the accumulator through shared memory and applies the bilinear blend + (x,y) ordering
//     + level interleave, writing fp16 pairs
// Roles per CTA (persistent, one per SM): warps 0.. consumers (TC_NG warpgroups taking edges round-robin, each issuing
// its own MMAs), then TC_NP producer warps (alternate edges, coords prefetched two edges ahead); one shared-memory
// stage per warpgroup, refilled as soon as its MMAs have retired, keeps TMA, tensor pipe and the blends overlapped.
#include "common.cuh"
#include "tc.cuh"
#include <cuda.h>
#include <cstring>
#include <cmath>

namespace dpvo {

constexpr int TC_L0_MAXDIM = 12, TC_L0_MAXROWS = 128;     // level-0 boxes: 8..12 per side, at most 128 pixels
constexpr int TC_L1_MAXDIM = 10;                          // level-1 boxes: 8..10 per side
constexpr int TC_L0_SHAPES = 5, TC_L1_SHAPES = 3;         // box sides per axis
constexpr int TC_WIN0_BYTES = 128 * 128;       // one 64-channel half of a level-0 box (<= 128 rows x 128 B)
constexpr int TC_WIN1_BYTES = 13 * 1024;       // level 1: <= 100 rows, rounded up to the 1024 B swizzle atom (the M=128
                                               // operand reads 3 KB past it into the next tile: padding rows, never used)
constexpr int TC_PAT_BYTES = 16 * 128;         // patch half: 16 rows (9 loaded) x 64 channels
constexpr int TC_PAT_TX = 9 * 128;
constexpr int TC_STAGE_BYTES = 2 * TC_WIN0_BYTES + 2 * TC_WIN1_BYTES + 2 * TC_PAT_BYTES;
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
static_assert(TC_STAGE_BYTES % 1024 == 0, "stages must keep the 1024 B swizzle alignment");

struct TcMaps {
  CUtensorMap l0[TC_L0_SHAPES * TC_L0_SHAPES];   // [bw - 8][bh - 8]
  CUtensorMap l1[TC_L1_SHAPES * TC_L1_SHAPES];
  CUtensorMap pat;
};

struct TcArgs {
  const float* coords;       // [M, 2, 3, 3]
  const int64_t* ii; const int64_t* jj;
  __half* out; int64_t out_row;
  float div1, inv1;          // inv1 = 1/div1 when div1 is a power of two (exact), else 0
  int M, H0, W0, H1, W1;
  int* fb_count; int* fb_list;   // edges whose windows do not fit the box
};

struct __align__(16) TcMeta {   // what the producer hands to the other roles, per edge
  int bx[2], by[2];             // box origin per level
  int pitch[2];                 // box width per level
  int uni;                      // 0: the edge goes to the list kernel
  int edge;
};

struct TcBars {
  uint64_t full[TC_STAGES], empty[TC_STAGES];
};

__device__ __forceinline__ uint32_t tc_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tc_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(tc_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void tc_mbar_arrive(uint64_t* bar) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.shared::cta.b64 st, [%0];\n}\n" ::"r"(tc_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tc_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n}\n" ::"r"(tc_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tc_mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}\n" ::"r"(tc_smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tc_tma_4d(uint32_t dst, const void* tmap, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];\n" ::"r"(dst),
               "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(tc_smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tc_tma_2d(uint32_t dst, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(dst),
               "l"(tmap), "r"(c0), "r"(c1), "r"(tc_smem_u32(bar))
               : "memory");
}
// level-1 coordinate: x / div (correlation is sampled at coords / 4, dpvo.py:206); a power-of-two divisor is
// applied as an exact multiplication
template <bool POW2> __device__ __forceinline__ float tc_level1(float x, const TcArgs& a) { return POW2 ? x * a.inv1 : x / a.div1; }

template <bool POW2>
__global__ void __launch_bounds__(TC_THREADS, 1)
corr_fwd_tc(const __grid_constant__ TcMaps maps, const TcArgs a) {
  extern __shared__ unsigned char tc_smem_raw[];
  // 1024-byte alignment by pointer arithmetic on the shared array (keeps LDS/STS; an integer round trip gives generic LD/ST)
  unsigned char* base = tc_smem_raw + ((1024u - (tc_smem_u32(tc_smem_raw) & 1023u)) & 1023u);
  unsigned char* stages = base;                                        // [TC_STAGES][TC_STAGE_BYTES]
  float* raw = reinterpret_cast<float*>(base + TC_STAGES * TC_STAGE_BYTES);      // [TC_NG][2 lev][9][TC_RAWP]
  TcMeta* meta = reinterpret_cast<TcMeta*>(raw + TC_NG * 2 * 9 * TC_RAWP);
  TcBars* bars = reinterpret_cast<TcBars*>(meta + TC_META);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    // a stage is handed back by lane 0 of each of the four warps of the consuming warpgroup
    for (int s = 0; s < TC_STAGES; ++s) { tc_mbar_init(&bars->full[s], 1); tc_mbar_init(&bars->empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (warp >= 4 * TC_NG) {
    const int pw = warp - 4 * TC_NG;                 // producer index
    // ================================================================================ producers
    // TC_NP warps take edges alternately.  Parity waits stay unambiguous because a producer that has issued
    // edge i (stage free => MMA of edge i - STAGES retired) next waits for the stage of edge i + NP, whose
    // previous user is edge i + NP - STAGES <= i: at most one phase behind.
    // lanes 0..17 hold the 18 coordinates of an edge, lanes 18/19 its patch / frame slot; fetched two
    // edges ahead so that the dependent global loads never sit on the critical path of the TMA issue
    auto fetch = [&](int e, float& cv, int& iv) {
      cv = 0.f; iv = 0;
      if (e < a.M) {
        if (lane < 18) cv = __ldg(a.coords + (int64_t)e * 18 + lane);
        else if (lane == 18) iv = (int)__ldg(a.ii + e);
        else if (lane == 19) iv = (int)__ldg(a.jj + e);
      }
    };
    float c0, c1, c2; int i0, i1, i2;
    const int G = gridDim.x * TC_NP;
    const int e_first = blockIdx.x + pw * gridDim.x;
    fetch(e_first, c0, i0);
    fetch(e_first + G, c1, i1);
    uint32_t it = pw;
    for (int e = e_first; e < a.M; e += G, it += TC_NP) {
      fetch(e + 2 * G, c2, i2);
      const uint32_t s = it % TC_STAGES, ph = (it / TC_STAGES) & 1;
      TcMeta& mt = meta[it % TC_META];
      const float xr = c0, yr = __shfl_down_sync(0xffffffffu, c0, 9);
      const int prow = __shfl_sync(0xffffffffu, i0, 18) * 9, slot = __shfl_sync(0xffffffffu, i0, 19);
      // box of the nine anchors per level: one warp-wide integer min / max each (lanes 0..8 hold the pixels);
      // the per-pixel weights are formed by the epilogue threads, off this warp's critical path
      int bx[2], by[2], bw[2], bh[2];
#pragma unroll
      for (int lev = 0; lev < 2; ++lev) {
        const float x = lev == 0 ? xr : tc_level1<POW2>(xr, a), y = lev == 0 ? yr : tc_level1<POW2>(yr, a);
        const int ax = safe_floor_int(x) - 3, ay = safe_floor_int(y) - 3;
        const bool px = lane < 9;
        bx[lev] = __reduce_min_sync(0xffffffffu, px ? ax : (1 << 28));
        by[lev] = __reduce_min_sync(0xffffffffu, px ? ay : (1 << 28));
        // spreads can be huge for degenerate projections: clamp before forming the box side
        bw[lev] = min(__reduce_max_sync(0xffffffffu, px ? ax : -(1 << 28)) - bx[lev], 64) + 8;
        bh[lev] = min(__reduce_max_sync(0xffffffffu, px ? ay : -(1 << 28)) - by[lev], 64) + 8;
      }
      const bool uni = bw[0] <= TC_L0_MAXDIM && bh[0] <= TC_L0_MAXDIM && bw[0] * bh[0] <= TC_L0_MAXROWS &&
                       bw[1] <= TC_L1_MAXDIM && bh[1] <= TC_L1_MAXDIM;
      if (lane == 0) {
        *reinterpret_cast<int4*>(&mt.bx[0]) = make_int4(bx[0], bx[1], by[0], by[1]);
        *reinterpret_cast<int4*>(&mt.pitch[0]) = make_int4(bw[0], bw[1], uni ? 1 : 0, e);
        if (!uni) { const int pos = atomicAdd(a.fb_count, 1); a.fb_list[pos] = e; }
      }
      __syncwarp();
      tc_mbar_wait(&bars->empty[s], ph ^ 1);
      if (lane == 0) {
        unsigned char* st = stages + (size_t)s * TC_STAGE_BYTES;
        const uint32_t w0a = tc_smem_u32(st), w1a = w0a + 2 * TC_WIN0_BYTES, pa = w1a + 2 * TC_WIN1_BYTES;
        if (uni) {
          tc_mbar_expect_tx(&bars->full[s], 2 * 128 * (bw[0] * bh[0] + bw[1] * bh[1]) + 2 * TC_PAT_TX);
          // clamp wild origins so the coordinates stay in int32 range; such boxes are entirely out of bounds
          const int x0 = max(min(bx[0], 1 << 20), -(1 << 20)), y0 = max(min(by[0], 1 << 20), -(1 << 20));
          const int x1 = max(min(bx[1], 1 << 20), -(1 << 20)), y1 = max(min(by[1], 1 << 20), -(1 << 20));
          const CUtensorMap* m0 = &maps.l0[(bw[0] - 8) * TC_L0_SHAPES + (bh[0] - 8)];
          const CUtensorMap* m1 = &maps.l1[(bw[1] - 8) * TC_L1_SHAPES + (bh[1] - 8)];
          tc_tma_4d(w0a, m0, 0, x0, y0, slot, &bars->full[s]);
          tc_tma_4d(w0a + TC_WIN0_BYTES, m0, 64, x0, y0, slot, &bars->full[s]);
          tc_tma_4d(w1a, m1, 0, x1, y1, slot, &bars->full[s]);
          tc_tma_4d(w1a + TC_WIN1_BYTES, m1, 64, x1, y1, slot, &bars->full[s]);
          tc_tma_2d(pa, &maps.pat, 0, prow, &bars->full[s]);
          tc_tma_2d(pa + TC_PAT_BYTES, &maps.pat, 64, prow, &bars->full[s]);
        } else {
          tc_mbar_arrive(&bars->full[s]);          // nothing to load: the stage passes through empty
        }
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
    // 36 shared-memory loads per (p, y) and level pair instead of 56 when every tap was blended on its own.
    const int u = et % 63, hx = et / 63;             // hx = 0: tap columns 0..3, hx = 1: tap columns 4..6
    const int p = u % 9, yrow = u / 9;
    const int x0 = hx * 4, nx = 4 - hx;
    float* rw = raw + eg * (2 * 9 * TC_RAWP);
    uint32_t it = 0;
    for (int e = blockIdx.x; e < a.M; e += gridDim.x, ++it) {
      if ((int)(it % TC_NG) != eg) continue;
      const uint32_t s = it % TC_STAGES, ph = (it / TC_STAGES) & 1;
      const TcMeta& mt = meta[it % TC_META];
      // this thread's patch pixel: anchor and bilinear weights per level (independent of the box, so the
      // loads and the arithmetic overlap the wait for the stage)
      const float xr = __ldg(a.coords + (int64_t)e * 18 + p), yr = __ldg(a.coords + (int64_t)e * 18 + 9 + p);
      int ax[2], ay[2];
      float4 w[2];
#pragma unroll
      for (int lev = 0; lev < 2; ++lev) {
        const float x = lev == 0 ? xr : tc_level1<POW2>(xr, a), y = lev == 0 ? yr : tc_level1<POW2>(yr, a);
        ax[lev] = safe_floor_int(x) - 3; ay[lev] = safe_floor_int(y) - 3;
        const float fx = x - floorf(x), fy = y - floorf(y);
        w[lev] = make_float4((1.f - fx) * (1.f - fy), fx * (1.f - fy), (1.f - fx) * fy, fx * fy);
      }
      tc_mbar_wait(&bars->full[s], ph);
      const int4 org = *reinterpret_cast<const int4*>(&mt.bx[0]);        // bx0 bx1 by0 by1
      const int4 shp = *reinterpret_cast<const int4*>(&mt.pitch[0]);     // pitch0 pitch1 uni edge
      if (!shp.z) {                                   // finished by the list kernel: just hand the stage back
        __syncwarp();
        if (lane == 0) tc_mbar_arrive(&bars->empty[s]);
        continue;
      }
      float acc[2][2][8];                             // [level][rows 0-63 | 64-127][fragment]
      {
        const uint32_t st = tc_smem_u32(stages + (size_t)s * TC_STAGE_BYTES);
        const uint32_t pa = st + 2 * TC_WIN0_BYTES + 2 * TC_WIN1_BYTES;
        wgmma_fence();
#pragma unroll
        for (int lev = 0; lev < 2; ++lev) {
          const uint32_t wa = lev == 0 ? st : st + 2 * TC_WIN0_BYTES;
          const uint32_t wstep = lev == 0 ? TC_WIN0_BYTES : TC_WIN1_BYTES;
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const uint64_t bd = wgmma_desc_sw128(pa + half * TC_PAT_BYTES);
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
              const uint64_t ad = wgmma_desc_sw128(wa + half * wstep + rh * 64 * 128);
#pragma unroll
              for (int k = 0; k < 4; ++k) wgmma_m64n16k16(acc[lev][rh], ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), (half | k) != 0);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int lev = 0; lev < 2; ++lev)
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) wgmma_fence_regs(acc[lev][rh]);
        __syncwarp();
        if (lane == 0) tc_mbar_arrive(&bars->empty[s]);
      }
      // transpose: raw[lev][p][r]   (rows past the box are padding); fragment i of row half rh: box pixel
      // r = 64 rh + 16 wq + lane / 4 + 8 ((i / 2) % 2), patch pixel 8 (i / 4) + 2 (lane % 4) + i % 2
#pragma unroll
      for (int lev = 0; lev < 2; ++lev)
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int r = rh * 64 + wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
            const int pp = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
            if (pp < 9) rw[(lev * 9 + pp) * TC_RAWP + r] = acc[lev][rh][i];
          }
      asm volatile("bar.sync %0, 128;\n" ::"r"(1 + eg) : "memory");
      if (et < 126) {
        __half2* orow = reinterpret_cast<__half2*>(a.out + (int64_t)e * a.out_row);
        const int p0 = shp.x, p1 = shp.y;
        const float* r0 = rw + p * TC_RAWP + (ay[0] - org.z + yrow) * p0 + (ax[0] - org.x) + x0;
        const float* r1 = rw + (9 + p) * TC_RAWP + (ay[1] - org.w + yrow) * p1 + (ax[1] - org.y) + x0;
        const float4 w0 = w[0], w1 = w[1];
        float a0[5], b0[5], a1[5], b1[5];            // rows y and y + 1 of the two levels, columns x0 .. x0 + nx
#pragma unroll
        for (int i = 0; i < 5; ++i) {
          if (i <= nx) { a0[i] = r0[i]; b0[i] = r0[p0 + i]; a1[i] = r1[i]; b1[i] = r1[p1 + i]; }
          else { a0[i] = b0[i] = a1[i] = b1[i] = 0.f; }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (i < nx) {
            const float o0 = w0.x * a0[i] + w0.y * a0[i + 1] + w0.z * b0[i] + w0.w * b0[i + 1];
            const float o1 = w1.x * a1[i] + w1.y * a1[i + 1] + w1.z * b1[i] + w1.w * b1[i + 1];
            orow[((x0 + i) * 7 + yrow) * 9 + p] = __floats2half2_rn(o0, o1);     // tap (x, y) -> feature (x * 7 + y) * 9 + p
          }
        }
      }
      asm volatile("bar.sync %0, 128;\n" ::"r"(1 + eg) : "memory");   // tile free for this group's next edge
    }
  }

}

typedef CUresult (*TcEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TcEncodeFn tc_encode() {
  static TcEncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (TcEncodeFn)p;
  }
  return fn;
}

// corr.cu: the mma.sync kernel run over a device-side list of edges
int corr_launch_fallback_list(const void* fmap1, const int64_t* s1, const void* l0, const int64_t* s20, int H0, int W0,
                              const void* l1, const int64_t* s21, int H1, int W1, float div1, const float* coords,
                              const int64_t* ii, const int64_t* jj, void* out, int64_t out_row, int M,
                              const int* list, const int* count, cudaStream_t st);

size_t corr_tc_smem_bytes() {
  return (size_t)TC_STAGES * TC_STAGE_BYTES + TC_NG * 2 * 9 * TC_RAWP * sizeof(float) + TC_META * sizeof(TcMeta) + sizeof(TcBars) + 1024;
}

// The tensor maps depend only on the ring buffers (pointer, strides, extents), which a VO front end allocates
// once: keep the last set per host thread and re-encode only when the buffers change.
struct TcMapKey {
  const void* p[3];
  int64_t s[8];
  int dims[6];
};
struct TcMapCache {
  bool valid = false;
  TcMapKey key;
  TcMaps maps;
};

static bool tc_build_maps(TcEncodeFn enc, TcMaps& m, const void* fmap1, int S1, const void* l0, const int64_t* s20, int H0, int W0,
                          const void* l1, const int64_t* s21, int H1, int W1, int S2) {
  auto level_map = [&](CUtensorMap* out, const void* ptr, const int64_t* s, int H, int W, int bw, int bh) -> bool {
    cuuint64_t dims[4] = {128, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)S2};
    cuuint64_t strides[3] = {(cuuint64_t)s[4] * 2, (cuuint64_t)s[3] * 2, (cuuint64_t)s[1] * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)bw, (cuuint32_t)bh, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  };
  memset(&m, 0, sizeof(m));
  for (int i = 0; i < TC_L0_SHAPES; ++i)
    for (int j = 0; j < TC_L0_SHAPES; ++j)
      if ((8 + i) * (8 + j) <= TC_L0_MAXROWS && !level_map(&m.l0[i * TC_L0_SHAPES + j], l0, s20, H0, W0, 8 + i, 8 + j)) return false;
  for (int i = 0; i < TC_L1_SHAPES; ++i)
    for (int j = 0; j < TC_L1_SHAPES; ++j)
      if (!level_map(&m.l1[i * TC_L1_SHAPES + j], l1, s21, H1, W1, 8 + i, 8 + j)) return false;
  cuuint64_t dims[2] = {128, (cuuint64_t)S1 * 9};
  cuuint64_t strides[1] = {256};
  cuuint32_t box[2] = {64, 9};
  cuuint32_t es[2] = {1, 1};
  return enc(&m.pat, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(fmap1), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// returns DPVO_OK, or DPVO_ERR_UNSUPPORTED when the inputs do not have the layout this kernel needs
int corr_tc_forward(const void* fmap1, const int64_t* s1, int S1, const void* l0, const int64_t* s20, int H0, int W0,
                    const void* l1, const int64_t* s21, int H1, int W1, int S2, float div1, const float* coords,
                    const int64_t* ii, const int64_t* jj, void* out, int64_t out_row, int M, void* scratch /* (M+1) ints */,
                    cudaStream_t st) {
  // layout requirements: channels-last rings, patch features [slot][3][3][128] contiguous
  if (s20[2] != 1 || s21[2] != 1 || s1[2] != 1 || s1[4] != 128 || s1[3] != 384 || s1[1] != 1152) return DPVO_ERR_UNSUPPORTED;
  if (((uintptr_t)fmap1 & 15) || ((uintptr_t)l0 & 15) || ((uintptr_t)l1 & 15) || ((uintptr_t)out & 3)) return DPVO_ERR_UNSUPPORTED;
  for (int d = 1; d < 5; ++d) if (d != 2 && ((s20[d] % 8) || (s21[d] % 8))) return DPVO_ERR_UNSUPPORTED;
  TcEncodeFn enc = tc_encode();
  if (!enc) return DPVO_ERR_UNSUPPORTED;
  static thread_local TcMapCache cache;
  TcMapKey key;
  memset(&key, 0, sizeof(key));
  key.p[0] = fmap1; key.p[1] = l0; key.p[2] = l1;
  key.s[0] = s20[1]; key.s[1] = s20[3]; key.s[2] = s20[4]; key.s[3] = s21[1]; key.s[4] = s21[3]; key.s[5] = s21[4];
  key.dims[0] = S1; key.dims[1] = S2; key.dims[2] = H0; key.dims[3] = W0; key.dims[4] = H1; key.dims[5] = W1;
  if (!cache.valid || memcmp(&cache.key, &key, sizeof(key)) != 0) {
    cache.valid = false;
    if (!tc_build_maps(enc, cache.maps, fmap1, S1, l0, s20, H0, W0, l1, s21, H1, W1, S2)) return DPVO_ERR_UNSUPPORTED;
    cache.key = key;
    cache.valid = true;
  }
  const size_t smem = corr_tc_smem_bytes();
  // per-device function attribute: set on every call
  if (cudaFuncSetAttribute(corr_fwd_tc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
      cudaFuncSetAttribute(corr_fwd_tc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    cudaGetLastError();
    return DPVO_ERR_UNSUPPORTED;
  }
  int* fb = reinterpret_cast<int*>(scratch);
  int rc = check_cuda(cudaMemsetAsync(fb, 0, sizeof(int), st), "corr_tc: memset");
  if (rc) return rc;
  TcArgs a;
  a.coords = coords; a.ii = ii; a.jj = jj; a.out = (__half*)out; a.out_row = out_row; a.div1 = div1;
  {
    int ex = 0;
    a.inv1 = (std::frexp(div1, &ex) == 0.5f) ? 1.0f / div1 : 0.f;
  }
  a.M = M; a.H0 = H0; a.W0 = W0; a.H1 = H1; a.W1 = W1; a.fb_count = fb; a.fb_list = fb + 1;
  const unsigned grid = (unsigned)std::min<int64_t>(M, sm_count());
  if (a.inv1 != 0.f) corr_fwd_tc<true><<<grid, TC_THREADS, smem, st>>>(cache.maps, a);
  else corr_fwd_tc<false><<<grid, TC_THREADS, smem, st>>>(cache.maps, a);
  DPVO_LAUNCH_CHECK("corr_fwd_tc");
  // edges whose reprojected patch is stretched beyond the box: same arithmetic on the mma.sync path
  return corr_launch_fallback_list(fmap1, s1, l0, s20, H0, W0, l1, s21, H1, W1, div1, coords, ii, jj, out, out_row, M, fb + 1, fb, st);
}

}  // namespace dpvo
