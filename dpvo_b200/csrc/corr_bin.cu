// Level-1 half of the two-level correlation, one shared-memory region per bin of edges (sm_90a).
//
// The quarter-resolution frame is small (30 x 40 pixels on the default config) and ~1,400 edges land in each target
// frame, so the per-edge boxes of level 1 overlap heavily: loading them edge by edge moves every level-1 pixel from L2
// about 80 times per update.  Here the edges are first binned on the device by (target ring slot, 7 x 7 tile of
// their level-1 box origin):
//   corr_bin_count    one thread per edge: both levels' boxes of the nine anchors (the same safe_floor_int / min-max
//                     as the level-0 producer of corr_tc.cu), edges that fit no box go to the list of the mma.sync
//                     kernel, the others get a bin key and their rank inside the bin (atomic histogram)
//   corr_bin_scan     one CTA: exclusive scan of the counters, and the work items (<= CB_ITEM edges of one bin)
//   corr_bin_scatter  edge ids in bin order
// and then corr_fwd_l1_tiles takes one work item per CTA: the bin's 16 x 16-pixel region (tile + 9-pixel apron, the
// reach of a <= 10 x 10 box; pixels outside the frame zero-filled, which is the reference's "out-of-bounds taps
// contribute 0") is loaded once with cp.async, and each warp correlates one edge at a time against it with
// mma.sync.m16n8k16 in exactly the k order and accumulation chains of corr_fwd_mma (corr.cu), followed by the same
// bilinear blend, so its values are bit-identical to the mma.sync kernel's level 1.  It writes the level-1 half of
// every (level 0, level 1) fp16 pair; corr_fwd_tc writes the other half, walking the edges in the same bin order.
// The two kernels run side by side on two streams: corr_fwd_tc is bound by the L2 -> SM feed of its per-edge boxes,
// this one by the latency of its per-edge MMA and blend chains, and one CTA of each fits an SM together (shared memory
// 82 + 121 KB, and per SM sub-partition 3 x 64 + 3 x 104 registers per lane).
// The bin order within a bin depends on atomic arrival order; every output depends on its own edge only.
#include "common.cuh"
#include "tc.cuh"

namespace dpvo {

constexpr int CB_T1 = 7;                       // level-1 tile side, in box origins
constexpr int CB_APRON = 9;                    // a level-1 box (<= 10 pixels per side) reaches 9 pixels past its origin
constexpr int CB_RS = CB_T1 + CB_APRON;        // region side: 16 x 16 pixels x 256 B = 64 KB
static_assert(CB_RS == 16, "the region indexing below uses shifts by 4");
constexpr int CB_ITEM = 48;                    // edges per work item (four per warp)
constexpr int CB_WARPS = 12;                   // 104 registers each (__maxnreg__ below)
constexpr int CB_RAWP = 105;                   // floats per patch pixel of the raw tile (odd pitch, as in corr_fwd_mma)
constexpr int CB_REGION_BYTES = CB_RS * CB_RS * 256;

struct __align__(16) CbWarpSmem {
  float raw[9 * CB_RAWP + 3];                  // raw[p][box pixel] = <patch pixel p, box pixel>
  __half stage[448];                           // blended level-1 outputs in output order
  float4 w[9];                                 // bilinear weights
  int base[9];                                 // index of tap (0,0) of pixel p inside the box
};
constexpr size_t CB_SMEM = CB_REGION_BYTES + 256 + CB_WARPS * sizeof(CbWarpSmem);

static int64_t cb_key_cap(int64_t M) { return 2 * M + 4096; }
static int64_t cb_item_cap(int64_t M) { return cb_key_cap(M) + (M + CB_ITEM - 1) / CB_ITEM; }

struct CbBinArgs {
  const float* coords; const int64_t* jj;
  float div1;
  int M, S2, nty, ntx;
  int* hdr; int* list; int* order; int* key; int* rank; int* cnt; int* off; int4* items;
};

// workspace, packed in int32 words: hdr[4] = {list count, binned count, item count, -} | list[M] | order[M] | key[M] |
// rank[M] | cnt[K] | off[K] | items[I] (int4: key, first index into order, edges), K = 2M + 4096 bins,
// I = K + ceil(M / CB_ITEM).  8M + 8196 words precede items: 16-byte aligned in a 16-byte aligned workspace.
static void cb_regions(int64_t M, WsLayout& L, CbBinArgs& b) {
  b.hdr = L.take<int>(4); b.list = L.take<int>(M); b.order = L.take<int>(M); b.key = L.take<int>(M); b.rank = L.take<int>(M);
  b.cnt = L.take<int>(cb_key_cap(M)); b.off = L.take<int>(cb_key_cap(M)); b.items = L.take<int4>(cb_item_cap(M));
}
int64_t corr_bin_workspace_bytes(int64_t M) { CbBinArgs b; WsLayout L(nullptr, sizeof(int)); cb_regions(M, L, b); return L.bytes() + 16; }

__global__ void __launch_bounds__(256) corr_bin_count(const CbBinArgs a) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.M) return;
  const float* c = a.coords + (int64_t)e * 18;
  int mnx[2] = {1 << 28, 1 << 28}, mny[2] = {1 << 28, 1 << 28}, mxx[2] = {-(1 << 28), -(1 << 28)}, mxy[2] = {-(1 << 28), -(1 << 28)};
#pragma unroll
  for (int p = 0; p < 9; ++p) {
    const float xr = c[p], yr = c[9 + p];
#pragma unroll
    for (int lev = 0; lev < 2; ++lev) {
      const float x = lev == 0 ? xr : xr / a.div1, y = lev == 0 ? yr : yr / a.div1;
      const int ax = safe_floor_int(x) - 3, ay = safe_floor_int(y) - 3;
      mnx[lev] = min(mnx[lev], ax); mxx[lev] = max(mxx[lev], ax);
      mny[lev] = min(mny[lev], ay); mxy[lev] = max(mxy[lev], ay);
    }
  }
  int bw[2], bh[2];
#pragma unroll
  for (int lev = 0; lev < 2; ++lev) { bw[lev] = min(mxx[lev] - mnx[lev], 64) + 8; bh[lev] = min(mxy[lev] - mny[lev], 64) + 8; }
  // the boxes corr_fwd_tc (level 0: 8..12 per side, <= 128 pixels) and corr_fwd_l1_tiles (level 1: 8..10) handle
  const bool boxed = bw[0] <= 12 && bh[0] <= 12 && bw[0] * bh[0] <= 128 && bw[1] <= 10 && bh[1] <= 10;
  const int64_t slot = a.jj[e];
  if (!boxed || slot < 0 || slot >= a.S2) {
    a.list[atomicAdd(&a.hdr[0], 1)] = e;
    a.key[e] = -1;
    return;
  }
  // tiles of origins start at -CB_APRON, the first origin whose box can reach the frame; origins beyond the tile grid
  // only see pixels outside the frame, which the border tiles give as zeros as well
  const int vy = mny[1] + CB_APRON, vx = mnx[1] + CB_APRON;
  const int ty = vy < 0 ? 0 : min(vy / CB_T1, a.nty - 1), tx = vx < 0 ? 0 : min(vx / CB_T1, a.ntx - 1);
  const int k = ((int)slot * a.nty + ty) * a.ntx + tx;
  a.key[e] = k;
  a.rank[e] = atomicAdd(&a.cnt[k], 1);
}

__global__ void __launch_bounds__(1024) corr_bin_scan(const CbBinArgs a, int nkeys) {
  __shared__ int s_c[32], s_i[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int carry_c = 0, carry_i = 0;
  for (int base = 0; base < nkeys; base += 1024) {
    const int k = base + tid;
    const int c = k < nkeys ? a.cnt[k] : 0, ni = (c + CB_ITEM - 1) / CB_ITEM;
    int ic = c, ii = ni;                       // inclusive warp scans
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int vc = __shfl_up_sync(0xffffffffu, ic, o), vi = __shfl_up_sync(0xffffffffu, ii, o);
      if (lane >= o) { ic += vc; ii += vi; }
    }
    if (lane == 31) { s_c[warp] = ic; s_i[warp] = ii; }
    __syncthreads();
    if (warp == 0) {
      int wc = s_c[lane], wi = s_i[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int vc = __shfl_up_sync(0xffffffffu, wc, o), vi = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) { wc += vc; wi += vi; }
      }
      s_c[lane] = wc; s_i[lane] = wi;
    }
    __syncthreads();
    const int ex_c = carry_c + (warp ? s_c[warp - 1] : 0) + ic - c;
    const int ex_i = carry_i + (warp ? s_i[warp - 1] : 0) + ii - ni;
    if (k < nkeys) {
      a.off[k] = ex_c;
      for (int j = 0; j < ni; ++j) a.items[ex_i + j] = make_int4(k, ex_c + j * CB_ITEM, min(CB_ITEM, c - j * CB_ITEM), 0);
    }
    carry_c += s_c[31]; carry_i += s_i[31];
    __syncthreads();
  }
  if (tid == 0) { a.hdr[1] = carry_c; a.hdr[2] = carry_i; }
}

__global__ void __launch_bounds__(256) corr_bin_scatter(const CbBinArgs a) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.M) return;
  const int k = a.key[e];
  if (k >= 0) a.order[a.off[k] + a.rank[e]] = e;
}

// ------------------------------------------------------------------------------------------------ level-1 pass
struct CbArgs {
  const __half* f1;          // patch features [slot][3][3][128]
  const __half* l1;          // level-1 ring, channels last
  int64_t s_slot, sy, sx;    // element strides of the level-1 ring
  const float* coords; const int64_t* ii;
  __half* out; int64_t out_row;
  float div1;
  int H1, W1, nty, ntx;
  const int* order; const int4* items; const int* item_count;
};

__device__ __forceinline__ uint4 cb_lds128(uint32_t a) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
  return r;
}
__device__ __forceinline__ uint4 cb_ldg128(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

// Region pixel q (row-major 16 x 16) holds its 16 channel chunks of 16 B with chunk c stored at position c ^ 4 (q & 1):
// a quarter-warp's 16-byte loads of the mma B fragments (two neighbouring box pixels x four chunks) then cover all 32
// banks whenever the two pixels are neighbours in the region.
__global__ void __maxnreg__(104)
corr_fwd_l1_tiles(const CbArgs a) {
  extern __shared__ __align__(128) unsigned char cb_smem[];
  if ((int)blockIdx.x >= *a.item_count) return;
  const int4 item = a.items[blockIdx.x];
  const int tiles = a.nty * a.ntx, t_in = item.x % tiles, slot = item.x / tiles;
  const int ry0 = (t_in / a.ntx) * CB_T1 - CB_APRON, rx0 = (t_in % a.ntx) * CB_T1 - CB_APRON;
  const uint32_t region = smem_u32(cb_smem), zero = region + CB_REGION_BYTES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  CbWarpSmem& sm = reinterpret_cast<CbWarpSmem*>(cb_smem + CB_REGION_BYTES + 256)[warp];

  {
    const __half* f2 = a.l1 + (int64_t)slot * a.s_slot;
    for (int idx = threadIdx.x; idx < CB_RS * CB_RS * 16; idx += CB_WARPS * 32) {
      const int q = idx >> 4, c = idx & 15;
      const int y = ry0 + (q >> 4), x = rx0 + (q & 15);
      const bool in = (unsigned)y < (unsigned)a.H1 && (unsigned)x < (unsigned)a.W1;
      const __half* src = in ? f2 + (int64_t)y * a.sy + (int64_t)x * a.sx + c * 8 : f2;
      cp_async16(region + q * 256 + ((c ^ ((q & 1) << 2)) << 4), src, in ? 16 : 0);
    }
    cp_async_commit();
    if (threadIdx.x < 16) asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};\n" ::"r"(zero + threadIdx.x * 16), "r"(0u) : "memory");
  }

  // A operand = patch pixels (row g; row 8 on the g == 0 lanes), K permuted as in corr_fwd_mma:
  // k-step s = 2 kb + h, logical k {2t, 2t+1 | 2t+8, 2t+9} <-> channel 32 kb + 8 t + 4 h + {0,1 | 2,3}.
  // The next edge's operand and coordinates are fetched while the current one is blended (and the first edge's while
  // the region lands); the edge ids and patch slots, one dependent load after another, are read once per item.
  uint4 PA[4], PB[4];
  float cx = 0.f, cy = 0.f;                     // lanes 0..8: the edge's nine reprojected pixels
  // lane k < CB_ITEM / CB_WARPS holds the id and patch slot of this warp's k-th edge, loaded once per item
  int my_e = 0, my_slot = 0;
  if (lane < CB_ITEM / CB_WARPS && warp + CB_WARPS * lane < item.z) {
    my_e = a.order[item.y + warp + CB_WARPS * lane];
    my_slot = (int)a.ii[my_e];
  }
  auto fetch = [&](int k) {
    const int e = __shfl_sync(0xffffffffu, my_e, k);
    const __half* pp = a.f1 + (int64_t)__shfl_sync(0xffffffffu, my_slot, k) * 1152;
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
      PA[kb] = cb_ldg128(pp + g * 128 + kb * 32 + t * 8);
      PB[kb] = g == 0 ? cb_ldg128(pp + 8 * 128 + kb * 32 + t * 8) : make_uint4(0u, 0u, 0u, 0u);
    }
    if (lane < 9) { cx = a.coords[(int64_t)e * 18 + lane]; cy = a.coords[(int64_t)e * 18 + 9 + lane]; }
  };
  if (warp < item.z) fetch(0);
  cp_async_wait<0>();
  __syncthreads();

  for (int j = warp, k = 0; j < item.z; j += CB_WARPS, ++k) {
    int ax = 1 << 28, ay = 1 << 28, axm = -(1 << 28), aym = -(1 << 28);
    float fx = 0.f, fy = 0.f;
    if (lane < 9) {
      const float x = cx / a.div1, y = cy / a.div1;
      ax = safe_floor_int(x) - 3; ay = safe_floor_int(y) - 3;
      axm = ax; aym = ay;
      fx = x - floorf(x); fy = y - floorf(y);
    }
    const int bx = __reduce_min_sync(0xffffffffu, ax), by = __reduce_min_sync(0xffffffffu, ay);
    const int bw = __reduce_max_sync(0xffffffffu, axm) - bx + 8, rows = bw * (__reduce_max_sync(0xffffffffu, aym) - by + 8);
    __syncwarp();                              // the previous edge's blend has read w / base
    if (lane < 9) {
      sm.w[lane] = make_float4((1.f - fx) * (1.f - fy), fx * (1.f - fy), (1.f - fx) * fy, fx * fy);
      sm.base[lane] = (ay - by) * bw + (ax - bx);
    }
    const int ntiles = (rows + 7) >> 3;
    // box pixel of this lane's B column: wp = nt * 8 + g, advanced incrementally (8 <= bw <= 10: one wrap at most)
    int wx = g, wy = 0;
    auto load_tile = [&](uint4 (&Q)[4], int wp) {
      const int y = by + wy - ry0, x = bx + wx - rx0;
      const bool ok = wp < rows && (unsigned)y < (unsigned)CB_RS && (unsigned)x < (unsigned)CB_RS;
      const int q = y * CB_RS + x;
      const uint32_t pa = ok ? region + q * 256 : zero;
      const uint32_t sw = ok ? (uint32_t)((q & 1) << 2) : 0u;
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) Q[kb] = cb_lds128(pa + ((((uint32_t)(4 * kb + t)) ^ sw) << 4));
      wx += 8; if (wx >= bw) { wx -= bw; ++wy; }
    };
    auto mma_tile = [&](const uint4 (&Q)[4], int nt) {
      float acc0[4] = {0.f, 0.f, 0.f, 0.f}, acc1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) {
        mma_m16n8k16(acc0, PA[kb].x, PB[kb].x, PA[kb].y, PB[kb].y, Q[kb].x, Q[kb].y);
        mma_m16n8k16(acc1, PA[kb].z, PB[kb].z, PA[kb].w, PB[kb].w, Q[kb].z, Q[kb].w);
      }
      const int col = nt * 8 + 2 * t;
      *reinterpret_cast<float2*>(&sm.raw[g * CB_RAWP + col + (g & 1)]) = make_float2(acc0[0] + acc1[0], acc0[1] + acc1[1]);
      if (g == 0) *reinterpret_cast<float2*>(&sm.raw[8 * CB_RAWP + col]) = make_float2(acc0[2] + acc1[2], acc0[3] + acc1[3]);
    };
    // one tile at a time: the warps of the CTA hide the shared-memory latency (a second register buffer would not fit
    // the register budget that lets one CTA of this kernel share an SM with corr_fwd_tc)
    for (int nt = 0; nt < ntiles; ++nt) {
      uint4 Q[4];
      load_tile(Q, nt * 8 + g);
      mma_tile(Q, nt);
    }
    const int e = __shfl_sync(0xffffffffu, my_e, k);
    if (j + CB_WARPS < item.z) fetch(k + 1);  // the A fragments are dead here
    __syncwarp();
    // bilinear blend: the arithmetic of corr_fwd_mma / corr_fwd_tc, rounded to fp16.  A lane takes (patch pixel p, tap
    // row y, half of the tap columns) tasks as corr_fwd_tc's epilogue does: the taps of a run share their corners, so
    // each raw value is read once per task
#pragma unroll 1
    for (int task = lane; task < 126; task += 32) {
      const int hx = task / 63, u = task - 63 * hx, p = u % 9, yrow = u / 9, x0 = hx * 4, nx = 4 - hx;
      const float4 w = sm.w[p];
      const float* r0 = &sm.raw[p * CB_RAWP + (p & 1) + sm.base[p] + yrow * bw + x0];
      float ra[5], rb[5];                         // rows y and y + 1, columns x0 .. x0 + nx
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        if (i <= nx) { ra[i] = r0[i]; rb[i] = r0[bw + i]; }
        else { ra[i] = rb[i] = 0.f; }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (i < nx)
          sm.stage[((x0 + i) * 7 + yrow) * 9 + p] = __float2half_rn(w.x * ra[i] + w.y * ra[i + 1] + w.z * rb[i] + w.w * rb[i + 1]);
    }
    __syncwarp();
    __half* orow = a.out + (int64_t)e * a.out_row + 1;          // odd halves: level 1 of each pair
    for (int q = lane; q < 441; q += 32) orow[2 * q] = sm.stage[q];
  }
}

static CbBinArgs cb_layout(void* workspace, int M, int S2, int H1, int W1, float div1) {
  CbBinArgs b;
  b.div1 = div1; b.M = M; b.S2 = S2;
  b.nty = (H1 + CB_APRON + CB_T1 - 1) / CB_T1; b.ntx = (W1 + CB_APRON + CB_T1 - 1) / CB_T1;
  WsLayout L(workspace, sizeof(int));
  cb_regions(M, L, b);
  return b;
}

// Bins the edges into the workspace (layout above): the list of the mma.sync kernel with its length (*list, *count),
// the other edges in bin order with theirs (*order, *ordered), and the level-1 work items.  Returns
// DPVO_ERR_UNSUPPORTED, before launching anything, when the bins of this ring do not fit the workspace.
int corr_bin_edges(const float* coords, const int64_t* jj, int M, int S2, int H1, int W1, float div1, void* workspace,
                   cudaStream_t st, int** list, int** count, int** order, int** ordered) {
  CbBinArgs b = cb_layout(workspace, M, S2, H1, W1, div1);
  const int64_t nkeys = (int64_t)S2 * b.nty * b.ntx;
  if (nkeys > cb_key_cap(M) || ((uintptr_t)workspace & 15)) return DPVO_ERR_UNSUPPORTED;
  if (cudaFuncSetAttribute(corr_fwd_l1_tiles, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) != cudaSuccess) {
    cudaGetLastError();
    return DPVO_ERR_UNSUPPORTED;
  }
  b.coords = coords; b.jj = jj;
  int rc = check_cuda(cudaMemsetAsync(b.hdr, 0, 4 * sizeof(int), st), "corr_bin: memset");
  if (!rc) rc = check_cuda(cudaMemsetAsync(b.cnt, 0, nkeys * sizeof(int), st), "corr_bin: memset");
  if (rc) return rc;
  const unsigned eg = (unsigned)((M + 255) / 256);
  rc = launch("corr_bin_count", corr_bin_count, eg, 256, 0, st, b);
  if (!rc) rc = launch("corr_bin_scan", corr_bin_scan, 1, 1024, 0, st, b, (int)nkeys);
  if (!rc) rc = launch("corr_bin_scatter", corr_bin_scatter, eg, 256, 0, st, b);
  if (rc) return rc;
  *list = b.list; *count = b.hdr; *order = b.order; *ordered = b.hdr + 1;
  return DPVO_OK;
}

// The level-1 pass over the work items corr_bin_edges left in the workspace.
int corr_bin_level1(const void* fmap1, const void* l1, const int64_t* s21, int H1, int W1, int S2, float div1,
                    const float* coords, const int64_t* ii, void* out, int64_t out_row, int M, void* workspace,
                    cudaStream_t st) {
  const CbBinArgs b = cb_layout(workspace, M, S2, H1, W1, div1);
  CbArgs a;
  a.f1 = reinterpret_cast<const __half*>(fmap1); a.l1 = reinterpret_cast<const __half*>(l1);
  a.s_slot = s21[1]; a.sy = s21[3]; a.sx = s21[4];
  a.coords = coords; a.ii = ii; a.out = reinterpret_cast<__half*>(out); a.out_row = out_row; a.div1 = div1;
  a.H1 = H1; a.W1 = W1; a.nty = b.nty; a.ntx = b.ntx; a.order = b.order; a.items = b.items; a.item_count = b.hdr + 2;
  const unsigned grid = (unsigned)((int64_t)S2 * b.nty * b.ntx + (M + CB_ITEM - 1) / CB_ITEM);     // bound on the items
  return launch("corr_fwd_l1_tiles", corr_fwd_l1_tiles, grid, CB_WARPS * 32, CB_SMEM, st, a);
}

}  // namespace dpvo
