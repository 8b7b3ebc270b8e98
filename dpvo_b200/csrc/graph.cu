// Patch-graph index structure, built on the device in ONE cooperative launch.
//
// The reference rebuilds the same information three times per update() on different paths:
//   * fastba.neighbors   ba.cpp:59-97      torch::_unique on GPU, D2H, per-group CPU stable_sort, H2D
//   * SoftAgg            blocks.py:41      torch.unique(return_inverse) x2 (host sync each)
//   * cuda_ba            ba_cuda.cu:447    torch::_unique(kk) (host sync)
// Here: a stable LSD radix sort of edge ids by (key_a, key_b, sec) over only the bits the value
// ranges need (ranges are found on the device), followed by boundary flagging and a scan that
// yields a CSR (order / group_start), the dense group id per edge and the group keys.  All
// phases run inside one persistent kernel separated by a software grid barrier; there are no
// floating-point or order-dependent atomics, so the result is bit-reproducible.
#include "common.cuh"
#include <cstring>

namespace dpvo {

constexpr int G_THREADS = 256;
constexpr int G_ITEMS = 4;
constexpr int G_TILE = G_THREADS * G_ITEMS;   // 1024 edge slots per tile
constexpr int G_WARPS = G_THREADS / 32;
constexpr int G_MAXBITS = 10;                 // radix digit width is chosen per sort, <= 10 bits
constexpr int G_BINS = 1 << G_MAXBITS;
constexpr int G_MAXPASS = 20;

// Header at the start of the workspace; the host wrapper memsets it to zero before the launch.
// Ranges are tracked as unsigned maxima of the order-preserving bias u = x ^ 2^63 and of ~u (giving
// the minimum), so zero is a valid initial value and no initialisation phase is needed.
struct GroupHeader {
  unsigned barrier; unsigned pad;
  unsigned long long amax, anmax, bmax, bnmax, smax, snmax;
};

struct GroupArgs {
  const int64_t* ka; const int64_t* kb; const int64_t* sec;
  int64_t E; int ntiles;
  int32_t* order; int32_t* group_of; int32_t* group_start;
  int64_t* group_key_a; int64_t* group_key_b; int32_t* n_groups;
  GroupHeader* hdr; int32_t* buf0; int32_t* buf1; unsigned* hist; int32_t* tile_sums;
};

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned& epoch) {
  __syncthreads();
  if (threadIdx.x == 0) {
    epoch += gridDim.x;
    __threadfence();
    atomicAdd(ctr, 1u);
    while (ld_acquire_u32(ctr) < epoch) { }
    __threadfence();
  }
  __syncthreads();
}

__device__ __forceinline__ int bits_needed(unsigned long long range) {
  return range == 0 ? 0 : 64 - __clzll(range);
}
__device__ __forceinline__ unsigned long long bias64(long long x) { return (unsigned long long)x ^ 0x8000000000000000ull; }

// exclusive scan of one int per thread across the block; returns the exclusive prefix and the total
__device__ __forceinline__ int block_excl_scan(int v, int* smem_warp /*[G_WARPS+1]*/, int& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  __syncthreads();
  if (lane == 31) smem_warp[w] = inc;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int i = 0; i < G_WARPS; ++i) { int t = smem_warp[i]; smem_warp[i] = run; run += t; }
    smem_warp[G_WARPS] = run;
  }
  __syncthreads();
  total = smem_warp[G_WARPS];
  return smem_warp[w] + inc - v;
}

// One persistent kernel: ranges -> [count, scatter] per radix pass -> boundary flags -> group ids.
// Two grid barriers per pass (every block derives its own scatter offsets from the tile-major
// histogram instead of waiting for a scan block), one after the ranges, one before the final phase.
// blockIdx.y selects one of (up to) two independent problems handled by the same launch: an update needs the edges
// grouped by patch and by (source, target) frame, and the kernel is bound by the latency of its grid barriers,
// not by work, so the second grouping rides along for free.  Barriers are per problem (own header, gridDim.x CTAs).
__global__ void __launch_bounds__(G_THREADS)
group_edges_kernel(const GroupArgs a0, const GroupArgs a1) {
  const GroupArgs& a = blockIdx.y ? a1 : a0;
  __shared__ unsigned warp_hist[G_WARPS][G_BINS];
  __shared__ int scan_tmp[G_WARPS + 1];
  __shared__ unsigned long long red[6];
  __shared__ int p_field[G_MAXPASS], p_shift[G_MAXPASS], p_bits[G_MAXPASS], n_pass;
  unsigned epoch = 0;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  GroupHeader* H = a.hdr;
  const int64_t E = a.E;

  // ---- phase 0: value ranges, identity permutation
  {
    unsigned long long mx[6] = {0, 0, 0, 0, 0, 0};
    for (int64_t i = (int64_t)blockIdx.x * G_THREADS + tid; i < E; i += (int64_t)gridDim.x * G_THREADS) {
      a.buf0[i] = (int32_t)i;
      const unsigned long long ua = bias64(a.ka[i]);
      mx[0] = max(mx[0], ua); mx[1] = max(mx[1], ~ua);
      if (a.kb) { const unsigned long long ub = bias64(a.kb[i]); mx[2] = max(mx[2], ub); mx[3] = max(mx[3], ~ub); }
      if (a.sec) { const unsigned long long us = bias64(a.sec[i]); mx[4] = max(mx[4], us); mx[5] = max(mx[5], ~us); }
    }
    if (tid < 6) red[tid] = 0ull;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 6; ++k) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx[k] = max(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
      if (lane == 0) atomicMax(&red[k], mx[k]);
    }
    __syncthreads();
    if (tid < 6) atomicMax(&H->amax + tid, red[tid]);
  }
  grid_barrier(&H->barrier, epoch);

  const unsigned long long amin = ~H->anmax, bmin = a.kb ? ~H->bnmax : 0, smin = a.sec ? ~H->snmax : 0;
  const int abits = bits_needed(H->amax - amin);
  const int bbits = a.kb ? bits_needed(H->bmax - bmin) : 0;
  const int sbits = a.sec ? bits_needed(H->smax - smin) : 0;
  const bool composite = abits + bbits + sbits <= 64;
  if (tid == 0) {
    // pass table (least significant first).  composite: one key  a_rel << (bbits+sbits) | b_rel << sbits | s_rel
    int np = 0;
    auto add_field = [&](int field, int bits) {
      if (bits == 0) return;
      const int passes = (bits + G_MAXBITS - 1) / G_MAXBITS, per = (bits + passes - 1) / passes;
      for (int sh = 0; sh < bits; sh += per) { p_field[np] = field; p_shift[np] = sh; p_bits[np] = min(per, bits - sh); ++np; }
    };
    if (composite) add_field(3, abits + bbits + sbits);
    else { add_field(0, sbits); add_field(1, bbits); add_field(2, abits); }
    n_pass = np;
  }
  __syncthreads();

  auto key_of = [&](int32_t e, int field) -> unsigned long long {
    if (field == 3) {
      unsigned long long k = bias64(a.ka[e]) - amin;
      if (a.kb) k = (k << bbits) | (bias64(a.kb[e]) - bmin);
      if (a.sec) k = (k << sbits) | (bias64(a.sec[e]) - smin);
      return k;
    }
    if (field == 0) return bias64(a.sec[e]) - smin;
    if (field == 1) return bias64(a.kb[e]) - bmin;
    return bias64(a.ka[e]) - amin;
  };

  int32_t* src = a.buf0;
  int32_t* dst = a.buf1;
  const int npass = n_pass;

  for (int pass = 0; pass < npass; ++pass) {
    const int field = p_field[pass], shift = p_shift[pass], nbins = 1 << p_bits[pass];
    const unsigned mask = (unsigned)nbins - 1u;

    // per-warp stable digit histograms of one tile (warp w owns 128 consecutive slots)
    auto warp_count = [&](int t) {
      for (int i = tid; i < G_WARPS * nbins; i += G_THREADS) warp_hist[i / nbins][i % nbins] = 0u;
      __syncthreads();
      const int64_t base = (int64_t)t * G_TILE + w * (G_TILE / G_WARPS);
#pragma unroll
      for (int c = 0; c < G_TILE / G_WARPS / 32; ++c) {
        const int64_t i = base + c * 32 + lane;
        unsigned d = 0xffffffffu;
        if (i < E) d = (unsigned)(key_of(src[i], field) >> shift) & mask;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        if (d != 0xffffffffu && lane == __ffs(peers) - 1) warp_hist[w][d] += __popc(peers);
        __syncwarp();
      }
      __syncthreads();
    };

    // ---- count
    for (int t = blockIdx.x; t < a.ntiles; t += gridDim.x) {
      warp_count(t);
      for (int b = tid; b < nbins; b += G_THREADS) {
        unsigned sum = 0;
#pragma unroll
        for (int k = 0; k < G_WARPS; ++k) sum += warp_hist[k][b];
        a.hist[(size_t)t * G_BINS + b] = sum;
      }
      __syncthreads();
    }
    grid_barrier(&H->barrier, epoch);

    // ---- scatter: every block derives the offsets of its own tiles from the tile-major histogram
    for (int t = blockIdx.x; t < a.ntiles; t += gridDim.x) {
      warp_count(t);
      const int bpt = (nbins + G_THREADS - 1) / G_THREADS;      // contiguous bins per thread
      unsigned before[G_BINS / G_THREADS], total[G_BINS / G_THREADS];
      int mine = 0;
#pragma unroll
      for (int k = 0; k < G_BINS / G_THREADS; ++k) {
        before[k] = 0; total[k] = 0;
        const int b = tid * bpt + k;
        if (k < bpt && b < nbins) {
          for (int tt = 0; tt < a.ntiles; ++tt) {
            const unsigned v = a.hist[(size_t)tt * G_BINS + b];
            if (tt < t) before[k] += v;
            total[k] += v;
          }
          mine += (int)total[k];
        }
      }
      int all;
      unsigned run = (unsigned)block_excl_scan(mine, scan_tmp, all);      // bins are contiguous per thread
#pragma unroll
      for (int k = 0; k < G_BINS / G_THREADS; ++k) {
        const int b = tid * bpt + k;
        if (k < bpt && b < nbins) {
          unsigned o = run + before[k];
          run += total[k];
#pragma unroll
          for (int q = 0; q < G_WARPS; ++q) { const unsigned v = warp_hist[q][b]; warp_hist[q][b] = o; o += v; }
        }
      }
      __syncthreads();
      const int64_t base = (int64_t)t * G_TILE + w * (G_TILE / G_WARPS);
#pragma unroll
      for (int c = 0; c < G_TILE / G_WARPS / 32; ++c) {
        const int64_t i = base + c * 32 + lane;
        unsigned d = 0xffffffffu;
        int32_t id = 0;
        if (i < E) { id = src[i]; d = (unsigned)(key_of(id, field) >> shift) & mask; }
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        unsigned pos = 0;
        if (d != 0xffffffffu && lane == leader) { pos = warp_hist[w][d]; warp_hist[w][d] = pos + __popc(peers); }
        pos = __shfl_sync(0xffffffffu, pos, leader);
        if (d != 0xffffffffu) dst[pos + __popc(peers & ((1u << lane) - 1u))] = id;
        __syncwarp();
      }
      __syncthreads();
    }
    grid_barrier(&H->barrier, epoch);
    int32_t* tmp = src; src = dst; dst = tmp;
  }

  // ---- boundaries: flag[i] = first position of a new (key_a, key_b) group
  auto is_head = [&](int64_t i) -> int {
    if (i == 0) return 1;
    const int32_t e = src[i], p = src[i - 1];
    if (a.ka[e] != a.ka[p]) return 1;
    if (a.kb && a.kb[e] != a.kb[p]) return 1;
    return 0;
  };
  for (int t = blockIdx.x; t < a.ntiles; t += gridDim.x) {
    int cnt = 0;
    const int64_t base = (int64_t)t * G_TILE + (int64_t)tid * G_ITEMS;
#pragma unroll
    for (int k = 0; k < G_ITEMS; ++k) if (base + k < E) cnt += is_head(base + k);
    int total;
    block_excl_scan(cnt, scan_tmp, total);
    if (tid == 0) a.tile_sums[t] = total;
    __syncthreads();
  }
  grid_barrier(&H->barrier, epoch);
  for (int t = blockIdx.x; t < a.ntiles; t += gridDim.x) {
    // groups before this tile (and, for the block owning tile 0, the grand total)
    int part = 0, whole = 0;
    for (int tt = tid; tt < a.ntiles; tt += G_THREADS) {
      const int v = a.tile_sums[tt];
      whole += v;
      if (tt < t) part += v;
    }
    int tot_part, tot_whole;
    block_excl_scan(part, scan_tmp, tot_part);
    block_excl_scan(whole, scan_tmp, tot_whole);
    if (t == 0 && tid == 0) { *a.n_groups = tot_whole; a.group_start[tot_whole] = (int32_t)E; }
    int flags[G_ITEMS];
    int cnt = 0;
    const int64_t base = (int64_t)t * G_TILE + (int64_t)tid * G_ITEMS;
#pragma unroll
    for (int k = 0; k < G_ITEMS; ++k) { flags[k] = (base + k < E) ? is_head(base + k) : 0; cnt += flags[k]; }
    int total;
    int gid = tot_part + block_excl_scan(cnt, scan_tmp, total) - 1;
#pragma unroll
    for (int k = 0; k < G_ITEMS; ++k) {
      const int64_t i = base + k;
      if (i < E) {
        const int32_t e = src[i];
        gid += flags[k];
        a.group_of[e] = gid;
        a.order[i] = e;
        if (flags[k]) {
          a.group_start[gid] = (int32_t)i;
          a.group_key_a[gid] = a.ka[e];
          if (a.group_key_b) a.group_key_b[gid] = a.kb ? a.kb[e] : 0;
        }
      }
    }
    __syncthreads();
  }
}

// neighbours inside a group in sorted order (ba.cpp:88-94)
__global__ void neighbors_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ group_of,
                                 int64_t E, int64_t* __restrict__ ix, int64_t* __restrict__ jx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t e = order[i];
    const int32_t g = group_of[e];
    int64_t prev = -1, next = -1;
    if (i > 0) { const int32_t p = order[i - 1]; if (group_of[p] == g) prev = p; }
    if (i + 1 < E) { const int32_t n = order[i + 1]; if (group_of[n] == g) next = n; }
    ix[e] = prev; jx[e] = next;
  }
}

// the grouping's workspace: header, the two permutation buffers of the radix passes, the tile-major digit histogram
// and the tile sums of the group-boundary scan
static void group_layout(int64_t E, WsLayout& L, GroupArgs& a) {
  const int64_t ntiles = (E + G_TILE - 1) / G_TILE;
  a.hdr = L.take<GroupHeader>(1); a.buf0 = L.take<int32_t>(E); a.buf1 = L.take<int32_t>(E);
  a.hist = L.take<unsigned>(ntiles * G_BINS); a.tile_sums = L.take<int32_t>(ntiles + 1);
}
static int64_t group_ws_bytes(int64_t E) { GroupArgs a; WsLayout L; group_layout(E, L, a); return L.bytes(); }

struct GroupProblem {
  const int64_t* ka; const int64_t* kb; const int64_t* sec; int64_t E;
  int32_t* order; int32_t* group_of; int32_t* group_start; int64_t* gka; int64_t* gkb; int32_t* n_groups;
  void* ws; int64_t ws_bytes;
};

static int group_fill(const GroupProblem& p, GroupArgs& a, cudaStream_t st) {
  const int64_t E = p.E;
  if (p.ws_bytes < group_ws_bytes(E)) {
    set_error("group_edges: workspace %lld B < required %lld B", (long long)p.ws_bytes, (long long)group_ws_bytes(E));
    return DPVO_ERR_WORKSPACE;
  }
  if (E >= (1ll << 31)) { set_error("group_edges: E too large"); return DPVO_ERR_UNSUPPORTED; }
  a.ka = p.ka; a.kb = p.kb; a.sec = p.sec; a.E = E; a.ntiles = (int)((E + G_TILE - 1) / G_TILE);
  a.order = p.order; a.group_of = p.group_of; a.group_start = p.group_start;
  a.group_key_a = p.gka; a.group_key_b = p.gkb; a.n_groups = p.n_groups;
  WsLayout L(p.ws);
  group_layout(E, L, a);
  int rc = check_cuda(cudaMemsetAsync(a.hdr, 0, sizeof(GroupHeader), st), "group_edges: memset");
  if (rc) return rc;
  if (E == 0) {
    rc = check_cuda(cudaMemsetAsync(p.n_groups, 0, 4, st), "group_edges: memset");
    if (rc) return rc;
    return check_cuda(cudaMemsetAsync(p.group_start, 0, 4, st), "group_edges: memset");
  }
  return DPVO_OK;
}

// one cooperative launch for one or two problems (second may be NULL)
static int group_launch_n(const GroupProblem* p0, const GroupProblem* p1, cudaStream_t st) {
  GroupArgs a0, a1;
  memset(&a0, 0, sizeof(a0)); memset(&a1, 0, sizeof(a1));
  int rc = group_fill(*p0, a0, st);
  if (rc) return rc;
  if (p1) { rc = group_fill(*p1, a1, st); if (rc) return rc; }
  const bool two = p1 && p1->E > 0;
  if (p0->E == 0 && !two) return DPVO_OK;
  if (p0->E == 0) { a0 = a1; }                       // only the second problem has work: run it alone
  const bool both = two && p0->E > 0;
  int per_sm = 0;                                     // per device: asked on every call (host-side table lookup)
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, group_edges_kernel, G_THREADS, 0);
  const int max_blocks = std::max(1, per_sm) * sm_count();
  // both y-slices use the same x extent; the tile loops stride by gridDim.x, so any extent >= 1 is correct
  const int want = both ? std::max(a0.ntiles, a1.ntiles) : a0.ntiles;
  const int grid = std::max(1, std::min(want, max_blocks / (both ? 2 : 1)));
  return launch<cudaLaunchAttributeCooperative>("group_edges_kernel", group_edges_kernel, dim3(grid, both ? 2 : 1), G_THREADS, 0, st, a0, a1);
}

}  // namespace dpvo

using namespace dpvo;

extern "C" int64_t dpvo_group_workspace_bytes(int64_t E) { return group_ws_bytes(E < 0 ? 0 : E); }

extern "C" int dpvo_group_edges(const int64_t* key_a, const int64_t* key_b, const int64_t* sec, int64_t E,
                                int32_t* order, int32_t* group_of, int32_t* group_start,
                                int64_t* group_key_a, int64_t* group_key_b, int32_t* n_groups,
                                void* workspace, int64_t workspace_bytes, void* stream) {
  DPVO_REQUIRE(E >= 0, "group_edges: negative E");
  DPVO_REQUIRE(order && group_of && group_start && group_key_a && n_groups && workspace, "group_edges: null pointer");
  DPVO_REQUIRE(E == 0 || key_a, "group_edges: null key");
  GroupProblem p{key_a, key_b, sec, E, order, group_of, group_start, group_key_a, group_key_b, n_groups, workspace, workspace_bytes};
  return group_launch_n(&p, nullptr, (cudaStream_t)stream);
}

extern "C" int dpvo_group_edges_pair(const int64_t* key_a0, const int64_t* key_b0, const int64_t* sec0,
                                     int32_t* order0, int32_t* group_of0, int32_t* group_start0,
                                     int64_t* group_key_a0, int64_t* group_key_b0, int32_t* n_groups0, void* workspace0,
                                     const int64_t* key_a1, const int64_t* key_b1, const int64_t* sec1,
                                     int32_t* order1, int32_t* group_of1, int32_t* group_start1,
                                     int64_t* group_key_a1, int64_t* group_key_b1, int32_t* n_groups1, void* workspace1,
                                     int64_t E, int64_t workspace_bytes_each, void* stream) {
  DPVO_REQUIRE(E >= 0, "group_edges_pair: negative E");
  DPVO_REQUIRE(order0 && group_of0 && group_start0 && group_key_a0 && n_groups0 && workspace0 && order1 && group_of1 && group_start1 &&
               group_key_a1 && n_groups1 && workspace1, "group_edges_pair: null pointer");
  DPVO_REQUIRE(E == 0 || (key_a0 && key_a1), "group_edges_pair: null key");
  DPVO_REQUIRE(workspace0 != workspace1, "group_edges_pair: the two problems need separate workspaces");
  GroupProblem p0{key_a0, key_b0, sec0, E, order0, group_of0, group_start0, group_key_a0, group_key_b0, n_groups0, workspace0, workspace_bytes_each};
  GroupProblem p1{key_a1, key_b1, sec1, E, order1, group_of1, group_start1, group_key_a1, group_key_b1, n_groups1, workspace1, workspace_bytes_each};
  return group_launch_n(&p0, &p1, (cudaStream_t)stream);
}

// dpvo_neighbors: the edges grouped by ii and ordered by jj -- the grouping's outputs, then its workspace
static GroupProblem neighbors_layout(const int64_t* ii, const int64_t* jj, int64_t E, WsLayout& L) {
  GroupProblem p{ii, nullptr, jj, E};
  p.order = L.take<int32_t>(E); p.group_of = L.take<int32_t>(E); p.group_start = L.take<int32_t>(E + 1);
  p.gka = L.take<int64_t>(E); p.n_groups = L.take<int32_t>(1); p.ws = L.take<char>(group_ws_bytes(E));
  return p;
}

extern "C" int64_t dpvo_neighbors_workspace_bytes(int64_t E) {
  WsLayout L;
  neighbors_layout(nullptr, nullptr, E < 0 ? 0 : E, L);
  return L.bytes();
}

extern "C" int dpvo_neighbors(const int64_t* ii, const int64_t* jj, int64_t E,
                              int64_t* ix, int64_t* jx,
                              void* workspace, int64_t workspace_bytes, void* stream) {
  DPVO_REQUIRE(E >= 0, "neighbors: negative E");
  if (E == 0) return DPVO_OK;
  DPVO_REQUIRE(ii && jj && ix && jx && workspace, "neighbors: null pointer");
  if (workspace_bytes < dpvo_neighbors_workspace_bytes(E)) {
    set_error("neighbors: workspace too small");
    return DPVO_ERR_WORKSPACE;
  }
  WsLayout L(workspace);
  GroupProblem p = neighbors_layout(ii, jj, E, L);
  p.ws_bytes = workspace_bytes - ((char*)p.ws - (char*)workspace);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = group_launch_n(&p, nullptr, st);
  if (rc) return rc;
  const int threads = 256;
  const unsigned blocks = (unsigned)std::min<int64_t>((E + threads - 1) / threads, (int64_t)sm_count() * 8);
  return launch("neighbors_kernel", neighbors_kernel, blocks, threads, 0, st, p.order, p.group_of, E, ix, jx);
}

extern "C" int dpvo_neighbors_from_groups(const int32_t* order, const int32_t* group_of, int64_t E,
                                          int64_t* ix, int64_t* jx, void* stream) {
  DPVO_REQUIRE(E >= 0, "neighbors_from_groups: negative E");
  if (E == 0) return DPVO_OK;
  DPVO_REQUIRE(order && group_of && ix && jx, "neighbors_from_groups: null pointer");
  const int threads = 256;
  const unsigned blocks = (unsigned)std::min<int64_t>((E + threads - 1) / threads, (int64_t)sm_count() * 8);
  return launch("neighbors_kernel", neighbors_kernel, blocks, threads, 0, (cudaStream_t)stream, order, group_of, E, ix, jx);
}
