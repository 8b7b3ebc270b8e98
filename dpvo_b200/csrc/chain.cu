// The row-local layer chains of the update operator (dpvo/net.py:74-92, dpvo/blocks.py:15-29) as ONE wgmma kernel
// each: a 64-edge tile goes through all dense layers of a chain without leaving the SM.
//
//   chain A  (net.py:76-77)   net = LN( net + inp[kk] + corr-MLP(corr) )          882->384 ReLU 384 LN ReLU 384
//   chain C  (net.py:83-85)   net = net + c( mask * net[ix] )                      384 ReLU 384   (c1 and c2)
//   chain G  (net.py:88-92)   net = GRU( net + h_kk[patch] + h_ij[pair] ); delta, weight   LN, gated res., LN, gated res., heads
//
// What the separate-layer path paid for and this kernel does not: every intermediate [E,384] activation written to
// and read back from global memory, one LayerNorm / gating / heads pass over the fp32 state per step, one launch
// (with its tail wave) per layer.
//
// One persistent CTA per SM, in clusters of CH_CL CTAs that work on CH_CL neighbouring tiles at a time and share
// every weight k-block: each CTA loads 1/CH_CL of its rows from L2 and multicasts them into the weight rings of all CTAs
// of the cluster, so L2 sends each weight byte once per cluster instead of once per CTA (at one 64-row tile per CTA a
// weight byte feeds only 64 FLOP: unshared, the weight feed asks more of L2 than the tensor pipe asks of it).  Roles:
//   warps 0-7  consumers   two warpgroups, warpgroup h owns column half h (192 columns) of the 64-row tile: it issues
//                          wgmma.m64n192k16 on shared-memory descriptors (a layer is 6 k-blocks x 4 instructions), keeps the
//                          64 x 192 fp32 accumulator in registers and runs the epilogue from them: bias, activation,
//                          LayerNorm (row statistics exchanged between the two warps that share a row), gating, heads; the
//                          fp16 result is written straight into the shared-memory operand tile of the NEXT layer in the
//                          SWIZZLE_128B K-major layout the descriptors expect.  All parameters sit in shared memory.
//                          A stage of the weight ring is handed back to every CTA of the cluster once its MMAs retired.
//   warp  8    W producer  streams its share of the weight k-blocks (192 x 64 fp16 = 24 KB each) of every layer of every
//                          tile through a 6-deep TMA ring, alternating the column halves; it depends on no data, so it
//                          runs ahead across layers and tiles, as far as the slowest CTA of the cluster has freed stages
//   warp  9    (chain A)   streams the 14 k-blocks of the 896-column correlation rows through the operand slots
//   warps 9-10 (chain C)   gather the neighbour rows net[ix] (masked) into the operand slots with cp.async
//   (warps 8-11 form the producer warpgroup; they hand most of their registers to the consumers)
// Every role of every CTA walks the same tile groups.  When the last group has fewer tiles than the cluster has CTAs,
// the CTAs without a tile still load their share of every weight k-block, and their consumers wait for and release each
// stage without computing.
// Shared memory: 6 operand slots of 64 rows x 64 halves (48 KB, one K=384 activation tile, overwritten in place by the
// layer's own output once both warpgroups' MMAs have retired), the weight ring (144 KB), the parameter vectors, 2 KB of
// exchange.  The fp32 recurrent state is read and written by the consumers directly: a warp's accesses cover 8 rows x
// 32 contiguous bytes, whole sectors.
// Row-private intermediates of chain G (the sigmoid gate, the fp32 LayerNorm output that the gated residual adds to)
// do not fit next to the accumulator in registers; they live in a per-CTA global scratch laid out fragment-major
// ([element pair][thread]) so that every access is a coalesced 256-byte warp transaction; it is rewritten every tile
// and stays in L2.
#include "common.cuh"
#include "tc.cuh"
#include <algorithm>
#include <atomic>
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace dpvo {

constexpr int CH_M = 64, CH_DIM = 384, CH_KB = 6, CH_NH = 192;
constexpr int CH_SLOT = CH_M * 128;            // one k-block of the operand tile: 64 rows x 128 bytes
constexpr int CH_WSTAGE = CH_NH * 128;         // one weight k-block of a column half: 192 rows x 128 bytes
constexpr int CH_WST = 6;                      // weight ring depth (even: each column half keeps to its own stages)
constexpr int CH_CL = 2;                       // CTAs per cluster, sharing every weight k-block
constexpr int CH_WBOX = CH_NH / CH_CL;         // rows of a weight k-block that one CTA of the cluster loads
static_assert(CH_WST % 2 == 0, "the column halves alternate through the weight ring");
// a CTA's share must be whole 8-row SWIZZLE_128B atoms at a 1024-byte aligned offset: the assembled stage is then
// byte-identical to one 192-row load
static_assert(CH_NH % CH_CL == 0 && CH_WBOX % 8 == 0, "weight share per CTA");
constexpr int CH_K0 = 896, CH_KB0 = CH_K0 / 64;
constexpr int CH_CONS_WARPS = 8, CH_CONS = CH_CONS_WARPS * 32, CH_W_WARP = 8, CH_A_WARP = 9;
constexpr int CH_GATHER_THREADS = 64;
constexpr float CH_EPS = 1e-3f;

enum { CHAIN_A = 0, CHAIN_C = 1, CHAIN_G = 2 };
// two consumer warpgroups and one producer warpgroup (whole warpgroups, so that registers can move between them)
constexpr int CH_THREADS = CH_CONS + 128;

struct ChainBars {
  uint64_t w_full[CH_WST], w_empty[CH_WST];
  uint64_t a_full[CH_KB], a_empty[CH_KB];
  uint64_t slots_free;                           // the tile's last MMAs on the operand slots have retired
};
template <int CHAIN> struct ChainCfg {
  static constexpr int NPARAM = CHAIN == 0 ? 7 * CH_DIM : (CHAIN == 1 ? 2 * CH_DIM : 14 * CH_DIM + 8);   // fp32 parameters kept in shared memory
  // weight k-blocks per tile and column half: A = the K = 896 first layer + 2 layers, C = 2 layers, G = 6 layers
  static constexpr int KBLOCKS = CHAIN == 0 ? CH_KB0 + 2 * CH_KB : (CHAIN == 1 ? 2 : 6) * CH_KB;
  static constexpr int XCH_BYTES = 2 * CH_M * 16;
  static constexpr int OFF_WRING = CH_KB * CH_SLOT;
  static constexpr int OFF_XCH = OFF_WRING + CH_WST * CH_WSTAGE;
  static constexpr int OFF_PARAM = OFF_XCH + XCH_BYTES;
  static constexpr int OFF_BARS = OFF_PARAM + NPARAM * 4;
  static constexpr int SMEM = OFF_BARS + (int)sizeof(ChainBars);
};
static_assert(ChainCfg<0>::SMEM <= 232448 && ChainCfg<1>::SMEM <= 232448 && ChainCfg<2>::SMEM <= 232448, "shared memory budget");
static_assert(ChainCfg<0>::OFF_BARS % 8 == 0 && ChainCfg<1>::OFF_BARS % 8 == 0 && ChainCfg<2>::OFF_BARS % 8 == 0, "barrier alignment");
constexpr int64_t CH_SCRATCH_GATE = (int64_t)CH_M * CH_DIM * 2, CH_SCRATCH_X = (int64_t)CH_M * CH_DIM * 4;
constexpr int64_t CH_SCRATCH_PER_CTA = CH_SCRATCH_GATE + CH_SCRATCH_X;

struct ChainArgs {
  int64_t rows;
  float* state;                // the fp32 recurrent state [rows, 384]
  __half* state16;             // A, C: fp16 copy of the new state [rows, 384]
  const float* p;              // fp32 parameter block, layout per chain (see the launchers)
  const __half* inp16;         // A: context table, row e uses inp16[inp_index ? inp_index[e] : e]
  const int64_t* inp_index;
  const __half* x16;           // C: gather source [rows, 384]
  const int64_t* gidx;         // C: source row per edge, -1 = masked (zero row)
  const __half* hij16;         // G: per-group rows added to the state before the first LayerNorm
  const int32_t* group_of;
  const __half* hkk16;         // G: a second table of per-group rows (the patch aggregation, net.py:87) and its group ids
  const int32_t* group_kk;
  const float* coords; int PP; int centre;
  float* delta; float* weight;
  unsigned char* scratch;
  int n_params;                // floats in p
};

__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
// two gates per SFU op: the pre-activations are rounded to fp16 first (which is where the reference's autocast computes
// its sigmoid, blocks.py:19 under dpvo.py:332), sigmoid(x) = 0.5 + 0.5 tanh(x / 2), tanh.approx.f16x2 has an absolute
// error of 2^-11, the gate is stored as fp16
__device__ __forceinline__ __half2 sigmoid_tanh_h2(float a, float b) {
  const __half2 x = __floats2half2_rn(0.5f * a, 0.5f * b);
  uint32_t t;
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(t) : "r"(*reinterpret_cast<const uint32_t*>(&x)));
  const __half2 half = __float2half2_rn(0.5f);
  return __hfma2(*reinterpret_cast<const __half2*>(&t), half, half);
}

template <int CHAIN>
__global__ void __cluster_dims__(CH_CL, 1, 1) __launch_bounds__(CH_THREADS, 1)
chain_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW0, const __grid_constant__ CUtensorMap tmW,
             const ChainArgs a) {
  using Cfg = ChainCfg<CHAIN>;
  extern __shared__ __align__(1024) unsigned char ch_smem[];
  unsigned char* slots = ch_smem;
  unsigned char* wring = ch_smem + Cfg::OFF_WRING;
  float4* xch = reinterpret_cast<float4*>(ch_smem + Cfg::OFF_XCH);
  float* sparam = reinterpret_cast<float*>(ch_smem + Cfg::OFF_PARAM);
  ChainBars* bars = reinterpret_cast<ChainBars*>(ch_smem + Cfg::OFF_BARS);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (int)((a.rows + CH_M - 1) / CH_M);                 // rows < 2^31 (the launchers check)
  // the CTAs of a cluster are consecutive in blockIdx.x, so the tiles blockIdx.x + k gridDim.x that a CTA takes are, for
  // each k, one group of CH_CL neighbouring tiles shared by its cluster.  Every role of every CTA walks the tile count
  // rounded up to whole groups: the CTAs of a cluster share the weight stages and must all run the same number of tiles
  cg::cluster_group cluster = cg::this_cluster();
  const uint32_t rank = cluster.block_rank();
  const int n_walk = (n_tiles + CH_CL - 1) / CH_CL * CH_CL;

  if (threadIdx.x == 0) {
    if ((smem_u32(ch_smem) & 1023u) != 0) { printf("chain_kernel: shared memory base is not 1024-byte aligned\n"); __trap(); }
    // a stage is released by every warp that read it, in every CTA of the cluster: 4 per column half and CTA
    for (int s = 0; s < CH_WST; ++s) { mbar_init(&bars->w_full[s], 1); mbar_init(&bars->w_empty[s], 4 * CH_CL); }
    for (int s = 0; s < CH_KB; ++s) { mbar_init(&bars->a_full[s], CHAIN == CHAIN_C ? CH_GATHER_THREADS : 1); mbar_init(&bars->a_empty[s], CH_CONS_WARPS); }
    mbar_init(&bars->slots_free, CH_CONS_WARPS);
    mbar_init_fence();
  }
  for (int i = threadIdx.x; i < Cfg::NPARAM; i += blockDim.x) sparam[i] = i < a.n_params ? a.p[i] : 0.f;
  cluster.sync();                                                    // no peer multicasts or arrives before the barriers exist
  // 168 registers per thread at launch (3 warpgroups); the consumers hold a 96-register accumulator next to their epilogue
  if (warp >= CH_CONS_WARPS) {
  warpgroup_reg_dealloc<56>();
  if (warp == CH_W_WARP) {
    // ===================================================================== weight producer
    if (lane == 0) {
      uint32_t wit = 0;
      // also a tile past the end: the peers need this CTA's share of its weights
      for (int tile = blockIdx.x; tile < n_walk; tile += gridDim.x) {
        for (int i = 0; i < Cfg::KBLOCKS; ++i) {
          // chain A: the 14 k-blocks of the K = 896 first layer (tmW0), then the K = 384 layers stacked in tmW
          const bool first = CHAIN == CHAIN_A && i < CH_KB0;
          const int j = (CHAIN == CHAIN_A && !first) ? i - CH_KB0 : i;
          const CUtensorMap* tm = first ? &tmW0 : &tmW;
          const int kcol = (first ? j : j % CH_KB) * 64, wrow = first ? 0 : j / CH_KB * CH_DIM;
          for (int h = 0; h < 2; ++h) {
            const uint32_t s = wit % CH_WST, ph = (wit / CH_WST) & 1;
            mbar_wait_bounded(&bars->w_empty[s], ph ^ 1);              // every CTA of the cluster has released the stage
            // armed for the whole k-block, this CTA's share and the peers'; a peer's share may complete bytes on this
            // phase before it is armed
            mbar_arrive_expect_tx(&bars->w_full[s], CH_WSTAGE);
            tma_load_2d_multicast(smem_u32(wring + s * CH_WSTAGE + rank * CH_WBOX * 128), tm, kcol, wrow + h * CH_NH + (int)rank * CH_WBOX,
                                  &bars->w_full[s], (uint16_t)((1u << CH_CL) - 1));
            ++wit;
          }
        }
      }
    }
  } else if (CHAIN == CHAIN_A && warp == CH_A_WARP) {
    // ===================================================================== chain A: correlation rows, 14 k-blocks
    if (lane == 0) {
      uint32_t ait = 0, ti = 0;
      for (int tile = blockIdx.x; tile < n_walk; tile += gridDim.x, ++ti) {
        if (tile >= n_tiles) continue;                               // past the end: nothing to load
        if (ti > 0) mbar_wait_bounded(&bars->slots_free, (ti - 1) & 1);   // the previous tile is done with the slots
        const int m0 = (int)(tile * CH_M);
        for (int kb = 0; kb < CH_KB0; ++kb, ++ait) {
          const uint32_t s = ait % CH_KB, ph = (ait / CH_KB) & 1;
          mbar_wait_bounded(&bars->a_empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&bars->a_full[s], CH_SLOT);
          tma_load_2d(smem_u32(slots + s * CH_SLOT), &tmX, kb * 64, m0, &bars->a_full[s]);
        }
      }
    }
  } else if (CHAIN == CHAIN_C && warp < CH_A_WARP + CH_GATHER_THREADS / 32) {
    // ===================================================================== chain C: masked row gather
    const int pt = threadIdx.x - CH_A_WARP * 32;
    const int ch = pt & 7;
    uint32_t ti = 0;
    auto src_of = [&](int64_t tile, int i) -> int64_t {
      const int64_t gr = tile * CH_M + (pt >> 3) + 8 * i;
      return (tile < n_tiles && gr < a.rows) ? a.gidx[gr] : -1;
    };
    int64_t src[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) src[i] = src_of(blockIdx.x, i);
    for (int tile = blockIdx.x; tile < n_walk; tile += gridDim.x, ++ti) {
      if (tile >= n_tiles) continue;                                 // past the end: nothing to gather
      if (ti > 0) mbar_wait_bounded(&bars->slots_free, (ti - 1) & 1);
#pragma unroll
      for (int kb = 0; kb < CH_KB; ++kb) {
        const uint32_t dst = smem_u32(slots + kb * CH_SLOT);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int row = (pt >> 3) + 8 * i;
          const bool ok = src[i] >= 0;
          cp_async16(dst + row * 128 + ((ch ^ (row & 7)) << 4), a.x16 + (ok ? src[i] : 0) * CH_DIM + kb * 64 + ch * 8, ok ? 16u : 0u);
        }
        cp_async_commit();
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) src[i] = src_of(tile + gridDim.x, i);     // next tile's indices while the rows arrive
      cp_async_wait<5>(); fence_proxy_async(); mbar_arrive(&bars->a_full[0]);
      cp_async_wait<4>(); fence_proxy_async(); mbar_arrive(&bars->a_full[1]);
      cp_async_wait<3>(); fence_proxy_async(); mbar_arrive(&bars->a_full[2]);
      cp_async_wait<2>(); fence_proxy_async(); mbar_arrive(&bars->a_full[3]);
      cp_async_wait<1>(); fence_proxy_async(); mbar_arrive(&bars->a_full[4]);
      cp_async_wait<0>(); fence_proxy_async(); mbar_arrive(&bars->a_full[5]);
    }
  }
  } else {
    // ===================================================================== consumers: MMA + epilogue
    warpgroup_reg_alloc<224>();
    // thread -> rows rl + 8 rr (rr = 0, 1) of the tile, columns colbase + 8 j + cl + {0, 1} (j = 0..23): acc[4 j + 2 rr + {0, 1}]
    const int h = warp >> 2, wq = warp & 3;
    const int rl = wq * 16 + (lane >> 2);
    const int cl = 2 * (lane & 3);
    const int colbase = h * CH_NH;
    float2* xch2 = reinterpret_cast<float2*>(xch);
    auto SP = [&](int vec) { return sparam + vec * CH_DIM; };
    float acc[96];
    uint32_t wit = h, ait = 0;                                       // weight stages alternate between the column halves
    auto cons_sync = [&]() { named_bar_sync(1, CH_CONS); };          // both warpgroups
    auto pair_sync = [&]() { named_bar_sync(2 + wq, 64); };          // the two warps that share this thread's rows
    auto warp_arrive = [&](uint64_t* bar) { __syncwarp(); if (lane == 0) mbar_arrive(bar); };
    // a weight stage is free once this warp of every CTA of the cluster is done with it: lane c arrives on CTA c's barrier
    auto release_w = [&](uint32_t ws) {
      __syncwarp();
      if (lane < CH_CL) mbar_arrive_cluster(&bars->w_empty[ws], lane);
    };
    auto next_w = [&]() {                                            // wait for this column half's next weight stage
      const uint32_t ws = wit % CH_WST;
      mbar_wait_bounded(&bars->w_full[ws], (wit / CH_WST) & 1);
      wit += 2;
      return ws;
    };
    // one k-block of this column half: 4 MMAs on the operand at a_smem, one weight stage; the previous k-block's
    // stages are handed back once its MMAs have retired
    uint32_t prev_w = 0, prev_a = 0;
    auto mma_kblock = [&](uint32_t a_smem, bool first) {
      const uint32_t ws = next_w();
      const uint64_t ad = wgmma_desc_sw128(a_smem), bd = wgmma_desc_sw128(smem_u32(wring + ws * CH_WSTAGE));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n192k16(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (!first || k) ? 1u : 0u);
      wgmma_commit();
      return ws;
    };
    auto mma_slots = [&]() {                                         // operand = the six slots
      for (int kb = 0; kb < CH_KB; ++kb) {
        const uint32_t ws = mma_kblock(smem_u32(slots + kb * CH_SLOT), kb == 0);
        if (kb > 0) { wgmma_wait<1>(); release_w(prev_w); }
        prev_w = ws;
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release_w(prev_w);
    };
    auto mma_gathered = [&](uint32_t ti) {                           // chain C: wait for each gathered k-block
      for (int kb = 0; kb < CH_KB; ++kb) {
        mbar_wait_bounded(&bars->a_full[kb], ti & 1);
        const uint32_t ws = mma_kblock(smem_u32(slots + kb * CH_SLOT), kb == 0);
        if (kb > 0) { wgmma_wait<1>(); release_w(prev_w); }
        prev_w = ws;
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release_w(prev_w);
    };
    auto mma_corr = [&]() {                                          // chain A: 14 k-blocks through the slot ring
      for (int kb = 0; kb < CH_KB0; ++kb, ++ait) {
        const uint32_t s = ait % CH_KB;
        mbar_wait_bounded(&bars->a_full[s], (ait / CH_KB) & 1);
        const uint32_t ws = mma_kblock(smem_u32(slots + s * CH_SLOT), kb == 0);
        if (kb > 0) { wgmma_wait<1>(); release_w(prev_w); warp_arrive(&bars->a_empty[prev_a]); }
        prev_w = ws; prev_a = s;
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release_w(prev_w);
      warp_arrive(&bars->a_empty[prev_a]);
    };
    // fp16 activation -> operand slots of the next layer (SWIZZLE_128B K-major).  Both warpgroups' MMAs must have
    // retired before the slots are overwritten, and the writes must be visible to the async proxy before the next MMAs.
    auto store_act = [&]() {
      cons_sync();
#pragma unroll
      for (int j = 0; j < 24; ++j) {
        const int col = colbase + 8 * j;
        unsigned char* slot = slots + (col >> 6) * CH_SLOT;
        const int chunk = (col & 63) >> 3;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int row = rl + 8 * rr;
          *reinterpret_cast<__half2*>(slot + row * 128 + ((chunk ^ (row & 7)) << 4) + cl * 2) = __floats2half2_rn(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
        }
      }
      fence_proxy_async();
      cons_sync();
    };
    auto add_bias = [&](const float* b) {
#pragma unroll
      for (int j = 0; j < 24; ++j) {
        const float2 bv = *reinterpret_cast<const float2*>(b + colbase + 8 * j + cl);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) { acc[4 * j + 2 * rr] += bv.x; acc[4 * j + 2 * rr + 1] += bv.y; }
      }
    };
    auto relu_all = [&]() {
#pragma unroll
      for (int i = 0; i < 96; ++i) acc[i] = fmaxf(acc[i], 0.f);
    };
    // LayerNorm over the 384 columns of each of this thread's two rows: 48 columns here, the rest in the 3 other lanes of
    // the quad and in the paired warp of the other column half.  One pass gives the row's sum S and sum of squares S2;
    // S2/n - mean^2 is accurate to 34 u of the variance (u = 2^-24) while 17 mean^2 <= S2/n.  Past that it cancels (by up to
    // all of its digits where |mean| >> spread), and the row takes a second pass, M2 = sum (x - mean)^2 about the mean of
    // the first, through a second exchange round; nn.LayerNorm does not cancel either.  Both halves of a row combine
    // their parts in the same order and so compute the same mean and rstd bits, and the two warps of a pair cover the
    // same rows, so both take the second round or neither (its barriers are theirs).
    auto layer_norm = [&](const float* g, const float* b) {
      float s[2] = {0.f, 0.f}, q[2] = {0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 24; ++j)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const float t0 = acc[4 * j + 2 * rr], t1 = acc[4 * j + 2 * rr + 1];
          s[rr] += t0 + t1;
          q[rr] += t0 * t0 + t1 * t1;
        }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr)
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) { s[rr] += __shfl_xor_sync(0xffffffffu, s[rr], o); q[rr] += __shfl_xor_sync(0xffffffffu, q[rr], o); }
      if ((lane & 3) == 0) { xch2[h * CH_M + rl] = make_float2(s[0], q[0]); xch2[h * CH_M + rl + 8] = make_float2(s[1], q[1]); }
      pair_sync();
      float mean[2], var[2];
      bool again = false;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const float2 o = xch2[(h ^ 1) * CH_M + rl + 8 * rr];
        const float S = h ? o.x + s[rr] : s[rr] + o.x, S2 = h ? o.y + q[rr] : q[rr] + o.y;     // same order in both halves
        mean[rr] = S * (1.0f / CH_DIM);
        const float ms = S2 * (1.0f / CH_DIM);
        var[rr] = ms - mean[rr] * mean[rr];
        again |= 17.0f * (mean[rr] * mean[rr]) > ms;
      }
      if (__any_sync(0xffffffffu, again)) {
        pair_sync();                                                 // both warps have read the first exchange
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          q[rr] = 0.f;
#pragma unroll
          for (int j = 0; j < 24; ++j) {
            const float d0 = acc[4 * j + 2 * rr] - mean[rr], d1 = acc[4 * j + 2 * rr + 1] - mean[rr];
            q[rr] += d0 * d0 + d1 * d1;
          }
#pragma unroll
          for (int o = 1; o <= 2; o <<= 1) q[rr] += __shfl_xor_sync(0xffffffffu, q[rr], o);
        }
        if ((lane & 3) == 0) { xch2[h * CH_M + rl].x = q[0]; xch2[h * CH_M + rl + 8].x = q[1]; }
        pair_sync();
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const float o = xch2[(h ^ 1) * CH_M + rl + 8 * rr].x;
          var[rr] = (h ? o + q[rr] : q[rr] + o) * (1.0f / CH_DIM);
        }
      }
      float rstd[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) rstd[rr] = rsqrtf(fmaxf(var[rr], 0.f) + CH_EPS);
      pair_sync();                                                   // exchange slots free for the next use
#pragma unroll
      for (int j = 0; j < 24; ++j) {
        const float2 gv = *reinterpret_cast<const float2*>(g + colbase + 8 * j + cl), bv = *reinterpret_cast<const float2*>(b + colbase + 8 * j + cl);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          acc[4 * j + 2 * rr] = (acc[4 * j + 2 * rr] - mean[rr]) * rstd[rr] * gv.x + bv.x;
          acc[4 * j + 2 * rr + 1] = (acc[4 * j + 2 * rr + 1] - mean[rr]) * rstd[rr] * gv.y + bv.y;
        }
      }
    };
    // acc += 384-wide fp16 table row (per row of this thread; src < 0: nothing)
    auto add_row16 = [&](const __half* tab, const int64_t (&src)[2]) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (src[rr] < 0) continue;
        const __half* p = tab + src[rr] * CH_DIM + colbase + cl;
#pragma unroll
        for (int j = 0; j < 24; ++j) {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(p + 8 * j));
          acc[4 * j + 2 * rr] += f.x; acc[4 * j + 2 * rr + 1] += f.y;
        }
      }
    };
    auto add_state = [&](const bool (&live)[2], const int64_t (&grow)[2]) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (!live[rr]) continue;
        const float* p = a.state + grow[rr] * CH_DIM + colbase + cl;
#pragma unroll
        for (int j = 0; j < 24; ++j) {
          const float2 x = *reinterpret_cast<const float2*>(p + 8 * j);
          acc[4 * j + 2 * rr] += x.x; acc[4 * j + 2 * rr + 1] += x.y;
        }
      }
    };
    auto emit_state = [&](const bool (&live)[2], const int64_t (&grow)[2], bool with16) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (!live[rr]) continue;
        float* p = a.state + grow[rr] * CH_DIM + colbase + cl;
        __half* p16 = with16 ? a.state16 + grow[rr] * CH_DIM + colbase + cl : nullptr;
#pragma unroll
        for (int j = 0; j < 24; ++j) {
          *reinterpret_cast<float2*>(p + 8 * j) = make_float2(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
          if (with16) *reinterpret_cast<__half2*>(p16 + 8 * j) = __floats2half2_rn(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
        }
      }
    };

    // chain G scratch (row-private, fragment-major): element pair (j, rr) of this thread
    float2* sc_x = a.scratch ? reinterpret_cast<float2*>(a.scratch + (int64_t)blockIdx.x * CH_SCRATCH_PER_CTA + CH_SCRATCH_GATE) : nullptr;
    __half2* sc_gate = a.scratch ? reinterpret_cast<__half2*>(a.scratch + (int64_t)blockIdx.x * CH_SCRATCH_PER_CTA) : nullptr;
    // this thread's element pair (j, rr) at a constant offset from one per-thread base: addresses formed per pair
    // would be loop-invariant across the two GRU blocks, hoisted and kept live next to the accumulator (register spills)
    if (sc_x) { sc_x += threadIdx.x; sc_gate += threadIdx.x; }
    auto sidx = [&](int j, int rr) { return (j * 2 + rr) * CH_CONS; };
    auto save_x = [&]() {
#pragma unroll
      for (int j = 0; j < 24; ++j)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) __stcg(sc_x + sidx(j, rr), make_float2(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]));
    };

    uint32_t ti = 0;
    for (int tile = blockIdx.x; tile < n_walk; tile += gridDim.x, ++ti) {
      if (tile >= n_tiles) {
        // past the end (only in the last group): every weight stage the tile would have used is filled for the peers,
        // so wait for each and hand it back, without MMAs, epilogue or global accesses
        for (int i = 0; i < Cfg::KBLOCKS; ++i) release_w(next_w());
        continue;
      }
      const int64_t m0 = (int64_t)tile * CH_M;
      int64_t grow[2]; bool live[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) { grow[rr] = m0 + rl + 8 * rr; live[rr] = grow[rr] < a.rows; }
      if constexpr (CHAIN == CHAIN_A) {
        // parameters: b0 | b2 | g3 | be3 | b5 | gN | beN
        mma_corr();                                                  // corr.0 + ReLU
        add_bias(SP(0)); relu_all(); store_act();
        mma_slots();                                                 // corr.2 -> LayerNorm -> ReLU
        add_bias(SP(1)); layer_norm(SP(2), SP(3)); relu_all(); store_act();
        mma_slots();                                                 // corr.5 ; net + inp + . ; norm
        warp_arrive(&bars->slots_free);
        int64_t irow[2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) irow[rr] = live[rr] ? (a.inp_index ? a.inp_index[grow[rr]] : grow[rr]) : -1;
        add_bias(SP(4)); add_state(live, grow); add_row16(a.inp16, irow);
        layer_norm(SP(5), SP(6));
        emit_state(live, grow, true);
      } else if constexpr (CHAIN == CHAIN_C) {
        // parameters: ba | bb
        mma_gathered(ti);
        add_bias(SP(0)); relu_all(); store_act();
        mma_slots();
        warp_arrive(&bars->slots_free);
        add_bias(SP(1)); add_state(live, grow);
        emit_state(live, grow, true);
      } else {
        // parameters: g0 | be0 | bg1 | ba1 | bb1 | g2 | be2 | bg2 | ba2 | bb2 | W4[4][384] | b4[4]
        {                                                            // prologue: x = LN(net + h_kk[patch] + h_ij[group])
          int64_t gk[2], gp[2];
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            gk[rr] = (live[rr] && a.group_kk) ? a.group_kk[grow[rr]] : -1;
            gp[rr] = (live[rr] && a.group_of) ? a.group_of[grow[rr]] : -1;
          }
#pragma unroll
          for (int i = 0; i < 96; ++i) acc[i] = 0.f;
          add_state(live, grow);
          add_row16(a.hkk16, gk);
          add_row16(a.hij16, gp);
          layer_norm(SP(0), SP(1));
          save_x();
          store_act();
        }
#pragma unroll 1
        for (int blk = 0; blk < 2; ++blk) {
          const int pv = 2 + 5 * blk;                                // bg | ba | bb | (g | be of the LayerNorm that follows block 0)
          mma_slots();                                               // gate = sigmoid(x Wg + bg) -> scratch
          add_bias(SP(pv));
#pragma unroll
          for (int j = 0; j < 24; ++j)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
              const __half2 g = sigmoid_tanh_h2(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
              __stcg(reinterpret_cast<unsigned int*>(sc_gate + sidx(j, rr)), *reinterpret_cast<const unsigned int*>(&g));
            }
          mma_slots();                                               // r1 = relu(x Wa + ba) -> operand tile (x is not needed as an operand again)
          add_bias(SP(pv + 1)); relu_all(); store_act();
          mma_slots();                                               // r2 = r1 Wb + bb;  v = x + gate * r2
          add_bias(SP(pv + 2));
#pragma unroll
          for (int j = 0; j < 24; ++j)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
              const float2 x = __ldcg(sc_x + sidx(j, rr));
              const unsigned int gu = __ldcg(reinterpret_cast<const unsigned int*>(sc_gate + sidx(j, rr)));
              const float2 g = __half22float2(*reinterpret_cast<const __half2*>(&gu));
              acc[4 * j + 2 * rr] = x.x + g.x * acc[4 * j + 2 * rr];
              acc[4 * j + 2 * rr + 1] = x.y + g.y * acc[4 * j + 2 * rr + 1];
            }
          if (blk == 0) {                                            // x' = LN(x + gate * r2): fp32 -> scratch, fp16 -> operand tile
            layer_norm(SP(pv + 3), SP(pv + 4));
            save_x();
            store_act();
          } else {                                                   // net = x + gate * r2 -> global; heads on relu(net)
            emit_state(live, grow, false);
            const float* W4 = SP(10);
            float hd[2][4];
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
              for (int o = 0; o < 4; ++o) hd[rr][o] = 0.f;
#pragma unroll
            for (int j = 0; j < 24; ++j)
#pragma unroll
              for (int o = 0; o < 4; ++o) {
                const float2 wv = *reinterpret_cast<const float2*>(W4 + o * CH_DIM + colbase + 8 * j + cl);
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) hd[rr][o] += fmaxf(acc[4 * j + 2 * rr], 0.f) * wv.x + fmaxf(acc[4 * j + 2 * rr + 1], 0.f) * wv.y;
              }
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
              for (int o = 0; o < 4; ++o) {
                hd[rr][o] += __shfl_xor_sync(0xffffffffu, hd[rr][o], 1);
                hd[rr][o] += __shfl_xor_sync(0xffffffffu, hd[rr][o], 2);
              }
            if ((lane & 3) == 0) {
#pragma unroll
              for (int rr = 0; rr < 2; ++rr) xch[h * CH_M + rl + 8 * rr] = make_float4(hd[rr][0], hd[rr][1], hd[rr][2], hd[rr][3]);
            }
            pair_sync();
            if (h == 0 && (lane & 3) == 0) {
              const float* b4 = W4 + 4 * CH_DIM;
#pragma unroll
              for (int rr = 0; rr < 2; ++rr) {
                if (!live[rr]) continue;
                const float4 o = xch[CH_M + rl + 8 * rr];
                float ctr0 = 0.f, ctr1 = 0.f;
                if (a.coords) { ctr0 = a.coords[grow[rr] * 2 * a.PP + a.centre]; ctr1 = a.coords[grow[rr] * 2 * a.PP + a.PP + a.centre]; }
                // target = centre + delta (dpvo.py:341)
                *reinterpret_cast<float2*>(a.delta + grow[rr] * 2) = make_float2(hd[rr][0] + o.x + b4[0] + ctr0, hd[rr][1] + o.y + b4[1] + ctr1);
                *reinterpret_cast<float2*>(a.weight + grow[rr] * 2) = make_float2(sigmoid_fast(hd[rr][2] + o.z + b4[2]), sigmoid_fast(hd[rr][3] + o.w + b4[3]));
              }
            }
            pair_sync();
          }
        }
      }
    }
  }
  cluster.sync();                                                    // no peer still arrives on or writes into this CTA
}

}  // namespace dpvo

using namespace dpvo;

struct ChainMaps { CUtensorMap X, W0, W; };

// how many CH_CL-CTA clusters of chain_kernel<CHAIN> the current device runs at once; queried once per device, after the
// shared-memory limit is raised
template <int CHAIN>
static int chain_max_clusters(int* n) {
  constexpr int kDevices = 64;
  static std::atomic<int> cached[kDevices];                          // 0 = not queried yet
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return check_cuda(e, "update chain: cudaGetDevice");
  if (dev < kDevices && (*n = cached[dev].load(std::memory_order_relaxed)) > 0) return DPVO_OK;
  if (int rc = allow_smem("update chain", chain_kernel<CHAIN>, ChainCfg<CHAIN>::SMEM)) return rc;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(CH_CL);
  cfg.blockDim = dim3(CH_THREADS);
  cfg.dynamicSmemBytes = ChainCfg<CHAIN>::SMEM;
  e = cudaOccupancyMaxActiveClusters(n, chain_kernel<CHAIN>, &cfg);
  if (e != cudaSuccess) return check_cuda(e, "update chain: cudaOccupancyMaxActiveClusters");
  if (*n < 1) {
    set_error("update chain: the device cannot run a cluster of %d chain CTAs (%d bytes of shared memory each)", CH_CL, ChainCfg<CHAIN>::SMEM);
    return DPVO_ERR_CUDA;
  }
  if (dev < kDevices) cached[dev].store(*n, std::memory_order_relaxed);
  return DPVO_OK;
}

template <int CHAIN>
static int chain_launch(const ChainMaps& m, const ChainArgs& a, cudaStream_t st) {
  int max_clusters = 0;
  if (int rc = chain_max_clusters<CHAIN>(&max_clusters)) return rc;
  const int64_t groups = ((a.rows + CH_M - 1) / CH_M + CH_CL - 1) / CH_CL;
  // at most one CTA per SM: chain G's scratch holds sm_count() CTA slots, indexed by blockIdx.x
  const int64_t clusters = std::min<int64_t>({groups, (int64_t)max_clusters, (int64_t)(sm_count() / CH_CL)});
  const unsigned grid = (unsigned)(clusters * CH_CL);
  return launch("chain_kernel", chain_kernel<CHAIN>, grid, CH_THREADS, ChainCfg<CHAIN>::SMEM, st, m.X, m.W0, m.W, a);
}

static bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

extern "C" int dpvo_update_corr_norm(const void* corr16, int64_t ld_corr, const void* W0, const void* W25, const float* params,
                                     float* net32, const void* inp16, const int64_t* inp_index, void* net16, int64_t E, void* stream) {
  DPVO_REQUIRE(E >= 0 && E < (1ll << 31) - CH_M, "update_corr_norm: bad edge count");
  if (E == 0) return DPVO_OK;
  DPVO_REQUIRE(corr16 && W0 && W25 && params && net32 && inp16 && net16, "update_corr_norm: null pointer");
  DPVO_REQUIRE(ld_corr >= CH_K0 && ld_corr % 8 == 0, "update_corr_norm: correlation rows must hold %d halves (zero padded) with a 16-byte aligned stride", CH_K0);
  DPVO_REQUIRE(al16(corr16) && al16(W0) && al16(W25) && al16(params) && al16(net32) && al16(inp16) && al16(net16), "update_corr_norm: pointers must be 16-byte aligned");
  ChainMaps m;
  memset(&m, 0, sizeof(m));
  int rc = encode_tmap_2d(&m.X, "update chain", corr16, E, CH_K0, ld_corr, CH_M);
  if (!rc) rc = encode_tmap_2d(&m.W0, "update chain", W0, CH_DIM, CH_K0, CH_K0, CH_WBOX);
  if (!rc) rc = encode_tmap_2d(&m.W, "update chain", W25, 2 * CH_DIM, CH_DIM, CH_DIM, CH_WBOX);
  if (rc) return rc;
  ChainArgs a;
  memset(&a, 0, sizeof(a));
  a.rows = E; a.state = net32; a.state16 = (__half*)net16; a.p = params; a.n_params = 7 * CH_DIM; a.inp16 = (const __half*)inp16; a.inp_index = inp_index;
  return chain_launch<CHAIN_A>(m, a, (cudaStream_t)stream);
}

extern "C" int dpvo_update_neighbor_mlp(const void* net16_in, const int64_t* index, const void* Wab, const float* params,
                                        float* net32, void* net16_out, int64_t E, void* stream) {
  DPVO_REQUIRE(E >= 0 && E < (1ll << 31) - CH_M, "update_neighbor_mlp: bad edge count");
  if (E == 0) return DPVO_OK;
  DPVO_REQUIRE(net16_in && index && Wab && params && net32 && net16_out, "update_neighbor_mlp: null pointer");
  DPVO_REQUIRE(net16_in != net16_out, "update_neighbor_mlp: the gathered source and the fp16 result must be different buffers");
  DPVO_REQUIRE(al16(net16_in) && al16(Wab) && al16(params) && al16(net32) && al16(net16_out), "update_neighbor_mlp: pointers must be 16-byte aligned");
  ChainMaps m;
  memset(&m, 0, sizeof(m));
  int rc = encode_tmap_2d(&m.W, "update chain", Wab, 2 * CH_DIM, CH_DIM, CH_DIM, CH_WBOX);
  if (rc) return rc;
  m.X = m.W; m.W0 = m.W;
  ChainArgs a;
  memset(&a, 0, sizeof(a));
  a.rows = E; a.state = net32; a.state16 = (__half*)net16_out; a.p = params; a.n_params = 2 * CH_DIM; a.x16 = (const __half*)net16_in; a.gidx = index;
  return chain_launch<CHAIN_C>(m, a, (cudaStream_t)stream);
}

extern "C" int64_t dpvo_update_gru_workspace_bytes(void) { return (int64_t)sm_count() * CH_SCRATCH_PER_CTA; }

extern "C" int dpvo_update_gru_heads(float* net32, const void* hij16, const int32_t* group_of, const void* hkk16, const int32_t* group_kk,
                                     const void* W6, const float* params, const float* coords, int P, float* delta, float* weight,
                                     void* workspace, int64_t E, void* stream) {
  DPVO_REQUIRE(E >= 0 && E < (1ll << 31) - CH_M, "update_gru_heads: bad edge count");
  if (E == 0) return DPVO_OK;
  DPVO_REQUIRE(net32 && W6 && params && delta && weight && workspace, "update_gru_heads: null pointer");
  DPVO_REQUIRE((hij16 == nullptr) == (group_of == nullptr) && (hkk16 == nullptr) == (group_kk == nullptr), "update_gru_heads: group rows and group ids come together");
  DPVO_REQUIRE(!hkk16 || al16(hkk16), "update_gru_heads: group rows must be 16-byte aligned");
  DPVO_REQUIRE(al16(net32) && al16(W6) && al16(params) && al16(workspace) && (!hij16 || al16(hij16)) && ((uintptr_t)delta & 7) == 0 && ((uintptr_t)weight & 7) == 0,
               "update_gru_heads: pointers must be 16-byte aligned (delta / weight: 8)");
  DPVO_REQUIRE(!coords || P >= 1, "update_gru_heads: patch size");
  ChainMaps m;
  memset(&m, 0, sizeof(m));
  int rc = encode_tmap_2d(&m.W, "update chain", W6, 6 * CH_DIM, CH_DIM, CH_DIM, CH_WBOX);
  if (rc) return rc;
  m.X = m.W; m.W0 = m.W;
  ChainArgs a;
  memset(&a, 0, sizeof(a));
  a.rows = E; a.state = net32; a.p = params; a.n_params = 14 * CH_DIM + 4; a.hij16 = (const __half*)hij16; a.group_of = group_of; a.hkk16 = (const __half*)hkk16; a.group_kk = group_kk; a.coords = coords;
  a.PP = P * P; a.centre = (P / 2) * P + P / 2; a.delta = delta; a.weight = weight; a.scratch = (unsigned char*)workspace;
  return chain_launch<CHAIN_G>(m, a, (cudaStream_t)stream);
}
