// Dense layers of the update operator on the Hopper tensor cores (wgmma, sm_90a).
//
//   Y[rows, N] = epilogue( X[rows, K] @ W[N, K]^T + bias )        fp16 operands, fp32 accumulate
//
// Persistent, warp-specialised kernel (one CTA per SM), tiles of 128 x 192:
//   warps 0-7  consumers    two warpgroups; warpgroup g issues wgmma.m64n192k16 for rows 64 g .. 64 g + 63 of the tile
//                           on shared-memory descriptors, keeps the 64 x 192 fp32 accumulator in registers and runs
//                           the epilogue (bias / activation / residual / gate, fp16 or fp32 store) straight from them
//   warps 8-11 producers    stage X and W k-blocks (64 halves = one 128-byte swizzle atom per row) into a
//                           5-deep shared-memory ring in the SWIZZLE_128B K-major layout the descriptors expect: by TMA
//                           (one elected thread), or with 16-byte cp.async when X rows are gathered through an index
//                           (net.py:84-85 `net[:, ix]` with mask) so the gather never touches HBM twice
// The weights (<= 0.7 MB per layer) stay L2 resident; X is read once per 192-column slice.
#include "common.cuh"
#include "tc.cuh"
#include <cuda.h>          // CUtensorMap types only; the encoder is fetched from the driver at run time

namespace dpvo {

constexpr int GM_M = 128;            // rows per tile (two warpgroups of 64)
constexpr int GM_N = 192;            // columns per tile (wgmma N)
constexpr int GM_K = 64;             // halves per k-block: 128 bytes, one swizzle atom
constexpr int GM_UK = 16;            // wgmma K for 16-bit operands
constexpr int GM_STAGES = 5;
// cp.async groups in flight per producer thread (gather mode).  A consumer returns the stage of k-block i - 1 only
// after it has issued the MMAs of k-block i, and a producer signals k-block i only once it has issued k-block
// i + LOOK, so LOOK must stay below ring depth - 1.
constexpr int GM_LOOK = GM_STAGES - 2;
constexpr int GM_CONS_WARPS = 8;     // two consumer warpgroups
constexpr int GM_CONS_THREADS = GM_CONS_WARPS * 32, GM_PROD_THREADS = 128;
constexpr int GM_THREADS = GM_CONS_THREADS + GM_PROD_THREADS;
constexpr int GM_A_BYTES = GM_M * 128, GM_B_BYTES = GM_N * 128;
constexpr int GM_WS_MAXKB = 6;       // weight-stationary mode: K <= 384 (6 k-blocks of the weight slice stay in smem)
constexpr int GM_WS_ASTAGES = 4;     // activation ring depth in weight-stationary mode
constexpr int GM_OUT_F16 = 0, GM_OUT_F32 = 1, GM_OUT_F32_F16 = 2;   // result: fp16 | fp32 | fp32 plus an fp16 copy

struct GemmArgs {
  const __half* X; int64_t ldx;
  const __half* W; int64_t ldw;
  const float* bias;
  const int64_t* gather;       // optional row indirection for X (-1 -> zero row)
  const void* res; int res_dtype; int64_t ldres;
  const __half* gate; int64_t ldgate;
  void* Y; int y_dtype; int64_t ldy;
  __half* Y16;                 // optional fp16 copy of the result (row stride ldy16)
  int64_t ldy16;
  int64_t rows; int N; int K; int epilogue;
};

struct GemmBars {
  uint64_t full[GM_STAGES], empty[GM_STAGES], wfull;
};

// GATHER = false: X and W tiles arrive by TMA (one elected thread, hardware swizzle, OOB rows zero).
// GATHER = true : X rows are fetched through an index with cp.async by 128 producer threads (W too).
// WS = true (weight stationary, K <= 384): a CTA works on ONE 192-column slice of the layer for its whole
// life, loads that slice of W once (<= 144 KB, resident) and streams only activation tiles.
template <bool GATHER, bool WS, int EPI, int OUT>
__global__ void __launch_bounds__(GM_THREADS, 1)
linear_f16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmArgs a) {
  extern __shared__ unsigned char gm_smem_raw[];
  constexpr int NST = WS ? GM_WS_ASTAGES : GM_STAGES;
  // 1024-byte alignment by pointer arithmetic on the shared array (an integer round trip would demote every
  // access through these pointers to generic LD/ST)
  unsigned char* base = gm_smem_raw + ((1024u - (smem_u32(gm_smem_raw) & 1023u)) & 1023u);
  unsigned char* sA = base;
  unsigned char* sB = base + NST * GM_A_BYTES;
  GemmBars* bars = reinterpret_cast<GemmBars*>(sB + (WS ? GM_WS_MAXKB : GM_STAGES) * GM_B_BYTES);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles_n = (a.N + GM_N - 1) / GM_N;
  const int64_t n_tiles_m = (a.rows + GM_M - 1) / GM_M;
  const int64_t n_tiles = n_tiles_m * n_tiles_n;
  const int KB = a.K / GM_K;

  if (threadIdx.x == 0) {
    for (int s = 0; s < GM_STAGES; ++s) { mbar_init(&bars->full[s], GATHER ? GM_PROD_THREADS : 1); mbar_init(&bars->empty[s], GM_CONS_WARPS); }
    mbar_init(&bars->wfull, 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (warp >= GM_CONS_WARPS) {
    // =========================================================================== producers
    if constexpr (!GATHER) {
      if (warp == GM_CONS_WARPS && lane == 0) {
        uint32_t it = 0;
        if constexpr (WS) {                  // the CTA's weight slice, once
          const int n0 = (int)(blockIdx.x % n_tiles_n) * GM_N;
          mbar_arrive_expect_tx(&bars->wfull, KB * GM_B_BYTES);
          for (int kb = 0; kb < KB; ++kb) tma_load_2d(smem_u32(sB + kb * GM_B_BYTES), &tmB, kb * GM_K, n0, &bars->wfull);
        }
        for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
          const int m0 = (int)((tile / n_tiles_n) * GM_M);
          const int n0 = (int)(tile % n_tiles_n) * GM_N;
          for (int kb = 0; kb < KB; ++kb, ++it) {
            const uint32_t s = it % NST, ph = (it / NST) & 1;
            mbar_wait(&bars->empty[s], ph ^ 1);
            mbar_arrive_expect_tx(&bars->full[s], WS ? GM_A_BYTES : GM_A_BYTES + GM_B_BYTES);
            tma_load_2d(smem_u32(sA + s * GM_A_BYTES), &tmA, kb * GM_K, m0, &bars->full[s]);
            if constexpr (!WS) tma_load_2d(smem_u32(sB + s * GM_B_BYTES), &tmB, kb * GM_K, n0, &bars->full[s]);
          }
        }
      }
    } else {
      const int pt = threadIdx.x - GM_CONS_THREADS;
      uint32_t it = 0;                       // k-block counter over all tiles of this CTA
      constexpr int LOOK = WS ? GM_WS_ASTAGES - 2 : GM_LOOK;
      if constexpr (WS) {
        if (pt == 0) {
          const int n0 = (int)(blockIdx.x % n_tiles_n) * GM_N;
          mbar_arrive_expect_tx(&bars->wfull, KB * GM_B_BYTES);
          for (int kb = 0; kb < KB; ++kb) tma_load_2d(smem_u32(sB + kb * GM_B_BYTES), &tmB, kb * GM_K, n0, &bars->wfull);
        }
      }
      // source rows of this thread's eight 16-byte chunks, fetched one tile ahead: the dependent index load would
      // otherwise open every tile with a global-memory latency during which nothing is in flight
      int64_t nsrc[8];
      auto fetch_rows = [&](int64_t tile) {
        const int64_t m0 = (tile / n_tiles_n) * GM_M;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int row = (pt + GM_PROD_THREADS * i) >> 3;
          int64_t src = m0 + row;
          if (tile >= n_tiles || src >= a.rows) src = -1;
          else if (a.gather) src = a.gather[src];
          nsrc[i] = src;
        }
      };
      fetch_rows(blockIdx.x);
      for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int n0 = (int)(tile % n_tiles_n) * GM_N;
        const __half* arow[8]; uint32_t aoff[8], abytes[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = pt + GM_PROD_THREADS * i, row = c >> 3, ch = c & 7;
          const int64_t src = nsrc[i];
          const bool ok = src >= 0;
          arow[i] = a.X + (ok ? src : 0) * a.ldx + ch * 8;
          abytes[i] = ok ? 16u : 0u;
          aoff[i] = row * 128 + ((ch ^ (row & 7)) << 4);
        }
        fetch_rows(tile + gridDim.x);
        const __half* brow[12]; uint32_t boff[12], bbytes[12];
#pragma unroll
        for (int i = 0; i < 12; ++i) {
          const int c = pt + GM_PROD_THREADS * i, row = c >> 3, ch = c & 7;
          const bool ok = n0 + row < a.N;
          brow[i] = a.W + (int64_t)(ok ? n0 + row : 0) * a.ldw + ch * 8;
          bbytes[i] = ok ? 16u : 0u;
          boff[i] = row * 128 + ((ch ^ (row & 7)) << 4);
        }
        for (int kb = 0; kb < KB; ++kb, ++it) {
          const uint32_t s = it % NST, ph = (it / NST) & 1;
          mbar_wait(&bars->empty[s], ph ^ 1);
          const uint32_t da = smem_u32(sA + s * GM_A_BYTES);
#pragma unroll
          for (int i = 0; i < 8; ++i) cp_async16(da + aoff[i], arow[i] + kb * GM_K, abytes[i]);
          if constexpr (!WS) {
            const uint32_t db = smem_u32(sB + s * GM_B_BYTES);
#pragma unroll
            for (int i = 0; i < 12; ++i) cp_async16(db + boff[i], brow[i] + kb * GM_K, bbytes[i]);
          }
          cp_async_commit();
          if (it >= LOOK) {                  // the group issued LOOK k-blocks ago has landed
            cp_async_wait<LOOK>();
            fence_proxy_async();
            mbar_arrive(&bars->full[(it - LOOK) % NST]);
          }
        }
      }
      cp_async_wait<0>();
      fence_proxy_async();
      for (uint32_t j = (it >= LOOK ? it - LOOK : 0); j < it; ++j) mbar_arrive(&bars->full[j % NST]);
    }
  } else {
    // =========================================================================== consumers: MMA + epilogue
    const int wg = warp >> 2, wq = warp & 3;
    uint32_t it = 0;
    float acc[96];
    if constexpr (WS) mbar_wait(&bars->wfull, 0);
    auto release = [&](uint32_t s) { __syncwarp(); if (lane == 0) mbar_arrive(&bars->empty[s]); };
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int64_t m0 = (tile / n_tiles_n) * GM_M;
      const int n0 = (int)(tile % n_tiles_n) * GM_N;
      uint32_t prev = 0;
      for (int kb = 0; kb < KB; ++kb, ++it) {
        const uint32_t s = it % NST, ph = (it / NST) & 1;
        mbar_wait(&bars->full[s], ph);
        const uint64_t ad = wgmma_desc_sw128(smem_u32(sA + s * GM_A_BYTES + wg * 64 * 128));
        const uint64_t bd = wgmma_desc_sw128(smem_u32(sB + (WS ? kb : (int)s) * GM_B_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GM_K / GM_UK; ++k) wgmma_m64n192k16(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (kb | k) != 0);
        wgmma_commit();
        if (kb > 0) { wgmma_wait<1>(); release(prev); }     // the previous k-block's MMAs have read their stage
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release(prev);

      // ---- epilogue from the accumulator registers: rows r0, r0 + 8; columns 8 j + 2 (lane % 4) + {0, 1}
      const int64_t r0 = m0 + wg * 64 + wq * 16 + (lane >> 2);
      const int cl = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < GM_N / 8; ++j) {
        const int col = n0 + 8 * j + cl;
        if (col >= a.N) continue;                              // N is a multiple of 32: uniform per 8-column block
        const float2 bv = a.bias ? *reinterpret_cast<const float2*>(a.bias + col) : make_float2(0.f, 0.f);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int64_t row = r0 + 8 * rr;
          if (row >= a.rows) continue;
          float v0 = acc[4 * j + 2 * rr] + bv.x, v1 = acc[4 * j + 2 * rr + 1] + bv.y;
          if constexpr (EPI == DPVO_EPI_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          else if constexpr (EPI == DPVO_EPI_SIGMOID) { v0 = __fdividef(1.0f, 1.0f + __expf(-v0)); v1 = __fdividef(1.0f, 1.0f + __expf(-v1)); }
          else if constexpr (EPI == DPVO_EPI_SIGMOID_RELU) {
            if (col < (a.N >> 1)) { v0 = __fdividef(1.0f, 1.0f + __expf(-v0)); v1 = __fdividef(1.0f, 1.0f + __expf(-v1)); }
            else { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          } else if constexpr (EPI == DPVO_EPI_RESADD || EPI == DPVO_EPI_GATEDRES) {
            // the residual may alias the output element for element (in-place `net += f(net)`): read before the write
            float2 rv;
            if (a.res_dtype == DPVO_F32) rv = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(a.res) + row * a.ldres + col);
            else rv = __half22float2(*reinterpret_cast<const __half2*>(reinterpret_cast<const __half*>(a.res) + row * a.ldres + col));
            if constexpr (EPI == DPVO_EPI_GATEDRES) {
              const float2 g = __half22float2(*reinterpret_cast<const __half2*>(a.gate + row * a.ldgate + col));
              v0 = rv.x + g.x * v0; v1 = rv.y + g.y * v1;
            } else {
              v0 += rv.x; v1 += rv.y;
            }
          }
          if constexpr (OUT == GM_OUT_F16) {
            *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(a.Y) + row * a.ldy + col) = __floats2half2_rn(v0, v1);
          } else {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(a.Y) + row * a.ldy + col) = make_float2(v0, v1);
            if constexpr (OUT == GM_OUT_F32_F16) *reinterpret_cast<__half2*>(a.Y16 + row * a.ldy16 + col) = __floats2half2_rn(v0, v1);
          }
        }
      }
    }
  }
}

}  // namespace dpvo

using namespace dpvo;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// row-major fp16 [rows, cols] with row stride ld (elements) -> tiles of box_rows x 64 columns, 128-byte swizzle
static int make_tmap(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  EncodeTiledFn fn = encode_tiled();
  if (!fn) { set_error("linear_f16: cuTensorMapEncodeTiled is not available from the driver"); return DPVO_ERR_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)GM_K, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("linear_f16: cuTensorMapEncodeTiled failed (%d)", (int)r); return DPVO_ERR_CUDA; }
  return DPVO_OK;
}

struct GemmMaps { CUtensorMap A, B; };

template <bool GATHER, bool WS, int EPI, int OUT>
static int launch_out(const GemmMaps& m, const GemmArgs& a, unsigned grid, cudaStream_t st) {
  const size_t smem = (WS ? (size_t)GM_WS_ASTAGES * GM_A_BYTES + (size_t)GM_WS_MAXKB * GM_B_BYTES
                          : (size_t)GM_STAGES * (GM_A_BYTES + GM_B_BYTES)) + sizeof(GemmBars) + 1024;
  // the opt-in is a per-device function attribute: set it on every launch (a cached flag would be wrong on the
  // second GPU of a process and is not worth a lock)
  cudaError_t e = cudaFuncSetAttribute(linear_f16_kernel<GATHER, WS, EPI, OUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return check_cuda(e, "linear_f16: cudaFuncSetAttribute");
  linear_f16_kernel<GATHER, WS, EPI, OUT><<<grid, GM_THREADS, smem, st>>>(m.A, m.B, a);
  DPVO_LAUNCH_CHECK("linear_f16_kernel");
  return DPVO_OK;
}

template <bool GATHER, bool WS, int EPI>
static int launch_epi(const GemmMaps& m, const GemmArgs& a, unsigned grid, cudaStream_t st) {
  if (a.y_dtype == DPVO_F16) return launch_out<GATHER, WS, EPI, GM_OUT_F16>(m, a, grid, st);
  if (a.Y16) return launch_out<GATHER, WS, EPI, GM_OUT_F32_F16>(m, a, grid, st);
  return launch_out<GATHER, WS, EPI, GM_OUT_F32>(m, a, grid, st);
}

template <bool GATHER, bool WS>
static int launch_variant(const GemmMaps& m, const GemmArgs& a, unsigned grid, cudaStream_t st) {
  switch (a.epilogue) {
    case DPVO_EPI_NONE: return launch_epi<GATHER, WS, DPVO_EPI_NONE>(m, a, grid, st);
    case DPVO_EPI_RELU: return launch_epi<GATHER, WS, DPVO_EPI_RELU>(m, a, grid, st);
    case DPVO_EPI_SIGMOID: return launch_epi<GATHER, WS, DPVO_EPI_SIGMOID>(m, a, grid, st);
    case DPVO_EPI_RESADD: return launch_epi<GATHER, WS, DPVO_EPI_RESADD>(m, a, grid, st);
    case DPVO_EPI_SIGMOID_RELU: return launch_epi<GATHER, WS, DPVO_EPI_SIGMOID_RELU>(m, a, grid, st);
    default: return launch_epi<GATHER, WS, DPVO_EPI_GATEDRES>(m, a, grid, st);
  }
}

static int linear_launch(GemmArgs& a, cudaStream_t st) {
  const int n_tiles_n = (a.N + GM_N - 1) / GM_N;
  const int64_t tiles = ((a.rows + GM_M - 1) / GM_M) * n_tiles_n;
  const bool ws = (a.K / GM_K) <= GM_WS_MAXKB;
  // weight-stationary CTAs keep their column slice: the grid must be a multiple of the slice count
  int64_t grid = std::min<int64_t>(tiles, sm_count());
  if (ws) grid = std::max<int64_t>(n_tiles_n, grid / n_tiles_n * n_tiles_n);
  GemmMaps m;
  memset(&m, 0, sizeof(m));
  int rc = make_tmap(&m.B, a.W, a.N, a.K, a.ldw, GM_N);
  if (rc) return rc;
  if (a.gather) return ws ? launch_variant<true, true>(m, a, (unsigned)grid, st) : launch_variant<true, false>(m, a, (unsigned)grid, st);
  rc = make_tmap(&m.A, a.X, a.rows, a.K, a.ldx, GM_M);
  if (rc) return rc;
  return ws ? launch_variant<false, true>(m, a, (unsigned)grid, st) : launch_variant<false, false>(m, a, (unsigned)grid, st);
}

extern "C" int dpvo_linear_f16(const void* X, int64_t ldx, const int64_t* gather, const void* W, int64_t ldw,
                               const float* bias, const void* res, int res_dtype, int64_t ldres,
                               const void* gate, int64_t ldgate, void* Y, int y_dtype, int64_t ldy,
                               void* Y16, int64_t ldy16,
                               int64_t rows, int N, int K, int epilogue, void* stream) {
  DPVO_REQUIRE(rows >= 0 && N > 0 && K > 0, "linear_f16: bad sizes");
  if (rows == 0) return DPVO_OK;
  DPVO_REQUIRE(X && W && Y, "linear_f16: null pointer");
  DPVO_REQUIRE(K % GM_K == 0, "linear_f16: K=%d must be a multiple of %d (pad the operands)", K, GM_K);
  DPVO_REQUIRE(N % 32 == 0, "linear_f16: N=%d must be a multiple of 32", N);
  DPVO_REQUIRE(rows < (1ll << 31), "linear_f16: too many rows");
  DPVO_REQUIRE(ldx % 8 == 0 && ldw % 8 == 0 && ((uintptr_t)X & 15) == 0 && ((uintptr_t)W & 15) == 0,
               "linear_f16: X / W rows must be 16-byte aligned");
  DPVO_REQUIRE(y_dtype == DPVO_F16 || y_dtype == DPVO_F32, "linear_f16: y dtype");
  DPVO_REQUIRE((y_dtype == DPVO_F16 ? ldy % 8 == 0 : ldy % 4 == 0) && ((uintptr_t)Y & 15) == 0, "linear_f16: Y rows must be 16-byte aligned");
  DPVO_REQUIRE(epilogue >= DPVO_EPI_NONE && epilogue <= DPVO_EPI_SIGMOID_RELU, "linear_f16: unknown epilogue %d", epilogue);
  DPVO_REQUIRE(epilogue != DPVO_EPI_SIGMOID_RELU || N % 32 == 0, "linear_f16: the split epilogue needs N/2 to be a multiple of 16");
  if (epilogue == DPVO_EPI_RESADD || epilogue == DPVO_EPI_GATEDRES)
    DPVO_REQUIRE(res && (res_dtype == DPVO_F16 || res_dtype == DPVO_F32), "linear_f16: residual operand missing");
  if (epilogue == DPVO_EPI_GATEDRES)
    DPVO_REQUIRE(gate && ldgate % 4 == 0 && ((uintptr_t)gate & 7) == 0, "linear_f16: gate operand missing, or rows not 8-byte aligned");
  DPVO_REQUIRE(!res || (ldres % 4 == 0 && ((uintptr_t)res & (res_dtype == DPVO_F32 ? 15 : 7)) == 0),
               "linear_f16: residual rows must be aligned to 4 elements");
  DPVO_REQUIRE(!bias || ((uintptr_t)bias & 15) == 0, "linear_f16: bias must be 16-byte aligned");
  GemmArgs a;
  a.X = (const __half*)X; a.ldx = ldx; a.W = (const __half*)W; a.ldw = ldw; a.bias = bias; a.gather = gather;
  a.res = res; a.res_dtype = res_dtype; a.ldres = ldres; a.gate = (const __half*)gate; a.ldgate = ldgate;
  DPVO_REQUIRE(!Y16 || (ldy16 % 8 == 0 && ((uintptr_t)Y16 & 15) == 0), "linear_f16: Y16 rows must be 16-byte aligned");
  DPVO_REQUIRE(!Y16 || y_dtype == DPVO_F32, "linear_f16: the fp16 copy accompanies an fp32 result (an fp16 result needs none)");
  a.Y16 = (__half*)Y16; a.ldy16 = ldy16;
  a.Y = Y; a.y_dtype = y_dtype; a.ldy = ldy; a.rows = rows; a.N = N; a.K = K; a.epilogue = epilogue;

  return linear_launch(a, (cudaStream_t)stream);
}
