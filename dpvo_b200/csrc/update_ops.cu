// Row-wise building blocks of the update operator (dpvo/net.py:74-92, dpvo/blocks.py:15-48).
//
// Everything that is not a dense layer is HBM-bound row streaming over [E, 384] activations, so
// each kernel here fuses a whole elementwise/normalisation group into ONE pass: one warp per row,
// 16-byte accesses, fp32 statistics, and -- where the next consumer is a tensor-core GEMM -- an fp16
// copy written in the same pass so the GEMM never re-reads fp32.
//
//   add_layernorm        y = LN(a + b + c) * gamma + beta (+ReLU)       net.py:77-78, 46-51, 53-60
//   gather_rows_masked   y[e] = idx[e] >= 0 ? x[idx[e]] : 0             net.py:81-85
//   residual_add         net += u                                        net.py:84-85
//   softagg_reduce       segment softmax-weighted sum                    blocks.py:40-43 (torch_scatter)
//   scatter_add_rows     net += h[group_of[e]]                           blocks.py:45-46 + net.py:87-88
//   gated_residual       x + sigmoid(g) * r                              blocks.py:28-29
//   heads                delta = Wd relu(net), weight = sigmoid(Ww relu(net))   net.py:62-71, 92
#include "common.cuh"
#include "tc.cuh"
#include <cstdlib>
#include <algorithm>

namespace dpvo {

// ---- 4-wide typed row access ---------------------------------------------------------------
__device__ __forceinline__ float4 load4(const void* base, int dtype, int64_t elem) {
  if (dtype == DPVO_F32) return *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem);
  const uint2 q = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(base) + elem);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&q.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&q.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void store4(void* base, int dtype, int64_t elem, float4 v) {
  if (dtype == DPVO_F32) { *reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + elem) = v; return; }
  __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  uint2 q; q.x = *reinterpret_cast<uint32_t*>(&a); q.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(base) + elem) = q;
}
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

template <int DT> __device__ __forceinline__ float4 load4t(const void* base, int64_t elem) {
  if constexpr (DT == DPVO_F32) return *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem);
  else {
    const uint2 q = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(base) + elem);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&q.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&q.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
}

constexpr int ROW_WARPS = 8;
constexpr int MAX_V4 = 8;     // up to 8 float4 per lane -> dim <= 1024

// ---- add + LayerNorm ------------------------------------------------------------------------
// NV = float4 per lane (dim = 128 NV, 3 for the update operator); a warp normalises RPW rows at a time so that
// the loads of all of them are in flight before the first reduction (one row per warp and 70 registers left
// the kernel at a third of the HBM rate: too few bytes in flight per SM).
// DA / DBC: element types of operand a and of operands b, c fixed at compile time (the three shapes the update
// operator uses), or -1 = decided at run time from da / db / dc.
template <int NV, int RPW, int DA, int DBC>
__global__ void __launch_bounds__(ROW_WARPS * 32, (NV * RPW <= 6) ? 3 : 2)
add_layernorm_kernel(const void* a, const void* b, const void* c, int da, int db, int dc,
                     const int64_t* __restrict__ b_index, const __half* __restrict__ cs, int64_t ld_cs,
                     const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                     float* y32, __half* y16, int relu, int64_t rows, int dim) {
  const int lane = threadIdx.x & 31;
  const int64_t wstride = (int64_t)gridDim.x * ROW_WARPS * RPW;
  for (int64_t r0 = ((int64_t)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5)) * RPW; r0 < rows; r0 += wstride) {
    float4 v[RPW][NV];
#pragma unroll
    for (int k = 0; k < RPW; ++k) {
      const int64_t r = r0 + k;
      const bool on = r < rows;
      const int64_t rb = (on && b_index) ? b_index[r] : r;      // operand b may be gathered (ctx = imap[kk], dpvo.py:334)
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (on) {
          const int64_t e = r * dim + (i * 32 + lane) * 4;
          if constexpr (DA >= 0) t = load4t<DA>(a, e); else t = load4(a, da, e);
          float4 cv = make_float4(0.f, 0.f, 0.f, 0.f);
          if constexpr (DBC >= 0) {
            if (b) t = add4(t, load4t<DBC>(b, rb * dim + (i * 32 + lane) * 4));
            if (c) cv = load4t<DBC>(c, e);
          } else {
            if (b) t = add4(t, load4(b, db, rb * dim + (i * 32 + lane) * 4));
            if (c) cv = load4(c, dc, e);
          }
          if (cs) {                                            // operand c enters scaled element-wise: a + cs * c
            const float4 g = load4t<DPVO_F16>(cs, r * ld_cs + (i * 32 + lane) * 4);
            cv = make_float4(cv.x * g.x, cv.y * g.y, cv.z * g.z, cv.w * g.w);
          }
          t = add4(t, cv);
        }
        v[k][i] = t;
      }
    }
    float mean[RPW], rstd[RPW];
#pragma unroll
    for (int k = 0; k < RPW; ++k) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) s += (v[k][i].x + v[k][i].y) + (v[k][i].z + v[k][i].w);
      mean[k] = s;
    }
#pragma unroll
    for (int k = 0; k < RPW; ++k) mean[k] = warp_sum(mean[k]) / (float)dim;
#pragma unroll
    for (int k = 0; k < RPW; ++k) {
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const float dx = v[k][i].x - mean[k], dy = v[k][i].y - mean[k], dz = v[k][i].z - mean[k], dw = v[k][i].w - mean[k];
        q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
      rstd[k] = q;
    }
#pragma unroll
    for (int k = 0; k < RPW; ++k) rstd[k] = rsqrtf(warp_sum(rstd[k]) / (float)dim + eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int col = (i * 32 + lane) * 4;
      const float4 g = *reinterpret_cast<const float4*>(gamma + col);
      const float4 bt = *reinterpret_cast<const float4*>(beta + col);
#pragma unroll
      for (int k = 0; k < RPW; ++k) {
        const int64_t r = r0 + k;
        if (r < rows) {
          float4 o;
          o.x = (v[k][i].x - mean[k]) * rstd[k] * g.x + bt.x;
          o.y = (v[k][i].y - mean[k]) * rstd[k] * g.y + bt.y;
          o.z = (v[k][i].z - mean[k]) * rstd[k] * g.z + bt.z;
          o.w = (v[k][i].w - mean[k]) * rstd[k] * g.w + bt.w;
          if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
          if (y32) store4(y32, DPVO_F32, r * dim + col, o);
          if (y16) store4(y16, DPVO_F16, r * dim + col, o);
        }
      }
    }
  }
}

// ---- add + LayerNorm, operands staged through shared memory by bulk copies ----------------------------------
// The register kernel above keeps one or two rows per warp in flight -- at 80 registers and three CTAs per SM that
// is ~36 KB per SM, a third of what the HBM latency-bandwidth product asks for -- so the dim = 384 shapes of the
// update operator take this path: rows are dense, a tile of LNB_ROWS rows of operand a (and c) is ONE contiguous
// range, fetched by a single cp.async.bulk per operand into a 4-deep ring by one thread; bytes in flight no longer
// cost registers.  Gathered operand b and the strided scale of c are read directly (L2-resident, small).
constexpr int LNB_ROWS = 16;          // rows per tile (two per warp)
constexpr int LNB_STAGES = 4;
constexpr int LNB_DIM = 384;
constexpr size_t LNB_SMEM_CAP = 200 * 1024;

// Block = ROW_WARPS consumer warps + one producer warp (its lane 0 issues the copies of the tile three iterations
// ahead while the consumers normalise the current one).
template <int DA, bool HAS_C>
__global__ void __launch_bounds__(ROW_WARPS * 32 + 32)
add_layernorm_bulk_kernel(const void* a, const void* b, const __half* c, int db, const int64_t* __restrict__ b_index,
                          const __half* __restrict__ cs, int64_t ld_cs,
                          const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                          float* y32, __half* y16, int relu, int64_t rows) {
  constexpr int ES = (DA == DPVO_F32) ? 4 : 2;
  constexpr int A_BYTES = LNB_ROWS * LNB_DIM * ES, C_BYTES = HAS_C ? LNB_ROWS * LNB_DIM * 2 : 0;
  extern __shared__ __align__(128) unsigned char lnb_smem[];
  constexpr int R_BYTES = LNB_ROWS * LNB_DIM * 2;                 // one fp16 tile (gathered b, scale of c)
  unsigned char* sA = lnb_smem;                                   // [LNB_STAGES][A_BYTES]
  unsigned char* sC = sA + LNB_STAGES * A_BYTES;                  // [LNB_STAGES][C_BYTES]
  unsigned char* sB = sC + LNB_STAGES * C_BYTES;                  // [LNB_STAGES][R_BYTES] when b is given (fp16)
  unsigned char* sS = sB + (b ? LNB_STAGES * R_BYTES : 0);        // [LNB_STAGES][R_BYTES] when cs is given
  uint64_t* full = reinterpret_cast<uint64_t*>(sS + (cs ? LNB_STAGES * R_BYTES : 0));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t n_tiles = (rows + LNB_ROWS - 1) / LNB_ROWS;
  if (threadIdx.x == 0) {
    for (int i = 0; i < LNB_STAGES; ++i) mbar_init(&full[i], 1);
    mbar_init_fence();
  }
  __syncthreads();
  // producer warp: lane 0 arms the barrier and copies the dense tiles of a and c with one bulk copy each; the rows
  // of the gathered operand b and of the strided scale of c are 768-byte copies, one per lane
  auto issue = [&](int64_t tile, int stage) {
    const int64_t r0 = tile * LNB_ROWS;
    const uint32_t nrow = (uint32_t)min((int64_t)LNB_ROWS, rows - r0);
    const uint32_t bar = smem_u32(&full[stage]);
    const uint32_t ba = nrow * LNB_DIM * ES, bc = HAS_C ? nrow * LNB_DIM * 2 : 0;
    const uint32_t brow = LNB_DIM * 2, bb = b ? nrow * brow : 0, bs = cs ? nrow * brow : 0;
    if (lane == 0) {
      mbar_arrive_expect_tx(&full[stage], ba + bc + bb + bs);
      bulk_load(smem_u32(sA + stage * A_BYTES), reinterpret_cast<const unsigned char*>(a) + r0 * LNB_DIM * ES, ba, bar);
      if constexpr (HAS_C) bulk_load(smem_u32(sC + stage * C_BYTES), reinterpret_cast<const unsigned char*>(c) + r0 * LNB_DIM * 2, bc, bar);
    }
    if ((uint32_t)lane < nrow) {
      const uint32_t q = (uint32_t)lane;
      if (b) {
        const int64_t src = b_index ? b_index[r0 + q] : r0 + q;
        bulk_load(smem_u32(sB + stage * R_BYTES + q * brow), reinterpret_cast<const unsigned char*>(b) + src * brow, brow, bar);
      }
      if (cs) bulk_load(smem_u32(sS + stage * R_BYTES + q * brow), reinterpret_cast<const unsigned char*>(cs) + (r0 + q) * ld_cs * 2, brow, bar);
    }
  };
  // gamma / beta of this lane's columns stay in registers
  float4 gm[3], bt[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    gm[i] = *reinterpret_cast<const float4*>(gamma + (i * 32 + lane) * 4);
    bt[i] = *reinterpret_cast<const float4*>(beta + (i * 32 + lane) * 4);
  }
  const bool producer = warp == ROW_WARPS;
  if (producer)
    for (int k = 0; k < LNB_STAGES - 1; ++k) {
      const int64_t t = (int64_t)blockIdx.x + (int64_t)k * gridDim.x;
      if (t < n_tiles) issue(t, k);
    }
  int64_t it = 0;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    const int stage = (int)(it % LNB_STAGES);
    if (producer) {                                               // into the stage freed by the previous iteration
      const int64_t t = tile + (int64_t)(LNB_STAGES - 1) * gridDim.x;
      if (t < n_tiles) issue(t, (int)((it + LNB_STAGES - 1) % LNB_STAGES));
      __syncthreads();
      continue;
    }
    mbar_wait(smem_u32(&full[stage]), (uint32_t)((it / LNB_STAGES) & 1));
    const unsigned char* ta = sA + stage * A_BYTES;
    const unsigned char* tc = sC + stage * C_BYTES;
    const unsigned char* tb = sB + stage * R_BYTES;
    const unsigned char* ts = sS + stage * R_BYTES;
    float4 v[2][3];
    int64_t rr[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int lr = warp * 2 + k;
      const int64_t r = tile * LNB_ROWS + lr;
      rr[k] = r;
      const bool on = r < rows;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const int col = (i * 32 + lane) * 4;
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (on) {
          if constexpr (DA == DPVO_F32) t = *reinterpret_cast<const float4*>(ta + ((size_t)lr * LNB_DIM + col) * 4);
          else t = load4t<DPVO_F16>(ta, (int64_t)lr * LNB_DIM + col);
          if (b) t = add4(t, load4t<DPVO_F16>(tb, (int64_t)lr * LNB_DIM + col));
          if constexpr (HAS_C) {
            float4 cv = load4t<DPVO_F16>(tc, (int64_t)lr * LNB_DIM + col);
            if (cs) {
              const float4 g = load4t<DPVO_F16>(ts, (int64_t)lr * LNB_DIM + col);
              cv = make_float4(cv.x * g.x, cv.y * g.y, cv.z * g.z, cv.w * g.w);
            }
            t = add4(t, cv);
          }
        }
        v[k][i] = t;
      }
    }
    float mean[2], rstd[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < 3; ++i) sum += (v[k][i].x + v[k][i].y) + (v[k][i].z + v[k][i].w);
      mean[k] = sum;
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) mean[k] = warp_sum(mean[k]) / (float)LNB_DIM;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const float dx = v[k][i].x - mean[k], dy = v[k][i].y - mean[k], dz = v[k][i].z - mean[k], dw = v[k][i].w - mean[k];
        q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
      rstd[k] = q;
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) rstd[k] = rsqrtf(warp_sum(rstd[k]) / (float)LNB_DIM + eps);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (rr[k] < rows) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const int col = (i * 32 + lane) * 4;
          float4 o;
          o.x = (v[k][i].x - mean[k]) * rstd[k] * gm[i].x + bt[i].x;
          o.y = (v[k][i].y - mean[k]) * rstd[k] * gm[i].y + bt[i].y;
          o.z = (v[k][i].z - mean[k]) * rstd[k] * gm[i].z + bt[i].z;
          o.w = (v[k][i].w - mean[k]) * rstd[k] * gm[i].w + bt[i].w;
          if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
          if (y32) store4(y32, DPVO_F32, rr[k] * LNB_DIM + col, o);
          if (y16) store4(y16, DPVO_F16, rr[k] * LNB_DIM + col, o);
        }
      }
    }
    __syncthreads();                                              // every warp is done with this stage
  }
}

template <int DA, bool HAS_C>
static int launch_ln_bulk(const void* a, const void* b, const void* c, int db, const int64_t* bi, const void* cs, int64_t ld_cs,
                          const float* gamma, const float* beta, float eps, void* y32, void* y16, int relu, int64_t rows, cudaStream_t st) {
  constexpr int ES = (DA == DPVO_F32) ? 4 : 2;
  const size_t smem = (size_t)LNB_STAGES * LNB_ROWS * LNB_DIM * (ES + (HAS_C ? 2 : 0) + (b ? 2 : 0) + (cs ? 2 : 0)) + LNB_STAGES * sizeof(uint64_t) + 128;
  if (smem > LNB_SMEM_CAP) return DPVO_ERR_UNSUPPORTED;          // all four operands at once: the register kernel takes it
  const int64_t n_tiles = (rows + LNB_ROWS - 1) / LNB_ROWS;
  const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (size_t)(200 * 1024) / smem));
  const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(n_tiles, (int64_t)sm_count() * per_sm));
  return launch("add_layernorm_bulk_kernel", add_layernorm_bulk_kernel<DA, HAS_C>, grid, ROW_WARPS * 32 + 32, smem, st, a, b, (const __half*)c, db,
                bi, (const __half*)cs, ld_cs, gamma, beta, eps, (float*)y32, (__half*)y16, relu, rows);
}

// ---- gather / residual / scatter / gate -------------------------------------------------------
__global__ void __launch_bounds__(ROW_WARPS * 32)
gather_rows_masked_kernel(const void* x, int dx, const int64_t* __restrict__ idx, void* y, int dy, int64_t rows, int dim) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (int64_t)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.x * ROW_WARPS) {
    const int64_t src = idx[r];
    for (int col = lane * 4; col < dim; col += 128) {
      const float4 v = (src >= 0) ? load4(x, dx, src * dim + col) : make_float4(0.f, 0.f, 0.f, 0.f);
      store4(y, dy, r * dim + col, v);
    }
  }
}

// net32[r] += u[src(r)]   (src = r, or group_of[r]);  optional fp16 copy of the result.  write_state = false: the sum is only
// emitted as fp16 (the state stays as it is; the consumer of the state adds u[src] itself)
__global__ void __launch_bounds__(ROW_WARPS * 32)
residual_add_kernel(float* net, const void* u, int du, const int32_t* __restrict__ group_of, __half* net16,
                    int64_t rows, int dim, bool write_state) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (int64_t)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.x * ROW_WARPS) {
    const int64_t src = group_of ? (int64_t)group_of[r] : r;
    for (int col = lane * 4; col < dim; col += 128) {
      const float4 v = add4(load4(net, DPVO_F32, r * dim + col), load4(u, du, src * dim + col));
      if (write_state) store4(net, DPVO_F32, r * dim + col, v);
      if (net16) store4(net16, DPVO_F16, r * dim + col, v);
    }
  }
}

// y = x + sigmoid(g) * res ; optional relu'd fp16 copy (input of the two heads)
__global__ void __launch_bounds__(ROW_WARPS * 32)
gated_residual_kernel(const float* x, const __half* g, const __half* res, float* y32, __half* y16_relu,
                      int64_t rows, int dim) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (int64_t)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.x * ROW_WARPS) {
    for (int col = lane * 4; col < dim; col += 128) {
      const int64_t e = r * dim + col;
      const float4 xv = load4(x, DPVO_F32, e), gv = load4(g, DPVO_F16, e), rv = load4(res, DPVO_F16, e);
      float4 o;
      o.x = xv.x + sigmoidf_(gv.x) * rv.x; o.y = xv.y + sigmoidf_(gv.y) * rv.y;
      o.z = xv.z + sigmoidf_(gv.z) * rv.z; o.w = xv.w + sigmoidf_(gv.w) * rv.w;
      store4(y32, DPVO_F32, e, o);
      if (y16_relu) store4(y16_relu, DPVO_F16, e, make_float4(fmaxf(o.x, 0.f), fmaxf(o.y, 0.f), fmaxf(o.z, 0.f), fmaxf(o.w, 0.f)));
    }
  }
}

// ---- SoftAgg: one CTA per group, SA_SPLIT threads per 2 channels -------------------------------------------
// Two passes over the group's (scattered) rows: the per-channel maximum of the logits with packed half2 compares,
// then exp / sum / weighted sum.  The single-pass online softmax this replaces was issue-bound (a rescale test and
// two extra exponentials per row); the second pass re-reads rows that are still in L1/L2.  The rows of a group are
// dealt round-robin to SA_SPLIT thread groups (a (source, target) group has ~100 rows and there are fewer such
// groups than CTA slots), partial maxima / sums are combined through shared memory in a fixed order, and four
// rows are requested before the first is consumed in both passes.
constexpr int SA_SPLIT = 2;
constexpr int SA_MAXPAIRS = 256;      // channel pairs per CTA pass (dim <= 512 per pass)

__global__ void __launch_bounds__(SA_SPLIT * SA_MAXPAIRS)
softagg_reduce_kernel(const __half* __restrict__ f, const __half* __restrict__ gl, int64_t ld,
                      const int32_t* __restrict__ order,
                      const int32_t* __restrict__ group_start, const int32_t* __restrict__ n_groups,
                      __half* __restrict__ y, int dim, int max_groups) {
  constexpr int PF = 4;
  constexpr float LOG2E = 1.4426950408889634f;
  __shared__ __half2 s_max[SA_SPLIT][SA_MAXPAIRS];
  __shared__ float4 s_part[SA_SPLIT][SA_MAXPAIRS];
  const int G = min(*n_groups, max_groups);                  // y holds max_groups rows (host hint): never write past it
  const int npairs = blockDim.x / SA_SPLIT;                 // channel pairs handled per pass
  const int pr = threadIdx.x % npairs, sp = threadIdx.x / npairs;
  for (int g = blockIdx.x; g < G; g += gridDim.x) {
    const int s = group_start[g], e = group_start[g + 1];
    for (int col0 = 0; col0 < dim; col0 += npairs * 2) {
      const int col = col0 + pr * 2;
      const bool on = col < dim;
      __half2 mx = __float2half2_rn(-INFINITY);
      if (on)
        for (int k0 = s + sp * PF; k0 < e; k0 += PF * SA_SPLIT) {
          __half2 gq[PF];
#pragma unroll
          for (int u = 0; u < PF; ++u)
            gq[u] = (k0 + u < e) ? *reinterpret_cast<const __half2*>(gl + (int64_t)order[k0 + u] * ld + col) : mx;
#pragma unroll
          for (int u = 0; u < PF; ++u) mx = __hmax2(mx, gq[u]);
        }
      s_max[sp][pr] = mx;
      __syncthreads();
#pragma unroll
      for (int q = 0; q < SA_SPLIT; ++q) mx = __hmax2(mx, s_max[q][pr]);
      const float2 m = __half22float2(mx);
      const float m0 = m.x * LOG2E, m1 = m.y * LOG2E;
      float z0 = 0.f, z1 = 0.f, a0 = 0.f, a1 = 0.f;
      if (on)
        for (int k0 = s + sp * PF; k0 < e; k0 += PF * SA_SPLIT) {
          __half2 gq[PF], fq[PF];
#pragma unroll
          for (int u = 0; u < PF; ++u) {
            if (k0 + u < e) {
              const int64_t row = (int64_t)order[k0 + u] * ld + col;
              gq[u] = *reinterpret_cast<const __half2*>(gl + row);
              fq[u] = *reinterpret_cast<const __half2*>(f + row);
            }
          }
#pragma unroll
          for (int u = 0; u < PF; ++u) {
            if (k0 + u < e) {
              const float2 gv = __half22float2(gq[u]), fv = __half22float2(fq[u]);
              const float w0 = exp2f(gv.x * LOG2E - m0), w1 = exp2f(gv.y * LOG2E - m1);   // exp(g - max), <= 1
              z0 += w0; a0 += w0 * fv.x;
              z1 += w1; a1 += w1 * fv.y;
            }
          }
        }
      s_part[sp][pr] = make_float4(z0, a0, z1, a1);
      __syncthreads();
      if (sp == 0 && on) {
        float zz0 = 0.f, aa0 = 0.f, zz1 = 0.f, aa1 = 0.f;
#pragma unroll
        for (int q = 0; q < SA_SPLIT; ++q) { const float4 p = s_part[q][pr]; zz0 += p.x; aa0 += p.y; zz1 += p.z; aa1 += p.w; }
        *reinterpret_cast<__half2*>(y + (int64_t)g * dim + col) = __floats2half2_rn(aa0 / zz0, aa1 / zz1);
      }
      __syncthreads();
    }
  }
  // y holds max_groups rows (a host-side bound): the rows past the true group count are defined (zero) as well, so that
  // the dense layer that follows reads no uninitialised memory and the caller needs no separate fill
  for (int g = G + blockIdx.x; g < max_groups; g += gridDim.x)
    for (int c = threadIdx.x * 2; c < dim; c += blockDim.x * 2) *reinterpret_cast<__half2*>(y + (int64_t)g * dim + c) = __float2half2_rn(0.f);
}

// ---- heads: out[r] = (Wd relu(net[r]) + bd, sigmoid(Ww relu(net[r]) + bw)) ---------------------
// NV = float4 per lane (dim = 128 NV).  The four weight rows live in shared memory and a warp takes two rows of net
// at a time (loads of both in flight before the first reduction).
// Optional gated input: the row is x + gate * res (GatedResidual, blocks.py:28-29, gate already a sigmoid) and is
// written back over x -- the last GatedResidual of the GRU folded into the pass that reads its output anyway.
template <int NV>
__global__ void __launch_bounds__(ROW_WARPS * 32)
heads_kernel(float* net, const __half* __restrict__ gate, int64_t ld_gate, const __half* __restrict__ res, int64_t ld_res,
             const float* __restrict__ W4, const float* __restrict__ b4,
             const float* __restrict__ coords, int PP, int centre,
             float* __restrict__ delta, float* __restrict__ weight, int64_t rows, int dim) {
  const int lane = threadIdx.x & 31;
  __shared__ float4 sw[4][NV * 32];                     // the four weight rows (6 KB at dim 384)
  for (int i = threadIdx.x; i < 4 * NV * 32; i += blockDim.x) sw[i / (NV * 32)][i % (NV * 32)] = *reinterpret_cast<const float4*>(W4 + (size_t)i * 4);
  __syncthreads();
  const float bias0 = b4[0], bias1 = b4[1], bias2 = b4[2], bias3 = b4[3];
  const int64_t wstride = (int64_t)gridDim.x * ROW_WARPS * 2;
  for (int64_t r0 = ((int64_t)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5)) * 2; r0 < rows; r0 += wstride) {
    float4 x[2][NV];
    uint2 gq[2][NV], rq[2][NV];
    // every load of both rows first (net may alias nothing here, but the compiler cannot know: a store between
    // the loads would serialise them)
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int64_t r = r0 + k;
        const int col = (i * 32 + lane) * 4;
        x[k][i] = make_float4(0.f, 0.f, 0.f, 0.f);
        gq[k][i] = make_uint2(0u, 0u); rq[k][i] = make_uint2(0u, 0u);
        if (r < rows) {
          x[k][i] = *reinterpret_cast<const float4*>(net + r * dim + col);
          if (gate) {
            gq[k][i] = *reinterpret_cast<const uint2*>(gate + r * ld_gate + col);
            rq[k][i] = *reinterpret_cast<const uint2*>(res + r * ld_res + col);
          }
        }
      }
    if (gate) {
#pragma unroll
      for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          const int64_t r = r0 + k;
          const float2 g0 = __half22float2(*reinterpret_cast<const __half2*>(&gq[k][i].x)), g1 = __half22float2(*reinterpret_cast<const __half2*>(&gq[k][i].y));
          const float2 q0 = __half22float2(*reinterpret_cast<const __half2*>(&rq[k][i].x)), q1 = __half22float2(*reinterpret_cast<const __half2*>(&rq[k][i].y));
          x[k][i] = make_float4(x[k][i].x + g0.x * q0.x, x[k][i].y + g0.y * q0.y, x[k][i].z + g1.x * q1.x, x[k][i].w + g1.y * q1.y);
          if (r < rows) *reinterpret_cast<float4*>(net + r * dim + (i * 32 + lane) * 4) = x[k][i];
        }
    }
    float acc[2][4];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
#pragma unroll
      for (int o = 0; o < 4; ++o) acc[k][o] = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const float4 v = make_float4(fmaxf(x[k][i].x, 0.f), fmaxf(x[k][i].y, 0.f), fmaxf(x[k][i].z, 0.f), fmaxf(x[k][i].w, 0.f));
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const float4 wv = sw[o][i * 32 + lane];
          acc[k][o] += (v.x * wv.x + v.y * wv.y) + (v.z * wv.z + v.w * wv.w);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int o = 0; o < 4; ++o) acc[k][o] = warp_sum(acc[k][o]);
    if (lane < 2 && r0 + lane < rows) {
      const int64_t r = r0 + lane;
      const float a0 = lane ? acc[1][0] : acc[0][0], a1 = lane ? acc[1][1] : acc[0][1];
      const float a2 = lane ? acc[1][2] : acc[0][2], a3 = lane ? acc[1][3] : acc[0][3];
      float d0 = a0 + bias0, d1 = a1 + bias1;
      if (coords) {      // target = reprojected patch centre + delta (dpvo.py:341)
        d0 += coords[r * 2 * PP + centre];
        d1 += coords[r * 2 * PP + PP + centre];
      }
      delta[r * 2 + 0] = d0;
      delta[r * 2 + 1] = d1;
      weight[r * 2 + 0] = sigmoidf_(a2 + bias2);
      weight[r * 2 + 1] = sigmoidf_(a3 + bias3);
    }
  }
}

static inline unsigned row_grid(int64_t rows) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((rows + ROW_WARPS - 1) / ROW_WARPS, (int64_t)sm_count() * 8));
}
static inline bool ok_dt(int d) { return d == DPVO_F16 || d == DPVO_F32; }

}  // namespace dpvo

using namespace dpvo;

extern "C" int dpvo_add_layernorm(const void* a, const void* b, const void* c, const int* in_dtypes,
                                  const int64_t* b_index, const void* c_scale, int64_t ld_c_scale,
                                  const float* gamma, const float* beta, float eps,
                                  void* y32, void* y16, int relu, int64_t rows, int dim, void* stream) {
  DPVO_REQUIRE(rows >= 0 && dim > 0, "add_layernorm: bad sizes");
  if (rows == 0) return DPVO_OK;
  DPVO_REQUIRE(a && in_dtypes && gamma && beta && (y32 || y16), "add_layernorm: null pointer");
  DPVO_REQUIRE(dim % 128 == 0 && dim <= 128 * MAX_V4, "add_layernorm: dim must be a multiple of 128, <= %d", 128 * MAX_V4);
  DPVO_REQUIRE(ok_dt(in_dtypes[0]) && (!b || ok_dt(in_dtypes[1])) && (!c || ok_dt(in_dtypes[2])), "add_layernorm: dtype");
  DPVO_REQUIRE(!c_scale || (c && ld_c_scale >= dim && ld_c_scale % 4 == 0 && ((uintptr_t)c_scale & 7) == 0),
               "add_layernorm: c_scale needs operand c and rows aligned to 4 elements");
  const int nv = dim / 128;
  const int db = b ? in_dtypes[1] : 0, dc = c ? in_dtypes[2] : 0;
  const int64_t* bi = b ? b_index : nullptr;
  cudaStream_t st = (cudaStream_t)stream;
#define DPVO_LN_LAUNCH_T(NV, RPW, DA, DBC)                                                                                   \
  return launch("add_layernorm_kernel", add_layernorm_kernel<NV, RPW, DA, DBC>, row_grid((rows + RPW - 1) / RPW), ROW_WARPS * 32, 0, st, a, b, c, \
                in_dtypes[0], db, dc, bi, (const __half*)c_scale, ld_c_scale, gamma, beta, eps, (float*)y32, (__half*)y16, relu, rows, dim)
#define DPVO_LN_LAUNCH(NV, RPW) DPVO_LN_LAUNCH_T(NV, RPW, -1, -1)
  // the update operator's shapes (dim 384): fp16 alone, fp32 alone, fp32 + fp16 (+ fp16)
  const bool bc16 = (!b || db == DPVO_F16) && (!c || dc == DPVO_F16);
  // dim 384, dense 16-byte aligned rows: operands a and c staged through shared memory by bulk copies
  if (nv == 3 && bc16 && ROW_WARPS * 2 == LNB_ROWS && ((uintptr_t)a & 15) == 0 &&
      (!c || ((uintptr_t)c & 15) == 0) && (!b || ((uintptr_t)b & 15) == 0) &&
      (!c_scale || (((uintptr_t)c_scale & 15) == 0 && (ld_c_scale * 2) % 16 == 0))) {
    int rc;
    if (in_dtypes[0] == DPVO_F16)
      rc = c ? launch_ln_bulk<DPVO_F16, true>(a, b, c, db, bi, c_scale, ld_c_scale, gamma, beta, eps, y32, y16, relu, rows, st)
             : launch_ln_bulk<DPVO_F16, false>(a, b, c, db, bi, c_scale, ld_c_scale, gamma, beta, eps, y32, y16, relu, rows, st);
    else
      rc = c ? launch_ln_bulk<DPVO_F32, true>(a, b, c, db, bi, c_scale, ld_c_scale, gamma, beta, eps, y32, y16, relu, rows, st)
             : launch_ln_bulk<DPVO_F32, false>(a, b, c, db, bi, c_scale, ld_c_scale, gamma, beta, eps, y32, y16, relu, rows, st);
    if (rc != DPVO_ERR_UNSUPPORTED) return rc;
  }
  if (nv == 3 && bc16) {
    if (in_dtypes[0] == DPVO_F16) DPVO_LN_LAUNCH_T(3, 2, DPVO_F16, DPVO_F16);
    DPVO_LN_LAUNCH_T(3, 2, DPVO_F32, DPVO_F16);
  }
  switch (nv) {
    case 1: DPVO_LN_LAUNCH(1, 4);
    case 2: DPVO_LN_LAUNCH(2, 2);
    case 3: DPVO_LN_LAUNCH(3, 2);
    case 4: DPVO_LN_LAUNCH(4, 2);
    case 5: DPVO_LN_LAUNCH(5, 1);
    case 6: DPVO_LN_LAUNCH(6, 1);
    case 7: DPVO_LN_LAUNCH(7, 1);
    default: DPVO_LN_LAUNCH(8, 1);
  }
#undef DPVO_LN_LAUNCH
#undef DPVO_LN_LAUNCH_T
}

extern "C" int dpvo_gather_rows_masked(const void* x, int x_dtype, const int64_t* idx,
                                       void* y, int y_dtype, int64_t rows, int dim, void* stream) {
  DPVO_REQUIRE(rows >= 0 && dim > 0 && dim % 4 == 0, "gather_rows_masked: bad sizes");
  if (rows == 0) return DPVO_OK;
  DPVO_REQUIRE(x && idx && y && ok_dt(x_dtype) && ok_dt(y_dtype), "gather_rows_masked: bad argument");
  return launch("gather_rows_masked_kernel", gather_rows_masked_kernel, row_grid(rows), ROW_WARPS * 32, 0, (cudaStream_t)stream, x, x_dtype, idx, y,
                y_dtype, rows, dim);
}

extern "C" int dpvo_residual_add(void* net32, const void* u, int u_dtype, const int32_t* group_of, void* net16,
                                 int64_t rows, int dim, void* stream) {
  DPVO_REQUIRE(rows >= 0 && dim > 0 && dim % 4 == 0, "residual_add: bad sizes");
  if (rows == 0) return DPVO_OK;
  DPVO_REQUIRE(net32 && u && ok_dt(u_dtype), "residual_add: bad argument");
  return launch("residual_add_kernel", residual_add_kernel, row_grid(rows), ROW_WARPS * 32, 0, (cudaStream_t)stream, (float*)net32, u, u_dtype,
                group_of, (__half*)net16, rows, dim, true);
}

extern "C" int dpvo_residual_sum16(const void* net32, const void* u, int u_dtype, const int32_t* group_of, void* net16,
                                   int64_t rows, int dim, void* stream) {
  DPVO_REQUIRE(rows >= 0 && dim > 0 && dim % 4 == 0, "residual_sum16: bad sizes");
  if (rows == 0) return DPVO_OK;
  DPVO_REQUIRE(net32 && u && net16 && ok_dt(u_dtype), "residual_sum16: bad argument");
  return launch("residual_add_kernel", residual_add_kernel, row_grid(rows), ROW_WARPS * 32, 0, (cudaStream_t)stream, (float*)const_cast<void*>(net32),
                u, u_dtype, group_of, (__half*)net16, rows, dim, false);
}

extern "C" int dpvo_gated_residual(const void* x32, const void* gate16, const void* res16, void* y32, void* y16_relu,
                                   int64_t rows, int dim, void* stream) {
  DPVO_REQUIRE(rows >= 0 && dim > 0 && dim % 4 == 0, "gated_residual: bad sizes");
  if (rows == 0) return DPVO_OK;
  DPVO_REQUIRE(x32 && gate16 && res16 && y32, "gated_residual: null pointer");
  return launch("gated_residual_kernel", gated_residual_kernel, row_grid(rows), ROW_WARPS * 32, 0, (cudaStream_t)stream,
                (const float*)x32, (const __half*)gate16, (const __half*)res16, (float*)y32, (__half*)y16_relu, rows, dim);
}

extern "C" int dpvo_softagg_reduce(const void* f16, const void* g16, int64_t ld, const int32_t* order, const int32_t* group_start,
                                   const int32_t* n_groups, int64_t max_groups, void* y16, int dim, void* stream) {
  DPVO_REQUIRE(max_groups >= 0 && dim > 0 && dim % 2 == 0, "softagg_reduce: bad sizes");
  if (max_groups == 0) return DPVO_OK;
  DPVO_REQUIRE(f16 && g16 && order && group_start && n_groups && y16, "softagg_reduce: null pointer");
  DPVO_REQUIRE(ld >= dim && ld % 2 == 0, "softagg_reduce: row stride must be even and >= dim");
  const unsigned grid = (unsigned)std::min<int64_t>(max_groups, (int64_t)sm_count() * 8);
  const int pairs = std::min(SA_MAXPAIRS, std::max(32, ((dim / 2 + 31) / 32) * 32));
  const int threads = pairs * SA_SPLIT;
  return launch("softagg_reduce_kernel", softagg_reduce_kernel, grid, threads, 0, (cudaStream_t)stream, (const __half*)f16, (const __half*)g16, ld,
                order, group_start, n_groups, (__half*)y16, dim, (int)max_groups);
}

extern "C" int dpvo_update_heads(void* net32, const void* gate16, int64_t ld_gate, const void* res16, int64_t ld_res,
                                 const float* W4, const float* b4, const float* coords, int P,
                                 float* delta, float* weight, int64_t rows, int dim, void* stream) {
  DPVO_REQUIRE(rows >= 0 && dim > 0 && dim % 128 == 0 && dim <= 512, "update_heads: dim must be a multiple of 128, <= 512");
  if (rows == 0) return DPVO_OK;
  DPVO_REQUIRE(net32 && W4 && b4 && delta && weight, "update_heads: null pointer");
  DPVO_REQUIRE((gate16 == nullptr) == (res16 == nullptr), "update_heads: gate and res come together");
  DPVO_REQUIRE(!gate16 || (ld_gate % 4 == 0 && ld_res % 4 == 0 && ((uintptr_t)gate16 & 7) == 0 && ((uintptr_t)res16 & 7) == 0),
               "update_heads: gate / res rows must be aligned to 4 elements");
  const unsigned grid = row_grid((rows + 1) / 2);
  const int PP = P * P, centre = (P / 2) * P + P / 2;
  decltype(&heads_kernel<1>) const kern[] = {heads_kernel<1>, heads_kernel<2>, heads_kernel<3>, heads_kernel<4>};
  return launch("heads_kernel", kern[dim / 128 - 1], grid, ROW_WARPS * 32, 0, (cudaStream_t)stream, (float*)net32, (const __half*)gate16, ld_gate,
                (const __half*)res16, ld_res, W4, b4, coords, PP, centre, delta, weight, rows, dim);
}
