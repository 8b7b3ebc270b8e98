// Patch <-> frame local correlation (altcorr) for sm_90a.
//
// Replaces dpvo/altcorr/correlation_kernel.cu:82-136 (raw 8x8 taps), :221-230 (bilinear blend,
// ~15 ATen launches over a [E,8,8,3,3] temporary) and :232 (permute) with ONE launch.
//
// Two code paths behind dpvo_corr_forward():
//   * corr_fwd_mma      fp16, C=128, P=3, R=3, channels-last frame features.  One warp per edge.
//                       The nine 8x8 tap windows of an edge overlap almost completely, so the warp
//                       reads the UNION box (<=10x10 pixels x 256 B) once, straight from global/L2
//                       into mma.sync B fragments with 16-byte loads (a K-permutation makes one
//                       LDG.128 == the fragment of two k-steps), multiplies it against the 9x128
//                       patch features held in registers as the A operand, and blends the raw taps
//                       bilinearly out of shared memory.  ~25.6 KB of loads per edge-level instead
//                       of the reference's ~295 KB of scalar requests.
//   * corr_fwd_generic  any dtype (f16/bf16/f32/f64), any strides (NCHW included), any C,
//                       P<=3, any R: one CTA per edge, union box staged in shared memory, fp32
//                       (fp64) FMA.  This is the training (fp32) path and the correctness anchor.
// Both fall back, per edge, to nine separate 8x8 boxes when the reprojected patch is stretched so
// much that the union box would not fit -- results are exact in every case.
#include "common.cuh"
#include <algorithm>
#include <cstdlib>

namespace dpvo {

// ------------------------------------------------------------------------------------------
// argument block shared by the forward kernels
// ------------------------------------------------------------------------------------------
struct CorrArgs {
  const void* fmap1;
  const void* fmap2[2];
  int64_t s1[5];        // element strides of logical [B,S1,C,P,P]
  int64_t s2[2][5];     // element strides of logical [B,S2,C,H2,W2] per level
  int H2[2], W2[2];
  float div[2];         // coords divisor per level (1, 4)
  const float* coords;  // [B,M,2,P,P]
  const int64_t* ii;
  const int64_t* jj;
  void* out;
  int64_t out_stride;   // element stride between consecutive logical outputs
  int64_t out_row;      // element stride between consecutive (b, m) rows
  int out_offset[2];    // element offset of each level inside one logical output slot
  int nlev;             // 1 or 2 levels handled by this launch
  int B, M, C, P, R;
  const int* list;       // optional device list of edge ids to process (B == 1), with its length on device
  const int* list_count;
};

// ==========================================================================================
// generic path
// ==========================================================================================
template <typename T, typename A> struct Vec4Load;
template <> struct Vec4Load<float, float> {
  static __device__ __forceinline__ void ld(const float* p, float (&v)[4]) {
    float4 q = *reinterpret_cast<const float4*>(p); v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  }
};
template <> struct Vec4Load<__half, float> {
  static __device__ __forceinline__ void ld(const __half* p, float (&v)[4]) {
    uint2 q = *reinterpret_cast<const uint2*>(p);
    float2 a = __half22float2(*reinterpret_cast<__half2*>(&q.x));
    float2 b = __half22float2(*reinterpret_cast<__half2*>(&q.y));
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
};
template <> struct Vec4Load<__nv_bfloat16, float> {
  static __device__ __forceinline__ void ld(const __nv_bfloat16* p, float (&v)[4]) {
    uint2 q = *reinterpret_cast<const uint2*>(p);
    float2 a = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&q.x));
    float2 b = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&q.y));
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
};
template <> struct Vec4Load<double, double> {
  static __device__ __forceinline__ void ld(const double* p, double (&v)[4]) {
    double2 a = *reinterpret_cast<const double2*>(p);
    double2 b = *reinterpret_cast<const double2*>(p + 2);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
};

constexpr int GEN_THREADS = 128;

// pad of the shared window row, in elements of T, so that consecutive rows start 16 B apart
// modulo 128 B (conflict-free 16-byte row-per-thread reads)
template <typename T> __host__ __device__ constexpr int row_pad() { return 16 / (int)sizeof(T); }

template <typename T, int P>
__global__ void __launch_bounds__(GEN_THREADS)
corr_fwd_generic(const CorrArgs a, int Cpad) {
  using A = typename acc_of<T>::type;
  constexpr int PP = P * P;
  const int R = a.R, D = 2 * R + 2, DD = D * D, BOX = D + 2, O = 2 * R + 1;
  const int C = a.C;
  const int pitch = Cpad + row_pad<T>();

  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* win = reinterpret_cast<T*>(smem_raw);                           // [BOX*BOX][pitch]
  A* pat = reinterpret_cast<A*>(win + (size_t)BOX * BOX * pitch);    // [PP][Cpad]
  A* raw = pat + PP * Cpad;                                          // [PP][DD]
  int* meta_i = reinterpret_cast<int*>(raw + PP * DD);               // ax[PP], ay[PP], box[6]
  float* meta_f = reinterpret_cast<float*>(meta_i + 2 * PP + 8);     // dx[PP], dy[PP]

  const int tid = threadIdx.x;
  const T* f1 = reinterpret_cast<const T*>(a.fmap1);
  T* out = reinterpret_cast<T*>(a.out);
  const int64_t nitems = (int64_t)a.B * a.M;

  for (int64_t item = blockIdx.x; item < nitems; item += gridDim.x) {
    const int b = (int)(item / a.M), m = (int)(item % a.M);
    const int64_t ix = a.ii[m], jx = a.jj[m];

    // ---- patch features -> shared (accumulate type), zero padded to Cpad
    for (int idx = tid; idx < PP * Cpad; idx += GEN_THREADS) {
      int p, c;
      if (a.s1[2] == 1) { c = idx % Cpad; p = idx / Cpad; } else { p = idx % PP; c = idx / PP; }
      A v = (A)0;
      if (c < C)
        v = to_acc<A, T>(f1[b * a.s1[0] + ix * a.s1[1] + c * a.s1[2] + (p / P) * a.s1[3] + (p % P) * a.s1[4]]);
      pat[p * Cpad + c] = v;
    }

    for (int lev = 0; lev < a.nlev; ++lev) {
      const T* f2 = reinterpret_cast<const T*>(a.fmap2[lev]) + b * a.s2[lev][0] + jx * a.s2[lev][1];
      const int64_t sc = a.s2[lev][2], sy = a.s2[lev][3], sx = a.s2[lev][4];
      const int H2 = a.H2[lev], W2 = a.W2[lev];

      __syncthreads();   // previous users of meta/raw/win are done
      if (tid < PP) {
        const float* cp = a.coords + ((int64_t)(b * a.M + m) * 2) * PP;
        float x = cp[tid], y = cp[PP + tid];
        if (a.div[lev] != 1.0f) { x = x / a.div[lev]; y = y / a.div[lev]; }
        meta_i[tid] = safe_floor_int(x) - R;
        meta_i[PP + tid] = safe_floor_int(y) - R;
        meta_f[tid] = x - floorf(x);
        meta_f[PP + tid] = y - floorf(y);
      }
      __syncthreads();
      if (tid == 0) {
        int x0 = meta_i[0], x1 = meta_i[0], y0 = meta_i[PP], y1 = meta_i[PP];
        for (int p = 1; p < PP; ++p) {
          x0 = min(x0, meta_i[p]); x1 = max(x1, meta_i[p]);
          y0 = min(y0, meta_i[PP + p]); y1 = max(y1, meta_i[PP + p]);
        }
        const bool uni = (x1 - x0 + D <= BOX) && (y1 - y0 + D <= BOX);
        meta_i[2 * PP + 0] = uni ? 1 : 0;
        meta_i[2 * PP + 1] = x0; meta_i[2 * PP + 2] = y0;
        meta_i[2 * PP + 3] = x1 - x0 + D; meta_i[2 * PP + 4] = y1 - y0 + D;
      }
      __syncthreads();
      const bool uni = meta_i[2 * PP + 0] != 0;
      const int npass = uni ? 1 : PP;

      for (int pass = 0; pass < npass; ++pass) {
        const int bx0 = uni ? meta_i[2 * PP + 1] : meta_i[pass];
        const int by0 = uni ? meta_i[2 * PP + 2] : meta_i[PP + pass];
        const int bw = uni ? meta_i[2 * PP + 3] : D;
        const int bh = uni ? meta_i[2 * PP + 4] : D;
        const int p_lo = uni ? 0 : pass, p_hi = uni ? PP : pass + 1;
        const int rows = bw * bh;

        if (pass > 0) __syncthreads();
        // ---- stage the box (zero outside the image: correlation_kernel.cu:121-122)
        for (int idx = tid; idx < rows * Cpad; idx += GEN_THREADS) {
          int r, c;
          if (sc == 1) { c = idx % Cpad; r = idx / Cpad; } else { r = idx % rows; c = idx / rows; }
          const int y = by0 + r / bw, x = bx0 + r % bw;
          T v = from_acc<T, A>((A)0);
          if (c < C && y >= 0 && y < H2 && x >= 0 && x < W2) v = f2[c * sc + (int64_t)y * sy + (int64_t)x * sx];
          win[r * pitch + c] = v;
        }
        __syncthreads();

        // ---- one box pixel per thread against all patch pixels
        for (int r = tid; r < rows; r += GEN_THREADS) {
          A acc[PP];
#pragma unroll
          for (int p = 0; p < PP; ++p) acc[p] = (A)0;
          const T* wr = win + r * pitch;
          for (int c = 0; c < Cpad; c += 4) {
            A w[4];
            Vec4Load<T, A>::ld(wr + c, w);
#pragma unroll
            for (int p = 0; p < PP; ++p) {
              A q[4];
              Vec4Load<A, A>::ld(pat + p * Cpad + c, q);
              acc[p] += w[0] * q[0]; acc[p] += w[1] * q[1]; acc[p] += w[2] * q[2]; acc[p] += w[3] * q[3];
            }
          }
          const int wy = r / bw, wx = r % bw;
#pragma unroll
          for (int p = 0; p < PP; ++p) {
            if (p >= p_lo && p < p_hi) {
              const int ty = wy - (meta_i[PP + p] - by0), tx = wx - (meta_i[p] - bx0);
              if (ty >= 0 && ty < D && tx >= 0 && tx < D) raw[p * DD + ty * D + tx] = acc[p];
            }
          }
        }
      }
      __syncthreads();

      // ---- bilinear blend (correlation_kernel.cu:221-230) + (x,y) offset order (:232)
      const int nout = O * O * PP;
      T* o = out + (int64_t)(b * a.M + m) * a.out_row + a.out_offset[lev];
      for (int q = tid; q < nout; q += GEN_THREADS) {
        const int p = q % PP, t = q / PP, yo = t % O, xo = t / O;
        const A dx = (A)meta_f[p], dy = (A)meta_f[PP + p];
        const A* rp = raw + p * DD + yo * D + xo;
        const A v = ((A)1 - dx) * ((A)1 - dy) * rp[0] + dx * ((A)1 - dy) * rp[1] +
                    ((A)1 - dx) * dy * rp[D] + dx * dy * rp[D + 1];
        o[(int64_t)q * a.out_stride] = from_acc<T, A>(v);
      }
    }
    __syncthreads();
  }
}

// ==========================================================================================
// fp16 tensor-core path (mma.sync m16n8k16, fp32 accumulate)
// ==========================================================================================
__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2,
                                         uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint4 ldg128(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

constexpr int MMA_WARPS = 8;
constexpr int MMA_PATP = 136;   // halves per patch-pixel row in shared (128 + 8 pad)
constexpr int MMA_BOX = 10;
constexpr int MMA_RAWP = 105;   // floats per patch pixel in the raw tile (odd pitch: conflict-free)

// per-warp shared memory: the patch staging buffer is dead once the A fragments are in registers,
// so the raw tap tile aliases it
struct __align__(16) MmaWarpSmem {
  union {
    __half patch[9 * MMA_PATP];       // 2448 B
    float raw[2][9 * MMA_RAWP + 3];   // per level: raw[p][box pixel] = <patch pixel p, box pixel>
  };
  uint32_t stage[444];                // blended outputs of one edge as half2 (level0, level1), output order
  float4 w[2][9];                     // bilinear weights (1-dx)(1-dy), dx(1-dy), (1-dx)dy, dx dy
  int base[2][9];                     // index of tap (0,0) of pixel p inside its box
  int pitch[2][9];                    // row pitch of that box (bw, or 8 in the per-pixel fallback)
};

// C = 128, P = 3, R = 3 (D = 8), fp16, fmap2 channels-last with 16-byte aligned pixels.
// Instruction budget matters more than bytes here (the first version issued 10k instructions per
// edge, 34 % of them integer multiply-adds from divisions and 64-bit address arithmetic):
//   * box coordinates advance incrementally per 8-pixel tile (no division in the loops)
//   * accumulators are stored densely as raw[p][box pixel]; the bilinear stage indexes the box
//   * per-lane output decomposition (q -> p, x-off, y-off) is computed once per kernel
//   * two independent HMMA accumulation chains per tile halve the dependent-issue latency
template <bool PAIR_OUT>
__global__ void __launch_bounds__(MMA_WARPS * 32, 2)
corr_fwd_mma(const CorrArgs a) {
  constexpr int D = 8, O = 7, NOUT = O * O * 9;   // 441
  extern __shared__ __align__(16) unsigned char mma_smem_raw[];
  MmaWarpSmem& sm = reinterpret_cast<MmaWarpSmem*>(mma_smem_raw)[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  // list mode (edges the wgmma kernel could not box): an item is ONE patch pixel of a listed edge -- its own 8x8
  // window on both levels and its 49 outputs -- so that the nine passes of a stretched edge spread over nine warps
  // instead of serialising in one (a handful of such edges used to cost 30 us of single-warp latency)
  const int64_t nitems = a.list ? (int64_t)*a.list_count * 9 : (int64_t)a.B * a.M;
  const int64_t wstride = (int64_t)gridDim.x * MMA_WARPS;
  const __half* f1 = reinterpret_cast<const __half*>(a.fmap1);
  __half* out = reinterpret_cast<__half*>(a.out);

  for (int64_t item = (int64_t)blockIdx.x * MMA_WARPS + (threadIdx.x >> 5); item < nitems; item += wstride) {
    const int b = a.list ? 0 : (int)(item / a.M), m = a.list ? a.list[item / 9] : (int)(item % a.M);
    const int psel = a.list ? (int)(item % 9) : -1;
    const int64_t ix = a.ii[m], jx = a.jj[m];

    // ---- patch features -> shared as [pixel][channel]
    __syncwarp();
    {
      const __half* src = f1 + b * a.s1[0] + ix * a.s1[1];
      if (a.s1[2] == 1 && (a.s1[3] % 8 == 0) && (a.s1[4] % 8 == 0)) {
        for (int idx = lane; idx < 9 * 16; idx += 32) {       // 16-byte chunks
          const int p = idx >> 4, ch = (idx & 15) * 8;
          *reinterpret_cast<uint4*>(&sm.patch[p * MMA_PATP + ch]) =
              *reinterpret_cast<const uint4*>(src + (p / 3) * a.s1[3] + (p % 3) * a.s1[4] + ch);
        }
      } else {
        for (int idx = lane; idx < 9 * 128; idx += 32) {
          int p, c;
          if (a.s1[2] == 1) { c = idx & 127; p = idx >> 7; } else { p = idx % 9; c = idx / 9; }
          sm.patch[p * MMA_PATP + c] = src[c * a.s1[2] + (p / 3) * a.s1[3] + (p % 3) * a.s1[4]];
        }
      }
    }
    __syncwarp();
    // A operand: rows = patch pixels (row g, and row 8 held by the g==0 lanes), K = channels in
    // the permuted order  k-step s=2*kb+h, logical k {2t,2t+1 | 2t+8,2t+9} <-> channel 32kb+8t+4h+{0,1 | 2,3}
    uint4 PA[4], PB[4];
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
      PA[kb] = *reinterpret_cast<const uint4*>(&sm.patch[g * MMA_PATP + kb * 32 + t * 8]);
      PB[kb] = (g == 0) ? *reinterpret_cast<const uint4*>(&sm.patch[8 * MMA_PATP + kb * 32 + t * 8])
                        : make_uint4(0u, 0u, 0u, 0u);
    }
    __syncwarp();                      // patch buffer is dead from here on (raw aliases it)

    for (int lev = 0; lev < a.nlev; ++lev) {
      float* raw = sm.raw[lev];
      const __half* f2 = reinterpret_cast<const __half*>(a.fmap2[lev]) + b * a.s2[lev][0] + jx * a.s2[lev][1];
      const int sy = (int)a.s2[lev][3], sx = (int)a.s2[lev][4];     // element strides inside one frame (< 2^31)
      const int H2 = a.H2[lev], W2 = a.W2[lev];

      // ---- anchors / fractions of the nine patch pixels (lanes 0..8)
      int ax = 1 << 28, ay = 1 << 28, axm = -(1 << 28), aym = -(1 << 28);
      float fx = 0.f, fy = 0.f;
      if (lane < 9) {
        const float* cp = a.coords + ((int64_t)(b * a.M + m) * 2) * 9;
        float x = cp[lane], y = cp[9 + lane];
        if (a.div[lev] != 1.0f) { x = x / a.div[lev]; y = y / a.div[lev]; }
        ax = safe_floor_int(x) - 3; ay = safe_floor_int(y) - 3;
        axm = ax; aym = ay;
        fx = x - floorf(x); fy = y - floorf(y);
      }
      const int bx_min = warp_min_i(ax), by_min = warp_min_i(ay);
      const int bx_max = warp_max_i(axm), by_max = warp_max_i(aym);
      const bool uni = psel < 0 && (bx_max - bx_min + D <= MMA_BOX) && (by_max - by_min + D <= MMA_BOX);
      const int ubw = bx_max - bx_min + D;
      if (lane < 9) {
        sm.w[lev][lane] = make_float4((1.f - fx) * (1.f - fy), fx * (1.f - fy), (1.f - fx) * fy, fx * fy);
        sm.base[lev][lane] = uni ? (ay - by_min) * ubw + (ax - bx_min) : 0;
        sm.pitch[lev][lane] = uni ? ubw : D;
      }

      const int pass0 = psel >= 0 ? psel : 0, npass = psel >= 0 ? psel + 1 : (uni ? 1 : 9);
      for (int pass = pass0; pass < npass; ++pass) {
        const int bx0 = uni ? bx_min : __shfl_sync(0xffffffffu, ax, pass);
        const int by0 = uni ? by_min : __shfl_sync(0xffffffffu, ay, pass);
        const int bw = uni ? ubw : D;
        const int rows = uni ? ubw * (by_max - by_min + D) : D * D;
        const int ntiles = (rows + 7) >> 3;

        // box pixel of this lane's B-operand column: wp = nt*8 + g, advanced incrementally
        int wx = g, wy = 0;
        if (wx >= bw) { wx -= bw; wy = 1; }
        auto load_tile = [&](uint4 (&Q)[4], int wp) {
          const int y = by0 + wy, x = bx0 + wx;
          const bool ok = (wp < rows) && ((unsigned)y < (unsigned)H2) && ((unsigned)x < (unsigned)W2);
          if (ok) {
            const __half* p = f2 + (y * sy + x * sx + t * 8);
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) Q[kb] = ldg128(p + kb * 32);
          } else {
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) Q[kb] = make_uint4(0u, 0u, 0u, 0u);
          }
          wx += 8; if (wx >= bw) { wx -= bw; ++wy; }          // 8 <= bw <= 10: at most one wrap
        };

        // one 8-pixel tile: 8 HMMAs (two independent accumulation chains) + dense store of the 16x8 block
        auto mma_tile = [&](const uint4 (&Q)[4], int nt) {
          float acc0[4] = {0.f, 0.f, 0.f, 0.f}, acc1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int kb = 0; kb < 4; ++kb) {
            mma16816(acc0, PA[kb].x, PB[kb].x, PA[kb].y, PB[kb].y, Q[kb].x, Q[kb].y);
            mma16816(acc1, PA[kb].z, PB[kb].z, PA[kb].w, PB[kb].w, Q[kb].z, Q[kb].w);
          }
          // rows of the accumulator tile = patch pixels g (c0,c1) and 8 (c2,c3; g==0 lanes);
          // columns = box pixels nt*8 + 2t, +1: stored densely, no per-tap logic
          const int col = nt * 8 + 2 * t;
          if (uni || g == pass)
            *reinterpret_cast<float2*>(&raw[g * MMA_RAWP + col + (g & 1)]) = make_float2(acc0[0] + acc1[0], acc0[1] + acc1[1]);
          if (g == 0 && (uni || pass == 8))
            *reinterpret_cast<float2*>(&raw[8 * MMA_RAWP + col]) = make_float2(acc0[2] + acc1[2], acc0[3] + acc1[3]);
        };
        // software pipeline with two register buffers used alternately (no register copies)
        uint4 Q0[4], Q1[4];
        load_tile(Q0, g);
        for (int nt = 0; nt < ntiles; nt += 2) {
          if (nt + 1 < ntiles) load_tile(Q1, (nt + 1) * 8 + g);
          mma_tile(Q0, nt);
          if (nt + 1 < ntiles) {
            if (nt + 2 < ntiles) load_tile(Q0, (nt + 2) * 8 + g);
            mma_tile(Q1, nt + 1);
          }
        }
      }
    }
    __syncwarp();

    // ---- bilinear blend of both levels.  Lanes own taps (two per lane, constant for the whole kernel),
    // the loop runs over the nine patch pixels, so box pitch / base / weights are warp-uniform and the
    // per-output cost is one multiply-add of indices, four shared loads and four FMAs.  Results are
    // staged in shared memory in output order and copied out with 16-byte stores.
    {
      __half2* stage = reinterpret_cast<__half2*>(sm.stage);
      const int tt0 = lane, tt1 = lane + 32;                  // taps 0..48 ; tap = xo*7 + yo
      const int xo0 = (tt0 * 37) >> 8, yo0 = tt0 - 7 * xo0;
      const int xo1 = (tt1 * 37) >> 8, yo1 = tt1 - 7 * xo1;
#pragma unroll 1
      for (int p = (psel >= 0 ? psel : 0); p < (psel >= 0 ? psel + 1 : 9); ++p) {
        float v0[2] = {0.f, 0.f}, v1[2] = {0.f, 0.f};
#pragma unroll
        for (int lev = 0; lev < 2; ++lev) {
          if (lev < a.nlev) {
            const int pitch = sm.pitch[lev][p];
            const float4 w = sm.w[lev][p];
            const float* rb = &sm.raw[lev][p * MMA_RAWP + (p & 1) + sm.base[lev][p]];
            const float* r0 = rb + yo0 * pitch + xo0;
            v0[lev] = w.x * r0[0] + w.y * r0[1] + w.z * r0[pitch] + w.w * r0[pitch + 1];
            if (tt1 < 49) {
              const float* r1 = rb + yo1 * pitch + xo1;
              v1[lev] = w.x * r1[0] + w.y * r1[1] + w.z * r1[pitch] + w.w * r1[pitch + 1];
            }
          }
        }
        stage[tt0 * 9 + p] = __floats2half2_rn(v0[0], v0[1]);
        if (tt1 < 49) stage[tt1 * 9 + p] = __floats2half2_rn(v1[0], v1[1]);
      }
      __syncwarp();
      if constexpr (PAIR_OUT) {
        __half* orow = out + (int64_t)(b * a.M + m) * a.out_row;
        if (psel >= 0) {                                       // one pixel: its 49 pairs, nine apart
          for (int tt = lane; tt < O * O; tt += 32) reinterpret_cast<__half2*>(orow)[tt * 9 + psel] = stage[tt * 9 + psel];
        } else if ((a.out_row & 7) == 0) {                            // 16-byte aligned rows (e.g. padded to 896)
          const uint4* s4 = reinterpret_cast<const uint4*>(stage);
          for (int i = lane; i < (NOUT * 4) / 16; i += 32) reinterpret_cast<uint4*>(orow)[i] = s4[i];
          if (lane == 0) reinterpret_cast<__half2*>(orow)[NOUT - 1] = stage[NOUT - 1];      // 441 = 4*110 + 1
        } else {
          for (int q = lane; q < NOUT; q += 32) reinterpret_cast<__half2*>(orow)[q] = stage[q];
        }
      } else {
        const __half* sh = reinterpret_cast<const __half*>(stage);
        for (int lev = 0; lev < a.nlev; ++lev)
          for (int q = lane; q < NOUT; q += 32)
            out[(int64_t)(b * a.M + m) * a.out_row + (int64_t)q * a.out_stride + a.out_offset[lev]] = sh[2 * q + lev];
      }
      __syncwarp();
    }
  }
}

// ==========================================================================================
// backward (training): fused bilinear-transpose + both feature gradients
// ==========================================================================================
// Replaces correlation_kernel.cu:252-269 (four zero-padded [E,8,8,3,3] temporaries) and the
// kernel at :139-190 (2*C global atomics per tap, 576 taps per edge).  One CTA per edge, one
// thread per channel: the thread walks the taps of every patch pixel once, accumulating the
// patch-feature gradient in registers and the window gradient in its own shared-memory column
// (no shared atomics), then issues one global atomic per touched (pixel, channel).
struct CorrBwdArgs {
  const void* fmap1; const void* fmap2;
  int64_t s1[5], s2[5], g1s[5], g2s[5];
  const float* coords; const int64_t* ii; const int64_t* jj;
  const void* grad;      // [B,M,O(x),O(y),P,P] contiguous
  void* g1; void* g2;
  int B, M, C, P, R, H2, W2;
};

template <typename T> __device__ __forceinline__ void atomic_add_any(T* p, T v) { atomicAdd(p, v); }

template <typename T, typename G, int P>
__global__ void __launch_bounds__(GEN_THREADS)
corr_bwd_generic(const CorrBwdArgs a, int Cpad) {
  using A = typename acc_of<T>::type;
  constexpr int PP = P * P;
  const int R = a.R, D = 2 * R + 2, DD = D * D, BOX = D + 2, O = 2 * R + 1;
  const int C = a.C;
  const int pitch = Cpad + row_pad<T>();

  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* win = reinterpret_cast<T*>(smem_raw);                              // [BOX*BOX][pitch]
  A* dwin = reinterpret_cast<A*>(win + (size_t)BOX * BOX * pitch);      // [BOX*BOX][Cpad]
  A* pat = dwin + (size_t)BOX * BOX * Cpad;                             // [PP][Cpad]
  A* graw = pat + PP * Cpad;                                            // [PP][DD]
  int* meta_i = reinterpret_cast<int*>(graw + PP * DD);
  float* meta_f = reinterpret_cast<float*>(meta_i + 2 * PP + 8);

  const int tid = threadIdx.x;
  const T* f1 = reinterpret_cast<const T*>(a.fmap1);
  const G* grad = reinterpret_cast<const G*>(a.grad);
  T* g1 = reinterpret_cast<T*>(a.g1);
  T* g2 = reinterpret_cast<T*>(a.g2);
  const int64_t nitems = (int64_t)a.B * a.M;

  for (int64_t item = blockIdx.x; item < nitems; item += gridDim.x) {
    const int b = (int)(item / a.M), m = (int)(item % a.M);
    const int64_t ix = a.ii[m], jx = a.jj[m];
    const T* f2 = reinterpret_cast<const T*>(a.fmap2) + b * a.s2[0] + jx * a.s2[1];
    const int64_t sc = a.s2[2], sy = a.s2[3], sx = a.s2[4];

    __syncthreads();
    for (int idx = tid; idx < PP * Cpad; idx += GEN_THREADS) {
      int p, c;
      if (a.s1[2] == 1) { c = idx % Cpad; p = idx / Cpad; } else { p = idx % PP; c = idx / PP; }
      A v = (A)0;
      if (c < C) v = to_acc<A, T>(f1[b * a.s1[0] + ix * a.s1[1] + c * a.s1[2] + (p / P) * a.s1[3] + (p % P) * a.s1[4]]);
      pat[p * Cpad + c] = v;
    }
    if (tid < PP) {
      const float* cp = a.coords + ((int64_t)(b * a.M + m) * 2) * PP;
      const float x = cp[tid], y = cp[PP + tid];
      meta_i[tid] = safe_floor_int(x) - R;
      meta_i[PP + tid] = safe_floor_int(y) - R;
      meta_f[tid] = x - floorf(x);
      meta_f[PP + tid] = y - floorf(y);
    }
    __syncthreads();
    if (tid == 0) {
      int x0 = meta_i[0], x1 = meta_i[0], y0 = meta_i[PP], y1 = meta_i[PP];
      for (int p = 1; p < PP; ++p) {
        x0 = min(x0, meta_i[p]); x1 = max(x1, meta_i[p]);
        y0 = min(y0, meta_i[PP + p]); y1 = max(y1, meta_i[PP + p]);
      }
      const bool uni = (x1 - x0 + D <= BOX) && (y1 - y0 + D <= BOX);
      meta_i[2 * PP + 0] = uni ? 1 : 0;
      meta_i[2 * PP + 1] = x0; meta_i[2 * PP + 2] = y0;
      meta_i[2 * PP + 3] = x1 - x0 + D; meta_i[2 * PP + 4] = y1 - y0 + D;
    }
    // ---- bilinear transpose: gradient of every raw tap (correlation_kernel.cu:252-269)
    {
      const G* gp = grad + (int64_t)(b * a.M + m) * O * O * PP;
      for (int q = tid; q < PP * DD; q += GEN_THREADS) {
        const int p = q / DD, ty = (q % DD) / D, tx = q % D;
        const A dx = (A)meta_f[p], dy = (A)meta_f[PP + p];
        A g = (A)0;
        // output (yo, xo) lives at gp[(xo*O + yo)*PP + p]
        if (ty < O && tx < O) g += ((A)1 - dx) * ((A)1 - dy) * to_acc<A, G>(gp[(tx * O + ty) * PP + p]);
        if (ty < O && tx >= 1) g += dx * ((A)1 - dy) * to_acc<A, G>(gp[((tx - 1) * O + ty) * PP + p]);
        if (ty >= 1 && tx < O) g += ((A)1 - dx) * dy * to_acc<A, G>(gp[(tx * O + ty - 1) * PP + p]);
        if (ty >= 1 && tx >= 1) g += dx * dy * to_acc<A, G>(gp[((tx - 1) * O + ty - 1) * PP + p]);
        // the reference casts the tap gradient to the feature dtype before use (:180)
        graw[q] = to_acc<A, T>(from_acc<T, A>(g));
      }
    }
    __syncthreads();
    const bool uni = meta_i[2 * PP + 0] != 0;
    const int npass = uni ? 1 : PP;

    A dP[PP];
#pragma unroll
    for (int p = 0; p < PP; ++p) dP[p] = (A)0;

    for (int pass = 0; pass < npass; ++pass) {
      const int bx0 = uni ? meta_i[2 * PP + 1] : meta_i[pass];
      const int by0 = uni ? meta_i[2 * PP + 2] : meta_i[PP + pass];
      const int bw = uni ? meta_i[2 * PP + 3] : D;
      const int bh = uni ? meta_i[2 * PP + 4] : D;
      const int rows = bw * bh;
      if (pass > 0) __syncthreads();
      for (int idx = tid; idx < rows * Cpad; idx += GEN_THREADS) {
        int r, c;
        if (sc == 1) { c = idx % Cpad; r = idx / Cpad; } else { r = idx % rows; c = idx / rows; }
        const int y = by0 + r / bw, x = bx0 + r % bw;
        T v = from_acc<T, A>((A)0);
        if (c < C && y >= 0 && y < a.H2 && x >= 0 && x < a.W2) v = f2[c * sc + (int64_t)y * sy + (int64_t)x * sx];
        win[r * pitch + c] = v;
        dwin[r * Cpad + c] = (A)0;
      }
      __syncthreads();
      for (int c = tid; c < Cpad; c += GEN_THREADS) {
#pragma unroll
        for (int p = 0; p < PP; ++p) {
          if (!uni && p != pass) continue;
          const A pc = pat[p * Cpad + c];
          const int r0 = (meta_i[PP + p] - by0) * bw + (meta_i[p] - bx0);
          A acc = (A)0;
          for (int ty = 0; ty < D; ++ty) {
            for (int tx = 0; tx < D; ++tx) {
              const A g = graw[p * DD + ty * D + tx];
              const int r = r0 + ty * bw + tx;
              acc += g * to_acc<A, T>(win[r * pitch + c]);
              dwin[r * Cpad + c] += g * pc;
            }
          }
          dP[p] += acc;
        }
        if (c < C) {
          for (int r = 0; r < rows; ++r) {
            const int y = by0 + r / bw, x = bx0 + r % bw;
            if (y >= 0 && y < a.H2 && x >= 0 && x < a.W2)
              atomic_add_any(&g2[b * a.g2s[0] + jx * a.g2s[1] + c * a.g2s[2] + (int64_t)y * a.g2s[3] + (int64_t)x * a.g2s[4]],
                             from_acc<T, A>(dwin[r * Cpad + c]));
          }
        }
      }
    }
    // one thread owns one channel when C <= GEN_THREADS; otherwise only the last strip's dP is
    // live, so wide feature maps are handled strip by strip below
    if (Cpad <= GEN_THREADS) {
      const int c = tid;
      if (c < C) {
#pragma unroll
        for (int p = 0; p < PP; ++p)
          atomic_add_any(&g1[b * a.g1s[0] + ix * a.g1s[1] + c * a.g1s[2] + (p / P) * a.g1s[3] + (p % P) * a.g1s[4]],
                         from_acc<T, A>(dP[p]));
      }
    }
  }
}

template <typename T, typename G>
static int launch_bwd(const CorrBwdArgs& a, cudaStream_t st) {
  using A = typename acc_of<T>::type;
  const int Cpad = (a.C + 3) & ~3;
  if (Cpad > GEN_THREADS) {
    set_error("corr_backward: C=%d > %d channels not supported", a.C, GEN_THREADS);
    return DPVO_ERR_UNSUPPORTED;
  }
  const int D = 2 * a.R + 2, BOX = D + 2, PP = a.P * a.P;
  size_t smem = (size_t)BOX * BOX * (Cpad + row_pad<T>()) * sizeof(T) + (size_t)BOX * BOX * Cpad * sizeof(A) +
                (size_t)PP * Cpad * sizeof(A) + (size_t)PP * D * D * sizeof(A) + (2 * PP + 8) * sizeof(int) +
                2 * PP * sizeof(float) + 16;
  smem = (smem + 15) & ~(size_t)15;
  if (smem > 227 * 1024) {
    set_error("corr_backward: needs %zu B shared memory per CTA (> 227 KB)", smem);
    return DPVO_ERR_UNSUPPORTED;
  }
  const int64_t nitems = (int64_t)a.B * a.M;
  if (nitems == 0) return DPVO_OK;
  auto go = [&](auto kern) -> int {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return check_cuda(e, "corr_backward: cudaFuncSetAttribute");
    int per_sm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, GEN_THREADS, smem);
    if (per_sm < 1) per_sm = 1;
    const int64_t grid = std::min<int64_t>(nitems, (int64_t)sm_count() * per_sm * 4);
    kern<<<(unsigned)grid, GEN_THREADS, smem, st>>>(a, Cpad);
    DPVO_LAUNCH_CHECK("corr_bwd_generic");
    return DPVO_OK;
  };
  switch (a.P) {
    case 1: return go(corr_bwd_generic<T, G, 1>);
    case 2: return go(corr_bwd_generic<T, G, 2>);
    case 3: return go(corr_bwd_generic<T, G, 3>);
  }
  set_error("corr_backward: patch size P=%d not supported (1..3)", a.P);
  return DPVO_ERR_UNSUPPORTED;
}

// ==========================================================================================
// host dispatch
// ==========================================================================================
template <typename T>
static int launch_generic(const CorrArgs& a, cudaStream_t st) {
  using A = typename acc_of<T>::type;
  const int Cpad = (a.C + 3) & ~3;
  const int D = 2 * a.R + 2, BOX = D + 2, PP = a.P * a.P;
  size_t smem = (size_t)BOX * BOX * (Cpad + row_pad<T>()) * sizeof(T) + (size_t)PP * Cpad * sizeof(A) +
                (size_t)PP * D * D * sizeof(A) + (2 * PP + 8) * sizeof(int) + 2 * PP * sizeof(float) + 16;
  smem = (smem + 15) & ~(size_t)15;
  if (smem > 227 * 1024) {
    set_error("corr_forward: C=%d radius=%d needs %zu B of shared memory per CTA (> 227 KB)", a.C, a.R, smem);
    return DPVO_ERR_UNSUPPORTED;
  }
  const int64_t nitems = (int64_t)a.B * a.M;
  if (nitems == 0) return DPVO_OK;
  auto go = [&](auto kern) -> int {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return check_cuda(e, "corr_forward: cudaFuncSetAttribute");
    int per_sm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, GEN_THREADS, smem);
    if (per_sm < 1) per_sm = 1;
    const int64_t grid = std::min<int64_t>(nitems, (int64_t)sm_count() * per_sm * 4);
    kern<<<(unsigned)grid, GEN_THREADS, smem, st>>>(a, Cpad);
    DPVO_LAUNCH_CHECK("corr_fwd_generic");
    return DPVO_OK;
  };
  switch (a.P) {
    case 1: return go(corr_fwd_generic<T, 1>);
    case 2: return go(corr_fwd_generic<T, 2>);
    case 3: return go(corr_fwd_generic<T, 3>);
  }
  set_error("corr_forward: patch size P=%d not supported (1..3)", a.P);
  return DPVO_ERR_UNSUPPORTED;
}

static bool mma_eligible(const CorrArgs& a, int dtype) {
  if (dtype != DPVO_F16 || a.C != 128 || a.P != 3 || a.R != 3) return false;
  if (((uintptr_t)a.fmap1 & 15) || ((uintptr_t)a.out & 3)) return false;
  for (int l = 0; l < a.nlev; ++l) {
    if ((uintptr_t)a.fmap2[l] & 15) return false;
    if (a.s2[l][2] != 1) return false;
    if ((a.s2[l][0] % 8) || (a.s2[l][1] % 8) || (a.s2[l][3] % 8) || (a.s2[l][4] % 8)) return false;
  }
  if ((a.s1[0] % 8) || (a.s1[1] % 8)) return false;   // 16-byte aligned patch records
  return true;
}

static int launch_mma(const CorrArgs& a, bool pair_out, cudaStream_t st) {
  const int64_t nitems = (int64_t)a.B * a.M;
  if (nitems == 0) return DPVO_OK;
  const int64_t need = (nitems + MMA_WARPS - 1) / MMA_WARPS;
  // list mode: the length lives on the device; one CTA per SM drains it
  const int64_t grid = std::min<int64_t>(need, (int64_t)sm_count() * (a.list ? 1 : 2));
  const size_t smem = sizeof(MmaWarpSmem) * MMA_WARPS;
  {   // per-device function attribute: set on every call
    cudaError_t e = pair_out ? cudaFuncSetAttribute(corr_fwd_mma<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                             : cudaFuncSetAttribute(corr_fwd_mma<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return check_cuda(e, "corr_forward: cudaFuncSetAttribute");
  }
  if (pair_out) corr_fwd_mma<true><<<(unsigned)grid, MMA_WARPS * 32, smem, st>>>(a);
  else corr_fwd_mma<false><<<(unsigned)grid, MMA_WARPS * 32, smem, st>>>(a);
  DPVO_LAUNCH_CHECK("corr_fwd_mma");
  return DPVO_OK;
}

// corr_tc.cu
int corr_tc_forward(const void* fmap1, const int64_t* s1, int S1, const void* l0, const int64_t* s20, int H0, int W0,
                    const void* l1, const int64_t* s21, int H1, int W1, int S2, float div1, const float* coords,
                    const int64_t* ii, const int64_t* jj, void* out, int64_t out_row, int M, void* scratch, cudaStream_t st);

int corr_launch_fallback_list(const void* fmap1, const int64_t* s1, const void* l0, const int64_t* s20, int H0, int W0,
                              const void* l1, const int64_t* s21, int H1, int W1, float div1, const float* coords,
                              const int64_t* ii, const int64_t* jj, void* out, int64_t out_row, int M,
                              const int* list, const int* count, cudaStream_t st) {
  CorrArgs a;
  memset(&a, 0, sizeof(a));
  a.fmap1 = fmap1; a.fmap2[0] = l0; a.fmap2[1] = l1;
  for (int i = 0; i < 5; ++i) { a.s1[i] = s1[i]; a.s2[0][i] = s20[i]; a.s2[1][i] = s21[i]; }
  a.H2[0] = H0; a.W2[0] = W0; a.H2[1] = H1; a.W2[1] = W1; a.div[0] = 1.0f; a.div[1] = div1;
  a.coords = coords; a.ii = ii; a.jj = jj; a.out = out; a.out_stride = 2;
  a.out_offset[0] = 0; a.out_offset[1] = 1; a.nlev = 2; a.B = 1; a.M = M; a.C = 128; a.P = 3; a.R = 3;
  a.out_row = out_row; a.list = list; a.list_count = count;
  return launch_mma(a, true, st);
}

static int corr_dispatch(const CorrArgs& a, int dtype, bool pair_out, cudaStream_t st) {
  if (mma_eligible(a, dtype)) return launch_mma(a, pair_out, st);
  switch (dtype) {
    case DPVO_F16: return launch_generic<__half>(a, st);
    case DPVO_BF16: return launch_generic<__nv_bfloat16>(a, st);
    case DPVO_F32: return launch_generic<float>(a, st);
    case DPVO_F64: return launch_generic<double>(a, st);
  }
  set_error("corr_forward: unknown dtype %d", dtype);
  return DPVO_ERR_INVALID;
}

}  // namespace dpvo

using namespace dpvo;

extern "C" int dpvo_corr_forward(const void* fmap1, const int64_t* fmap1_strides,
                                 const void* fmap2, const int64_t* fmap2_strides,
                                 const float* coords, const int64_t* ii, const int64_t* jj,
                                 void* out, int64_t out_elem_stride,
                                 int dtype, int B, int M, int C, int P,
                                 int S1, int S2, int H2, int W2, int radius, void* stream) {
  DPVO_REQUIRE(B >= 0 && M >= 0 && C > 0 && P > 0 && radius >= 0 && H2 > 0 && W2 > 0 && out_elem_stride > 0,
               "corr_forward: bad sizes B=%d M=%d C=%d P=%d R=%d H2=%d W2=%d", B, M, C, P, radius, H2, W2);
  if ((int64_t)B * M == 0) return DPVO_OK;
  DPVO_REQUIRE(fmap1 && fmap2 && coords && ii && jj && out && fmap1_strides && fmap2_strides,
               "corr_forward: null pointer");
  (void)S1; (void)S2;
  CorrArgs a;
  memset(&a, 0, sizeof(a));
  a.fmap1 = fmap1; a.fmap2[0] = fmap2;
  for (int i = 0; i < 5; ++i) { a.s1[i] = fmap1_strides[i]; a.s2[0][i] = fmap2_strides[i]; }
  a.H2[0] = H2; a.W2[0] = W2; a.div[0] = 1.0f;
  a.coords = coords; a.ii = ii; a.jj = jj; a.out = out; a.out_stride = out_elem_stride;
  a.out_offset[0] = 0; a.nlev = 1; a.B = B; a.M = M; a.C = C; a.P = P; a.R = radius;
  a.out_row = (int64_t)(2 * radius + 1) * (2 * radius + 1) * P * P * out_elem_stride;
  return corr_dispatch(a, dtype, false, (cudaStream_t)stream);
}

extern "C" int dpvo_corr_forward_pyramid2(const void* fmap1, const int64_t* fmap1_strides,
                                          const void* fmap2_l0, const int64_t* l0_strides, int H0, int W0,
                                          const void* fmap2_l1, const int64_t* l1_strides, int H1, int W1,
                                          float lvl1_div,
                                          const float* coords, const int64_t* ii, const int64_t* jj,
                                          void* out, int64_t out_row_stride,
                                          int dtype, int B, int M, int C, int P,
                                          int S1, int S2, int radius,
                                          void* workspace, int64_t workspace_bytes, void* stream) {
  DPVO_REQUIRE(B >= 0 && M >= 0 && C > 0 && P > 0 && radius >= 0 && H0 > 0 && W0 > 0 && H1 > 0 && W1 > 0,
               "corr_forward_pyramid2: bad sizes");
  DPVO_REQUIRE(lvl1_div > 0.f, "corr_forward_pyramid2: lvl1_div must be > 0");
  DPVO_REQUIRE(out_row_stride >= 2 * (int64_t)(2 * radius + 1) * (2 * radius + 1) * P * P && out_row_stride % 2 == 0,
               "corr_forward_pyramid2: bad out_row_stride");
  if ((int64_t)B * M == 0) return DPVO_OK;
  DPVO_REQUIRE(fmap1 && fmap2_l0 && fmap2_l1 && coords && ii && jj && out && fmap1_strides && l0_strides && l1_strides,
               "corr_forward_pyramid2: null pointer");
  CorrArgs a;
  memset(&a, 0, sizeof(a));
  a.fmap1 = fmap1; a.fmap2[0] = fmap2_l0; a.fmap2[1] = fmap2_l1;
  for (int i = 0; i < 5; ++i) { a.s1[i] = fmap1_strides[i]; a.s2[0][i] = l0_strides[i]; a.s2[1][i] = l1_strides[i]; }
  a.H2[0] = H0; a.W2[0] = W0; a.H2[1] = H1; a.W2[1] = W1; a.div[0] = 1.0f; a.div[1] = lvl1_div;
  a.coords = coords; a.ii = ii; a.jj = jj; a.out = out; a.out_stride = 2;
  a.out_offset[0] = 0; a.out_offset[1] = 1; a.nlev = 2; a.B = B; a.M = M; a.C = C; a.P = P; a.R = radius;
  a.out_row = out_row_stride;
  // wgmma + TMA path: fp16 channels-last rings, batch 1, caller-provided scratch for the edge list
  if (workspace && workspace_bytes >= dpvo_corr_pyramid2_workspace_bytes(M) && B == 1 && S1 > 0 && S2 > 0 &&
      mma_eligible(a, dtype)) {
    const int rc = corr_tc_forward(fmap1, a.s1, S1, fmap2_l0, a.s2[0], H0, W0, fmap2_l1, a.s2[1], H1, W1, S2, lvl1_div, coords, ii, jj,
                                   out, out_row_stride, M, workspace, (cudaStream_t)stream);
    if (rc != DPVO_ERR_UNSUPPORTED) return rc;
  }
  return corr_dispatch(a, dtype, true, (cudaStream_t)stream);
}

extern "C" int64_t dpvo_corr_pyramid2_workspace_bytes(int64_t M) { return (M + 1) * (int64_t)sizeof(int) + 16; }

extern "C" int dpvo_corr_backward(const void* fmap1, const int64_t* fmap1_strides,
                                  const void* fmap2, const int64_t* fmap2_strides,
                                  const float* coords, const int64_t* ii, const int64_t* jj,
                                  const void* grad, int grad_dtype,
                                  void* fmap1_grad, const int64_t* fmap1_grad_strides,
                                  void* fmap2_grad, const int64_t* fmap2_grad_strides,
                                  int dtype, int B, int M, int C, int P,
                                  int S1, int S2, int H2, int W2, int radius, void* stream) {
  DPVO_REQUIRE(B >= 0 && M >= 0 && C > 0 && P > 0 && radius >= 0 && H2 > 0 && W2 > 0, "corr_backward: bad sizes");
  if ((int64_t)B * M == 0) return DPVO_OK;
  DPVO_REQUIRE(fmap1 && fmap2 && coords && ii && jj && grad && fmap1_grad && fmap2_grad && fmap1_strides &&
               fmap2_strides && fmap1_grad_strides && fmap2_grad_strides, "corr_backward: null pointer");
  (void)S1; (void)S2;
  CorrBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.fmap1 = fmap1; a.fmap2 = fmap2; a.coords = coords; a.ii = ii; a.jj = jj; a.grad = grad;
  a.g1 = fmap1_grad; a.g2 = fmap2_grad;
  for (int i = 0; i < 5; ++i) {
    a.s1[i] = fmap1_strides[i]; a.s2[i] = fmap2_strides[i];
    a.g1s[i] = fmap1_grad_strides[i]; a.g2s[i] = fmap2_grad_strides[i];
  }
  a.B = B; a.M = M; a.C = C; a.P = P; a.R = radius; a.H2 = H2; a.W2 = W2;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DPVO_F32 && grad_dtype == DPVO_F32) return launch_bwd<float, float>(a, st);
  if (dtype == DPVO_F64 && grad_dtype == DPVO_F64) return launch_bwd<double, double>(a, st);
  if (dtype == DPVO_F64 && grad_dtype == DPVO_F32) return launch_bwd<double, float>(a, st);
  if (dtype == DPVO_F16 && grad_dtype == DPVO_F32) return launch_bwd<__half, float>(a, st);
  if (dtype == DPVO_F16 && grad_dtype == DPVO_F16) return launch_bwd<__half, __half>(a, st);
  if (dtype == DPVO_BF16 && grad_dtype == DPVO_F32) return launch_bwd<__nv_bfloat16, float>(a, st);
  if (dtype == DPVO_BF16 && grad_dtype == DPVO_BF16) return launch_bwd<__nv_bfloat16, __nv_bfloat16>(a, st);
  set_error("corr_backward: unsupported dtype pair (features %d, grad %d)", dtype, grad_dtype);
  return DPVO_ERR_UNSUPPORTED;
}
