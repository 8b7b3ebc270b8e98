// Frame encoders (dpvo/extractor.py:200-264 BasicEncoder4, dpvo/net.py:95-157 Patchifier) for inference:
// a uint8 camera image in, the new frame's ring-buffer slots (fmap1, fmap2, gmap, imap, patches) out.
//
// Every convolution is an implicit GEMM on the tensor cores (mma.sync m16n8k16, fp16 operands, fp32 accumulation) over
// an NHWC fp16 activation.  A CTA (4 warps) owns an 8 x 16 tile of output pixels and a slice of <= 64 output channels:
//   - the input halo of the tile is staged in shared memory channel-chunk-major, [8-channel chunk][halo y][halo x], 16 B
//     per pixel and chunk.  The A fragment of tap (ky, kx) is then 16 output pixels of one row, read by ldmatrix from
//     16-byte rows at halo (y * s + ky, x * s + kx): no im2col copy, and a stride-2 tap is the same address rule with
//     s = 2.  For stride 1 the 8 rows of an ldmatrix phase are 128 contiguous bytes (no bank conflict), for stride 2
//     every second 16-byte row (two-way).
//   - the weights of the slice are staged as [tap][chunk][cout][8], which is how FrameEncoder.pack() stores them, so
//     the B fragments are conflict-free ldmatrix reads too.
//   - the 7x7/2 stem (3 input channels) builds an explicit im2col tile [20 chunks][128 pixels][8] (K = 147 -> 160) from
//     the normalised image halo.
// The prologue applies the pending transform of the producing layer while it stages the halo: instance norm + ReLU
// relu((x - mean) * rstd), ReLU alone (inet), or the residual join relu(skip' + that) where skip' is the block input or
// the normalised 1x1/2 projection.  Pixels outside the image are staged as 0 after the transform, as nn.Conv2d pads
// its (already transformed) input.  A join can write the joined block output of the pixels the CTA owns, so the next
// block reads it as its skip.
// The epilogue adds the bias, scales (1/4 on the output convolutions, net.py:112), rounds to fp16 and stores.  A
// normalised layer also leaves per-CTA per-channel (count, mean, M2) of the fp16-rounded outputs in a fixed slot; the
// last CTA to finish (integer ticket) merges the slots in tile order with Chan's formula and writes (mean, rstd) for
// the next launch.  No float atomics: two launches give identical bits.
// A launch covers B images x nenc encoders, blockIdx.z = nenc * image + encoder.  Image b owns block b of the workspace
// (its activations, statistics partials, (mean, rstd) slots and tickets), so each (image, encoder) z-slice reads,
// writes and merges exactly what a single-image launch does, and its outputs are bit-identical to encoding it alone.
#include <type_traits>

#include "common.cuh"
#include "tc.cuh"

namespace dpvo {

constexpr int EC_TH = 8, EC_TW = 16, EC_PIX = EC_TH * EC_TW;   // output tile (one m16 fragment = one tile row)
constexpr int EC_THREADS = 128;                                // 4 warps, warp w: tile rows 2w, 2w + 1
constexpr int EC_STEM_K = 147, EC_STEM_KC = 20;                // 3 x 7 x 7 taps, padded to 20 chunks of 8
constexpr int EC_NLAYERS = 11;
constexpr int EC_BIAS_STRIDE = 384;
constexpr float EC_EPS = 1e-5f;
constexpr int EC_MAX_IMAGES = 64;                              // images per launch: gridDim.z <= 128, rows fit the params

// Pointers are image 0's.  Image b's are y + row[b] y_sr and pool + row[b] pool_sr (elements), the stem's x + b x_sb
// (elements), and every other pointer + b ws_sb (bytes: its block of the workspace).
struct EncSide {
  const void* x;                   // stem: uint8 [3, H, W] (strides xs); otherwise fp16 NHWC [Hin, Win, CIN] dense
  int64_t xs_c, xs_y, xs_x;
  const float* x_stats;            // [2][CIN] (mean, rstd) of x, or null: no normalisation
  int x_relu;
  const __half* skip;              // residual join: relu(skip' + x'), skip fp16 NHWC [Hin, Win, CIN] dense
  const float* skip_stats;
  int skip_relu;
  __half* joined;                  // optional: the joined input of the pixels this CTA owns
  const __half* w;                 // [taps][CIN / 8][COUT][8]
  const float* bias;               // [COUT]
  __half* y;                       // [Hout, Wout, COUT] with pixel strides y_sy, y_sx, channel stride 1
  int64_t y_sy, y_sx, y_sr;
  __half* pool;                    // optional 4x4 average of y (fmap2): strides pool_sy, pool_sx
  int64_t pool_sy, pool_sx, pool_sr;
  float* part;                     // [tiles][3][COUT] per-CTA (count, mean, M2), with stats
  float* stats;                    // optional [2][COUT] (mean, rstd) of y
  int* ticket;
  float scale;
};

struct EncConvParams {
  EncSide e[2];
  int Hin, Win, Hout, Wout, tiles_x;
  int nenc;                        // encoders per image
  int64_t x_sb, ws_sb;
  int row[EC_MAX_IMAGES];          // destination row of each image's y / pool
};

// blockIdx.z read where it is used: volatile, so the image index is not held in registers across the MMA loop
__device__ __forceinline__ int cta_z() {
  int z;
  asm volatile("mov.u32 %0, %%ctaid.z;" : "=r"(z));
  return z;
}

// image b's copy of a workspace pointer (null stays null).  Byte-pointer arithmetic, not an integer round trip, so the
// compiler keeps the kernel parameter's global address space (LDG / STG rather than generic loads and stores).
template <class T>
__device__ __forceinline__ T* img_ptr(T* q, int64_t bytes) {
  using Byte = typename std::conditional<std::is_const<T>::value, const char, char>::type;
  return q == nullptr ? q : reinterpret_cast<T*>(reinterpret_cast<Byte*>(q) + bytes);
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

// the normalised image value of dpvo.py:389 as the fp16 operand of the stem
__device__ __forceinline__ __half image_value(uint8_t u) {
  return __float2half_rn(__fsub_rn(__fmul_rn(2.0f, __fdiv_rn((float)u, 255.0f)), 0.5f));
}

// Chan's merge of (n, mean, M2) partials
__device__ __forceinline__ void chan_merge(float& n, float& mean, float& m2, float nb, float mb, float m2b) {
  if (nb == 0.f) return;
  const float nn = n + nb, d = mb - mean;
  mean = mean + d * (nb / nn);
  m2 = m2 + m2b + d * d * (n * (nb / nn));
  n = nn;
}

template <int KS, int S, int CIN, int NT, bool STEM>
struct EncCfg {
  static constexpr int PAD = KS / 2;
  static constexpr int HH = STEM ? (EC_TH - 1) * 2 + 7 : (EC_TH - 1) * S + KS;
  static constexpr int HWD = STEM ? (EC_TW - 1) * 2 + 7 : (EC_TW - 1) * S + KS;
  static constexpr int HALO = HH * HWD;
  static constexpr int KC = STEM ? EC_STEM_KC : CIN / 8;
  static constexpr int TAPS = STEM ? 1 : KS * KS;
  static constexpr int A_BYTES = STEM ? EC_STEM_KC * EC_PIX * 16 : KC * HALO * 16;
  static constexpr int W_BYTES = TAPS * KC * NT * 16;
  static constexpr int IMG_BYTES = STEM ? ((3 * HH * HWD * 2 + 15) / 16) * 16 : 0;
  static constexpr int OST = NT + 8;                                      // staged output row (halves), pooling
  static constexpr int O_BYTES = EC_PIX * OST * 2;
  static constexpr int A_REGION = A_BYTES > O_BYTES ? A_BYTES : O_BYTES;
  static constexpr int SMEM = A_REGION + W_BYTES + IMG_BYTES;
};

template <int KS, int S, int CIN, int NT, bool STEM>
__global__ void __launch_bounds__(EC_THREADS, 2)
enc_conv_kernel(const __grid_constant__ EncConvParams p, const int cout) {
  using C = EncCfg<KS, S, CIN, NT, STEM>;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* As = smem;
  uint8_t* Ws = smem + C::A_REGION;
  __half* img = reinterpret_cast<__half*>(smem + C::A_REGION + C::W_BYTES);
  __shared__ float s_xm[64], s_xr[64], s_sm[64], s_sr[64];
  __shared__ float s_red[4][NT], s_mean[NT];
  __shared__ float s_mrg[EC_THREADS][3];
  __shared__ int s_last;

  const EncSide& E = p.e[blockIdx.z % p.nenc];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tile = blockIdx.x, n0 = blockIdx.y * NT;
  const int oy0 = (tile / p.tiles_x) * EC_TH, ox0 = (tile % p.tiles_x) * EC_TW;

  // ---- weights of the channel slice
  for (int i = tid; i < C::TAPS * C::KC * NT; i += EC_THREADS) {
    const int tk = i / NT, n = i % NT;
    reinterpret_cast<uint4*>(Ws)[i] = reinterpret_cast<const uint4*>(E.w)[(int64_t)tk * cout + n0 + n];
  }

  // ---- input halo
  if constexpr (STEM) {
    const uint8_t* im = static_cast<const uint8_t*>(E.x) + (cta_z() / p.nenc) * p.x_sb;
    const int iy0 = oy0 * 2 - 3, ix0 = ox0 * 2 - 3;
    for (int i = tid; i < 3 * C::HALO; i += EC_THREADS) {
      const int c = i / C::HALO, hp = i % C::HALO, iy = iy0 + hp / C::HWD, ix = ix0 + hp % C::HWD;
      __half v = __float2half_rn(0.f);
      if (iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win) v = image_value(im[c * E.xs_c + iy * E.xs_y + ix * E.xs_x]);
      img[i] = v;
    }
    __syncthreads();
    // im2col: thread = tile pixel, k = (c * 7 + ky) * 7 + kx as in the [cout][3][7][7] weight
    const int r = tid / EC_TW, q = tid % EC_TW;
#pragma unroll
    for (int kc = 0; kc < EC_STEM_KC; ++kc) {
      __align__(16) __half v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = kc * 8 + j;
        if (k < EC_STEM_K) {
          const int c = k / 49, ky = (k % 49) / 7, kx = k % 7;
          v[j] = img[c * C::HALO + (r * 2 + ky) * C::HWD + q * 2 + kx];
        } else {
          v[j] = __float2half_rn(0.f);
        }
      }
      reinterpret_cast<uint4*>(As)[kc * EC_PIX + tid] = *reinterpret_cast<uint4*>(v);
    }
  } else {
    const int64_t wo = (cta_z() / p.nenc) * p.ws_sb;
    const float* x_stats = img_ptr(E.x_stats, wo);
    const float* skip_stats = img_ptr(E.skip_stats, wo);
    if (tid < CIN) {
      s_xm[tid] = x_stats ? x_stats[tid] : 0.f;
      s_xr[tid] = x_stats ? x_stats[CIN + tid] : 1.f;
      s_sm[tid] = skip_stats ? skip_stats[tid] : 0.f;
      s_sr[tid] = skip_stats ? skip_stats[CIN + tid] : 1.f;
    }
    __syncthreads();
    const __half* X = img_ptr(static_cast<const __half*>(E.x), wo);
    const __half* skip = img_ptr(E.skip, wo);
    const bool norm_x = x_stats != nullptr, norm_s = skip_stats != nullptr, join = skip != nullptr;
    __half* joined = (E.joined != nullptr && blockIdx.y == 0) ? img_ptr(E.joined, wo) : nullptr;
    const int iy0 = oy0 * S - C::PAD, ix0 = ox0 * S - C::PAD;
    for (int i = tid; i < C::HALO * C::KC; i += EC_THREADS) {
      const int hp = i / C::KC, kc = i % C::KC, iy = iy0 + hp / C::HWD, ix = ix0 + hp % C::HWD;
      uint4 out = make_uint4(0, 0, 0, 0);
      if (iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win) {
        const int64_t off = ((int64_t)iy * p.Win + ix) * CIN + kc * 8;
        uint4 raw = *reinterpret_cast<const uint4*>(X + off);
        uint4 sraw = join ? *reinterpret_cast<const uint4*>(skip + off) : make_uint4(0, 0, 0, 0);
        const __half* xv = reinterpret_cast<const __half*>(&raw);
        const __half* sv = reinterpret_cast<const __half*>(&sraw);
        __align__(16) __half o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = kc * 8 + j;
          float f = __half2float(xv[j]);
          if (norm_x) f = __fmul_rn(__fsub_rn(f, s_xm[c]), s_xr[c]);
          if (E.x_relu) f = fmaxf(f, 0.f);
          if (join) {
            float s = __half2float(sv[j]);
            if (norm_s) s = __fmul_rn(__fsub_rn(s, s_sm[c]), s_sr[c]);
            if (E.skip_relu) s = fmaxf(s, 0.f);
            f = fmaxf(__fadd_rn(s, f), 0.f);
          }
          o[j] = __float2half_rn(f);
        }
        out = *reinterpret_cast<uint4*>(o);
        if (joined && iy >= oy0 * S && iy < (oy0 + EC_TH) * S && ix >= ox0 * S && ix < (ox0 + EC_TW) * S)
          *reinterpret_cast<uint4*>(joined + off) = out;
      }
      reinterpret_cast<uint4*>(As)[kc * C::HALO + hp] = out;
    }
  }
  __syncthreads();

  // ---- MMA: warp w computes tile rows 2w, 2w + 1 (one m16 fragment each) x NT channels
  constexpr int NB = NT / 8;
  float acc[2][NB][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[mt][nb][j] = 0.f;

  const uint32_t a_base = smem_u32(As), w_base = smem_u32(Ws);
  const int lr = lane & 15, lk = lane >> 4;                              // A: row of the fragment, chunk half
  const int bn = (lane & 7) + ((lane >> 4) << 3), bk = (lane >> 3) & 1;  // B: channel within 16, chunk half
#pragma unroll 1
  for (int tap = 0; tap < C::TAPS; ++tap) {
    const int ky = tap / KS, kx = tap % KS;
#pragma unroll
    for (int kc = 0; kc < C::KC; kc += 2) {
      uint32_t a[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int row = 2 * warp + mt;
        uint32_t addr;
        if constexpr (STEM) addr = a_base + ((kc + lk) * EC_PIX + row * EC_TW + lr) * 16;
        else addr = a_base + ((kc + lk) * C::HALO + (row * S + ky) * C::HWD + lr * S + kx) * 16;
        ldsm_x4(addr, a[mt][0], a[mt][1], a[mt][2], a[mt][3]);
      }
#pragma unroll
      for (int np = 0; np < NT / 16; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(w_base + ((tap * C::KC + kc + bk) * NT + np * 16 + bn) * 16, b0, b1, b2, b3);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma_m16n8k16(acc[mt][2 * np], a[mt][0], a[mt][1], a[mt][2], a[mt][3], b0, b1);
          mma_m16n8k16(acc[mt][2 * np + 1], a[mt][0], a[mt][1], a[mt][2], a[mt][3], b2, b3);
        }
      }
    }
  }

  // ---- epilogue: bias, scale, fp16, store
  const int g = lane >> 2, cq = 2 * (lane & 3);
  const int vh = min(EC_TH, p.Hout - oy0), vw = min(EC_TW, p.Wout - ox0);
  const bool want_stats = E.stats != nullptr, want_pool = E.pool != nullptr;
  const int image = cta_z() / p.nenc;
  const int64_t wo = image * p.ws_sb;
  __half* const Y = E.y + p.row[image] * E.y_sr;
  float sum[NB][2];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) sum[nb][0] = sum[nb][1] = 0.f;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
    const int row = 2 * warp + mt, oy = oy0 + row;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int col = g + 8 * hr, ox = ox0 + col;
      const bool valid = row < vh && col < vw;
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) {
        const int n = nb * 8 + cq;
        const float v0 = (acc[mt][nb][2 * hr] + E.bias[n0 + n]) * E.scale;
        const float v1 = (acc[mt][nb][2 * hr + 1] + E.bias[n0 + n + 1]) * E.scale;
        const __half2 h = __floats2half2_rn(v0, v1);
        const float2 f = __half22float2(h);
        acc[mt][nb][2 * hr] = f.x;                                         // keep the rounded value for the statistics
        acc[mt][nb][2 * hr + 1] = f.y;
        if (valid) {
          *reinterpret_cast<__half2*>(Y + oy * E.y_sy + ox * E.y_sx + n0 + n) = h;
          sum[nb][0] += f.x;
          sum[nb][1] += f.y;
        }
      }
    }
  }

  if (want_pool) {
    // F.avg_pool2d(y, 4, 4) of the written tile: 16 fp16 values summed in fp32, rows then columns, / 16
    __syncthreads();                                                       // every warp is done with the A tile
    __half* ost = reinterpret_cast<__half*>(As);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int hr = 0; hr < 2; ++hr)
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
          const int px = (2 * warp + mt) * EC_TW + g + 8 * hr;
          *reinterpret_cast<__half2*>(ost + px * C::OST + nb * 8 + cq) = __floats2half2_rn(acc[mt][nb][2 * hr], acc[mt][nb][2 * hr + 1]);
        }
    __syncthreads();
    const int ch = p.Hout / 4, cw = p.Wout / 4;
    __half* const pool = E.pool + p.row[image] * E.pool_sr;
    for (int i = tid; i < (EC_TH / 4) * (EC_TW / 4) * NT; i += EC_THREADS) {
      const int cell = i / NT, c = i % NT, cy = cell / (EC_TW / 4), cx = cell % (EC_TW / 4);
      const int gy = oy0 / 4 + cy, gx = ox0 / 4 + cx;
      if (gy < ch && gx < cw) {
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int q = 0; q < 4; ++q) s += __half2float(ost[((cy * 4 + r) * EC_TW + cx * 4 + q) * C::OST + c]);
        pool[gy * E.pool_sy + gx * E.pool_sx + n0 + c] = __float2half_rn(s / 16.f);
      }
    }
  }

  if (!want_stats) return;
  // ---- per-CTA statistics of the fp16 outputs: mean first, then M2 around it (two exact passes over registers)
  const float cnt = (float)(vh * vw);
#pragma unroll
  for (int nb = 0; nb < NB; ++nb)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      float s = sum[nb][j];
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      s += __shfl_xor_sync(0xffffffffu, s, 8);
      s += __shfl_xor_sync(0xffffffffu, s, 16);
      if (g == 0) s_red[warp][nb * 8 + cq + j] = s;
    }
  __syncthreads();
  if (tid < NT) s_mean[tid] = (((s_red[0][tid] + s_red[1][tid]) + s_red[2][tid]) + s_red[3][tid]) / cnt;
  __syncthreads();
#pragma unroll
  for (int nb = 0; nb < NB; ++nb)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float m = s_mean[nb * 8 + cq + j];
      float s = 0.f;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const bool valid = (2 * warp + mt) < vh && (g + 8 * hr) < vw;
          const float d = acc[mt][nb][2 * hr + j] - m;
          if (valid) s += d * d;
        }
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      s += __shfl_xor_sync(0xffffffffu, s, 8);
      s += __shfl_xor_sync(0xffffffffu, s, 16);
      if (g == 0) s_red[warp][nb * 8 + cq + j] = s;
    }
  __syncthreads();
  float* const parts = img_ptr(E.part, wo);
  int* const ticket = img_ptr(E.ticket, wo);
  if (tid < NT) {
    float* slot = parts + (int64_t)tile * 3 * cout;
    slot[n0 + tid] = cnt;
    slot[cout + n0 + tid] = s_mean[tid];
    slot[2 * cout + n0 + tid] = ((s_red[0][tid] + s_red[1][tid]) + s_red[2][tid]) + s_red[3][tid];
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(ticket, 1) == (int)(gridDim.x * gridDim.y) - 1;   // this (image, encoder)
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // last CTA: G threads per channel merge contiguous tile ranges in order, then the G results in order
  const int tiles = gridDim.x, G = EC_THREADS / cout;                   // cout <= 64 for normalised layers
  const int c = tid / G, part = tid % G;
  if (c < cout) {
    const int t0 = tiles * part / G, t1 = tiles * (part + 1) / G;
    float n = 0.f, mean = 0.f, m2 = 0.f;
    for (int t = t0; t < t1; ++t) {
      const float* slot = parts + (int64_t)t * 3 * cout;
      chan_merge(n, mean, m2, __ldcg(slot + c), __ldcg(slot + cout + c), __ldcg(slot + 2 * cout + c));
    }
    s_mrg[tid][0] = n; s_mrg[tid][1] = mean; s_mrg[tid][2] = m2;
  }
  __syncthreads();
  if (c < cout && part == 0) {
    float n = 0.f, mean = 0.f, m2 = 0.f;
    for (int q = 0; q < G; ++q) chan_merge(n, mean, m2, s_mrg[tid + q][0], s_mrg[tid + q][1], s_mrg[tid + q][2]);
    float* const stats = img_ptr(E.stats, wo);
    stats[c] = mean;
    stats[cout + c] = 1.0f / sqrtf(m2 / n + EC_EPS);
  }
  if (tid == 0) *ticket = 0;                                             // ready for the next launch
}

// inet's output convolution at the M centroids, the gmap windows of the written fmap1 slot, the patch grids and
// (optional) the viewer colours.  Block (m, b): centroid m of image b, whose rows are frame_row[b] (fmap1),
// feat_row[b] + m (gmap, imap) and patch_row[b] + m (patches, colours).
struct EncCentroidParams {
  const float* coords;             // [B, M, 2]
  const float* depth;              // [B, M] or null: depth 1
  int M, h, w, cout;
  const __half* b3;                // image 0's level-2 block output and t9 (+ b ws_sb bytes for image b)
  const __half* t9;
  int64_t ws_sb;
  const __half* W;
  const float* bias;
  const __half* fmap1;
  int64_t f_sr, f_sy, f_sx;
  __half* gmap;
  int64_t g_sm, g_sy, g_sx;
  __half* imap;
  int64_t i_sm;
  float* patches;                  // rows of 27
  uint8_t* colors;                 // rows of 3, or null: no colours
  const uint8_t* image;            // image 0 (+ b x_sb for image b), element strides xs_c, xs_y, xs_x
  int64_t x_sb, xs_c, xs_y, xs_x;
  int img_h, img_w;
  int frame_row[EC_MAX_IMAGES], feat_row[EC_MAX_IMAGES], patch_row[EC_MAX_IMAGES];
};

// The viewer colour of dpvo.py:392-404, channel c (BGR -> RGB: image channel 2 - c) of the centroid (fx, fy):
//   clr = patchify(2 (img / 255.0) - 0.5, 4 (coords + 0.5), 0)     the bilinear form of altcorr.patchify
//   byte = uint8((clr + 0.5) * 127.5)                               truncating, through int64 as torch converts
// Every step is one fp32 operation rounded to nearest, in torch's order, so that nothing is contracted into an FMA.
// img / 255.0 is the product with the fp32 reciprocal of 255: that is how PyTorch's CUDA kernel divides a tensor by a
// scalar (the CPU kernel divides, and differs for the bytes 24..31).  Pixels outside the image read 0 (the normalised
// value, not the byte), as patchify zero-fills its window.
__device__ __forceinline__ uint8_t centroid_color(const uint8_t* im, int64_t sc, int64_t sy, int64_t sx, int H, int W, float fx,
                                                  float fy, int c) {
  constexpr float kInv255 = 1.0f / 255.0f;
  const float px = __fmul_rn(4.0f, __fadd_rn(fx, 0.5f)), py = __fmul_rn(4.0f, __fadd_rn(fy, 0.5f));
  const float flx = floorf(px), fly = floorf(py);
  const float dx = __fsub_rn(px, flx), dy = __fsub_rn(py, fly);
  const int x0 = (int)flx, y0 = (int)fly;
  const uint8_t* plane = im + (int64_t)(2 - c) * sc;
  float v[2][2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int y = y0 + i, x = x0 + j;
      v[i][j] = (y >= 0 && y < H && x >= 0 && x < W)
                    ? __fsub_rn(__fmul_rn(2.0f, __fmul_rn((float)plane[y * sy + x * sx], kInv255)), 0.5f) : 0.0f;
    }
  const float omx = __fsub_rn(1.0f, dx), omy = __fsub_rn(1.0f, dy);
  const float x00 = __fmul_rn(__fmul_rn(omy, omx), v[0][0]);
  const float x01 = __fmul_rn(__fmul_rn(omy, dx), v[0][1]);
  const float x10 = __fmul_rn(__fmul_rn(dy, omx), v[1][0]);
  const float x11 = __fmul_rn(__fmul_rn(dy, dx), v[1][1]);
  const float clr = __fadd_rn(__fadd_rn(__fadd_rn(x00, x01), x10), x11);
  return (uint8_t)__float2ll_rz(__fmul_rn(__fadd_rn(clr, 0.5f), 127.5f));
}

__global__ void __launch_bounds__(128)
enc_centroid_kernel(const __grid_constant__ EncCentroidParams p) {
  __shared__ float xin[64];
  const int m = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, h = p.h, w = p.w;
  const int64_t bm = (int64_t)b * p.M + m;
  const float fx = p.coords[2 * bm], fy = p.coords[2 * bm + 1];
  const int x = (int)floorf(fx), y = (int)floorf(fy);
  const bool inside = x >= 0 && x < w && y >= 0 && y < h;
  if (tid < 64) {
    float v = 0.f;
    if (inside) {
      const __half* b3 = img_ptr(p.b3, b * p.ws_sb);
      const __half* t9 = img_ptr(p.t9, b * p.ws_sb);
      const int64_t off = ((int64_t)y * w + x) * 64 + tid;                 // block 4 of inet: relu(b3 + relu(t9))
      v = __half2float(__float2half_rn(fmaxf(__fadd_rn(__half2float(b3[off]), fmaxf(__half2float(t9[off]), 0.f)), 0.f)));
    }
    xin[tid] = v;
  }
  __syncthreads();
  const int64_t fr = p.feat_row[b] + (int64_t)m;
  __half* const imap = p.imap + fr * p.i_sm;
  for (int co = tid; co < p.cout; co += 128) {
    float a = 0.f;
#pragma unroll 8
    for (int ci = 0; ci < 64; ++ci) a = fmaf(xin[ci], __half2float(p.W[((ci >> 3) * p.cout + co) * 8 + (ci & 7)]), a);
    imap[co] = __float2half_rn((a + p.bias[co]) * 0.25f);
  }
  const __half* const fmap1 = p.fmap1 + p.frame_row[b] * p.f_sr;
  __half* const gmap = p.gmap + fr * p.g_sm;
  for (int i = tid; i < 9 * 16; i += 128) {
    const int tap = i / 16, c8 = i % 16, dy = tap / 3, dx = tap % 3, yy = y + dy - 1, xx = x + dx - 1;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (yy >= 0 && yy < h && xx >= 0 && xx < w) v = *reinterpret_cast<const uint4*>(fmap1 + yy * p.f_sy + xx * p.f_sx + c8 * 8);
    *reinterpret_cast<uint4*>(gmap + dy * p.g_sy + dx * p.g_sx + c8 * 8) = v;
  }
  if (tid < 27) {
    const int c = tid / 9, i = (tid / 3) % 3, j = tid % 3;
    const float d = p.depth ? p.depth[bm] : 1.0f;
    p.patches[(p.patch_row[b] + (int64_t)m) * 27 + tid] = c == 0 ? fx + (float)(j - 1) : c == 1 ? fy + (float)(i - 1) : d;
  } else if (tid >= 32 && tid < 35 && p.colors != nullptr) {
    const int c = tid - 32;
    p.colors[(p.patch_row[b] + (int64_t)m) * 3 + c] =
        centroid_color(p.image + b * p.x_sb, p.xs_c, p.xs_y, p.xs_x, p.img_h, p.img_w, fx, fy, c);
  }
}

// ------------------------------------------------------------------------------------------- host side
struct ShapeInfo { int ks, s, cin, cout; };
static const ShapeInfo kShapes[] = {
    {7, 2, 3, 32},     // DPVO_ENC_STEM
    {3, 1, 32, 32},    // DPVO_ENC_C3_32
    {3, 2, 32, 64},    // DPVO_ENC_C3S2_32_64
    {1, 2, 32, 64},    // DPVO_ENC_C1S2_32_64
    {3, 1, 64, 64},    // DPVO_ENC_C3_64
    {1, 1, 64, 128},   // DPVO_ENC_OUT_128
    {1, 1, 64, 384},   // DPVO_ENC_OUT_384
};
constexpr int EC_NSHAPES = sizeof(kShapes) / sizeof(kShapes[0]);
// shape of each layer of an encoder in checkpoint order (the last one is fnet's; inet's is DPVO_ENC_OUT_384)
static const int kLayerShape[EC_NLAYERS] = {DPVO_ENC_STEM, DPVO_ENC_C3_32, DPVO_ENC_C3_32, DPVO_ENC_C3_32, DPVO_ENC_C3_32,
                                            DPVO_ENC_C3S2_32_64, DPVO_ENC_C1S2_32_64, DPVO_ENC_C3_64, DPVO_ENC_C3_64,
                                            DPVO_ENC_C3_64, DPVO_ENC_OUT_128};

static inline int out_size(int n, int ks, int s) { return (n + 2 * (ks / 2) - ks) / s + 1; }
static inline int64_t layer_halves(int shape) {
  const ShapeInfo& si = kShapes[shape];
  const int taps = shape == DPVO_ENC_STEM ? 1 : si.ks * si.ks, kc = shape == DPVO_ENC_STEM ? EC_STEM_KC : si.cin / 8;
  return (int64_t)taps * kc * si.cout * 8;
}
static inline int64_t ntiles(int ho, int wo) { return (int64_t)((ho + EC_TH - 1) / EC_TH) * ((wo + EC_TW - 1) / EC_TW); }

template <int KS, int S, int CIN, int NT, bool STEM>
static int launch_conv(const EncConvParams& p, int nimg, int cout, const char* name, cudaStream_t st) {
  using C = EncCfg<KS, S, CIN, NT, STEM>;
  dim3 grid((unsigned)ntiles(p.Hout, p.Wout), (unsigned)(cout / NT), (unsigned)(nimg * p.nenc));
  return launch(name, enc_conv_kernel<KS, S, CIN, NT, STEM>, grid, EC_THREADS, C::SMEM, st, p, cout);
}

// one launch of layer `shape` over nimg images x p.nenc encoders
static int launch_shape(int shape, const EncConvParams& p, int nimg, cudaStream_t st) {
  switch (shape) {
    case DPVO_ENC_STEM: return launch_conv<7, 2, 8, 32, true>(p, nimg, 32, "encoder_conv stem", st);
    case DPVO_ENC_C3_32: return launch_conv<3, 1, 32, 32, false>(p, nimg, 32, "encoder_conv 3x3/1 32", st);
    case DPVO_ENC_C3S2_32_64: return launch_conv<3, 2, 32, 64, false>(p, nimg, 64, "encoder_conv 3x3/2 32->64", st);
    case DPVO_ENC_C1S2_32_64: return launch_conv<1, 2, 32, 64, false>(p, nimg, 64, "encoder_conv 1x1/2 32->64", st);
    case DPVO_ENC_C3_64: return launch_conv<3, 1, 64, 64, false>(p, nimg, 64, "encoder_conv 3x3/1 64", st);
    case DPVO_ENC_OUT_128: return launch_conv<1, 1, 64, 64, false>(p, nimg, 128, "encoder_conv 1x1 64->128", st);
    case DPVO_ENC_OUT_384: return launch_conv<1, 1, 64, 64, false>(p, nimg, 384, "encoder_conv 1x1 64->384", st);
  }
  set_error("encoder_conv: unknown shape %d", shape);
  return DPVO_ERR_INVALID;
}

static bool al16(const void* q) { return ((uintptr_t)q & 15) == 0; }

}  // namespace dpvo

using namespace dpvo;

extern "C" int64_t dpvo_encoder_conv_workspace_bytes(int shape, int H, int W) {
  if (shape < 0 || shape >= EC_NSHAPES || H <= 0 || W <= 0) return 0;
  const ShapeInfo& si = kShapes[shape];
  return 2 * (ntiles(out_size(H, si.ks, si.s), out_size(W, si.ks, si.s)) * 3 * si.cout * (int64_t)sizeof(float) + 64);
}

extern "C" int dpvo_encoder_conv(int shape, int H, int W, int nenc, const dpvo_encoder_conv_io* io, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
  DPVO_REQUIRE(shape >= 0 && shape < EC_NSHAPES, "encoder_conv: unknown shape %d", shape);
  DPVO_REQUIRE(nenc == 1 || nenc == 2, "encoder_conv: nenc must be 1 or 2");
  DPVO_REQUIRE(io != nullptr, "encoder_conv: null io");
  DPVO_REQUIRE(H >= 1 && W >= 1 && (int64_t)H * W < (1ll << 28), "encoder_conv: bad image size %dx%d", H, W);
  const ShapeInfo& si = kShapes[shape];
  const bool stem = shape == DPVO_ENC_STEM, normalised = si.cout <= 64;
  EncConvParams p{};
  p.Hin = H; p.Win = W; p.Hout = out_size(H, si.ks, si.s); p.Wout = out_size(W, si.ks, si.s);
  p.tiles_x = (p.Wout + EC_TW - 1) / EC_TW;
  p.nenc = nenc;
  const int64_t tiles = ntiles(p.Hout, p.Wout);
  const int64_t part_bytes = tiles * 3 * si.cout * (int64_t)sizeof(float);
  bool any_stats = false;
  for (int e = 0; e < nenc; ++e) {
    const dpvo_encoder_conv_io& q = io[e];
    DPVO_REQUIRE(q.x && q.w && q.bias && q.y, "encoder_conv: null pointer (x, w, bias and y are required)");
    DPVO_REQUIRE(al16(q.x) && al16(q.w) && al16(q.y) && (!q.skip || al16(q.skip)) && (!q.joined || al16(q.joined)),
                 "encoder_conv: x, w, y, skip and joined must be 16-byte aligned");
    DPVO_REQUIRE(q.y_sy % 8 == 0 && q.y_sx % 8 == 0 && q.y_sx >= si.cout && q.y_sy >= (int64_t)p.Wout * q.y_sx,
                 "encoder_conv: y pixel strides must be multiples of 8 and cover %d channels", si.cout);
    DPVO_REQUIRE(!stem || (!q.x_stats && !q.skip && !q.joined), "encoder_conv: the stem reads the uint8 image and has no prologue");
    DPVO_REQUIRE(!q.joined || (q.skip && si.ks == 3), "encoder_conv: joined needs a residual join (skip) on a 3x3 layer");
    DPVO_REQUIRE(!q.stats || normalised, "encoder_conv: statistics are produced for layers of at most 64 channels");
    DPVO_REQUIRE(!q.pool || (q.pool_sy >= 0 && q.pool_sx >= si.cout), "encoder_conv: bad pool strides");
    any_stats |= q.stats != nullptr;
    EncSide& s = p.e[e];
    s.x = q.x; s.xs_c = q.x_strides[0]; s.xs_y = q.x_strides[1]; s.xs_x = q.x_strides[2];
    s.x_stats = q.x_stats; s.x_relu = q.x_relu; s.skip = (const __half*)q.skip; s.skip_stats = q.skip_stats; s.skip_relu = q.skip_relu;
    s.joined = (__half*)q.joined; s.w = (const __half*)q.w; s.bias = q.bias; s.y = (__half*)q.y; s.y_sy = q.y_sy; s.y_sx = q.y_sx;
    s.pool = (__half*)q.pool; s.pool_sy = q.pool_sy; s.pool_sx = q.pool_sx; s.stats = q.stats; s.scale = q.scale;
  }
  if (any_stats) {
    DPVO_REQUIRE(workspace && ((uintptr_t)workspace & 15) == 0, "encoder_conv: statistics need a 16-byte aligned workspace");
    DPVO_REQUIRE(workspace_bytes >= dpvo_encoder_conv_workspace_bytes(shape, H, W), "encoder_conv: workspace %lld B < required %lld B",
                 (long long)workspace_bytes, (long long)dpvo_encoder_conv_workspace_bytes(shape, H, W));
    uint8_t* ws = (uint8_t*)workspace;
    for (int e = 0; e < nenc; ++e) {
      p.e[e].part = (float*)(ws + e * part_bytes);
      p.e[e].ticket = (int*)(ws + 2 * part_bytes) + e;
    }
    cudaError_t ce = cudaMemsetAsync(ws + 2 * part_bytes, 0, 2 * sizeof(int), (cudaStream_t)stream);
    if (ce != cudaSuccess) return check_cuda(ce, "encoder_conv: ticket reset");
  }
  return launch_shape(shape, p, 1, (cudaStream_t)stream);
}

// ---- whole frame
namespace {
struct FrameLayout {
  int H1, W1, H2, W2;
  int64_t l1, l2, part, bytes;     // bytes of a level-1 / level-2 buffer, of the partials, of the whole workspace
  int64_t x[2][4], y[2][4], parts, stats, tickets;
};
FrameLayout frame_layout(int H, int W) {
  FrameLayout L{};
  L.H1 = out_size(H, 7, 2); L.W1 = out_size(W, 7, 2);
  L.H2 = out_size(L.H1, 3, 2); L.W2 = out_size(L.W1, 3, 2);
  L.l1 = align256((int64_t)L.H1 * L.W1 * 32 * 2);
  L.l2 = align256((int64_t)L.H2 * L.W2 * 64 * 2);
  L.part = align256(std::max(ntiles(L.H1, L.W1) * 3 * 32, ntiles(L.H2, L.W2) * 3 * 64) * (int64_t)sizeof(float));
  int64_t o = 0;
  for (int e = 0; e < 2; ++e) {
    for (int i = 0; i < 4; ++i) { L.x[e][i] = o; o += L.l1; }
    for (int i = 0; i < 4; ++i) { L.y[e][i] = o; o += L.l2; }
  }
  L.parts = o; o += 2 * L.part;
  L.stats = o; o += align256(2 * EC_NLAYERS * 2 * 64 * sizeof(float));
  L.tickets = o; o += 256;
  L.bytes = o;
  return L;
}
}  // namespace

extern "C" int64_t dpvo_encode_frames_workspace_bytes(int B, int H, int W) {
  if (B < 1 || B > EC_MAX_IMAGES || H < 1 || W < 1) return 0;
  return B * frame_layout(H, W).bytes;
}

extern "C" int64_t dpvo_encode_frame_workspace_bytes(int H, int W) { return dpvo_encode_frames_workspace_bytes(1, H, W); }

// offset (halves) of layer `layer` of encoder `encoder` (0 fnet, 1 inet) in the packed weight blob
static int64_t weight_offset(int encoder, int layer) {
  int64_t o = 0;
  for (int e = 0; e <= encoder; ++e)
    for (int l = 0; l < EC_NLAYERS; ++l) {
      if (e == encoder && l == layer) return o;
      o += layer_halves(e == 1 && l == EC_NLAYERS - 1 ? DPVO_ENC_OUT_384 : kLayerShape[l]);
    }
  return o;
}

// rows [a, a + n) and [b, b + n) share a row
static bool rows_overlap(int64_t a, int64_t b, int64_t n) { return a < b + n && b < a + n; }

static int encode_frames(const uint8_t* images, int64_t s_b, int64_t s_c, int64_t s_y, int64_t s_x, int B, int H, int W,
                         const void* w16, const float* b32, const float* coords, int M,
                         void* fmap1, int64_t f1_sr, int64_t f1_sy, int64_t f1_sx,
                         void* fmap2, int64_t f2_sr, int64_t f2_sy, int64_t f2_sx, int64_t frame_rows,
                         void* gmap, int64_t g_sm, int64_t g_sy, int64_t g_sx, void* imap, int64_t i_sm, int64_t feat_rows,
                         float* patches, int64_t patch_rows,
                         const int64_t* frame_row, const int64_t* feat_row, const int64_t* patch_row,
                         const float* depth, uint8_t* colors, void* workspace, int64_t workspace_bytes, void* stream) {
  DPVO_REQUIRE(B >= 1 && B <= EC_MAX_IMAGES, "encode_frames: B=%d images, 1 to %d per call", B, EC_MAX_IMAGES);
  DPVO_REQUIRE(images && w16 && b32 && coords && fmap1 && fmap2 && gmap && imap && patches && frame_row && feat_row && patch_row &&
               workspace, "encode_frames: null pointer");
  DPVO_REQUIRE(H >= 16 && W >= 16 && (int64_t)H * W < (1ll << 26), "encode_frames: image size %dx%d outside [16, 2^26 pixels]", H, W);
  DPVO_REQUIRE(M >= 1 && M < (1 << 20), "encode_frames: M=%d", M);
  DPVO_REQUIRE(s_b >= 0 && s_c >= 0 && s_y >= 0 && s_x >= 0, "encode_frames: negative image strides");
  DPVO_REQUIRE(al16(w16) && al16(fmap1) && al16(fmap2) && al16(gmap) && al16(workspace) && ((uintptr_t)b32 & 3) == 0 &&
               ((uintptr_t)coords & 3) == 0 && ((uintptr_t)imap & 1) == 0 && ((uintptr_t)patches & 3) == 0 &&
               ((uintptr_t)depth & 3) == 0 && f1_sr % 8 == 0 && f2_sr % 8 == 0,
               "encode_frames: misaligned pointer (w16, fmap1, fmap2, gmap, workspace and the fmap1 / fmap2 rows need 16 bytes)");
  DPVO_REQUIRE(f1_sx >= 128 && f1_sx % 8 == 0 && f1_sy % 8 == 0 && f2_sx >= 128 && f2_sx % 8 == 0 && f2_sy % 8 == 0,
               "encode_frames: fmap1 / fmap2 must be channels-last (channel stride 1) with pixel strides that are multiples of 8");
  DPVO_REQUIRE(g_sx >= 128 && g_sx % 8 == 0 && g_sy % 8 == 0 && g_sm % 8 == 0 && i_sm >= 384,
               "encode_frames: gmap must be [M, 3, 3, 128] channels-last with strides that are multiples of 8, imap [M, 384]");
  DPVO_REQUIRE(frame_rows >= 1 && frame_rows < (1ll << 31) && feat_rows >= 1 && feat_rows < (1ll << 31) && patch_rows >= 1 &&
               patch_rows < (1ll << 31), "encode_frames: ring sizes must be 1 to 2^31 - 1 rows");
  for (int b = 0; b < B; ++b) {
    DPVO_REQUIRE(frame_row[b] >= 0 && frame_row[b] < frame_rows, "encode_frames: image %d: frame row %lld outside the %lld-row fmap1 / fmap2 ring",
                 b, (long long)frame_row[b], (long long)frame_rows);
    DPVO_REQUIRE(feat_row[b] >= 0 && feat_row[b] + M <= feat_rows, "encode_frames: image %d: patch-feature rows [%lld, %lld) outside the "
                 "%lld-row gmap / imap ring", b, (long long)feat_row[b], (long long)feat_row[b] + M, (long long)feat_rows);
    DPVO_REQUIRE(patch_row[b] >= 0 && patch_row[b] + M <= patch_rows, "encode_frames: image %d: patch rows [%lld, %lld) outside the "
                 "%lld patches", b, (long long)patch_row[b], (long long)patch_row[b] + M, (long long)patch_rows);
    for (int a = 0; a < b; ++a) {
      DPVO_REQUIRE(frame_row[a] != frame_row[b], "encode_frames: images %d and %d write the same destination fmap1 / fmap2 row %lld",
                   a, b, (long long)frame_row[b]);
      DPVO_REQUIRE(!rows_overlap(feat_row[a], feat_row[b], M), "encode_frames: images %d and %d write the same destination gmap / imap "
                   "rows (first rows %lld and %lld, M=%d)", a, b, (long long)feat_row[a], (long long)feat_row[b], M);
      DPVO_REQUIRE(!rows_overlap(patch_row[a], patch_row[b], M), "encode_frames: images %d and %d write the same destination patch "
                   "rows (first rows %lld and %lld, M=%d)", a, b, (long long)patch_row[a], (long long)patch_row[b], M);
    }
  }
  const FrameLayout L = frame_layout(H, W);
  DPVO_REQUIRE(workspace_bytes >= B * L.bytes, "encode_frames: workspace %lld B < required %lld B", (long long)workspace_bytes,
               (long long)(B * L.bytes));
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* ws = (uint8_t*)workspace;
  const __half* wh = (const __half*)w16;
  // every image's tickets (256 bytes at the same offset of each workspace block): one strided memset for the batch
  cudaError_t ce = cudaMemset2DAsync(ws + L.tickets, (size_t)L.bytes, 0, 256, (size_t)B, st);
  if (ce != cudaSuccess) return check_cuda(ce, "encode_frames: ticket reset");

  auto X = [&](int e, int i) { return (__half*)(ws + L.x[e][i]); };
  auto Y = [&](int e, int i) { return (__half*)(ws + L.y[e][i]); };
  auto S = [&](int e, int l) { return e == 0 ? (float*)(ws + L.stats) + (e * EC_NLAYERS + l) * 128 : (float*)nullptr; };
  auto Wt = [&](int e, int l) { return wh + weight_offset(e, l); };
  auto Bt = [&](int e, int l) { return b32 + (e * EC_NLAYERS + l) * EC_BIAS_STRIDE; };

  // one launch per layer for both encoders of every image; (input, input stats, skip, skip stats, skip relu, joined) -> output
  struct Step { int layer; int lvl_in; int x, skip, joined; int lvl_out; int y; bool skip_norm, skip_relu; };
  // buffer index: 0..3 = level-1 buffers X, 4..7 = level-2 buffers Y, -1 = none
  const Step steps[] = {
      {0, 0, -1, -1, -1, 1, 0, false, false},        // stem -> s0 (X0)
      {1, 1, 0, -1, -1, 1, 1, false, false},         // layer1.0.conv1: act(s0) -> t1 (X1)
      {2, 1, 1, -1, -1, 1, 2, false, false},         // layer1.0.conv2: act(t1) -> t2 (X2)
      {3, 1, 2, 0, 1, 1, 3, true, true},             // layer1.1.conv1: b1 = relu(act(s0) + act(t2)) (X1) -> t3 (X3)
      {4, 1, 3, -1, -1, 1, 0, false, false},         // layer1.1.conv2: act(t3) -> t4 (X0)
      {5, 1, 0, 1, 2, 2, 4, false, false},           // layer2.0.conv1: b2 = relu(b1 + act(t4)) (X2) -> t5 (Y0)
      {6, 1, 2, -1, -1, 2, 5, false, false},         // layer2.0.downsample: b2 -> p6 (Y1)
      {7, 2, 4, -1, -1, 2, 6, false, false},         // layer2.0.conv2: act(t5) -> t7 (Y2)
      {8, 2, 6, 5, 4, 2, 7, true, false},            // layer2.1.conv1: b3 = relu(norm(p6) + act(t7)) (Y0) -> t8 (Y3)
      {9, 2, 7, -1, -1, 2, 5, false, false},         // layer2.1.conv2: act(t8) -> t9 (Y1)
  };
  auto buf = [&](int e, int lvl, int i) -> __half* { return i < 0 ? nullptr : lvl == 1 ? X(e, i) : Y(e, i - 4); };
  for (const Step& s : steps) {
    const int shape = kLayerShape[s.layer];
    const ShapeInfo& si = kShapes[shape];
    const int Hin = s.layer == 0 ? H : s.lvl_in == 1 ? L.H1 : L.H2, Win = s.layer == 0 ? W : s.lvl_in == 1 ? L.W1 : L.W2;
    EncConvParams p{};
    p.Hin = Hin; p.Win = Win; p.Hout = out_size(Hin, si.ks, si.s); p.Wout = out_size(Win, si.ks, si.s);
    p.tiles_x = (p.Wout + EC_TW - 1) / EC_TW;
    p.nenc = 2; p.x_sb = s_b; p.ws_sb = L.bytes;
    for (int b = 0; b < B; ++b) p.row[b] = b;                            // y: image b's workspace block
    for (int e = 0; e < 2; ++e) {
      EncSide& d = p.e[e];
      // the producer of x (and of skip) is the layer that wrote that buffer; its stats slot is the layer index
      d.x = s.layer == 0 ? (const void*)images : buf(e, s.lvl_in, s.x);
      d.xs_c = s_c; d.xs_y = s_y; d.xs_x = s_x;
      d.x_relu = 1;
      d.w = Wt(e, s.layer); d.bias = Bt(e, s.layer);
      d.y = buf(e, s.lvl_out, s.y); d.y_sy = (int64_t)p.Wout * si.cout; d.y_sx = si.cout; d.y_sr = L.bytes / 2;
      d.stats = S(e, s.layer); d.part = (float*)(ws + L.parts + e * L.part); d.ticket = (int*)(ws + L.tickets) + e * 16 + s.layer;
      d.scale = 1.0f;
    }
    // the transform of each input: which layer produced it (for its statistics)
    switch (s.layer) {
      case 0: for (int e = 0; e < 2; ++e) p.e[e].x_relu = 0; break;
      case 1: for (int e = 0; e < 2; ++e) p.e[e].x_stats = S(e, 0); break;
      case 2: for (int e = 0; e < 2; ++e) p.e[e].x_stats = S(e, 1); break;
      case 3: for (int e = 0; e < 2; ++e) { p.e[e].x_stats = S(e, 2); p.e[e].skip_stats = S(e, 0); } break;
      case 4: for (int e = 0; e < 2; ++e) p.e[e].x_stats = S(e, 3); break;
      case 5: for (int e = 0; e < 2; ++e) p.e[e].x_stats = S(e, 4); break;
      case 6: for (int e = 0; e < 2; ++e) p.e[e].x_relu = 0; break;       // b2 is already a block output
      case 7: for (int e = 0; e < 2; ++e) p.e[e].x_stats = S(e, 5); break;
      case 8: for (int e = 0; e < 2; ++e) { p.e[e].x_stats = S(e, 7); p.e[e].skip_stats = S(e, 6); } break;
      case 9: for (int e = 0; e < 2; ++e) p.e[e].x_stats = S(e, 8); break;
    }
    for (int e = 0; e < 2; ++e) {
      p.e[e].skip = buf(e, s.lvl_in, s.skip);
      p.e[e].skip_relu = s.skip_relu;
      if (!s.skip_norm) p.e[e].skip_stats = nullptr;
      p.e[e].joined = buf(e, s.lvl_in, s.joined);
    }
    const int rc = launch_shape(shape, p, B, st);
    if (rc != DPVO_OK) return rc;
  }
  {  // fnet output: b4 = relu(b3 + act(t9)) -> (. W + b) / 4 -> fmap1 slot and its 4x4 average -> fmap2 slot
    EncConvParams p{};
    p.Hin = p.Hout = L.H2; p.Win = p.Wout = L.W2; p.tiles_x = (L.W2 + EC_TW - 1) / EC_TW;
    p.nenc = 1; p.ws_sb = L.bytes;
    for (int b = 0; b < B; ++b) p.row[b] = (int)frame_row[b];
    EncSide& d = p.e[0];
    d.x = Y(0, 1); d.x_stats = S(0, 9); d.x_relu = 1; d.skip = Y(0, 0);
    d.w = Wt(0, 10); d.bias = Bt(0, 10);
    d.y = (__half*)fmap1; d.y_sy = f1_sy; d.y_sx = f1_sx; d.y_sr = f1_sr;
    d.pool = (__half*)fmap2; d.pool_sy = f2_sy; d.pool_sx = f2_sx; d.pool_sr = f2_sr;
    d.scale = 0.25f;
    const int rc = launch_shape(DPVO_ENC_OUT_128, p, B, st);
    if (rc != DPVO_OK) return rc;
  }
  EncCentroidParams c{};
  c.coords = coords; c.depth = depth; c.M = M; c.h = L.H2; c.w = L.W2; c.cout = 384;
  c.b3 = Y(1, 0); c.t9 = Y(1, 1); c.ws_sb = L.bytes; c.W = Wt(1, 10); c.bias = Bt(1, 10);
  c.fmap1 = (const __half*)fmap1; c.f_sr = f1_sr; c.f_sy = f1_sy; c.f_sx = f1_sx;
  c.gmap = (__half*)gmap; c.g_sm = g_sm; c.g_sy = g_sy; c.g_sx = g_sx;
  c.imap = (__half*)imap; c.i_sm = i_sm; c.patches = patches;
  c.colors = colors; c.image = images; c.x_sb = s_b; c.xs_c = s_c; c.xs_y = s_y; c.xs_x = s_x; c.img_h = H; c.img_w = W;
  for (int b = 0; b < B; ++b) {
    c.frame_row[b] = (int)frame_row[b]; c.feat_row[b] = (int)feat_row[b]; c.patch_row[b] = (int)patch_row[b];
  }
  return launch("enc_centroid_kernel", enc_centroid_kernel, dim3(M, B), 128, 0, st, c);
}

extern "C" int dpvo_encode_frames(const uint8_t* images, int64_t s_b, int64_t s_c, int64_t s_y, int64_t s_x, int B, int H, int W,
                                  const void* w16, const float* b32, const float* coords, int M,
                                  void* fmap1, int64_t f1_sr, int64_t f1_sy, int64_t f1_sx,
                                  void* fmap2, int64_t f2_sr, int64_t f2_sy, int64_t f2_sx, int64_t frame_rows,
                                  void* gmap, int64_t g_sm, int64_t g_sy, int64_t g_sx, void* imap, int64_t i_sm, int64_t feat_rows,
                                  float* patches, int64_t patch_rows,
                                  const int64_t* frame_row, const int64_t* feat_row, const int64_t* patch_row,
                                  const float* depth, void* workspace, int64_t workspace_bytes, void* stream) {
  return encode_frames(images, s_b, s_c, s_y, s_x, B, H, W, w16, b32, coords, M, fmap1, f1_sr, f1_sy, f1_sx, fmap2, f2_sr, f2_sy,
                       f2_sx, frame_rows, gmap, g_sm, g_sy, g_sx, imap, i_sm, feat_rows, patches, patch_rows, frame_row, feat_row,
                       patch_row, depth, nullptr, workspace, workspace_bytes, stream);
}

// dpvo_encode_frames that also writes the viewer colours: uint8 rows [patch_row[b], patch_row[b] + M) of colors
// [patch_rows, 3], the rows of the patches
extern "C" int dpvo_encode_frames_colors(const uint8_t* images, int64_t s_b, int64_t s_c, int64_t s_y, int64_t s_x, int B, int H,
                                         int W, const void* w16, const float* b32, const float* coords, int M,
                                         void* fmap1, int64_t f1_sr, int64_t f1_sy, int64_t f1_sx,
                                         void* fmap2, int64_t f2_sr, int64_t f2_sy, int64_t f2_sx, int64_t frame_rows,
                                         void* gmap, int64_t g_sm, int64_t g_sy, int64_t g_sx, void* imap, int64_t i_sm,
                                         int64_t feat_rows, float* patches, int64_t patch_rows,
                                         const int64_t* frame_row, const int64_t* feat_row, const int64_t* patch_row,
                                         const float* depth, uint8_t* colors, void* workspace, int64_t workspace_bytes,
                                         void* stream) {
  DPVO_REQUIRE(colors, "encode_frames_colors: null colour destination (dpvo_encode_frames writes none)");
  return encode_frames(images, s_b, s_c, s_y, s_x, B, H, W, w16, b32, coords, M, fmap1, f1_sr, f1_sy, f1_sx, fmap2, f2_sr, f2_sy,
                       f2_sx, frame_rows, gmap, g_sm, g_sy, g_sx, imap, i_sm, feat_rows, patches, patch_rows, frame_row, feat_row,
                       patch_row, depth, colors, workspace, workspace_bytes, stream);
}

// one image: the B = 1 case of dpvo_encode_frames, its slots the single rows of rings of one frame and M patches
extern "C" int dpvo_encode_frame(const uint8_t* image, int64_t s_c, int64_t s_y, int64_t s_x, int H, int W,
                                 const void* w16, const float* b32, const float* coords, int M,
                                 void* fmap1, int64_t f1_sy, int64_t f1_sx, void* fmap2, int64_t f2_sy, int64_t f2_sx,
                                 void* gmap, int64_t g_sm, int64_t g_sy, int64_t g_sx, void* imap, int64_t i_sm,
                                 float* patches, void* workspace, int64_t workspace_bytes, void* stream) {
  const int64_t row0 = 0;
  return dpvo_encode_frames(image, 0, s_c, s_y, s_x, 1, H, W, w16, b32, coords, M, fmap1, 0, f1_sy, f1_sx, fmap2, 0, f2_sy, f2_sx, 1,
                            gmap, g_sm, g_sy, g_sx, imap, i_sm, M, patches, M, &row0, &row0, &row0, nullptr, workspace,
                            workspace_bytes, stream);
}
