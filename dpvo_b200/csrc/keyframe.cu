// Keyframe culling on the device (dpvo/dpvo.py:257-300 DPVO.keyframe, :166-198 get_pose / terminate, :400-444 the
// timestamp bookkeeping) for one stream or the B streams of a stacked batch:
//   * dpvo_keyframe_motion   the motion test of frame k = n - KI from the edges (i, j) and (j, i), i = n - KI - 1,
//                            j = n - KI + 1; under the decision it records frame k's relative pose in the delta table and
//                            decrements the device frame counter
//   * dpvo_keyframe_shift    the KI - 1 slot copies t + 1 -> t, t = k .. n - 2, of every per-frame buffer and ring
//                            (dpvo_keyframe_shift_bytes: also slots of any byte count, e.g. the 3 M-byte colour rows)
//   * dpvo_keyframe_count    add_frame (tstamp[n - 1] = counter++) and skip_frame (delta[c] = (c - 1, identity))
//   * dpvo_keyframe_trajectory  one pose per timestamp t < counter, through the live keyframes and the delta chains
// Every call reads the frame counters from device memory, so a frame's add_frame + cull can be captured in a CUDA graph.
// The edges' renumbering is pgraph.cu's dpvo_pgraph_remove rule 1 under the decision flag.
#include "common.cuh"
#include "flow.cuh"

namespace dpvo {

constexpr int KF_THREADS = 256;
constexpr int KF_MAX_BUFS = 9;
constexpr int KF_PARTS = 64;                 // CTAs per stream of the motion test's partial sums

struct KfBufs {
  char* base[KF_MAX_BUFS];
  int64_t row_bytes[KF_MAX_BUFS];
  int64_t rows[KF_MAX_BUFS];
  int vec[KF_MAX_BUFS];                         // bytes per copy: 16, 8, 4 or 1
  int nbuf;
};

// the motion test in two launches.  Partial sums: grid (KF_PARTS, B); CTA p of stream b owns the p-th contiguous chunk
// of the stream's slots, thread t its slots t, t + KF_THREADS, ... (neighbouring lanes read neighbouring slots), and
// sums them in that order: the flow of all 9 pixels of every active (i, j) and (j, i) edge in fp64.  A fixed butterfly
// and a fixed walk over the warps give the CTA's (sum_ij, sum_ji, count_ij, count_ji).  Validity is ignored, as
// flow.mean() ignores it (dpvo.py:265).
__global__ void __launch_bounds__(KF_THREADS)
keyframe_motion_partial_kernel(const float* __restrict__ poses, const float* __restrict__ patches, const float* __restrict__ intr,
                               int64_t F, const int64_t* __restrict__ ii, const int64_t* __restrict__ jj,
                               const int64_t* __restrict__ kk, const uint8_t* __restrict__ active, int64_t slots,
                               const int64_t* __restrict__ n_dev, int ki, double* __restrict__ partial) {
  __shared__ double ssum[2][KF_THREADS / 32];
  __shared__ int scnt[2][KF_THREADS / 32];
  const int b = blockIdx.y, part = blockIdx.x;
  const int64_t f0 = (int64_t)b * F;
  const int64_t n = n_dev[b];
  const int64_t i = n - ki - 1, j = n - ki + 1;
  const int64_t gi = f0 + i, gj = f0 + j;
  const bool any = i >= 0 && j < F;
  const int64_t chunk = (slots + KF_PARTS - 1) / KF_PARTS;
  const int64_t c0s = min(slots, (int64_t)part * chunk), c1s = min(slots, c0s + chunk);
  const int64_t base = (int64_t)b * slots;
  double s0 = 0.0, s1 = 0.0;
  int c0 = 0, c1 = 0;
  if (any) {
    for (int64_t e = base + c0s + threadIdx.x; e < base + c1s; e += KF_THREADS) {
      if (!active[e]) continue;
      const int64_t a = ii[e], c = jj[e];
      const int set = (a == gi && c == gj) ? 0 : (a == gj && c == gi) ? 1 : -1;
      if (set < 0) continue;
      const int64_t p = kk[e];
      double s = 0.0;
#pragma unroll 1
      for (int px = 0; px < 9; ++px) {
        bool ok;
        s += (double)patch_flow(poses, patches, intr, a, c, p, px, ok);
      }
      if (set == 0) { s0 += s; ++c0; } else { s1 += s; ++c1; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    c0 += __shfl_xor_sync(0xffffffffu, c0, o);
    c1 += __shfl_xor_sync(0xffffffffu, c1, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { ssum[0][w] = s0; ssum[1][w] = s1; scnt[0][w] = c0; scnt[1][w] = c1; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double t0 = 0.0, t1 = 0.0, n0 = 0.0, n1 = 0.0;
  for (int q = 0; q < KF_THREADS / 32; ++q) { t0 += ssum[0][q]; t1 += ssum[1][q]; n0 += scnt[0][q]; n1 += scnt[1][q]; }
  double* out = partial + 4 * ((int64_t)b * KF_PARTS + part);
  out[0] = t0; out[1] = t1; out[2] = n0; out[3] = n1;
}

// the decision, one thread per stream: the partials summed in chunk order (two launches give identical bits), then
// m = mean(i, j) + mean(j, i) and m / 2 < thresh in fp64; under it the delta record and n -= 1
__global__ void keyframe_motion_kernel(const float* __restrict__ poses, int64_t F, int B, const double* __restrict__ partial,
                                       int64_t* n_dev, const int64_t* __restrict__ tstamp, float* delta, int64_t* delta_src,
                                       int64_t T, int ki, double thresh, int32_t* flag, int64_t* k_out, double* m_out,
                                       int32_t* overflow) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t f0 = (int64_t)b * F;
  const int64_t n = n_dev[b];
  const int64_t k = n - ki;
  double t0 = 0.0, t1 = 0.0, n0 = 0.0, n1 = 0.0;
  for (int p = 0; p < KF_PARTS; ++p) {
    const double* q = partial + 4 * ((int64_t)b * KF_PARTS + p);
    t0 += q[0]; t1 += q[1]; n0 += q[2]; n1 += q[3];
  }
  // an empty set has a NaN mean (flow.mean() of no element), and m / 2 < thresh is then false: the frame is kept
  const double mean0 = n0 > 0.0 ? t0 / (9.0 * n0) : (double)NAN;
  const double mean1 = n1 > 0.0 ? t1 / (9.0 * n1) : (double)NAN;
  const double m = mean0 + mean1;
  const bool removed = m / 2.0 < thresh;
  flag[b] = removed ? 1 : 0;
  k_out[b] = f0 + k;
  m_out[b] = m;
  if (!removed) return;
  // dpvo.py:274-278: delta[tstamp[k]] = (tstamp[k - 1], P_k P_{k-1}^-1), read before the shift moves slot k
  using namespace lie;
  const int64_t ts1 = tstamp[f0 + k], ts0 = tstamp[f0 + k - 1];
  if (ts1 >= 0 && ts1 < T) {
    const SE3<float> dP = se3_mul(se3_load(poses + 7 * (f0 + k)), se3_inv(se3_load(poses + 7 * (f0 + k - 1))));
    se3_store(dP, delta + 7 * ((int64_t)b * T + ts1));
    delta_src[(int64_t)b * T + ts1] = ts0;
  } else {
    overflow[b] = 1;
  }
  n_dev[b] = n - 1;                                       // dpvo.py:297: a removal issued next sees n - 1
}

// step `step` of the shift: slot t + 1 -> slot t of every buffer, t = k + step; buffer q's slot t is row
// b rows + t mod rows.  Grid (x, B); a stream whose flag is clear returns at once.
__global__ void __launch_bounds__(256)
keyframe_shift_kernel(KfBufs bufs, int64_t F, int step, const int32_t* __restrict__ flag, const int64_t* __restrict__ k_glob) {
  const int b = blockIdx.y;
  if (!flag[b]) return;
  const int64_t t = k_glob[b] - (int64_t)b * F + step;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  for (int q = 0; q < bufs.nbuf; ++q) {
    const int64_t R = bufs.rows[q], rb = bufs.row_bytes[q];
    char* dst = bufs.base[q] + ((int64_t)b * R + t % R) * rb;
    const char* src = bufs.base[q] + ((int64_t)b * R + (t + 1) % R) * rb;
    if (bufs.vec[q] == 16) {
      for (int64_t x = tid; x < rb / 16; x += stride) reinterpret_cast<uint4*>(dst)[x] = reinterpret_cast<const uint4*>(src)[x];
    } else if (bufs.vec[q] == 8) {
      for (int64_t x = tid; x < rb / 8; x += stride) reinterpret_cast<uint2*>(dst)[x] = reinterpret_cast<const uint2*>(src)[x];
    } else if (bufs.vec[q] == 4) {
      for (int64_t x = tid; x < rb / 4; x += stride) reinterpret_cast<uint32_t*>(dst)[x] = reinterpret_cast<const uint32_t*>(src)[x];
    } else {
      for (int64_t x = tid; x < rb; x += stride) dst[x] = src[x];
    }
  }
}

// mode 0, add_frame (dpvo.py:400, 440): tstamp[n - 1] = counter, counter += 1
// mode 1, skip_frame (dpvo.py:441-444): delta[c] = (c - 1, identity), counter = c + 1
// A timestamp at or beyond the delta table sets overflow.
__global__ void keyframe_count_kernel(int mode, const int64_t* __restrict__ n_dev, int64_t* tstamp, int64_t F, int B,
                                      int64_t* counter, float* delta, int64_t* delta_src, int64_t T, int32_t* overflow) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t c = counter[b];
  if (c < 0 || c >= T) overflow[b] = 1;
  if (mode == 0) {
    const int64_t n = n_dev[b];
    if (n >= 1 && n <= F) tstamp[(int64_t)b * F + n - 1] = c;
    else overflow[b] = 1;
  } else if (c >= 0 && c < T) {
    float* d = delta + 7 * ((int64_t)b * T + c);
    for (int q = 0; q < 6; ++q) d[q] = 0.f;
    d[6] = 1.f;
    delta_src[(int64_t)b * T + c] = c - 1;
  }
  counter[b] = c + 1;
}

// terminate()'s interpolation (dpvo.py:181-195), one CTA per stream: an inverse map of tstamp[0:n], then one thread per
// timestamp t < counter walks its delta chain, pose(t) = dP_t dP_t0 ... pose(live keyframe), and writes pose(t)^-1.
// A chain that leaves the table, meets an unrecorded timestamp or runs longer than T steps writes NaN and sets error[b].
__global__ void __launch_bounds__(256)
keyframe_trajectory_kernel(const float* __restrict__ poses, const int64_t* __restrict__ tstamp, const int64_t* __restrict__ n_dev,
                           int64_t F, const float* __restrict__ delta, const int64_t* __restrict__ delta_src, int64_t T,
                           const int64_t* __restrict__ counter, int32_t* map, float* out, int32_t* error) {
  using namespace lie;
  const int b = blockIdx.x;
  int32_t* mp = map + (int64_t)b * T;
  for (int64_t t = threadIdx.x; t < T; t += blockDim.x) mp[t] = -1;
  __syncthreads();
  const int64_t n = min(n_dev[b], F);
  for (int64_t s = threadIdx.x; s < n; s += blockDim.x) {
    const int64_t ts = tstamp[(int64_t)b * F + s];
    if (ts >= 0 && ts < T) mp[ts] = (int32_t)s;         // timestamps of live frames are distinct
  }
  __syncthreads();
  const int64_t cnt = min(counter[b], T);
  for (int64_t t = threadIdx.x; t < cnt; t += blockDim.x) {
    SE3<float> acc;
    acc.t = v3<float>(0.f, 0.f, 0.f);
    acc.q.x = acc.q.y = acc.q.z = 0.f; acc.q.w = 1.f;
    int64_t cur = t, steps = 0;
    bool ok = true;
    while (true) {
      if (cur < 0 || cur >= T || steps > T) { ok = false; break; }
      if (mp[cur] >= 0) break;
      const int64_t src = delta_src[(int64_t)b * T + cur];
      if (src < 0) { ok = false; break; }
      acc = se3_mul(acc, se3_load(delta + 7 * ((int64_t)b * T + cur)));
      cur = src;
      ++steps;
    }
    float* o = out + 7 * ((int64_t)b * T + t);
    if (ok) {
      se3_store(se3_inv(se3_mul(acc, se3_load(poses + 7 * ((int64_t)b * F + mp[cur])))), o);
    } else {
      for (int q = 0; q < 7; ++q) o[q] = NAN;
      error[b] = 1;
    }
  }
}

}  // namespace dpvo

using namespace dpvo;

extern "C" int64_t dpvo_keyframe_motion_workspace_bytes(int B) { return B > 0 ? (int64_t)B * KF_PARTS * 4 * 8 : 0; }

extern "C" int dpvo_keyframe_motion(const float* poses, const float* patches, const float* intrinsics, int64_t F, int B,
                                    const int64_t* ii, const int64_t* jj, const int64_t* kk, const uint8_t* active,
                                    int64_t slots, int64_t* n, const int64_t* tstamp, float* delta, int64_t* delta_src,
                                    int64_t T, int ki, double thresh, int32_t* flag, int64_t* k, double* m,
                                    int32_t* overflow, void* workspace, int64_t workspace_bytes, void* stream) {
  DPVO_REQUIRE(ki >= 1, "keyframe_motion: keyframe_index=%d must be at least 1", ki);
  DPVO_REQUIRE(B >= 1 && F >= 2 && slots >= 0, "keyframe_motion: bad sizes (B=%d, frames=%lld, slots=%lld)", B, (long long)F,
               (long long)slots);
  DPVO_REQUIRE(T >= F, "keyframe_motion: a delta table of %lld timestamps is smaller than the %lld frame slots", (long long)T,
               (long long)F);
  DPVO_REQUIRE(poses && patches && intrinsics && n && tstamp && delta && delta_src && flag && k && m && overflow && workspace &&
               (slots == 0 || (ii && jj && kk && active)), "keyframe_motion: null pointer");
  DPVO_REQUIRE(workspace_bytes >= dpvo_keyframe_motion_workspace_bytes(B), "keyframe_motion: workspace of %lld bytes, %lld needed",
               (long long)workspace_bytes, (long long)dpvo_keyframe_motion_workspace_bytes(B));
  cudaStream_t st = (cudaStream_t)stream;
  double* partial = (double*)workspace;
  const int rc = launch("keyframe_motion_partial_kernel", keyframe_motion_partial_kernel, dim3(KF_PARTS, B), KF_THREADS, 0, st, poses, patches,
                        intrinsics, F, ii, jj, kk, active, slots, n, ki, partial);
  if (rc) return rc;
  return launch("keyframe_motion_kernel", keyframe_motion_kernel, (B + 63) / 64, 64, 0, st, poses, F, B, partial, n, tstamp, delta, delta_src, T,
                ki, thresh, flag, k, m, overflow);
}

// any_bytes: rows of any positive byte count at any alignment, copied 1 byte at a time where 4 does not divide them
static int keyframe_shift(void* const* bases, const int64_t* row_bytes, const int64_t* rows, int nbuf, int64_t F, int B, int ki,
                          const int32_t* flag, const int64_t* k, bool any_bytes, void* stream) {
  DPVO_REQUIRE(ki >= 1, "keyframe_shift: keyframe_index=%d must be at least 1", ki);
  DPVO_REQUIRE(nbuf >= 0 && nbuf <= KF_MAX_BUFS && B >= 1 && F >= 2, "keyframe_shift: bad sizes (buffers=%d, B=%d, frames=%lld)",
               nbuf, B, (long long)F);
  DPVO_REQUIRE(flag && k && (nbuf == 0 || (bases && row_bytes && rows)), "keyframe_shift: null pointer");
  KfBufs bufs{};
  int64_t most = 0;
  for (int q = 0; q < nbuf; ++q) {
    DPVO_REQUIRE(bases[q], "keyframe_shift: null pointer (buffer %d)", q);
    if (any_bytes)
      DPVO_REQUIRE(row_bytes[q] > 0, "keyframe_shift: buffer %d has %lld-byte slots, a positive count is needed", q,
                   (long long)row_bytes[q]);
    else
      DPVO_REQUIRE(row_bytes[q] > 0 && row_bytes[q] % 4 == 0, "keyframe_shift: buffer %d has %lld-byte slots, a positive multiple of 4 is needed",
                   q, (long long)row_bytes[q]);
    DPVO_REQUIRE(rows[q] >= ki, "keyframe_shift: buffer %d holds %lld slots per stream, fewer than keyframe_index=%d", q,
                 (long long)rows[q], ki);
    const uintptr_t a = (uintptr_t)bases[q];
    bufs.base[q] = (char*)bases[q];
    bufs.row_bytes[q] = row_bytes[q];
    bufs.rows[q] = rows[q];
    bufs.vec[q] = (a % 16 == 0 && row_bytes[q] % 16 == 0) ? 16 : (a % 8 == 0 && row_bytes[q] % 8 == 0) ? 8
                : (a % 4 == 0 && row_bytes[q] % 4 == 0) ? 4 : 1;
    DPVO_REQUIRE(any_bytes || a % 4 == 0, "keyframe_shift: buffer %d is not 4-byte aligned", q);
    most = std::max(most, row_bytes[q] / bufs.vec[q]);
  }
  bufs.nbuf = nbuf;
  const int64_t want = std::max<int64_t>(1, std::min<int64_t>((most + 255) / 256, ((int64_t)sm_count() * 4 + B - 1) / B));
  for (int s = 0; s < ki - 1; ++s) {
    const int rc = launch("keyframe_shift_kernel", keyframe_shift_kernel, dim3((unsigned)want, (unsigned)B), 256, 0, (cudaStream_t)stream, bufs, F,
                          s, flag, k);
    if (rc) return rc;
  }
  return DPVO_OK;
}

extern "C" int dpvo_keyframe_shift(void* const* bases, const int64_t* row_bytes, const int64_t* rows, int nbuf, int64_t F, int B,
                                   int ki, const int32_t* flag, const int64_t* k, void* stream) {
  return keyframe_shift(bases, row_bytes, rows, nbuf, F, B, ki, flag, k, false, stream);
}

extern "C" int dpvo_keyframe_shift_bytes(void* const* bases, const int64_t* row_bytes, const int64_t* rows, int nbuf, int64_t F,
                                         int B, int ki, const int32_t* flag, const int64_t* k, void* stream) {
  return keyframe_shift(bases, row_bytes, rows, nbuf, F, B, ki, flag, k, true, stream);
}

extern "C" int dpvo_keyframe_count(int mode, const int64_t* n, int64_t* tstamp, int64_t F, int B, int64_t* counter, float* delta,
                                   int64_t* delta_src, int64_t T, int32_t* overflow, void* stream) {
  DPVO_REQUIRE(mode == 0 || mode == 1, "keyframe_count: mode %d is neither add (0) nor skip (1)", mode);
  DPVO_REQUIRE(B >= 1 && F >= 2 && T >= F, "keyframe_count: bad sizes (B=%d, frames=%lld, timestamps=%lld)", B, (long long)F,
               (long long)T);
  DPVO_REQUIRE(counter && overflow && (mode == 1 || (n && tstamp)) && (mode == 0 || (delta && delta_src)),
               "keyframe_count: null pointer");
  return launch("keyframe_count_kernel", keyframe_count_kernel, (B + 63) / 64, 64, 0, (cudaStream_t)stream, mode, n, tstamp, F, B, counter, delta,
                delta_src, T, overflow);
}

extern "C" int dpvo_keyframe_trajectory(const float* poses, const int64_t* tstamp, const int64_t* n, int64_t F, int B,
                                        const float* delta, const int64_t* delta_src, int64_t T, const int64_t* counter,
                                        int32_t* map, float* out, int32_t* error, void* stream) {
  DPVO_REQUIRE(B >= 1 && F >= 2 && T >= F, "keyframe_trajectory: bad sizes (B=%d, frames=%lld, timestamps=%lld)", B, (long long)F,
               (long long)T);
  DPVO_REQUIRE(T <= INT32_MAX, "keyframe_trajectory: %lld timestamps exceed the int32 map", (long long)T);
  DPVO_REQUIRE(poses && tstamp && n && delta && delta_src && counter && map && out && error, "keyframe_trajectory: null pointer");
  return launch("keyframe_trajectory_kernel", keyframe_trajectory_kernel, B, 256, 0, (cudaStream_t)stream, poses, tstamp, n, F, delta, delta_src,
                T, counter, map, out, error);
}
