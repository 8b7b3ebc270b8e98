// Camera-image preparation (dpvo/stream.py:image_stream / video_stream, evaluate_tum.py:tum_image_stream) in front of
// the frame encoders: cv2.undistort, the optional cv2.resize(fx = fy = 0.5, INTER_AREA) and the crop, as one launch.
//
// The work is OpenCV's exact integer specification (DESIGN §3.8):
//   map     the destination pixel (j, i) reads the source point (u, v) of the float64 pinhole model with k1, k2, p1, p2,
//           k3, evaluated left to right with explicit __dmul_rn / __dadd_rn (nothing is contracted into an FMA), and
//           fixed to iu = rint(32 u), iv = rint(32 v) after clamping 32 u to +-UD_MAP_LIMIT (far outside any image).
//   remap   the fixed-point bilinear on the taps (iu >> 5, iv >> 5) + {0, 1}^2 with the weights 32 (32 - tx)(32 - ty),
//           32 tx (32 - ty), 32 (32 - tx) ty, 32 tx ty (tx = iu & 31, ty = iv & 31; they sum to 2^15), a tap outside
//           the image contributing 0: (sum w p + 2^14) >> 15.
//   halve   (the four undistorted pixels of the 2 x 2 block + 2) >> 2.
// The map is computed where it is used: no map tensor, no set-up launch.  Every image's camera comes by value in the
// kernel parameters (up to 64 cameras, 6.7 KB: sm_90 takes up to 32 KB of parameters), so a captured graph keeps them.
// A thread owns one output pixel of the crop window and its three channels; it evaluates the map only there (four
// times when halving).  No workspace, no atomics, no host synchronisation.
#include <cmath>

#include "common.cuh"

namespace dpvo {

constexpr int UD_MAX_IMAGES = 64;
constexpr double UD_MAP_LIMIT = 1073741824.0;                   // 2^30 = |32 u| of a point 2^25 pixels out
constexpr int UD_BX = 32, UD_BY = 8;                            // output pixels of a CTA: 32 columns x 8 rows

struct UdCamera {
  double fx, fy, cx, cy, k1, k2, p1, p2, k3;
  double ir0, ir2, ir4, ir5;                                    // 1 / fx, -cx / fx, 1 / fy, -cy / fy
};

struct UndistortParams {
  const uint8_t* src;                                           // image b at src + b s_b, element strides s_c, s_y, s_x
  int64_t s_b, s_c, s_y, s_x;
  int H, W;
  uint8_t* dst;                                                 // image b's window at dst + b d_b, strides d_y, d_x, d_c
  int64_t d_b, d_y, d_x, d_c;
  int Ho, Wo, y0, x0, half;
  UdCamera cam[UD_MAX_IMAGES];
};

__device__ __forceinline__ int ud_fixed(double s) {
  return __double2int_rn(fmin(fmax(s, -UD_MAP_LIMIT), UD_MAP_LIMIT));   // fmax(NaN, -L) = -L: NaN is far outside
}

// the fixed-point source point (32 u, 32 v) of destination pixel (column j, row i)
__device__ __forceinline__ void ud_map(const UdCamera& c, int i, int j, int& iu, int& iv) {
  const double x = __dadd_rn(__dmul_rn(c.ir0, (double)j), c.ir2);
  const double y = __dadd_rn(__dmul_rn(c.ir4, (double)i), c.ir5);
  const double x2 = __dmul_rn(x, x), y2 = __dmul_rn(y, y);
  const double r2 = __dadd_rn(x2, y2);
  const double xy2 = __dmul_rn(__dmul_rn(2.0, x), y);
  const double kr = __dadd_rn(1.0, __dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(c.k3, r2), c.k2), r2), c.k1), r2));
  const double xd = __dadd_rn(__dadd_rn(__dmul_rn(x, kr), __dmul_rn(c.p1, xy2)), __dmul_rn(c.p2, __dadd_rn(r2, __dmul_rn(2.0, x2))));
  const double yd = __dadd_rn(__dadd_rn(__dmul_rn(y, kr), __dmul_rn(c.p1, __dadd_rn(r2, __dmul_rn(2.0, y2)))), __dmul_rn(c.p2, xy2));
  iu = ud_fixed(__dmul_rn(__dadd_rn(__dmul_rn(c.fx, xd), c.cx), 32.0));
  iv = ud_fixed(__dmul_rn(__dadd_rn(__dmul_rn(c.fy, yd), c.cy), 32.0));
}

// the three channels of the undistorted pixel (column j, row i) of image `im`
__device__ __forceinline__ void ud_pixel(const UndistortParams& p, const uint8_t* im, const UdCamera& c, int i, int j, int out[3]) {
  int iu, iv;
  ud_map(c, i, j, iu, iv);
  const int xs = iu >> 5, ys = iv >> 5, tx = iu & 31, ty = iv & 31;
  int acc[3] = {1 << 14, 1 << 14, 1 << 14};
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int yy = ys + dy, xx = xs + dx;
      if (yy < 0 || yy >= p.H || xx < 0 || xx >= p.W) continue;
      const int w = 32 * (dx ? tx : 32 - tx) * (dy ? ty : 32 - ty);
      const uint8_t* q = im + yy * p.s_y + xx * p.s_x;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) acc[ch] += w * (int)q[ch * p.s_c];
    }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) out[ch] = acc[ch] >> 15;
}

__global__ void __launch_bounds__(UD_BX * UD_BY)
undistort_kernel(const __grid_constant__ UndistortParams p) {
  const int ox = blockIdx.x * UD_BX + threadIdx.x, oy = blockIdx.y * UD_BY + threadIdx.y, b = blockIdx.z;
  if (ox >= p.Wo || oy >= p.Ho) return;
  const UdCamera& c = p.cam[b];
  const uint8_t* im = p.src + b * p.s_b;
  const int X = p.x0 + ox, Y = p.y0 + oy;                      // in the (halved) undistorted image
  int v[3];
  if (p.half) {
    int s[3] = {2, 2, 2};
#pragma unroll 1
    for (int k = 0; k < 4; ++k) {
      int q[3];
      ud_pixel(p, im, c, 2 * Y + (k >> 1), 2 * X + (k & 1), q);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) s[ch] += q[ch];
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) v[ch] = s[ch] >> 2;
  } else {
    ud_pixel(p, im, c, Y, X, v);
  }
  uint8_t* d = p.dst + b * p.d_b + oy * p.d_y + ox * p.d_x;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) d[ch * p.d_c] = (uint8_t)v[ch];
}

}  // namespace dpvo

using namespace dpvo;

extern "C" int dpvo_undistort_frames(const uint8_t* images, int64_t s_b, int64_t s_c, int64_t s_y, int64_t s_x, int B, int H,
                                     int W, const dpvo_camera* cameras, int half, int y0, int x0, int Ho, int Wo, uint8_t* out,
                                     int64_t o_sb, int64_t o_sy, int64_t o_sx, int64_t o_sc, void* stream) {
  DPVO_REQUIRE(B >= 1 && B <= UD_MAX_IMAGES, "undistort_frames: B=%d images, 1 to %d per call", B, UD_MAX_IMAGES);
  DPVO_REQUIRE(images && cameras && out, "undistort_frames: null pointer");
  DPVO_REQUIRE(H >= 1 && W >= 1 && H <= 32767 && W <= 32767, "undistort_frames: image size %dx%d outside [1, 32767]", H, W);
  DPVO_REQUIRE(s_b >= 0 && s_c >= 0 && s_y >= 0 && s_x >= 0 && o_sb >= 0 && o_sy >= 0 && o_sx >= 0 && o_sc >= 0,
               "undistort_frames: negative strides");
  DPVO_REQUIRE(half == 0 || half == 1, "undistort_frames: half must be 0 or 1");
  DPVO_REQUIRE(!half || (H % 2 == 0 && W % 2 == 0), "undistort_frames: halving needs an even-sized image, got %dx%d", H, W);
  DPVO_REQUIRE(Ho >= 1 && Wo >= 1, "undistort_frames: empty output window %dx%d", Ho, Wo);
  const int Hh = half ? H / 2 : H, Wh = half ? W / 2 : W;
  DPVO_REQUIRE(y0 >= 0 && x0 >= 0 && (int64_t)y0 + Ho <= Hh && (int64_t)x0 + Wo <= Wh,
               "undistort_frames: window (y0 %d, x0 %d, %dx%d) outside the %dx%d %simage", y0, x0, Ho, Wo, Hh, Wh,
               half ? "halved " : "");
  UndistortParams p{};
  p.src = images; p.s_b = s_b; p.s_c = s_c; p.s_y = s_y; p.s_x = s_x; p.H = H; p.W = W;
  p.dst = out; p.d_b = o_sb; p.d_y = o_sy; p.d_x = o_sx; p.d_c = o_sc;
  p.Ho = Ho; p.Wo = Wo; p.y0 = y0; p.x0 = x0; p.half = half;
  for (int b = 0; b < B; ++b) {
    const dpvo_camera& q = cameras[b];
    DPVO_REQUIRE(std::isfinite(q.fx) && std::isfinite(q.fy) && q.fx > 0 && q.fy > 0,
                 "undistort_frames: camera %d: focal lengths must be finite and positive (fx %g, fy %g)", b, q.fx, q.fy);
    DPVO_REQUIRE(std::isfinite(q.cx) && std::isfinite(q.cy) && std::isfinite(q.k1) && std::isfinite(q.k2) &&
                 std::isfinite(q.p1) && std::isfinite(q.p2) && std::isfinite(q.k3),
                 "undistort_frames: camera %d: non-finite principal point or distortion coefficient", b);
    UdCamera& c = p.cam[b];
    c.fx = q.fx; c.fy = q.fy; c.cx = q.cx; c.cy = q.cy; c.k1 = q.k1; c.k2 = q.k2; c.p1 = q.p1; c.p2 = q.p2; c.k3 = q.k3;
    c.ir0 = 1.0 / q.fx; c.ir2 = -q.cx / q.fx; c.ir4 = 1.0 / q.fy; c.ir5 = -q.cy / q.fy;
  }
  const dim3 grid((unsigned)((Wo + UD_BX - 1) / UD_BX), (unsigned)((Ho + UD_BY - 1) / UD_BY), (unsigned)B);
  return launch("undistort_kernel", undistort_kernel, grid, dim3(UD_BX, UD_BY), 0, (cudaStream_t)stream, p);
}
