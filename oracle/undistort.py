"""ORACLE (test infrastructure): numpy restatement of the camera-image preparation of the reference's readers,
dpvo/stream.py:image_stream / video_stream and evaluate_tum.py:tum_image_stream:

    cv2.undistort(image, K, d)                                    (when the calibration row has coefficients)
    cv2.resize(image, None, fx=0.5, fy=0.5, INTER_AREA)           (video_stream only)
    image[y0:y0 + h, x0:x0 + w]                                   (crop to multiples of 16, or TUM's [8:-8, 16:-16])

written from OpenCV's documented semantics, as exact integer arithmetic on top of a float64 map:

  map     x = ir0 j + ir2, y = ir4 i + ir5 (ir0 = 1 / fx, ir2 = -cx / fx, ir4 = 1 / fy, ir5 = -cy / fy),
          r2 = x x + y y, kr = 1 + ((k3 r2 + k2) r2 + k1) r2,
          u = fx (x kr + p1 2xy + p2 (r2 + 2 x x)) + cx,  v = fy (y kr + p1 (r2 + 2 y y) + p2 2xy) + cy,
          float64, left to right, nothing fused; iu = rint(32 u), iv = rint(32 v) (half to even), 32 u clamped to
          +-MAP_LIMIT first (a point that far out has every tap outside the image, as cv2 has).
  remap   tx = iu & 31, ty = iv & 31, weights 32 (32 - tx)(32 - ty), 32 tx (32 - ty), 32 (32 - tx) ty, 32 tx ty (sum
          32768) on the taps (iu >> 5, iv >> 5) + {0, 1}^2, a tap outside the image contributing 0;
          out = (sum w p + 2^14) >> 15.
  halve   (sum of the 2 x 2 block + 2) >> 2.

cv2 evaluates the map in its own operation order, so at an entry where 32 u lies within a few ulps of a .5 tie it may
round the other way and differ from this restatement by one 1/32-pixel step; tie_entries() lists those entries.  Nothing here imports cv2 or the
reference.
"""
import numpy as np

MAP_LIMIT = float(1 << 30)                 # |32 u| beyond this is far outside any image
TIE_TOL = 1e-9                             # a few hundred float64 ulps of 32 u at 1080p


def calib_row(calib):
    """the 9 values (fx, fy, cx, cy, k1, k2, p1, p2, k3) of a reference calibration row of 4, 8 or 9 numbers"""
    c = [float(v) for v in calib]
    if len(c) not in (4, 8, 9):
        raise ValueError("a calibration row is fx fy cx cy [k1 k2 p1 p2 [k3]], got %d numbers" % len(c))
    return np.array(c + [0.0] * (9 - len(c)), dtype=np.float64)


def undistort_map(calib, H, W):
    """(u, v) float64 [H, W]: the source point of every destination pixel"""
    fx, fy, cx, cy, k1, k2, p1, p2, k3 = calib_row(calib)
    ir0, ir2, ir4, ir5 = 1.0 / fx, -cx / fx, 1.0 / fy, -cy / fy
    x = np.broadcast_to(ir0 * np.arange(W, dtype=np.float64)[None, :] + ir2, (H, W))
    y = np.broadcast_to(ir4 * np.arange(H, dtype=np.float64)[:, None] + ir5, (H, W))
    with np.errstate(all="ignore"):
        x2, y2 = x * x, y * y
        r2 = x2 + y2
        xy2 = (2.0 * x) * y
        kr = 1.0 + ((k3 * r2 + k2) * r2 + k1) * r2
        u = fx * ((x * kr + p1 * xy2) + p2 * (r2 + 2.0 * x2)) + cx
        v = fy * ((y * kr + p1 * (r2 + 2.0 * y2)) + p2 * xy2) + cy
    return u, v


def fixed_point(u):
    """rint(32 u) as int64 after the clamp (NaN counts as far outside)"""
    with np.errstate(all="ignore"):
        s = np.fmin(np.fmax(u * 32.0, -MAP_LIMIT), MAP_LIMIT)
    return np.rint(s).astype(np.int64)


def tie_entries(calib, H, W, tol=TIE_TOL):
    """bool [H, W]: the map entries where 32 u or 32 v lies within `tol` of a .5 tie, so close that the order of the
    float64 operations decides which way it rounds"""
    u, v = undistort_map(calib, H, W)
    with np.errstate(all="ignore"):
        su, sv = u * 32.0, v * 32.0
        return (np.abs(su - np.floor(su) - 0.5) <= tol) | (np.abs(sv - np.floor(sv) - 0.5) <= tol)


def remap(image, iu, iv):
    """the fixed-point bilinear of uint8 image [H, W, C] at the map (iu, iv) [Ho, Wo] -> uint8 [Ho, Wo, C]"""
    H, W = image.shape[:2]
    x0, y0 = iu >> 5, iv >> 5
    tx, ty = iu & 31, iv & 31
    acc = np.full(iu.shape + image.shape[2:], 1 << 14, dtype=np.int64)
    for dy, wy in ((0, 32 - ty), (1, ty)):
        for dx, wx in ((0, 32 - tx), (1, tx)):
            yy, xx = y0 + dy, x0 + dx
            inside = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            p = image[np.where(inside, yy, 0), np.where(inside, xx, 0)].astype(np.int64)
            w = np.where(inside, 32 * wx * wy, 0)
            acc += w[..., None] * p if image.ndim == 3 else w * p
    return (acc >> 15).astype(np.uint8)


def undistort(image, calib):
    """cv2.undistort(image, K, d) of uint8 image [H, W, C]; a row without coefficients leaves the image as it is"""
    H, W = image.shape[:2]
    u, v = undistort_map(calib, H, W)
    return remap(image, fixed_point(u), fixed_point(v))


def halve(image):
    """cv2.resize(image, None, fx=0.5, fy=0.5, interpolation=INTER_AREA) of an even-sized uint8 image"""
    H, W = image.shape[:2]
    if H % 2 or W % 2:
        raise ValueError("halving needs an even-sized image, got %dx%d" % (H, W))
    s = image.astype(np.int32)
    return ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)


def default_crop(H, W, half=False):
    """the readers' crop: the top-left (h - h % 16, w - w % 16) of the (halved) image, as (y0, x0, h, w)"""
    if half:
        H, W = H // 2, W // 2
    return 0, 0, H - H % 16, W - W % 16


def prepare(image, calib, half=False, crop=None):
    """undistort, halve if asked, crop: uint8 [H, W, C] -> uint8 [h, w, C]"""
    out = undistort(image, calib) if len(calib) > 4 else image
    if half:
        out = halve(out)
    y0, x0, h, w = default_crop(image.shape[0], image.shape[1], half) if crop is None else crop
    return np.ascontiguousarray(out[y0:y0 + h, x0:x0 + w])


def intrinsics(calib, half=False, crop=None, H=None, W=None):
    """the prepared image's (fx, fy, cx, cy) as the readers compute them (float64): halved, then shifted by the crop"""
    fx, fy, cx, cy = calib_row(calib)[:4]
    if half:
        fx, fy, cx, cy = fx * .5, fy * .5, cx * .5, cy * .5
    y0, x0 = (0, 0) if crop is None else crop[:2]
    return np.array([fx, fy, cx - x0, cy - y0], dtype=np.float64)
