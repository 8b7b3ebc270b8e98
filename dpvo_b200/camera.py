"""Calibrated camera images prepared on the device: the image preparation of the reference's readers
(dpvo/stream.py:image_stream and video_stream, evaluate_tum.py:tum_image_stream) on the sm_90a kernel of
csrc/undistort.cu, in front of the frame encoders:

    cv2.undistort(image, K, calib[4:])                         when the calibration row has coefficients
    cv2.resize(image, None, fx=0.5, fy=0.5, INTER_AREA)        half=True (video_stream)
    image[y0:y0 + h, x0:x0 + w]                                crop (default: top-left, to multiples of 16)

A Camera holds one calibration, raw image size and preparation; `undistort` prepares one raw uint8 CUDA image and
`undistort_frames` several of one raw size in one launch.  The result is bit-identical to OpenCV's integer arithmetic
(DESIGN §3.8).  Images must already be on the device.
"""
import math

import torch

from . import camera_extension

MAX_IMAGES = 64                     # images per launch (csrc/undistort.cu)
MAX_SIZE = 32767                    # raw image side


class Camera:
    """One camera's image preparation.

    calib   a reference calibration row: fx fy cx cy, fx fy cx cy k1 k2 p1 p2, or the same plus k3 (OpenCV's 0-, 4- and
            5-coefficient pinhole models; the rational, thin-prism and tilt models are not supported).
    width, height   the raw image size.
    half    halve the undistorted image with the 2x2 area average (video_stream); needs an even-sized raw image.
    crop    (y0, x0, h, w) in the (halved) image; default: the readers' top-left crop to multiples of 16.

    size        (h, w) of the prepared image
    intrinsics  its fp32 [fx, fy, cx, cy]: halved with the image, the principal point shifted by the crop -- what the
                readers put on their queues with the image
    """

    def __init__(self, calib, width, height, half=False, crop=None):
        vals = [float(v) for v in calib]
        if len(vals) not in (4, 8, 9):
            raise ValueError("Camera: a calibration row is fx fy cx cy [k1 k2 p1 p2 [k3]] (4, 8 or 9 numbers), got %d; the "
                             "rational, thin-prism and tilt models are not supported" % len(vals))
        if not all(math.isfinite(v) for v in vals):
            raise ValueError("Camera: non-finite calibration value in %s" % vals)
        if not (vals[0] > 0 and vals[1] > 0):
            raise ValueError("Camera: focal lengths must be positive, got fx %g, fy %g" % (vals[0], vals[1]))
        self.width, self.height, self.half = int(width), int(height), bool(half)
        if not (1 <= self.width <= MAX_SIZE and 1 <= self.height <= MAX_SIZE):
            raise ValueError("Camera: raw image size %dx%d outside [1, %d]" % (self.width, self.height, MAX_SIZE))
        if self.half and (self.width % 2 or self.height % 2):
            raise ValueError("Camera: halving needs an even-sized image, got %dx%d" % (self.width, self.height))
        hh, wh = (self.height // 2, self.width // 2) if self.half else (self.height, self.width)
        if crop is None:
            crop = (0, 0, hh - hh % 16, wh - wh % 16)
        y0, x0, h, w = (int(v) for v in crop)
        if h < 1 or w < 1:
            raise ValueError("Camera: empty crop window %dx%d" % (h, w))
        if y0 < 0 or x0 < 0 or y0 + h > hh or x0 + w > wh:
            raise ValueError("Camera: crop (y0 %d, x0 %d, %dx%d) outside the %dx%d %simage"
                             % (y0, x0, h, w, hh, wh, "halved " if self.half else ""))
        self.calib = tuple(vals)
        self.crop = (y0, x0, h, w)
        self.values = vals + [0.0] * (9 - len(vals))          # fx fy cx cy k1 k2 p1 p2 k3
        fx, fy, cx, cy = vals[:4]
        if self.half:
            fx, fy, cx, cy = fx * .5, fy * .5, cx * .5, cy * .5
        self.intrinsics = torch.tensor([fx, fy, cx - x0, cy - y0], dtype=torch.float64).float()
        self._ring_intrinsics = {}

    @property
    def size(self):
        return self.crop[2], self.crop[3]

    def ring_intrinsics(self, device):
        """intrinsics / 4 (dpvo.py:401, intrinsics / RES) on `device`, made once per device so that writing it into a
        state is a device-to-device copy (capturable)"""
        key = torch.device(device)
        if key not in self._ring_intrinsics:
            self._ring_intrinsics[key] = (self.intrinsics / 4).to(key)
        return self._ring_intrinsics[key]

    def _key(self):
        return self.width, self.height, self.half, self.crop

    def __repr__(self):
        return "Camera(%s, %d, %d, half=%s, crop=%s)" % (list(self.calib), self.width, self.height, self.half, self.crop)

    def undistort(self, image, out=None):
        """prepare one raw uint8 CUDA image [3, H, W] (CHW or the permuted HWC view) -> uint8 [h, w, 3] (into `out`, any
        strides, when given)"""
        if not isinstance(image, torch.Tensor) or image.dim() != 3:
            raise RuntimeError("Camera.undistort: the image must be a uint8 tensor [3, H, W]")
        res = undistort_frames(image[None], [self], None if out is None else out[None])
        return res[0]


def undistort_frames(images, cameras, out=None):
    """Prepare B raw uint8 CUDA images [B, 3, H, W] (CHW or HWC strides) in one launch, image b with cameras[b].  The
    cameras share the raw size, `half` and the crop window; their calibrations may differ.  Returns uint8 [B, h, w, 3]
    (`out`, any strides, when given)."""
    cameras = list(cameras)
    B = len(cameras)
    if not 1 <= B <= MAX_IMAGES:
        raise ValueError("undistort_frames: %d cameras, 1 to %d per call" % (B, MAX_IMAGES))
    if any(c._key() != cameras[0]._key() for c in cameras):
        raise ValueError("undistort_frames: the cameras of one call share the raw size, half and crop: %s" % cameras)
    if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8 or images.dim() != 4 or images.shape[1] != 3:
        raise RuntimeError("undistort_frames: the images must be uint8 [B, 3, H, W], got %s" % (
            "%s %s" % (images.dtype, tuple(images.shape)) if isinstance(images, torch.Tensor) else type(images).__name__))
    if not images.is_cuda:
        raise RuntimeError("undistort_frames: the images must be a CUDA tensor (there is no CPU path)")
    cam = cameras[0]
    if images.shape[0] != B or (images.shape[2], images.shape[3]) != (cam.height, cam.width):
        raise RuntimeError("undistort_frames: %d cameras of %dx%d images, got images %s" % (B, cam.width, cam.height, tuple(images.shape)))
    h, w = cam.size
    if out is None:
        out = torch.empty(B, h, w, 3, dtype=torch.uint8, device=images.device)
    elif tuple(out.shape) != (B, h, w, 3):
        raise RuntimeError("undistort_frames: out must be uint8 [%d, %d, %d, 3], got %s" % (B, h, w, tuple(out.shape)))
    camera_extension().undistort_frames(images, [v for c in cameras for v in c.values], cam.half, cam.crop[0], cam.crop[1], out)
    return out
