"""ORACLE fixture (test infrastructure): run OpenCV's own image preparation once for each camera recipe of the
reference's readers and store what pins oracle/undistort.py to it in tests/golden/undistort_ref.pt, so that
tests/test_undistort_cpu.py checks the restatement against OpenCV without OpenCV.

    python oracle/make_golden_undistort.py      (needs cv2)

Each recipe stores the calibration row, the raw size, the seed of the torch CPU generator that draws the raw BGR
image (torch.randint(0, 256, (H, W, 3), uint8)), the half / crop of the reader, the SHA-256 of cv2's prepared image,
and the positions (row, column of the prepared image) and cv2 values of the pixels where the restatement differs.
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import undistort as OU  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "undistort_ref.pt")

EUROC = [458.654, 457.296, 367.215, 248.375, -0.28340811, 0.07395907, 0.00019359, 1.76187114e-05]
IPHONE = [1660.0, 1660.0, 960.0, 540.0, 0.07, -0.08, 0.0, 0.0]
BARN = [1161.545689, 1161.545689, 960.0, 540.0, -0.025158, 0.0, 0.0, 0.0]
TUM = [517.3, 516.5, 318.6, 255.3, 0.2624, -0.9531, -0.0054, 0.0026, 1.1633]
KITTI = [718.8, 718.8, 607.0, 185.0]
EXTREME = [458.654, 457.296, 367.215, 248.375, 1000.0, 0.0, 0.0, 0.0]

# name: (calibration row, width, height, half, crop or None for the readers' top-left crop to multiples of 16, seed)
RECIPES = {
    "euroc_image": (EUROC, 752, 480, False, None, 11),
    "iphone_image": (IPHONE, 1920, 1080, False, None, 12),
    "iphone_video": (IPHONE, 1920, 1080, True, None, 13),
    "barn_image": (BARN, 1920, 1080, False, None, 14),
    "barn_video": (BARN, 1920, 1080, True, None, 15),
    "tum": (TUM, 640, 480, False, (8, 16, 464, 608), 16),
    "kitti": (KITTI, 1241, 376, False, None, 17),
    "extreme": (EXTREME, 752, 480, False, None, 18),
}


def raw_image(H, W, seed):
    """the raw BGR image of a recipe, uint8 [H, W, 3]"""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).numpy()


def cv2_prepare(cv2, img, calib, half, crop):
    """the readers' preparation with OpenCV (image_stream, video_stream, tum_image_stream)"""
    fx, fy, cx, cy = calib[:4]
    K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
    if len(calib) > 4:
        img = cv2.undistort(img, K, np.array(calib[4:], dtype=np.float64))
    if half:
        img = cv2.resize(img, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA)
    h, w = img.shape[:2]
    y0, x0, ch, cw = (0, 0, h - h % 16, w - w % 16) if crop is None else crop
    return np.ascontiguousarray(img[y0:y0 + ch, x0:x0 + cw])


def main():
    import cv2
    out = dict(opencv=cv2.__version__, recipes={})
    for name, (calib, W, H, half, crop, seed) in RECIPES.items():
        img = raw_image(H, W, seed)
        ref = cv2_prepare(cv2, img, calib, half, crop)
        mine = OU.prepare(img, calib, half, crop)
        assert ref.shape == mine.shape, (name, ref.shape, mine.shape)
        rows, cols = np.nonzero(np.any(ref != mine, axis=-1))
        out["recipes"][name] = dict(calib=list(calib), width=W, height=H, half=half, crop=crop, seed=seed,
                                    sha256=hashlib.sha256(ref.tobytes()).hexdigest(), shape=tuple(ref.shape),
                                    diff_rc=torch.from_numpy(np.stack([rows, cols], 1).astype(np.int64)),
                                    diff_values=torch.from_numpy(ref[rows, cols].copy()))
        print("%-13s %4dx%-4d half=%d -> %s  %d pixels differ from the restatement" % (name, W, H, half, ref.shape, len(rows)))
    torch.save(out, OUT)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
