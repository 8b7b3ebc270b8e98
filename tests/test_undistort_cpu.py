"""Camera-image preparation on the host side: oracle/undistort.py pinned to OpenCV through tests/golden/undistort_ref.pt
(and to live cv2 where it imports), Camera's intrinsics against the reference readers' arithmetic, and every argument
the host rejects before a launch."""
import ctypes
import hashlib
import math
import os

import numpy as np
import pytest
import torch

import dpvo_b200
from dpvo_b200.camera import Camera, undistort_frames
from oracle import undistort as OU

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "undistort_ref.pt")


def _fixture():
    return torch.load(GOLDEN, weights_only=False)


RECIPES = sorted(_fixture()["recipes"])


def raw_image(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).numpy()


def tie_pixels(r):
    """bool [h, w] of the prepared image: the pixels computed from a map entry within a few ulps of a .5 tie"""
    t = OU.tie_entries(r["calib"], r["height"], r["width"]) if len(r["calib"]) > 4 else np.zeros((r["height"], r["width"]), bool)
    if r["half"]:
        t = t[0::2, 0::2] | t[0::2, 1::2] | t[1::2, 0::2] | t[1::2, 1::2]
    y0, x0, h, w = OU.default_crop(r["height"], r["width"], r["half"]) if r["crop"] is None else r["crop"]
    return t[y0:y0 + h, x0:x0 + w]


@pytest.mark.parametrize("name", RECIPES)
def test_oracle_matches_opencv_from_the_fixture(name):
    r = _fixture()["recipes"][name]
    out = OU.prepare(raw_image(r["height"], r["width"], r["seed"]), r["calib"], r["half"], r["crop"])
    assert out.shape == tuple(r["shape"])
    rc, vals = r["diff_rc"].numpy(), r["diff_values"].numpy()
    differs = np.zeros(out.shape[:2], bool)
    differs[rc[:, 0], rc[:, 1]] = True
    assert np.any(out[rc[:, 0], rc[:, 1]] != vals, axis=-1).all()          # each listed pixel does differ
    patched = out.copy()
    patched[rc[:, 0], rc[:, 1]] = vals
    assert hashlib.sha256(patched.tobytes()).hexdigest() == r["sha256"]
    ties = tie_pixels(r)
    # every pixel where OpenCV differs comes from a near-tie map entry; without halving those are exactly the entries
    assert not (differs & ~ties).any()
    if not r["half"]:
        assert np.array_equal(differs, ties)
    assert len(rc) <= (4 if name.startswith("iphone") else 0)


@pytest.mark.parametrize("name", RECIPES)
def test_oracle_matches_live_opencv(name):
    cv2 = pytest.importorskip("cv2")
    from oracle.make_golden_undistort import cv2_prepare
    r = _fixture()["recipes"][name]
    img = raw_image(r["height"], r["width"], r["seed"])
    ref = cv2_prepare(cv2, img, r["calib"], r["half"], r["crop"])
    out = OU.prepare(img, r["calib"], r["half"], r["crop"])
    assert hashlib.sha256(ref.tobytes()).hexdigest() == r["sha256"]
    assert not ((np.any(ref != out, axis=-1)) & ~tie_pixels(r)).any()


def test_opencv_map_far_outside_and_area_halving():
    """cv2's map does not wrap for points far outside the image (the clamp gives its result), and INTER_AREA halving is
    (sum + 2) >> 2"""
    cv2 = pytest.importorskip("cv2")
    img = raw_image(96, 128, 3)
    for d in ([1000.0, 0, 0, 0], [1e6, 1e6, 1e6, 1e6, 1e6], [-50.0, 30.0, 0.5, -0.5, 7.0]):
        calib = [90.0, 91.0, 63.5, 47.5] + d
        K = np.array([[90.0, 0, 63.5], [0, 91.0, 47.5], [0, 0, 1.0]])
        assert np.array_equal(cv2.undistort(img, K, np.array(d)), OU.undistort(img, calib))
    assert np.array_equal(cv2.resize(img, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA), OU.halve(img))


# ---------------------------------------------------------------------------------------------- Camera
def _reader_intrinsics(calib, reader):
    """what the reference readers put on their queues, float64 then fp32 (dpvo/stream.py, evaluate_tum.py)"""
    fx, fy, cx, cy = np.array(calib[:4], dtype=np.float64)
    if reader == "image":
        intr = np.array([fx, fy, cx, cy])
    elif reader == "video":
        intr = np.array([fx * .5, fy * .5, cx * .5, cy * .5])
    else:
        intr = np.asarray([fx, fy, cx, cy])
        intr[2] -= 16
        intr[3] -= 8
    return torch.as_tensor(intr, dtype=torch.float)


@pytest.mark.parametrize("name", RECIPES)
def test_camera_intrinsics_and_size_follow_the_readers(name):
    r = _fixture()["recipes"][name]
    cam = Camera(r["calib"], r["width"], r["height"], half=r["half"], crop=r["crop"])
    assert cam.size == tuple(r["shape"][:2])
    reader = "tum" if name == "tum" else "video" if r["half"] else "image"
    assert torch.equal(cam.intrinsics, _reader_intrinsics(r["calib"], reader))
    assert cam.intrinsics.dtype == torch.float32
    assert torch.equal((cam.intrinsics / 4), cam.intrinsics.double().div(4).float())
    assert np.array_equal(cam.intrinsics.numpy(), OU.intrinsics(r["calib"], r["half"], r["crop"]).astype(np.float32))


def test_camera_default_crop_and_coefficients():
    cam = Camera([718.8, 718.8, 607, 185], 1241, 376)
    assert cam.size == (368, 1232) and cam.crop == (0, 0, 368, 1232)
    assert cam.values == [718.8, 718.8, 607.0, 185.0, 0, 0, 0, 0, 0]
    cam = Camera([1660.0, 1660.0, 960, 540, 0.07, -0.08, 0, 0], 1920, 1080, half=True)
    assert cam.size == (528, 960)
    assert Camera([500, 500, 320, 240, 0.1, 0.2, 0.01, 0.02, 0.3], 640, 480).values[4:] == [0.1, 0.2, 0.01, 0.02, 0.3]


@pytest.mark.parametrize("calib", [[500, 500, 320], [500, 500, 320, 240, 0.1], [500, 500, 320, 240, 0.1, 0.2, 0, 0, 0.3, 0.4],
                                   [500, 500, 320, 240] + [0.0] * 8, [500, 500, 320, 240] + [0.0] * 10])
def test_camera_rejects_calibration_lengths(calib):
    with pytest.raises(ValueError, match="4, 8 or 9"):
        Camera(calib, 640, 480)


@pytest.mark.parametrize("calib, match", [([0.0, 500, 320, 240], "positive"), ([500, -1.0, 320, 240], "positive"),
                                          ([math.inf, 500, 320, 240], "non-finite"), ([500, math.nan, 320, 240], "non-finite"),
                                          ([500, 500, 320, 240, math.nan, 0, 0, 0], "non-finite"),
                                          ([500, 500, math.inf, 240], "non-finite")])
def test_camera_rejects_bad_values(calib, match):
    with pytest.raises(ValueError, match=match):
        Camera(calib, 640, 480)


def test_camera_rejects_sizes_and_crops():
    calib = [500, 500, 320, 240]
    with pytest.raises(ValueError, match="even-sized"):
        Camera(calib, 641, 480, half=True)
    with pytest.raises(ValueError, match="even-sized"):
        Camera(calib, 640, 481, half=True)
    with pytest.raises(ValueError, match="outside"):
        Camera(calib, 0, 480)
    with pytest.raises(ValueError, match="outside"):
        Camera(calib, 640, 480, crop=(8, 16, 480, 608))
    with pytest.raises(ValueError, match="outside"):
        Camera(calib, 640, 480, crop=(-1, 0, 16, 16))
    with pytest.raises(ValueError, match="outside"):
        Camera(calib, 640, 480, half=True, crop=(0, 0, 241, 320))
    with pytest.raises(ValueError, match="empty"):
        Camera(calib, 640, 480, crop=(0, 0, 0, 16))
    Camera(calib, 640, 480, half=True, crop=(0, 0, 240, 320))                      # the whole halved image


def test_undistort_frames_rejects_batches_and_tensors():
    cam = Camera([500, 500, 320, 240], 64, 48)
    img = torch.zeros(1, 3, 48, 64, dtype=torch.uint8)
    with pytest.raises(ValueError, match="1 to 64"):
        undistort_frames(img[:0], [])
    with pytest.raises(ValueError, match="1 to 64"):
        undistort_frames(img.expand(65, 3, 48, 64), [cam] * 65)
    with pytest.raises(ValueError, match="share"):
        undistort_frames(img.expand(2, 3, 48, 64), [cam, Camera([500, 500, 320, 240], 64, 48, crop=(0, 0, 32, 32))])
    with pytest.raises(RuntimeError, match="CUDA"):
        undistort_frames(img, [cam])
    with pytest.raises(RuntimeError, match="CUDA"):
        cam.undistort(img[0])
    with pytest.raises(RuntimeError, match="uint8"):
        undistort_frames(img.float(), [cam])
    with pytest.raises(RuntimeError, match="uint8"):
        cam.undistort(img[0, :2])


def test_shim_refuses_cpu_tensors_and_dtypes():
    ex = dpvo_b200.camera_extension()
    img, out = torch.zeros(1, 3, 48, 64, dtype=torch.uint8), torch.zeros(1, 48, 64, 3, dtype=torch.uint8)
    cam = [500.0, 500, 32, 24, 0, 0, 0, 0, 0]
    with pytest.raises(RuntimeError, match="no CPU path"):
        ex.undistort_frames(img, cam, False, 0, 0, out)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ex.undistort_frames(img.float(), cam, False, 0, 0, out)


def _abi():
    lib = dpvo_b200.library()
    f = lib.dpvo_undistort_frames
    i64, i32 = ctypes.c_int64, ctypes.c_int
    f.argtypes = [ctypes.c_void_p, i64, i64, i64, i64, i32, i32, i32, ctypes.c_void_p, i32, i32, i32, i32, i32, ctypes.c_void_p,
                  i64, i64, i64, i64, ctypes.c_void_p]
    return lib, f


class _Camera(ctypes.Structure):
    _fields_ = [(n, ctypes.c_double) for n in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3")]


@pytest.mark.parametrize("change, match", [
    (dict(B=0), b"1 to 64"), (dict(B=65), b"1 to 64"),
    (dict(fx=0.0), b"focal"), (dict(fy=-2.0), b"focal"), (dict(fx=math.nan), b"focal"), (dict(fy=math.inf), b"focal"),
    (dict(k3=math.inf), b"non-finite"), (dict(cx=math.nan), b"non-finite"),
    (dict(half=1, W=641), b"even-sized"), (dict(half=1, H=481), b"even-sized"),
    (dict(y0=1), b"outside"), (dict(x0=-1), b"outside"), (dict(half=1, Ho=241), b"outside"), (dict(Wo=641), b"outside"),
    (dict(Ho=0), b"empty"), (dict(Wo=0), b"empty"),
])
def test_library_rejects_arguments_before_any_launch(change, match):
    """the C-ABI rejects each bad argument on the host: these run without a GPU"""
    lib, f = _abi()
    a = dict(B=1, H=480, W=640, half=0, y0=0, x0=0, Ho=480, Wo=640, fx=500.0, fy=500.0, cx=320.0, cy=240.0, k3=0.0)
    a.update(change)
    cams = (_Camera * 65)()
    for c in cams:
        c.fx, c.fy, c.cx, c.cy, c.k3 = a["fx"], a["fy"], a["cx"], a["cy"], a["k3"]
    buf = (ctypes.c_char * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    rc = f(p, 0, 1, 640, 1, a["B"], a["H"], a["W"], ctypes.cast(cams, ctypes.c_void_p), a["half"], a["y0"], a["x0"], a["Ho"], a["Wo"], p,
           0, 640 * 3, 3, 1, None)
    assert rc == 1, lib.dpvo_last_error()
    assert match in lib.dpvo_last_error()
