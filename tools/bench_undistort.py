"""What preparing a calibrated camera image costs on one GPU (csrc/undistort.cu, dpvo_b200/camera.py):
    kernel   Camera.undistort / undistort_frames for one EuRoC frame, eight EuRoC frames in one call, one 1080p iPhone
             video_stream frame (undistort + half-size area resize + crop) and one TUM frame: device time per call
             (CUDA events over REPS calls after warm-up, median of ROUNDS rounds), the bytes the preparation must move
             (each raw pixel read once, each prepared pixel written once) and that over the time against the H100
             SXM's 3.35 TB/s.
    cv2      cv2.undistort (+ the resize) of the same frames on this machine's CPU, when cv2 is present.
    ingest   UpdateRunner.ingest_image(raw, camera=...) against ingest_image(prepared) with given centroids and depth,
             alternated: the added device time per frame.
The card's name and power limit are read in the same run; one JSON line per row.

    python tools/bench_undistort.py
"""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from dpvo_b200 import frontend, synthetic
from dpvo_b200.camera import Camera, undistort_frames
from dpvo_b200.runner import UpdateRunner

REPS, ROUNDS = int(os.environ.get("REPS", 200)), int(os.environ.get("ROUNDS", 11))
DEV = "cuda"
HBM = 3.35e12

EUROC = [458.654, 457.296, 367.215, 248.375, -0.28340811, 0.07395907, 0.00019359, 1.76187114e-05]
IPHONE = [1660.0, 1660.0, 960.0, 540.0, 0.07, -0.08, 0.0, 0.0]
TUM = [517.3, 516.5, 318.6, 255.3, 0.2624, -0.9531, -0.0054, 0.0026, 1.1633]


def smi():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def timed(fs, reps=REPS, rounds=ROUNDS):
    """median over rounds of the mean ms per call of each f, the fs alternated within a round"""
    for f in fs:
        for _ in range(10):
            f()
    torch.cuda.synchronize()
    ts = [[] for _ in fs]
    for _ in range(rounds):
        for f, out in zip(fs, ts):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                f()
            b.record()
            b.synchronize()
            out.append(a.elapsed_time(b) / reps)
    return [statistics.median(t) for t in ts]


def raw(B, H, W, seed=0):
    """B raw BGR frames as [B, 3, H, W] views of HWC storage (what a decoded frame is after its H2D copy)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(0, 256, (B, H, W, 3), generator=g, device=DEV, dtype=torch.uint8).permute(0, 3, 1, 2)


CASES = [
    ("euroc_x1", EUROC, 752, 480, False, None, 1),
    ("euroc_x8", EUROC, 752, 480, False, None, 8),
    ("iphone_video_1080p", IPHONE, 1920, 1080, True, None, 1),
    ("tum", TUM, 640, 480, False, (8, 16, 464, 608), 1),
]


def cv2_ms(cv2, calib, W, H, half, crop, B):
    import numpy as np
    img = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8).numpy()
    fx, fy, cx, cy = calib[:4]
    K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
    d = np.array(calib[4:])

    def f():
        x = cv2.undistort(img, K, d)
        if half:
            x = cv2.resize(x, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA)
        return x
    for _ in range(3):
        f()
    n = 20
    t = time.perf_counter()
    for _ in range(n * B):
        f()
    return (time.perf_counter() - t) / n * 1e3


def main():
    assert torch.cuda.is_available(), "bench_undistort measures on a CUDA device"
    card = smi()
    try:
        import cv2
    except ImportError:
        cv2 = None
    for name, calib, W, H, half, crop, B in CASES:
        cams = [Camera(calib, W, H, half=half, crop=crop)] * B
        src = raw(B, H, W)
        h, w = cams[0].size
        out = torch.empty(B, h, w, 3, dtype=torch.uint8, device=DEV)
        ms, = timed([lambda: undistort_frames(src, cams, out)])
        nbytes = B * (H * W * 3 + h * w * 3)
        row = dict(bench="undistort", case=name, B=B, raw="%dx%d" % (W, H), out="%dx%d" % (w, h), half=half,
                   us_per_call=round(ms * 1e3, 2), us_per_frame=round(ms * 1e3 / B, 2), bytes=nbytes,
                   GBps=round(nbytes / (ms * 1e-3) / 1e9, 1), share_of_hbm=round(nbytes / (ms * 1e-3) / HBM, 3),
                   cpu_cv2_ms=round(cv2_ms(cv2, calib, W, H, half, crop, B), 3) if cv2 is not None else "not measured",
                   cpu_threads=(cv2.getNumThreads() if cv2 is not None else None), card=card)
        print(json.dumps(row), flush=True)

    # ingest_image with a camera against ingest_image of the prepared frame (fast configuration, EuRoC camera)
    torch.manual_seed(0)
    st = synthetic.make_state("fast", 8, device=DEV, buffer=16, mem=10, map=True)
    run = UpdateRunner(st, encoder=frontend.FrameEncoder(frontend.Patchifier().cuda().eval()))
    cam = Camera(EUROC, 752, 480)
    src = raw(1, 480, 752)[0]
    prepared = cam.undistort(src).permute(2, 0, 1)
    M = st.cfg["M"]
    coords = run.encoder.centroids(prepared, M, "RANDOM")
    depth = torch.rand(M, 1, 1, device=DEV)
    t_cam, t_plain = timed([lambda: run.ingest_image(src, coords=coords, depth=depth, camera=cam),
                            lambda: run.ingest_image(prepared, coords=coords, depth=depth)], reps=50)
    print(json.dumps(dict(bench="undistort", case="ingest_image_euroc", us_with_camera=round(t_cam * 1e3, 1),
                          us_prepared=round(t_plain * 1e3, 1), us_added=round((t_cam - t_plain) * 1e3, 1), card=card)),
          flush=True)


if __name__ == "__main__":
    main()
