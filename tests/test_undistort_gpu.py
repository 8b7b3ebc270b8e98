"""Camera-image preparation on the sm_90a kernel (csrc/undistort.cu): bit-identical to oracle/undistort.py (pinned to
OpenCV by tests/test_undistort_cpu.py) for every camera recipe of tests/golden/undistort_ref.pt with CHW and HWC
sources, crop windows at every edge, nothing written outside the window, batches of mixed cameras equal to single
calls, CUDA-graph replay, and UpdateRunner.ingest_image(s) with a camera equal to ingesting the prepared image."""
import os

import numpy as np
import pytest
import torch

from dpvo_b200 import camera_extension, extensions, frontend, synthetic
from dpvo_b200.camera import Camera, undistort_frames
from dpvo_b200.net import Update
from dpvo_b200.runner import UpdateRunner
from dpvo_b200.streams import StreamBatch
from oracle import undistort as OU

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "undistort_ref.pt")
RECIPES = torch.load(GOLDEN, weights_only=False)["recipes"]
EUROC = RECIPES["euroc_image"]["calib"]
EXTREME = RECIPES["extreme"]["calib"]
TUM = RECIPES["tum"]["calib"]


@pytest.fixture(scope="module")
def ex():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return extensions()[3]


def raw_image(H, W, seed):
    """uint8 [H, W, 3] on the host, the fixture's draw"""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8)


def on_device(img, hwc):
    """[3, H, W] on the device: the permuted view of HWC storage, or CHW storage"""
    d = img.to(DEV)
    return d.permute(2, 0, 1) if hwc else d.permute(2, 0, 1).contiguous()


def oracle(img, cam):
    return torch.from_numpy(OU.prepare(img.numpy(), list(cam.calib), cam.half, cam.crop))


@pytest.mark.parametrize("hwc", [False, True], ids=["chw", "hwc"])
@pytest.mark.parametrize("name", sorted(RECIPES))
def test_bit_identical_to_the_oracle(ex, name, hwc):
    r = RECIPES[name]
    cam = Camera(r["calib"], r["width"], r["height"], half=r["half"], crop=r["crop"])
    img = raw_image(r["height"], r["width"], r["seed"])
    out = cam.undistort(on_device(img, hwc))
    assert out.shape == (*cam.size, 3)
    assert torch.equal(out.cpu(), oracle(img, cam))


@pytest.mark.parametrize("half", [False, True], ids=["full", "half"])
def test_crop_windows_at_every_edge(ex, half):
    H, W = 480, 752
    img = raw_image(H, W, 5)
    d = on_device(img, True)
    hh, wh = (H // 2, W // 2) if half else (H, W)
    windows = [(0, 0, 16, 16), (0, wh - 16, 16, 16), (hh - 16, 0, 16, 16), (hh - 16, wh - 16, 16, 16), (0, 0, hh, wh),
               (0, 5, 1, wh - 5), (hh - 1, 0, 1, wh), (3, wh - 1, hh - 3, 1), (0, 0, hh, 1), (7, 9, 33, 65)]
    for calib in (EUROC, EXTREME, EUROC[:4]):
        for crop in windows:
            cam = Camera(calib, W, H, half=half, crop=crop)
            assert torch.equal(cam.undistort(d).cpu(), oracle(img, cam)), (calib, crop)


def test_bytes_outside_the_window_are_untouched(ex):
    cam = Camera(TUM, 640, 480, crop=(8, 16, 464, 608))
    img = raw_image(480, 640, 6)
    buf = torch.full((2, 464 + 5, 608 + 7, 5), 0xA5, dtype=torch.uint8, device=DEV)
    before = buf.clone()
    view = buf[1, 2:2 + 464, 3:3 + 608, 1:4]
    out = cam.undistort(on_device(img, False), out=view)
    assert out.data_ptr() == view.data_ptr()
    torch.cuda.synchronize()
    assert torch.equal(view.cpu(), oracle(img, cam))
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[1, 2:2 + 464, 3:3 + 608, 1:4] = False
    assert torch.equal(buf[mask], before[mask])


def _mixed_cameras(B, W=752, H=480):
    """EuRoC, the extreme k1 = 1000 camera, a coefficient-free one, TUM's coefficients, ... cycled"""
    rows = [EUROC, EXTREME, [700.0, 690.0, 380.0, 236.0], TUM[:4] + [c * 0.5 for c in TUM[4:]],
            [EUROC[0] * 1.1, EUROC[1] * 0.9, 360.0, 250.0, 0.1, -0.05, 0.002, -0.001, 0.01]]
    return [Camera(rows[b % len(rows)], W, H) for b in range(B)]


@pytest.mark.parametrize("hwc", [False, True], ids=["chw", "hwc"])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_batch_of_mixed_cameras_equals_single_calls(ex, B, hwc):
    cams = _mixed_cameras(B)
    raws = [raw_image(480, 752, 40 + b) for b in range(B)]
    imgs = torch.stack([r.to(DEV) for r in raws])                        # [B, H, W, 3]
    imgs = imgs.permute(0, 3, 1, 2) if hwc else imgs.permute(0, 3, 1, 2).contiguous()
    n0 = ex.launch_count()
    out = undistort_frames(imgs, cams)
    assert ex.launch_count() - n0 == 1
    for b in range(B):
        assert torch.equal(out[b], cams[b].undistort(imgs[b]))
        assert torch.equal(out[b].cpu(), oracle(raws[b], cams[b]))


def test_half_batch_and_64_images(ex):
    cams = [Camera(c.calib, 752, 480, half=True) for c in _mixed_cameras(64)]
    raws = [raw_image(480, 752, 90 + b % 5) for b in range(64)]
    imgs = torch.stack([r.to(DEV) for r in raws]).permute(0, 3, 1, 2)
    out = undistort_frames(imgs, cams)
    for b in (0, 1, 2, 3, 4, 37, 63):
        assert torch.equal(out[b].cpu(), oracle(raws[b], cams[b])), b


def test_captured_graph_replays_bit_identically(ex):
    cams = _mixed_cameras(3)
    src = torch.stack([raw_image(480, 752, 60 + b).to(DEV) for b in range(3)]).permute(0, 3, 1, 2).contiguous()
    out = torch.empty(3, 480, 752, 3, dtype=torch.uint8, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        undistort_frames(src, cams, out)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        undistort_frames(src, cams, out)
    src.copy_(torch.stack([raw_image(480, 752, 70 + b).to(DEV) for b in range(3)]).permute(0, 3, 1, 2))
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, undistort_frames(src, cams))


def test_device_rejections(ex):
    cam = Camera(EUROC, 752, 480)
    img = on_device(raw_image(480, 752, 1), True)
    with pytest.raises(RuntimeError, match="images"):
        cam.undistort(on_device(raw_image(480, 640, 1), True))
    with pytest.raises(RuntimeError, match="out must be"):
        cam.undistort(img, out=torch.empty(480, 752, 4, dtype=torch.uint8, device=DEV))
    with pytest.raises(RuntimeError, match="uint8"):
        camera_extension().undistort_frames(img[None], cam.values, False, 0, 0, torch.empty(1, 480, 752, 3, device=DEV))
    with pytest.raises(RuntimeError, match="9 camera values"):
        camera_extension().undistort_frames(img[None], cam.values[:8], False, 0, 0, torch.empty(1, 480, 752, 3, dtype=torch.uint8, device=DEV))
    with pytest.raises(RuntimeError, match="no CPU path"):
        camera_extension().undistort_frames(img[None], cam.values, False, 0, 0, torch.empty(1, 480, 752, 3, dtype=torch.uint8))
    bad = list(cam.values)
    bad[0] = float("nan")
    with pytest.raises(RuntimeError, match="focal"):
        camera_extension().undistort_frames(img[None], bad, False, 0, 0, torch.empty(1, 480, 752, 3, dtype=torch.uint8, device=DEV))


# ------------------------------------------------------------------------------------------------ ingest
@pytest.fixture(scope="module")
def update(ex):
    torch.manual_seed(1234)
    return Update(3).to(DEV).eval()


def _encoder(seed=4):
    torch.manual_seed(seed)
    return frontend.FrameEncoder(frontend.Patchifier().cuda().eval())


SLOTS = ("fmap1", "fmap2", "gmap", "imap", "patches", "colors", "intrinsics")


def _single(update):
    st = synthetic.make_state("fast", 8, device=DEV, seed=11, buffer=16, mem=10, map=True)
    return UpdateRunner(st, update=update, encoder=_encoder()), st


def test_ingest_image_with_camera_equals_ingesting_the_prepared_image(ex, update):
    cam = Camera(EUROC, 752, 480)
    raw = raw_image(480, 752, 21)
    prepared = oracle(raw, cam).to(DEV).permute(2, 0, 1)
    M = synthetic.CONFIGS["fast"]["M"]
    g = torch.Generator(device=DEV).manual_seed(3)
    coords = torch.stack([torch.randint(1, 188 - 1, (M,), generator=g, device=DEV),
                          torch.randint(1, 120 - 1, (M,), generator=g, device=DEV)], -1).float()
    depth = torch.rand(M, 1, 1, device=DEV, generator=g)
    rA, sA = _single(update)
    rB, sB = _single(update)
    intr0 = sB.intrinsics.clone()
    rA.ingest_image(on_device(raw, True), coords=coords, depth=depth, camera=cam)
    rB.ingest_image(prepared, coords=coords, depth=depth)
    torch.cuda.synchronize()
    for k in SLOTS[:-1]:
        assert torch.equal(getattr(sA, k), getattr(sB, k)), k
    expect = intr0.clone()
    expect.view(-1, 4)[sB.n - 1] = cam.intrinsics.to(DEV) / 4
    assert torch.equal(sA.intrinsics, expect)
    assert torch.equal(sB.intrinsics, intr0)                             # no camera: intrinsics untouched


def test_ingest_image_with_camera_draws_as_the_prepared_image(ex, update):
    """without coords / depth the generator is drawn from the prepared image, as ingest_image(prepared) draws it"""
    cam = Camera(EXTREME, 752, 480)
    raw = raw_image(480, 752, 22)
    prepared = oracle(raw, cam).to(DEV).permute(2, 0, 1)
    rA, sA = _single(update)
    rB, sB = _single(update)
    torch.manual_seed(8)
    cA = rA.ingest_image(on_device(raw, False), camera=cam)
    rng_a = torch.cuda.get_rng_state()
    torch.manual_seed(8)
    cB = rB.ingest_image(prepared)
    assert torch.equal(cA, cB) and torch.equal(rng_a, torch.cuda.get_rng_state())
    for k in SLOTS[:-1]:
        assert torch.equal(getattr(sA, k), getattr(sB, k)), k


def test_captured_ingest_image_with_camera_equals_eager(ex, update):
    cam = Camera(EUROC, 752, 480)
    raw = on_device(raw_image(480, 752, 23), True)
    run, st = _single(update)
    M = st.cfg["M"]
    torch.manual_seed(5)
    coords = run.encoder.centroids(cam.undistort(raw).permute(2, 0, 1), M, "RANDOM")
    depth = torch.rand(M, 1, 1, device=DEV)
    snap = {k: getattr(st, k).clone() for k in SLOTS}

    def restore():
        for k in SLOTS:
            getattr(st, k).copy_(snap[k])

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run.ingest_image(raw, coords=coords, depth=depth, camera=cam)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    restore()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run.ingest_image(raw, coords=coords, depth=depth, camera=cam)
    restore()
    g.replay()
    torch.cuda.synchronize()
    res_g = {k: getattr(st, k).clone() for k in SLOTS}
    restore()
    run.ingest_image(raw, coords=coords, depth=depth, camera=cam)
    torch.cuda.synchronize()
    for k in SLOTS:
        assert torch.equal(res_g[k], getattr(st, k)), k


def _batch(update, B, n_frames):
    batch = StreamBatch(B, synthetic.CONFIGS["fast"], 16, 4, device=DEV, map=True)
    for b in range(B):
        batch.stream(b).n = n_frames[b]
    batch.set_edges()
    return UpdateRunner(batch, update=update, encoder=_encoder()), batch


@pytest.mark.parametrize("B,streams", [(1, None), (3, None), (8, [6, 1, 3])], ids=["B1", "B3", "B8-subset"])
def test_ingest_images_with_cameras_equal_per_stream_calls(ex, update, B, streams):
    n_frames = [3 + (b % 4) for b in range(B)]
    sel = list(range(B)) if streams is None else streams
    cams = _mixed_cameras(len(sel))
    raws = torch.stack([raw_image(480, 752, 30 + i).to(DEV) for i in range(len(sel))]).permute(0, 3, 1, 2)
    rA, bA = _batch(update, B, n_frames)
    rB, bB = _batch(update, B, n_frames)
    torch.manual_seed(9)
    cA = rA.ingest_images(raws, streams=streams, cameras=cams)
    rng_a = torch.cuda.get_rng_state()
    torch.manual_seed(9)
    cB = torch.stack([rB.ingest_image(raws[i], stream=b, camera=cams[i]) for i, b in enumerate(sel)])
    assert torch.equal(cA, cB) and torch.equal(rng_a, torch.cuda.get_rng_state())
    torch.cuda.synchronize()
    for k in SLOTS:
        assert torch.equal(getattr(bA, k), getattr(bB, k)), k
    for i, b in enumerate(sel):
        s = bA.stream(b)
        assert torch.equal(s.intrinsics[s.n - 1].cpu(), cams[i].intrinsics / 4)


def test_ingest_without_camera_is_unchanged(ex, update):
    """no camera: the call writes what it wrote before and leaves the intrinsics alone"""
    raw = on_device(raw_image(480, 752, 24), True)
    rA, sA = _single(update)
    intr0 = sA.intrinsics.clone()
    torch.manual_seed(4)
    rA.ingest_image(raw)
    torch.cuda.synchronize()
    assert torch.equal(sA.intrinsics, intr0)
    assert getattr(rA, "_prepared", None) is None
