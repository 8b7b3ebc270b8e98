"""DPVO's map on the device: the patch colours the encoders write (csrc/encoder.cu) against Patchifier.forward's
return_color and dpvo.py:404, the patch points every update writes (csrc/map.cu) against pops.point_cloud and a float64
restatement, the colours Keyframes.cull moves against the reference's own DPVO.keyframe, and map=False unchanged."""

import pytest
import torch

from dpvo_b200 import extensions, frontend, synthetic
from dpvo_b200 import projective_ops as pops
from dpvo_b200.altcorr import patchify
from dpvo_b200.keyframe import Keyframes
from dpvo_b200.lietorch import SE3
from dpvo_b200.loop import LoopClosure
from dpvo_b200.net import Update
from dpvo_b200.patchgraph import DevicePatchGraph
from dpvo_b200.runner import UpdateRunner
from dpvo_b200.streams import StreamBatch

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT_C, SENT_P = 171, -7.5          # sentinels of rows nothing may write


@pytest.fixture(scope="module")
def ex():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return extensions()[3]


@pytest.fixture(scope="module")
def update(ex):
    torch.manual_seed(1234)
    return Update(3).to(DEV).eval()


def _encoder(strategy="RANDOM", seed=4):
    torch.manual_seed(seed)
    return frontend.FrameEncoder(frontend.Patchifier().cuda().eval(), strategy=strategy)


def _image(H, W, seed, hwc=False):
    """a structured image with noise on top, and every byte value 0..255 somewhere near the top left"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    ys = torch.linspace(0, 1, H, device=DEV)[:, None]
    xs = torch.linspace(0, 1, W, device=DEV)[None, :]
    base = torch.stack([200 * xs + 40 * ys, 230 * ys * (1 - xs) + 10, 128 + 120 * torch.sin(12 * xs + 7 * ys)])
    img = (base + 40 * torch.randn(3, H, W, device=DEV, generator=g)).clamp(0, 255).to(torch.uint8)
    img[:, :16, :16] = torch.randint(0, 256, (3, 16, 16), device=DEV, generator=g, dtype=torch.uint8)
    img[:, 0, :256 if W >= 256 else W] = torch.arange(256, device=DEV, dtype=torch.uint8)[:min(W, 256)]
    return img.permute(1, 2, 0).contiguous().permute(2, 0, 1) if hwc else img


def _ref_colors(img, coords):
    """Patchifier.forward(return_color=True)'s clr (frontend.py, net.py:142-143) and dpvo.py:404 on the GPU"""
    images = 2 * (img[None, None] / 255.0) - 0.5                          # dpvo.py:389
    clr = patchify(images[0], 4 * (coords[None] + 0.5), 0).view(1, -1, 3)
    return ((clr[0, :, [2, 1, 0]] + 0.5) * (255.0 / 2)).to(torch.uint8)


def _single_runner(update, config="default", strategy="RANDOM", n=8):
    st = synthetic.make_state(config, n, device=DEV, seed=11, buffer=16, mem=10, map=True)
    st.colors.fill_(SENT_C)
    return UpdateRunner(st, update=update, encoder=_encoder(strategy)), st


# ------------------------------------------------------------------------------------------------ colours
@pytest.mark.parametrize("hwc", [False, True], ids=["chw", "hwc"])
@pytest.mark.parametrize("strategy", ["RANDOM", "GRADIENT_BIAS"])
def test_ingest_image_colours_equal_patchifier_return_color(ex, update, strategy, hwc):
    run, st = _single_runner(update, strategy=strategy)
    M = run.M
    img = _image(480, 640, 5, hwc)
    torch.manual_seed(21)
    coords = run.ingest_image(img)
    torch.manual_seed(21)                                                  # the same centroid draws
    images = 2 * (img[None, None] / 255.0) - 0.5
    out = run.encoder.patchifier(images, patches_per_image=M, centroid_sel_strat=strategy, return_color=True)
    assert torch.equal(out[3][0, :, :2, 1, 1], coords), "the centroids differ from Patchifier.forward's"
    ref = ((out[5][0, :, [2, 1, 0]] + 0.5) * (255.0 / 2)).to(torch.uint8)  # dpvo.py:403-404
    torch.cuda.synchronize()
    assert torch.equal(st.colors[st.n - 1], ref)
    others = torch.ones(st.colors.shape[0], dtype=torch.bool, device=DEV)
    others[st.n - 1] = False
    assert (st.colors[others] == SENT_C).all(), "a row of another frame was written"


@pytest.mark.parametrize("hwc", [False, True], ids=["chw", "hwc"])
@pytest.mark.parametrize("kind", ["integer", "fractional", "border"])
def test_ingest_image_colours_at_given_coords(ex, update, kind, hwc):
    run, st = _single_runner(update)
    M = run.M
    h, w = st.fmap1.shape[3], st.fmap1.shape[4]
    g = torch.Generator(device=DEV).manual_seed(3)
    if kind == "integer":
        coords = torch.stack([torch.randint(0, w, (M,), generator=g, device=DEV),
                              torch.randint(0, h, (M,), generator=g, device=DEV)], -1).float()
        coords[:8] = torch.tensor([[0, 0], [1, 0], [2, 0], [3, 0], [w - 1, 0], [0, h - 1], [w - 1, h - 1], [63, 0]],
                                  device=DEV, dtype=torch.float)
    elif kind == "fractional":
        coords = torch.rand(M, 2, generator=g, device=DEV) * torch.tensor([w - 1.0, h - 1.0], device=DEV)
    else:                                   # windows that leave the image on each side (zero-filled pixels)
        t = torch.rand(M, generator=g, device=DEV)
        side = torch.arange(M, device=DEV) % 4
        x = torch.where(side == 0, -0.6 + 0.3 * t, torch.where(side == 1, w - 0.6 + 0.5 * t, t * (w - 1)))
        y = torch.where(side == 2, -0.6 + 0.3 * t, torch.where(side == 3, h - 0.6 + 0.5 * t, t * (h - 1)))
        coords = torch.stack([x, y], -1)
    img = _image(480, 640, 9, hwc)
    run.ingest_image(img, coords=coords, depth=torch.ones(M, 1, 1, device=DEV))
    torch.cuda.synchronize()
    assert torch.equal(st.colors[st.n - 1], _ref_colors(img, coords))


def _batch(update, B, n_frames, strategy="RANDOM"):
    cfg = synthetic.CONFIGS["fast"]
    batch = StreamBatch(B, cfg, 16, 4, device=DEV, map=True)
    for b in range(B):
        batch.stream(b).n = n_frames[b]
    batch.set_edges()
    batch.colors.fill_(SENT_C)
    return UpdateRunner(batch, update=update, encoder=_encoder(strategy)), batch


@pytest.mark.parametrize("B,streams", [(1, None), (3, None), (8, None), (8, [6, 1, 3])], ids=["B1", "B3", "B8", "B8-subset"])
def test_ingest_images_colours_equal_per_image_calls(ex, update, B, streams):
    frames = [3 + (5 * b) % 11 for b in range(B)]
    run, batch = _batch(update, B, frames)
    M = batch.M
    sel = list(range(B)) if streams is None else streams
    imgs = torch.stack([_image(480, 752, 40 + i) for i in range(len(sel))])
    if B == 3:                                                             # the permuted [B, H, W, 3] view
        imgs = imgs.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    g = torch.Generator(device=DEV).manual_seed(7)
    h, w = batch.fmap1.shape[3], batch.fmap1.shape[4]
    coords = torch.rand(len(sel), M, 2, generator=g, device=DEV) * torch.tensor([w + 0.8, h + 0.8], device=DEV) - 0.6
    coords[:, :M // 2] = coords[:, :M // 2].floor().clamp(min=0)           # half of them integer
    run.ingest_images(imgs, depth=torch.ones(len(sel), M, device=DEV), coords=coords, streams=streams)
    torch.cuda.synchronize()
    written = torch.zeros(batch.colors.shape[0], dtype=torch.bool, device=DEV)
    for i, b in enumerate(sel):
        s = batch.stream(b)
        # the same image alone through encode_into (ingest_image's call) into a fresh slot
        one = torch.full((M, 3), SENT_C, dtype=torch.uint8, device=DEV)
        hh, ww = frontend.encoder_output_size(480, 752)
        enc = run.encoder
        enc.encode_into(imgs[i], M, "RANDOM", torch.zeros(hh, ww, 128, device=DEV, dtype=torch.half),
                        torch.zeros(hh // 4, ww // 4, 128, device=DEV, dtype=torch.half),
                        torch.zeros(M, 3, 3, 128, device=DEV, dtype=torch.half), torch.zeros(M, 384, device=DEV, dtype=torch.half),
                        torch.zeros(M, 3, 3, 3, device=DEV), coords=coords[i], colors_slot=one)
        torch.cuda.synchronize()
        assert torch.equal(s.colors[s.n - 1], one), "stream %d" % b
        assert torch.equal(one, _ref_colors(imgs[i], coords[i])), "stream %d" % b
        written[b * batch.F + s.n - 1] = True
    assert (batch.colors[~written] == SENT_C).all(), "a row of another frame or stream was written"


def test_captured_ingest_images_with_colours_equals_eager(ex, update):
    run, batch = _batch(update, 3, [4, 7, 5])
    M = batch.M
    imgs = torch.stack([_image(480, 752, 70 + i) for i in range(3)])
    coords = torch.rand(3, M, 2, device=DEV) * 20
    depth = torch.ones(3, M, device=DEV)
    run.ingest_images(imgs, depth=depth, coords=coords)
    eager = batch.colors.clone()
    batch.colors.fill_(SENT_C)
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run.ingest_images(imgs, depth=depth, coords=coords)
    torch.cuda.current_stream().wait_stream(side)
    batch.colors.fill_(SENT_C)
    with torch.cuda.graph(g):
        run.ingest_images(imgs, depth=depth, coords=coords)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(batch.colors, eager)


# ------------------------------------------------------------------------------------------------ points
def _ref_points(poses, patches, intrinsics, n, M):
    """dpvo.py:358-360 with this package's pops.point_cloud"""
    ix = torch.arange(n, device=poses.device).repeat_interleave(M)
    pts = pops.point_cloud(SE3(poses.view(1, -1, 7)), patches.view(1, -1, 3, 3, 3)[:, :n * M], intrinsics.view(1, -1, 4), ix)
    return (pts[..., 1, 1, :3] / pts[..., 1, 1, 3:]).reshape(-1, 3)


def _f64_points(poses, patches, intrinsics, n, M):
    """the same points in float64 from the camera model: X_world = R^T (X_cam - t), X_cam = ((x - cx)/fx, (y - cy)/fy, 1) / d"""
    P = poses[:n].double().cpu()
    q = P[:, 3:] / P[:, 3:].norm(dim=1, keepdim=True)
    x, y, z, w = q.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    c = patches[:n * M, :, 1, 1].double().cpu()
    K = intrinsics[:n].double().cpu().repeat_interleave(M, 0)
    d = c[:, 2:3]
    Xc = torch.stack([(c[:, 0] - K[:, 2]) / K[:, 0], (c[:, 1] - K[:, 3]) / K[:, 1], torch.ones(n * M, dtype=torch.float64)], 1) / d
    f = torch.arange(n).repeat_interleave(M)
    return torch.einsum("kji,kj->ki", R[f], Xc - P[f, :3])


def _check_points(points, poses, patches, intrinsics, n, M):
    ref = _ref_points(poses, patches, intrinsics, n, M)
    assert torch.equal(points[:n * M], ref), "%d of %d points differ, by up to %g" % (
        int((points[:n * M] != ref).any(dim=1).sum()), n * M, (points[:n * M] - ref).abs().max().item())
    r64 = _f64_points(poses, patches, intrinsics, n, M)
    err = ((points[:n * M].double().cpu() - r64).norm(dim=1) / r64.norm(dim=1)).max().item()
    assert err <= 1e-6, err
    assert (points[n * M:] == SENT_P).all(), "a row at or above n M was written"


@pytest.mark.parametrize("config", ["default", "fast"])
def test_step_writes_the_point_cloud_of_the_post_ba_state(ex, update, config):
    st = synthetic.make_state(config, 20, device=DEV, seed=3, noise=0.02, map=True)
    st.points.fill_(SENT_P)
    run = UpdateRunner(st, update=update)
    run.step()
    torch.cuda.synchronize()
    _check_points(st.points, st.poses, st.patches, st.intrinsics, st.n, st.cfg["M"])
    pts, clr = run.map()
    assert pts.data_ptr() == st.points.data_ptr() and pts.shape == (st.n * st.cfg["M"], 3) and clr.shape == pts.shape


def test_batch_points_per_stream_at_its_own_n(ex, update):
    batch = synthetic.make_batch("fast", 3, n_frames=[12, 9, 14], device=DEV, frames_per_stream=24, mem=16, map=True)
    batch.points.fill_(SENT_P)
    run = UpdateRunner(batch, update=update)
    run.step()
    torch.cuda.synchronize()
    for b in range(3):
        s = batch.stream(b)
        _check_points(s.points, s.poses, s.patches, s.intrinsics, s.n, batch.M)
        pts, _ = run.map(stream=b)
        assert pts.shape[0] == s.n * batch.M


def test_step_graph_equals_eager(ex, update):
    sA = synthetic.make_state("fast", 16, device=DEV, seed=4, noise=0.02, map=True)
    sB = synthetic.make_state("fast", 16, device=DEV, seed=4, noise=0.02, map=True)
    rA, rB = UpdateRunner(sA, update=update), UpdateRunner(sB, update=update)
    rB.capture()
    rB.reset()
    rB.net.zero_()
    sB.points.fill_(SENT_P)
    rA.step()
    rB.step_graph()
    torch.cuda.synchronize()
    assert torch.equal(sA.poses, sB.poses) and torch.equal(sA.patches, sB.patches)
    assert torch.equal(sA.points[:sA.n * rA.M], sB.points[:sB.n * rB.M])
    _check_points(sB.points, sB.poses, sB.patches, sB.intrinsics, sB.n, rB.M)


def test_map_off_launches_and_computes_what_it_did(ex, update):
    """map=False: no buffers, no launch; the step's outputs are those of the same step with map=True"""
    sA = synthetic.make_state("fast", 16, device=DEV, seed=8)
    sB = synthetic.make_state("fast", 16, device=DEV, seed=8, map=True)
    assert sA.points is None and sA.colors is None
    rA, rB = UpdateRunner(sA, update=update), UpdateRunner(sB, update=update)
    rA.step()                                                              # first calls: lazy workspaces
    rB.step()
    torch.cuda.synchronize()
    c0 = ex.launch_count()
    tA, wA = rA.step()
    c1 = ex.launch_count()
    tB, wB = rB.step()
    c2 = ex.launch_count()
    torch.cuda.synchronize()
    assert c2 - c1 == c1 - c0 + 1
    assert torch.equal(sA.poses, sB.poses) and torch.equal(sA.patches, sB.patches)
    assert torch.equal(tA, tB) and torch.equal(wA, wB) and torch.equal(rA.net, rB.net)


def test_loop_closure_global_ba_frame_gets_the_normalized_map(ex, update):
    st = synthetic.make_loop_state("fast", 40, period=12, radius=1.0, max_edge_age=64, device=DEV)
    synthetic.add_map(st)
    st.points.fill_(SENT_P)
    M, cap = st.cfg["M"], st.E + 1024
    g = DevicePatchGraph(cap, M, st.poses.shape[0] - 1, DEV, loop_pairs=64, inactive_capacity=100000)
    lc = LoopClosure(st.cfg, g, max_edge_age=64)
    g.append(st.ii, st.jj, st.kk)
    run = UpdateRunner(st, update=update, graph=g, loop=lc)
    run.step()
    lc.propose(st.poses, st.patches, st.intrinsics, torch.tensor([st.n], dtype=torch.long, device=DEV))
    assert lc.read_flags(st.n)[1], "the closed loop must give a long-range loop edge"
    run.step()
    torch.cuda.synchronize()
    assert st.n in lc.ran_global_ba
    _check_points(st.points, st.poses, st.patches, st.intrinsics, st.n, M)
    # the normalized map: the first pose is the identity (PatchGraph.normalize, dpvo.py:352) up to the BA's own update
    assert torch.isfinite(st.points[:st.n * M]).all()


# ------------------------------------------------------------------------------------------------ culling
def _graph(st):
    M = st.cfg["M"]
    g = DevicePatchGraph(2 * st.E + 4 * M * st.cfg["lifetime"], M, st.poses.shape[0] - 1, DEV)
    g.append(st.ii, st.jj, st.kk)
    return g


def _edges(g):
    a = g.active.bool().cpu()
    return sorted(zip(g.ii.cpu()[a].tolist(), g.jj.cpu()[a].tolist(), g.kk.cpu()[a].tolist()))


@pytest.mark.parametrize("M", [96, 42])
def test_cull_moves_colours_as_the_reference_dpvo_keyframe(ex, M):
    """DPVO.keyframe of the reference's unmodified Python (on our native modules) on a DPVO object built on a copy of
    the same state, colours included, against Keyframes.cull: bit-identical colours, for culled and for kept frames"""
    from oracle import keyframe as OK
    from oracle import refimport
    if not refimport.staged():
        pytest.skip("the reference's Python package is not staged in oracle/_ref")
    cfg = dict(synthetic.CONFIGS["fast"], M=M)
    outcomes = set()
    for n, seed, mem in [(22, 5, 10), (14, 6, 10), (27, 8, 36), (31, 9, 7), (20, 3, 8), (25, 4, 9)]:
        st = synthetic.make_stop_go_state(cfg, n, total=40, mem=mem, device=DEV, seed=seed)
        synthetic.add_map(st)
        st.colors.copy_(torch.randint(0, 256, st.colors.shape, device=DEV, dtype=torch.uint8,
                                      generator=torch.Generator(device=DEV).manual_seed(seed)))
        g = _graph(st)
        kf = Keyframes(st.cfg, st, g)
        edges = torch.tensor(_edges(g), dtype=torch.long)
        with refimport.reference_python():
            ref = OK.reference_dpvo(st, edges, n, kf.tstamp[0], 4, 15.0)
            ref.pg.colors_[:] = st.colors
            ref.keyframe()
            torch.cuda.synchronize()
            r_n, r_colors, r_poses = ref.pg.n, ref.pg.colors_.clone(), ref.pg.poses_.clone()
        kf.cull()
        g.remove_old(kf.n_dev, st.cfg["removal"])
        (removed, _), = kf.read()
        assert removed == (r_n == n - 1) and st.n == r_n
        assert torch.equal(st.poses, r_poses)
        assert torch.equal(st.colors, r_colors), (n, seed, removed)
        outcomes.add(removed)
    assert outcomes == {True, False}, "cover both a culled and a kept frame"


def test_tracking_loop_with_culling_returns_the_replayed_map(ex, update):
    """60 frames of add_frame, step, cull, window removal; the caller writes each frame's colours.  map() against a host
    replay of the reference's bookkeeping: colors_ shifted with the culled frames (dpvo.py:289), points_ written by the
    last update and not shifted (dpvo.py:358-360)"""
    frames, n0, ki = 60, 16, 4
    st = synthetic.make_stop_go_state("fast", n0, total=n0 + frames, stop=8, go=6, mem=36, device=DEV, seed=7)
    synthetic.add_map(st)
    cfg, M = st.cfg, st.cfg["M"]
    st.colors[:n0] = torch.arange(n0, device=DEV, dtype=torch.uint8)[:, None, None]
    g = _graph(st)
    run = UpdateRunner(st, update=update, graph=g)
    kf = Keyframes(cfg, st, g)
    host = st.colors.cpu().clone()
    culled = 0
    for f in range(frames):
        c = int(kf.counter[0])
        st.n += 1
        kf.n_dev += 1
        n = st.n
        st.poses[n - 1] = st.extras["trajectory"][c]
        st.patches[(n - 1) * M:n * M] = st.extras["patches"][c * M:(c + 1) * M]
        clr = ((c * 37 + torch.arange(M * 3, device=DEV)) % 256).to(torch.uint8).view(M, 3)
        st.colors[n - 1] = clr
        host[n - 1] = clr.cpu()
        kf.add_frame()
        g.append_frame_edges(kf.n_dev, cfg["lifetime"])
        st.t0 = max(n - cfg["opt_window"], 1)
        run.step()
        points = _ref_points(st.poses, st.patches, st.intrinsics, n, M)
        kf.cull()
        (removed, _), = kf.read()
        if removed:
            k = n - ki
            host[k:n - 1] = host[k + 1:n].clone()
            culled += 1
        g.remove_old(kf.n_dev, cfg["removal"])
        pts, cols = run.map()
        assert torch.equal(pts, points[:st.n * M]), "frame %d: %d points differ" % (f, int((pts != points[:st.n * M]).any(dim=1).sum()))
        assert torch.equal(cols.cpu(), host.view(-1, 3)[:st.n * M]), "frame %d" % f
    assert culled >= 10, culled
