"""Synthetic DPVO state for benchmarks and parity tests (no datasets, no checkpoint).

Replays the reference's edge rules (dpvo/dpvo.py:362-375 __edges_forw/__edges_back, :457-459
append order, :305-310 removal of edges whose patch left the REMOVAL_WINDOW) to obtain the patch
graph exactly as `DPVO.update()` sees it in steady state, and fills the state tensors with the shapes
and dtypes of dpvo/dpvo.py:58-73 and dpvo/patchgraph.py:26-35:

    default.yaml (config/default.yaml:4-7): M=96, lifetime 13, removal 22, optimisation 10
        -> E = 47,712 edges over 2,208 live patches inside update() (SURVEY 8, table)
    fast.yaml: M=48, lifetime 11, removal 16, optimisation 7 -> E = 14,496

Everything is seeded; tensors are created on `device`.
"""
import math
from dataclasses import dataclass, field

import torch

CONFIGS = {
    "default": dict(M=96, lifetime=13, removal=22, opt_window=10, ht=480, wd=640,
                    intrinsics=(320.0, 320.0, 320.0, 240.0)),
    "fast": dict(M=48, lifetime=11, removal=16, opt_window=7, ht=480, wd=752,
                 intrinsics=(458.654, 457.296, 367.215, 248.375)),
}


def replay_edges(n_frames, M, lifetime, removal):
    """Edge lists (ii, jj, kk) at the entry of update() after `n_frames` frames were added, assuming
    no keyframe is dropped (the upper bound of SURVEY 8).  CPU int64 tensors, reference order."""
    ii = torch.zeros(0, dtype=torch.long)
    jj = torch.zeros(0, dtype=torch.long)
    kk = torch.zeros(0, dtype=torch.long)

    def append(k, j):
        nonlocal ii, jj, kk
        kg, jg = torch.meshgrid(k, j, indexing="ij")
        kg, jg = kg.reshape(-1), jg.reshape(-1)
        jj = torch.cat([jj, jg])
        kk = torch.cat([kk, kg])
        ii = torch.cat([ii, kg // M])

    n = 0
    for _ in range(n_frames):
        if n > 0 or True:
            n += 1
            # forward: live patches of the previous `lifetime` frames -> new frame (n-1)
            append(torch.arange(M * max(n - lifetime, 0), M * max(n - 1, 0)), torch.arange(n - 1, n))
            # backward: patches of the new frame -> previous `lifetime` frames (and itself)
            append(torch.arange(M * max(n - 1, 0), M * n), torch.arange(max(n - lifetime, 0), n))
        if _ < n_frames - 1:
            keep = (kk // M) >= n - removal        # keyframe(): drop edges outside the removal window
            ii, jj, kk = ii[keep], jj[keep], kk[keep]
    return ii, jj, kk


@dataclass
class SyntheticState:
    cfg: dict
    n: int                      # number of frames (t1 of the BA window)
    t0: int                     # first free pose of the BA window
    ii: torch.Tensor            # [E] int64 source frame of each edge
    jj: torch.Tensor            # [E] int64 target frame
    kk: torch.Tensor            # [E] int64 patch id (frame * M + slot)
    poses: torch.Tensor         # [N,7] fp32
    patches: torch.Tensor       # [N*M,3,3,3] fp32
    intrinsics: torch.Tensor    # [N,4] fp32 (already /4)
    fmap1: torch.Tensor = None  # [1,mem,128,h,w]   logical NCHW, memory per `channels_last`
    fmap2: torch.Tensor = None  # [1,mem,128,h/4,w/4]
    gmap: torch.Tensor = None   # [1,mem*M,128,3,3]
    imap: torch.Tensor = None   # [1,mem*M,384]
    net: torch.Tensor = None    # [1,E,384]
    extras: dict = field(default_factory=dict)
    points: torch.Tensor = None  # [N*M,3] fp32 world points of the patch centres (pg.points_), or None: no map
    colors: torch.Tensor = None  # [N,M,3] uint8 viewer colours of the patches (pg.colors_), or None

    @property
    def E(self):
        return self.ii.numel()


def _trajectory(n, device, dtype=torch.float32):
    """Smooth camera path: 0.05 units/frame along x, 1 degree/frame yaw (SURVEY 8(d)).  [n,7]"""
    out = torch.zeros(n, 7, dtype=torch.float64)
    for t in range(n):
        yaw = math.radians(1.0) * t
        out[t, 0] = -0.05 * t
        out[t, 2] = 0.01 * t
        out[t, 4] = math.sin(0.5 * yaw)      # rotation about y
        out[t, 6] = math.cos(0.5 * yaw)
    return out.to(device=device, dtype=dtype)


def add_map(state):
    """give `state` the map buffers of dpvo.py:68-72, in the reference's layouts: points fp32 [N M, 3] (pg.points_) and
    colors uint8 [N, M, 3] (pg.colors_), N = its pose slots; zero-filled.  Returns the state."""
    N, M = state.poses.shape[0], int(state.cfg["M"])
    state.points = torch.zeros(N * M, 3, device=state.poses.device)
    state.colors = torch.zeros(N, M, 3, dtype=torch.uint8, device=state.poses.device)
    return state


def check_map(state, what):
    """reject map buffers that are not in the layouts add_map gives (state: one stream, or a StreamBatch whose pose
    rows are all its streams' frames)"""
    N, M, dev = state.poses.shape[0], int(state.cfg["M"]), state.poses.device
    for name, shape, dtype in (("points", (N * M, 3), torch.float32), ("colors", (N, M, 3), torch.uint8)):
        t = getattr(state, name, None)
        if t is None:
            continue
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != shape or t.dtype != dtype or not t.is_contiguous() or t.device != dev:
            got = (tuple(t.shape), t.dtype, str(t.device)) if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError("%s: %s must be a contiguous %s tensor %s on %s (the state's %d pose slots x M=%d), got %s"
                             % (what, name, dtype, list(shape), dev, N, M, got))


def make_state(config="default", n_frames=30, device="cuda", seed=1234, features=True, dtype=torch.half,
               channels_last=True, buffer=64, mem=36, noise=0.0, map=False):
    """Build a steady-state synthetic DPVO state.  `buffer` is the number of pose slots allocated
    (the reference allocates 4096); `mem` the feature ring size (dpvo.py:58).  map=True adds the map buffers
    (`add_map`): UpdateRunner then writes the patch points every step and the encoders the patch colours."""
    cfg = dict(CONFIGS[config]) if isinstance(config, str) else dict(config)
    M = cfg["M"]
    g = torch.Generator(device="cpu").manual_seed(seed)
    ii, jj, kk = replay_edges(n_frames, M, cfg["lifetime"], cfg["removal"])
    n = n_frames
    assert n < buffer and n <= mem, "synthetic state keeps all live frames inside the ring buffers"
    h, w = cfg["ht"] // 4, cfg["wd"] // 4
    fx, fy, cx, cy = [v / 4.0 for v in cfg["intrinsics"]]

    poses = torch.zeros(buffer, 7)
    poses[:, 6] = 1.0
    poses[:n] = _trajectory(n, "cpu")
    if noise > 0:
        poses[1:n, :3] += noise * torch.randn(n - 1, 3, generator=g)
    px = torch.randint(1, w - 1, (buffer * M,), generator=g).float()
    py = torch.randint(1, h - 1, (buffer * M,), generator=g).float()
    offs = torch.tensor([-1.0, 0.0, 1.0])
    patches = torch.zeros(buffer * M, 3, 3, 3)
    patches[:, 0] = px[:, None, None] + offs[None, None, :]
    patches[:, 1] = py[:, None, None] + offs[None, :, None]
    patches[:, 2] = (0.25 + 0.75 * torch.rand(buffer * M, generator=g))[:, None, None]
    intr = torch.tensor([fx, fy, cx, cy]).repeat(buffer, 1)

    st = SyntheticState(cfg=cfg, n=n, t0=max(n - cfg["opt_window"], 1),
                        ii=ii.to(device), jj=jj.to(device), kk=kk.to(device),
                        poses=poses.to(device), patches=patches.to(device), intrinsics=intr.to(device))
    if features:
        gd = torch.Generator(device=device).manual_seed(seed + 1)
        # features are generated directly on the device (177 MB for the default level-0 pyramid)
        if channels_last:
            f1 = (torch.randn(1, mem, h, w, 128, generator=gd, device=device, dtype=torch.float32) / 4).to(dtype).permute(0, 1, 4, 2, 3)
        else:
            f1 = (torch.randn(1, mem, 128, h, w, generator=gd, device=device, dtype=torch.float32) / 4).to(dtype)
        f2 = torch.nn.functional.avg_pool2d(f1[0].float(), 4, 4).to(dtype)[None]
        if channels_last:
            f2 = f2.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
            gm = (torch.randn(1, mem * M, 3, 3, 128, generator=gd, device=device) / 4).to(dtype).permute(0, 1, 4, 2, 3)
        else:
            gm = (torch.randn(1, mem * M, 128, 3, 3, generator=gd, device=device) / 4).to(dtype)
        st.fmap1, st.fmap2, st.gmap = f1, f2, gm
        st.imap = (torch.randn(1, mem * M, 384, generator=gd, device=device) / 4).to(dtype)
        st.net = torch.zeros(1, st.E, 384, device=device, dtype=dtype)
    if map:
        add_map(st)
    return st


def make_batch(config="default", B=2, seeds=None, n_frames=30, device="cuda", frames_per_stream=64, mem=36, map=False):
    """B independent steady-state streams in one streams.StreamBatch: stream b is make_state(config, n_frames[b],
    seed=seeds[b]) (an int n_frames serves every stream), with frames_per_stream pose slots and a ring of `mem`.
    map=True gives the batch (and every stream) the map buffers."""
    from .streams import StreamBatch
    cfg = dict(CONFIGS[config]) if isinstance(config, str) else dict(config)
    seeds = [1234 + 17 * b for b in range(B)] if seeds is None else list(seeds)
    frames = [n_frames] * B if isinstance(n_frames, int) else list(n_frames)
    if len(seeds) != B or len(frames) != B:
        raise ValueError("make_batch: one seed and one frame count per stream")
    batch = StreamBatch(B, cfg, frames_per_stream, mem, mem, device=device, map=map)
    for b in range(B):
        batch.load(b, make_state(cfg, frames[b], device=device, seed=seeds[b], buffer=frames_per_stream, mem=mem))
    batch.set_edges()
    return batch


def _look(t, period, radius, dtype=torch.float64):
    """world -> camera pose of frame t on a closed loop: the camera centre circles (radius) in the x-z plane once per
    `period` frames while the heading swings by +-0.1 rad, so frame t and t + period see the scene from the same place"""
    th = 2.0 * math.pi * t / period
    c = torch.tensor([radius * (math.cos(th) - 1.0), 0.0, radius * math.sin(th)], dtype=dtype)
    yaw = 0.1 * math.sin(th)
    q = torch.tensor([0.0, math.sin(0.5 * yaw), 0.0, math.cos(0.5 * yaw)], dtype=dtype)   # camera -> world rotation
    R = torch.tensor([[math.cos(yaw), 0.0, math.sin(yaw)], [0.0, 1.0, 0.0], [-math.sin(yaw), 0.0, math.cos(yaw)]], dtype=dtype)
    # world -> camera: R^T (X - c);  as [t, q]: t = -R^T c, q = conj(q)
    out = torch.zeros(7, dtype=dtype)
    out[:3] = -(R.T @ c)
    out[3:6] = -q[:3]
    out[6] = q[3]
    return out


def make_loop_state(config="fast", n_frames=60, period=20, radius=2.0, noise=1e-3, max_edge_age=1000, buffer=None,
                    mem=36, device="cuda", seed=1234, features=True, dtype=torch.half):
    """A stream that drives a closed loop again and again (one lap per `period` frames), for loop closure: the patches
    of every frame are M points of ONE 3-D scene (points at depth 4..8 in front of the loop) with their true pixel
    positions and inverse depths, so frame t and frame t + period reproject onto each other and their loop score is
    close to zero, while frames half a lap apart score tens of pixels.  `noise` jitters every pose's translation so
    that no two candidate scores tie.  The rings hold `mem` frames of feature maps and pmem = max_edge_age frames of
    patch features (dpvo.py:58-61); the edge lists are the steady-state window of replay_edges.  buffer (pose slots)
    defaults to n_frames + 2, the last slot being free for DevicePatchGraph's dummy frame."""
    cfg = dict(CONFIGS[config]) if isinstance(config, str) else dict(config)
    cfg["max_edge_age"] = int(max_edge_age)
    M = cfg["M"]
    buffer = n_frames + 2 if buffer is None else int(buffer)
    assert n_frames < buffer
    g = torch.Generator(device="cpu").manual_seed(seed)
    h, w = cfg["ht"] // 4, cfg["wd"] // 4
    fx, fy, cx, cy = [v / 4.0 for v in cfg["intrinsics"]]
    scene = torch.empty(20000, 3, dtype=torch.float64)
    scene[:, 0] = (torch.rand(20000, generator=g, dtype=torch.float64) - 0.5) * 16.0 - radius
    scene[:, 1] = (torch.rand(20000, generator=g, dtype=torch.float64) - 0.5) * 8.0
    scene[:, 2] = 4.0 + 4.0 * torch.rand(20000, generator=g, dtype=torch.float64) + radius
    poses = torch.zeros(buffer, 7, dtype=torch.float64)
    poses[:, 6] = 1.0
    patches = torch.zeros(buffer * M, 3, 3, 3)
    offs = torch.tensor([-1.0, 0.0, 1.0])
    for t in range(n_frames):
        P = _look(t, period, radius)
        tq, q = P[:3], P[3:]
        # rotate the scene into the camera: q_rot(q, X) + t
        v = q[:3].expand_as(scene)
        uv = 2.0 * torch.cross(v, scene, dim=1)
        Xc = scene + q[3] * uv + torch.cross(v, uv, dim=1) + tq
        u = fx * Xc[:, 0] / Xc[:, 2] + cx
        vv = fy * Xc[:, 1] / Xc[:, 2] + cy
        ok = (Xc[:, 2] > 1.0) & (u > 1) & (u < w - 2) & (vv > 1) & (vv < h - 2)
        idx = torch.nonzero(ok).view(-1)
        assert idx.numel() >= M, "make_loop_state: too few scene points in view"
        pick = idx[torch.randperm(idx.numel(), generator=g)[:M]]
        k = slice(t * M, (t + 1) * M)
        patches[k, 0] = (u[pick].float()[:, None, None] + offs[None, None, :])
        patches[k, 1] = (vv[pick].float()[:, None, None] + offs[None, :, None])
        patches[k, 2] = (1.0 / Xc[pick, 2]).float()[:, None, None]
        poses[t] = P
    if noise > 0:
        poses[:n_frames, :3] += noise * torch.randn(n_frames, 3, generator=g, dtype=torch.float64)
    intr = torch.tensor([fx, fy, cx, cy]).repeat(buffer, 1)
    ii, jj, kk = replay_edges(n_frames, M, cfg["lifetime"], cfg["removal"])
    st = SyntheticState(cfg=cfg, n=n_frames, t0=max(n_frames - cfg["opt_window"], 1), ii=ii.to(device), jj=jj.to(device),
                        kk=kk.to(device), poses=poses.float().to(device), patches=patches.to(device), intrinsics=intr.to(device))
    if features:
        pmem = int(max_edge_age)
        gd = torch.Generator(device=device).manual_seed(seed + 1)
        f1 = (torch.randn(1, mem, h, w, 128, generator=gd, device=device) / 4).to(dtype).permute(0, 1, 4, 2, 3)
        f2 = torch.nn.functional.avg_pool2d(f1[0].float(), 4, 4).to(dtype)[None]
        st.fmap1 = f1
        st.fmap2 = f2.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
        st.gmap = (torch.randn(1, pmem * M, 3, 3, 128, generator=gd, device=device) / 4).to(dtype).permute(0, 1, 4, 2, 3)
        st.imap = (torch.randn(1, pmem * M, 384, generator=gd, device=device) / 4).to(dtype)
        st.net = torch.zeros(1, st.E, 384, device=device, dtype=dtype)
    return st


def make_stop_go_state(config="fast", n_frames=16, total=200, stop=8, go=8, speed=0.4, yaw_deg=0.5, buffer=None, mem=36,
                       device="cuda", seed=1234, features=True, dtype=torch.half):
    """A camera that stops and goes, for keyframe culling: over `total` timestamps it alternates `stop` frames standing
    still (a 1e-4 jitter) with `go` frames moving `speed` units per frame sideways while turning `yaw_deg` per frame.
    DPVO's motion test between frames two apart then gives about 0 px while stopped and tens of px while moving
    (fx / 4 * speed * 2 * inverse depth, inverse depths 0.25..1), far from the 15 px threshold on both sides.
    The state holds the first `n_frames` timestamps as frames (edges: replay_edges); extras["trajectory"] [total, 7]
    and extras["patches"] [total M, 3, 3, 3] hold every timestamp's pose and patches for a tracking loop to add.
    buffer (pose slots) defaults to total + 2, the last slot being free for DevicePatchGraph's dummy frame; the rings
    hold `mem` frames (pmem = mem)."""
    cfg = dict(CONFIGS[config]) if isinstance(config, str) else dict(config)
    M = cfg["M"]
    buffer = total + 2 if buffer is None else int(buffer)
    assert n_frames <= total < buffer
    g = torch.Generator(device="cpu").manual_seed(seed)
    h, w = cfg["ht"] // 4, cfg["wd"] // 4
    fx, fy, cx, cy = [v / 4.0 for v in cfg["intrinsics"]]
    traj = torch.zeros(total, 7, dtype=torch.float64)
    x, yaw = 0.0, 0.0
    for t in range(total):
        if t > 0 and (t - 1) % (stop + go) >= stop:            # timestamps stop + 1 .. stop + go of each period move
            x += speed
            yaw += math.radians(yaw_deg)
        traj[t, 0] = -x
        traj[t, 4] = math.sin(0.5 * yaw)
        traj[t, 6] = math.cos(0.5 * yaw)
    traj[:, :3] += 1e-4 * torch.randn(total, 3, generator=g, dtype=torch.float64)
    traj = traj.float()
    px = torch.randint(1, w - 1, (total * M,), generator=g).float()
    py = torch.randint(1, h - 1, (total * M,), generator=g).float()
    offs = torch.tensor([-1.0, 0.0, 1.0])
    allp = torch.zeros(total * M, 3, 3, 3)
    allp[:, 0] = px[:, None, None] + offs[None, None, :]
    allp[:, 1] = py[:, None, None] + offs[None, :, None]
    allp[:, 2] = (0.25 + 0.75 * torch.rand(total * M, generator=g))[:, None, None]
    poses = torch.zeros(buffer, 7)
    poses[:, 6] = 1.0
    poses[:n_frames] = traj[:n_frames]
    patches = torch.zeros(buffer * M, 3, 3, 3)
    patches[:, 2] = 1.0
    patches[:n_frames * M] = allp[:n_frames * M]
    intr = torch.tensor([fx, fy, cx, cy]).repeat(buffer, 1)
    ii, jj, kk = replay_edges(n_frames, M, cfg["lifetime"], cfg["removal"])
    st = SyntheticState(cfg=cfg, n=n_frames, t0=max(n_frames - cfg["opt_window"], 1), ii=ii.to(device), jj=jj.to(device),
                        kk=kk.to(device), poses=poses.to(device), patches=patches.to(device), intrinsics=intr.to(device))
    st.extras["trajectory"] = traj.to(device)
    st.extras["patches"] = allp.to(device)
    if features:
        gd = torch.Generator(device=device).manual_seed(seed + 1)
        f1 = (torch.randn(1, mem, h, w, 128, generator=gd, device=device) / 4).to(dtype).permute(0, 1, 4, 2, 3)
        f2 = torch.nn.functional.avg_pool2d(f1[0].float(), 4, 4).to(dtype)[None]
        st.fmap1 = f1
        st.fmap2 = f2.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
        st.gmap = (torch.randn(1, mem * M, 3, 3, 128, generator=gd, device=device) / 4).to(dtype).permute(0, 1, 4, 2, 3)
        st.imap = (torch.randn(1, mem * M, 384, generator=gd, device=device) / 4).to(dtype)
        st.net = torch.zeros(1, st.E, 384, device=device, dtype=dtype)
    return st
