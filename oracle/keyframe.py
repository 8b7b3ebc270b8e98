"""ORACLE: host restatement of DPVO's keyframe culling (dpvo/dpvo.py:257-300 motionmag / keyframe, :166-198 get_pose /
terminate, :400-444 the timestamp bookkeeping, dpvo/patchgraph.py:84-91 normalize's delta scaling).

    flow9 / motionmag     flow_mag (beta = 0.5) of all 9 pixels of a set of edges, and the mean of one (i, j) set (fp64)
    motion                m = motionmag(i, j) + motionmag(j, i) and the decision m / 2 < thresh
    HostKeyframes         one stream's buffers, rings, edges (oracle.loop.HostGraph) and delta record: keyframe() with
                          every slot copy, the stale slot n - 1 included, add_frame / skip_frame
    scale_deltas          normalize's dP.scale(s)
    terminate             get_pose / terminate's interpolation, poses.inv() (fp64)
"""
import math

import torch

from oracle.loop import HostGraph, _act, _inv, _mul, _norm


def flow9(poses, patches, intrinsics, ii, jj, kk):
    """[E, 9] fp64 flow of every pixel of patches kk from frames ii to jj (projective_ops.py:flow_mag, beta = 0.5);
    the origin is the patch reprojected through P_i P_i^-1 with frame i's intrinsics, as flow_mag's coords0"""
    ii, jj, kk = (torch.as_tensor(x, dtype=torch.long) for x in (ii, jj, kk))
    poses = _norm(poses.double())
    pt = patches.double()[kk].reshape(-1, 3, 9)                  # [E, (x, y, d), 9]
    x, y, d = pt[:, 0], pt[:, 1], pt[:, 2]
    Ki, Kj = intrinsics.double()[ii][:, None, :], intrinsics.double()[jj][:, None, :]
    p = torch.stack([(x - Ki[..., 2]) / Ki[..., 0], (y - Ki[..., 3]) / Ki[..., 1], torch.ones_like(x)], -1)   # [E, 9, 3]
    Pi, Pj = poses[ii][:, None, :].expand(-1, 9, 7), poses[jj][:, None, :].expand(-1, 9, 7)

    def proj(G, K, tonly=False):
        X = (p if tonly else _act(G[..., 3:], torch.zeros_like(p), p)) + d[..., None] * G[..., :3]
        z = X[..., 2].clamp(min=0.1)
        return torch.stack([K[..., 0] * X[..., 0] / z + K[..., 2], K[..., 1] * X[..., 1] / z + K[..., 3]], -1)

    c0 = proj(_mul(Pi, _inv(Pi)), Ki)
    Gij = _mul(Pj, _inv(Pi))
    c1 = proj(Gij, Kj)
    c2 = proj(Gij, Kj, tonly=True)
    return 0.5 * (c1 - c0).norm(dim=-1) + 0.5 * (c2 - c0).norm(dim=-1)


def motionmag(poses, patches, intrinsics, edges, i, j):
    """DPVO.motionmag (dpvo.py:257-264) over an edge list [[ii, jj, kk], ...]: the mean flow of all 9 pixels of the
    edges with (ii, jj) = (i, j); NaN without one"""
    sel = [e for e in edges if e[0] == i and e[1] == j]
    if not sel:
        return float("nan")
    ii, jj, kk = zip(*sel)
    return float(flow9(poses, patches, intrinsics, ii, jj, kk).mean())


def motion(poses, patches, intrinsics, edges, n, ki, thresh):
    """(m, removed) of DPVO.keyframe (dpvo.py:266-272) at frame count n"""
    i, j = n - ki - 1, n - ki + 1
    m = motionmag(poses, patches, intrinsics, edges, i, j) + motionmag(poses, patches, intrinsics, edges, j, i)
    return m, m / 2 < thresh


def rel_pose(Pk, Pk1):
    """dP = P_k P_{k-1}^-1 (fp64)"""
    return _mul(_norm(Pk.double()[None]), _inv(_norm(Pk1.double()[None])))[0]


class HostKeyframes:
    """one stream as DPVO holds it: per-frame buffers (poses [F, 7], patches [F M, 3, 3, 3], intrinsics [F, 4],
    tstamp [F]), the rings (fmap1 / fmap2 [1, mem, ...], gmap / imap [1, pmem M, ...]; None when absent), the edge
    lists of an oracle.loop.HostGraph, n, counter and the delta record {t: (t0, dP fp64 [7])}.  The buffers are CPU
    tensors in the dtypes the device holds, so every copy is exact."""

    def __init__(self, M, poses, patches, intrinsics, n, fmap1=None, fmap2=None, gmap=None, imap=None, tstamp=None,
                 counter=None, graph=None):
        self.M, self.n = int(M), int(n)
        self.poses, self.patches, self.intrinsics = poses.clone(), patches.clone(), intrinsics.clone()
        self.fmap1, self.fmap2 = (None if x is None else x.clone() for x in (fmap1, fmap2))
        self.gmap, self.imap = (None if x is None else x.clone() for x in (gmap, imap))
        F = self.poses.shape[0]
        if tstamp is None:
            tstamp = torch.zeros(F, dtype=torch.long)
            tstamp[:self.n] = torch.arange(self.n)
        self.tstamp = tstamp.clone()
        self.counter = self.n if counter is None else int(counter)
        self.graph = graph
        self.delta = {}

    def add_frame(self):
        self.tstamp[self.n - 1] = self.counter
        self.counter += 1

    def skip_frame(self):
        self.delta[self.counter] = (self.counter - 1, torch.tensor([0, 0, 0, 0, 0, 0, 1.0], dtype=torch.float64))
        self.counter += 1

    def motion(self, ki, thresh):
        return motion(self.poses, self.patches, self.intrinsics, self.graph.act, self.n, ki, thresh)

    def keyframe(self, ki, thresh, removed=None):
        """DPVO.keyframe without the window removal; `removed` overrides the decision (to follow the device's).
        Returns (m, removed)"""
        m, dec = self.motion(ki, thresh)
        removed = dec if removed is None else bool(removed)
        if not removed:
            return m, False
        M, k = self.M, self.n - ki
        t0, t1 = int(self.tstamp[k - 1]), int(self.tstamp[k])
        self.delta[t1] = (t0, rel_pose(self.poses[k], self.poses[k - 1]))
        if self.graph is not None:
            self.graph.remove_keyframe(k)
        for t in range(k, self.n - 1):
            self.tstamp[t] = self.tstamp[t + 1]
            self.poses[t] = self.poses[t + 1]
            self.patches[t * M:(t + 1) * M] = self.patches[(t + 1) * M:(t + 2) * M]
            self.intrinsics[t] = self.intrinsics[t + 1]
            for ring in (self.fmap1, self.fmap2):
                if ring is not None:
                    mem = ring.shape[1]
                    ring[0, t % mem] = ring[0, (t + 1) % mem]
            for ring in (self.gmap, self.imap):
                if ring is not None:
                    pmem = ring.shape[1] // M
                    a, b = (t % pmem) * M, ((t + 1) % pmem) * M
                    ring[0, a:a + M] = ring[0, b:b + M]
        self.n -= 1
        return m, True


def scale_deltas(delta, s):
    """PatchGraph.normalize's dP.scale(s) of every record"""
    out = {}
    for t, (t0, dP) in delta.items():
        dP = dP.clone()
        dP[:3] *= s
        out[t] = (t0, dP)
    return out


def terminate(poses, tstamp, n, delta, counter):
    """get_pose / terminate (dpvo.py:166-198): [counter, 7] fp64, pose(t)^-1 for t < counter"""
    traj = {int(tstamp[i]): _norm(poses[i].double()[None])[0] for i in range(n)}

    def get_pose(t):
        chain = []
        while t not in traj:
            t0, dP = delta[t]
            chain.append(dP)
            t = t0
        P = traj[t]
        for dP in reversed(chain):
            P = _mul(dP[None], P[None])[0]
        return P

    return torch.stack([_inv(get_pose(t)[None])[0] for t in range(counter)])


def pose_distance(A, B):
    """per-row (translation error, rotation angle in rad) between two [N, 7] pose lists"""
    A, B = _norm(A.double()), _norm(B.double())
    dt = (A[:, :3] - B[:, :3]).norm(dim=-1)
    dot = (A[:, 3:] * B[:, 3:]).sum(-1).abs().clamp(max=1.0)
    return dt, 2.0 * torch.acos(dot)


def chain_bar(length, scale=1.0):
    """the fp32 error bar of a pose reached through `length` relative poses: one fp32 rounding of each product, a few
    ulps per step, with the translation scale of the trajectory"""
    return 2e-6 * (length + 1) * max(1.0, scale) + 1e-6 * math.sqrt(length + 1)


def reference_dpvo(st, edges, n, tstamp, ki, thresh):
    """the reference's own DPVO object (dpvo/dpvo.py), built with __new__ on copies of one stream's state, for
    DPVO.keyframe: its PatchGraph holds poses, patches, intrinsics, timestamps and the active edges (ii, jj, kk device
    int64, zero state rows, targets and weights), its rings are copies of the state's in the reference's shapes.  Call
    inside oracle.refimport.reference_python(); LOOP_CLOSURE and CLASSIC_LOOP_CLOSURE are off."""
    import numpy as np
    import dpvo.dpvo as RD
    from dpvo.config import cfg as base
    from dpvo.patchgraph import PatchGraph
    cfg = base.clone()
    M, N = int(st.cfg["M"]), st.poses.shape[0]
    cfg.PATCHES_PER_FRAME, cfg.BUFFER_SIZE = M, N
    cfg.KEYFRAME_INDEX, cfg.KEYFRAME_THRESH = int(ki), float(thresh)
    cfg.REMOVAL_WINDOW, cfg.OPTIMIZATION_WINDOW = int(st.cfg["removal"]), int(st.cfg["opt_window"])
    cfg.LOOP_CLOSURE = cfg.CLASSIC_LOOP_CLOSURE = False
    s = RD.DPVO.__new__(RD.DPVO)
    s.cfg, s.M, s.N, s.P, s.DIM = cfg, M, N, 3, 384
    s.mem, s.pmem = st.fmap1.shape[1], st.gmap.shape[1] // M
    pg = PatchGraph(cfg, 3, 384, s.pmem, device="cuda", dtype=torch.half)
    pg.n, pg.m = int(n), int(n) * M
    pg.tstamps_[:] = np.asarray(tstamp.cpu(), dtype=np.int64)
    pg.poses_[:] = st.poses
    pg.patches_[:] = st.patches.view(N, M, 3, 3, 3)
    pg.intrinsics_[:] = st.intrinsics
    pg.index_[:] = torch.arange(N, device="cuda")[:, None]
    pg.ii, pg.jj, pg.kk = (edges[:, c].to("cuda").contiguous() for c in range(3))
    E = pg.ii.numel()
    pg.net = torch.zeros(1, E, 384, device="cuda", dtype=torch.half)
    pg.weight = torch.zeros(1, E, 2, device="cuda")
    pg.target = torch.zeros(1, E, 2, device="cuda")
    s.pg = pg
    s.imap_ = st.imap.clone()[0].view(s.pmem, M, 384)
    s.gmap_ = st.gmap.clone()[0].unflatten(0, (s.pmem, M))
    s.fmap1_, s.fmap2_ = st.fmap1.clone(), st.fmap2.clone()
    return s
