"""ORACLE: host restatement of proximity loop closure (dpvo/patchgraph.py:56-91, dpvo/dpvo.py:223-238, 266-310,
312-326, 449-459, loop_closure/optim_utils.py:23-61) on the candidate layout of dpvo_b200/csrc/loop.cu.

    loop_range / scores   the candidate pairs and their flow scores (fp64)
    select                reduce_edges on a score vector: (i, j) pairs in acceptance order
    HostGraph             the edge lists of the reference (active, loop and inactive), its removal rule, keyframe
                          renumbering and loop proposal
    normalize             PatchGraph.normalize (fp64)
"""
import torch

MIN_GAP = 30


def loop_range(n, removal, max_age, freq, kf_index):
    """(i0, ni, j0, J): sources i0 .. i0 + ni - 1, targets j0 .. j0 + J - 1"""
    l = n - removal
    i0 = max(l - max_age, 0)
    ni = l - i0 if l > 0 else 0
    return i0, ni, n - freq, freq - kf_index


def _act(q, t, X):
    """SE3 [t, q] acting on points X [..., 3]"""
    v = q[..., :3].expand_as(X)
    uv = 2.0 * torch.cross(v, X, dim=-1)
    return X + q[..., 3:4] * uv + torch.cross(v, uv, dim=-1) + t


def _qmul(a, b):
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                        aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], -1)


def _inv(P):
    q = torch.cat([-P[..., 3:6], P[..., 6:7]], -1)
    return torch.cat([-_act(q, torch.zeros_like(P[..., :3]), P[..., :3]), q], -1)


def _mul(A, B):
    q = _qmul(A[..., 3:], B[..., 3:])
    return torch.cat([A[..., :3] + _act(A[..., 3:], torch.zeros_like(B[..., :3]), B[..., :3]), q], -1)


def _norm(P):
    P = P.clone()
    P[..., 3:] = P[..., 3:] / P[..., 3:].norm(dim=-1, keepdim=True)
    return P


def flow(poses, patches, intrinsics, i, j, k):
    """centre-pixel flow of patches k from frames i to j (projective_ops.py:120-130, beta = 0.5) and validity"""
    poses = _norm(poses.double())
    c = patches.double()[k][:, :, 1, 1]                     # [E, 3] (x, y, d)
    Ki, Kj = intrinsics.double()[i], intrinsics.double()[j]
    p = torch.stack([(c[:, 0] - Ki[:, 2]) / Ki[:, 0], (c[:, 1] - Ki[:, 3]) / Ki[:, 1], torch.ones_like(c[:, 0])], -1)
    d = c[:, 2:3]
    Pi, Pj = poses[i], poses[j]

    def proj(G, K, tonly=False):
        X = (p if tonly else _act(G[:, 3:], torch.zeros_like(p), p)) + d * G[:, :3]
        z = X[:, 2].clamp(min=0.1)
        return torch.stack([K[:, 0] * X[:, 0] / z + K[:, 2], K[:, 1] * X[:, 1] / z + K[:, 3]], -1), X[:, 2]

    c0, _ = proj(_mul(Pi, _inv(Pi)), Ki)
    Gij = _mul(Pj, _inv(Pi))
    c1, Z = proj(Gij, Kj)
    c2, _ = proj(Gij, Kj, tonly=True)
    return 0.5 * (c1 - c0).norm(dim=-1) + 0.5 * (c2 - c0).norm(dim=-1), Z > 0.2


def scores(poses, patches, intrinsics, n, M, removal, max_age, freq, kf_index, last_ba=-1000):
    """fp64 [J * max_age] in the layout of dpvo_loop_scores: +inf outside the range or when no proposal is due"""
    i0, ni, j0, J = loop_range(n, removal, max_age, freq, kf_index)
    out = torch.full((J * max_age,), float("inf"), dtype=torch.float64)
    if n - last_ba < freq or ni <= 0:
        return out
    jr, ir = torch.meshgrid(torch.arange(J), torch.arange(ni), indexing="ij")
    jr, ir = jr.reshape(-1), ir.reshape(-1)
    keep = (j0 + jr) >= 0
    jr, ir = jr[keep], ir[keep]
    i = (i0 + ir).repeat_interleave(M)
    j = (j0 + jr).repeat_interleave(M)
    k = i * M + torch.arange(M).repeat(jr.numel())
    f, v = flow(poses, patches, intrinsics, i, j, k)
    f, v = f.view(-1, M), v.view(-1, M)
    cnt = v.sum(1)
    s = torch.where(cnt > 0.75 * M, (f * v).sum(1) / cnt.clamp(min=1), torch.full_like(cnt, float("inf"), dtype=torch.float64))
    out[jr * max_age + ir] = s
    return out


def select(sc, n, removal, max_age, freq, kf_index, thresh=64.0, max_pairs=1000):
    """reduce_edges over a candidate score vector: pairs (i, j) in acceptance order"""
    i0, ni, j0, J = loop_range(n, removal, max_age, freq, kf_index)
    sc = torch.as_tensor(sc).double()
    slots = [s for s in range(J * max_age) if sc[s] < thresh and sc[s] < 1000]
    slots.sort(key=lambda s: (float(sc[s]), s))
    sup, out = set(), []
    for s in slots:
        if len(out) >= max_pairs:
            break
        jr, ir = divmod(s, max_age)
        i, j = i0 + ir, j0 + jr
        if j - i < MIN_GAP or (i, j) in sup:
            continue
        out.append((i, j))
        sup.update({(i - 1, j), (i, j), (i + 1, j)})
    return out


def normalize(poses, patches, n, M):
    """PatchGraph.normalize in fp64: returns (poses [N, 7], patches [K, 3, P, P]) with frames [0, n) normalized"""
    poses, patches = poses.double().clone(), patches.double().clone()
    s = patches[:n * M, 2].mean()
    patches[:n * M, 2] /= s
    poses[:n, :3] *= s
    poses[:n] = _mul(_norm(poses[:n]), _inv(_norm(poses[0:1])).expand(n, 7))
    return poses, patches


class HostGraph:
    """the reference's growing edge lists: active (ii, jj, kk, target, weight) and inactive ones, in list order"""

    def __init__(self, M, removal, opt_window):
        self.M, self.removal, self.opt_window = M, removal, opt_window
        self.act = []            # [ii, jj, kk]
        self.inac = []           # [ii, jj, kk, target (2), weight (2)]

    def append(self, ii, jj, kk):
        self.act += [[int(a), int(b), int(c)] for a, b, c in zip(ii, jj, kk)]

    def append_pairs(self, pairs):
        for i, j in pairs:
            self.append([i] * self.M, [j] * self.M, [i * self.M + m for m in range(self.M)])

    def remove_window(self, n, target_of):
        """dpvo.py:300-310 with LOOP_CLOSURE: target_of(edge) -> (target, weight) of an active edge"""
        keep = []
        for e in self.act:
            i, j, k = e
            drop = k // self.M < n - self.removal and not ((j - i) > MIN_GAP and j > n - self.opt_window)
            if drop:
                self.inac.append(e + list(target_of(e)))
            else:
                keep.append(e)
        self.act = keep

    def remove_keyframe(self, k):
        """dpvo.py:279-286: the inactive lists are untouched"""
        keep = []
        for i, j, kk in self.act:
            if i == k or j == k:
                continue
            if i > k:
                i, kk = i - 1, kk - self.M
            if j > k:
                j -= 1
            keep.append([i, j, kk])
        self.act = keep
