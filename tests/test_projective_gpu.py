"""dpvo_b200.projective_ops (interface of dpvo/projective_ops.py:19-130) on the device kernels vs the oracle
restatement (oracle/ba.py:transform, pinned bit-exactly to the reference file on the CPU), including the
closed-form Jacobians, autograd through the lietorch kernels, the Sim3 column and flow_mag / point_cloud."""
import pytest
import torch

from oracle import ba as OB, lie as OL
from dpvo_b200 import synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _state(seed=5, n=14):
    st = synthetic.make_state("fast", n, device="cpu", features=False, seed=seed, noise=0.03)
    g = torch.Generator().manual_seed(seed)
    st.patches[:, 2] *= 0.5 + torch.rand(st.patches.shape[0], 1, 1, generator=g)
    return st


def test_transform_and_jacobians_match_oracle(ext):
    from dpvo_b200 import projective_ops as pops
    from dpvo_b200.lietorch import SE3
    st = _state()
    dev = [t.to(DEV) for t in (st.poses[None], st.patches[None], st.intrinsics[None], st.ii, st.jj, st.kk)]
    x, v, (Ji, Jj, Jz) = pops.transform(SE3(dev[0]), *dev[1:], jacobian=True)
    ox, ov, (oJi, oJj, oJz) = OB.transform(st.poses.double()[None], st.patches.double()[None], st.intrinsics.double()[None],
                                           st.ii, st.jj, st.kk, jacobian=True)
    assert x.shape == ox.shape and Ji.shape == oJi.shape and Jj.shape == oJj.shape and Jz.shape == oJz.shape
    for mine, theirs, nm in ((x, ox, "coords"), (v, ov, "valid"), (Ji, oJi, "Ji"), (Jj, oJj, "Jj"), (Jz, oJz, "Jz")):
        err = (mine.cpu().double() - theirs).abs().max().item()
        assert err <= 2e-4 * max(1.0, theirs.abs().max().item()), (nm, err)
    # valid / depth variants
    x2, v2 = pops.transform(SE3(dev[0]), *dev[1:], valid=True)
    o2, ov2 = OB.transform(st.poses.double()[None], st.patches.double()[None], st.intrinsics.double()[None], st.ii, st.jj, st.kk, valid=True)
    assert torch.equal(x2, x) and (v2.cpu().double() - ov2).abs().max().item() == 0
    x3 = pops.transform(SE3(dev[0]), *dev[1:], depth=True)
    assert x3.shape[-1] == 3 and torch.equal(x3[..., :2], x)
    # the fused inference kernel is the same map in the layout corr consumes
    xf = pops.transform_fused(SE3(dev[0]), *dev[1:])
    assert (xf.permute(0, 1, 3, 4, 2) - x).abs().max().item() < 2e-3


def test_transform_autograd_matches_oracle_autograd(ext):
    """d(sum w * coords)/d(patches) through our lietorch backward kernels vs autograd through the fp64 oracle"""
    from dpvo_b200 import projective_ops as pops
    from dpvo_b200.lietorch import SE3
    st = _state(seed=6, n=10)
    g = torch.Generator().manual_seed(1)
    w = torch.randn(1, st.E, 3, 3, 2, generator=g)
    q = st.patches[None].to(DEV).requires_grad_(True)
    x = pops.transform(SE3(st.poses[None].to(DEV)), q, st.intrinsics[None].to(DEV), st.ii.to(DEV), st.jj.to(DEV), st.kk.to(DEV))
    (x * w.to(DEV)).sum().backward()
    q64 = st.patches.double()[None].requires_grad_(True)
    ox = OB.transform(st.poses.double()[None], q64, st.intrinsics.double()[None], st.ii, st.jj, st.kk)
    (ox * w.double()).sum().backward()
    assert (q.grad.cpu().double() - q64.grad).abs().max().item() <= 2e-4 * q64.grad.abs().max().item()


def test_sim3_jacobian_column_by_finite_differences(ext):
    """Sim3 poses with unit scale reproduce the SE3 columns; the 7th (scale) column is checked numerically"""
    from dpvo_b200 import projective_ops as pops
    from dpvo_b200.lietorch import SE3, Sim3
    st = _state(seed=7, n=9)
    P = st.poses.double()[None].to(DEV)
    S = torch.cat([P, torch.ones_like(P[..., :1])], -1)
    args = (st.patches.double()[None].to(DEV), st.intrinsics.double()[None].to(DEV), st.ii.to(DEV), st.jj.to(DEV), st.kk.to(DEV))
    x_se, _, (Ji_se, Jj_se, Jz_se) = pops.transform(SE3(P), *args, jacobian=True)
    x_si, _, (Ji, Jj, Jz) = pops.transform(Sim3(S), *args, jacobian=True)
    assert Jj.shape[-1] == 7 and (x_si - x_se).abs().max().item() < 1e-9
    assert (Jj[..., :6] - Jj_se).abs().max().item() < 1e-9 and (Ji[..., :6] - Ji_se).abs().max().item() < 1e-9
    assert (Jz - Jz_se).abs().max().item() < 1e-9
    # numeric derivative of the centre pixel w.r.t. a left scale perturbation of pose j:  G_j <- Exp(0,0,eps) G_j
    eps = 1e-6
    xi = torch.zeros(1, P.shape[1], 7, dtype=torch.float64, device=DEV)
    xi[..., 6] = eps
    moved = Sim3.exp(xi) * Sim3(S)
    # only frame-j poses move: build per-edge poses by hand
    def centre(pose_i, pose_j):
        Gij = pose_j * pose_i.inv()
        X = Gij[:, :, None, None] * pops.iproj(args[0][:, args[4]], args[1][:, args[2]])
        return pops.proj(X, args[1][:, args[3]])[:, :, 1, 1]
    base = centre(Sim3(S)[:, args[2]], Sim3(S)[:, args[3]])
    pert = centre(Sim3(S)[:, args[2]], moved[:, args[3]])
    num = (pert - base) / eps
    assert (num - Jj[..., 6]).abs().max().item() <= 1e-4 * max(1.0, Jj[..., 6].abs().max().item())


def test_flow_mag_and_point_cloud(ext):
    from dpvo_b200 import projective_ops as pops
    from dpvo_b200.lietorch import SE3
    st = _state(seed=8, n=12)
    poses, patches, intr = st.poses.double()[None], st.patches.double()[None], st.intrinsics.double()[None]
    sel = (st.ii == 6) & (st.jj == 8)
    ii, jj, kk = st.ii[sel], st.jj[sel], st.kk[sel]
    # oracle flow_mag (projective_ops.py:120-130 restated with the oracle transform; tonly = rotation dropped)
    c0 = OB.transform(poses, patches, intr, ii, ii, kk)
    c1, val = OB.transform(poses, patches, intr, ii, jj, kk, valid=True)
    Gij = OL.GROUPS[3].mul(poses[:, jj], OL.GROUPS[3].inv(poses[:, ii])).clone()
    Gij[..., 3:] = torch.tensor([0, 0, 0, 1.0], dtype=torch.float64)
    X1 = OL.GROUPS[3].act4(Gij[:, :, None, None], OB.iproj(patches[:, kk], intr[:, ii]))
    c2 = OB.proj(X1, intr[:, jj])
    ref = 0.5 * (c1 - c0).norm(dim=-1) + 0.5 * (c2 - c0).norm(dim=-1)
    mag, ok = pops.flow_mag(SE3(poses.float().to(DEV)), patches.float().to(DEV), intr.float().to(DEV), ii.to(DEV), jj.to(DEV), kk.to(DEV), beta=0.5)
    assert (mag.cpu().double() - ref).abs().max().item() < 2e-3
    assert torch.equal(ok.cpu(), val > 0.5)
    ix = (torch.arange(st.n * st.cfg["M"]) // st.cfg["M"])
    pc = pops.point_cloud(SE3(poses.float().to(DEV)), patches[:, :ix.numel()].float().to(DEV), intr.float().to(DEV), ix.to(DEV))
    refpc = OL.GROUPS[3].act4(OL.GROUPS[3].inv(poses[:, ix])[:, :, None, None], OB.iproj(patches[:, :ix.numel()], intr[:, ix]))
    assert (pc.cpu().double() - refpc).abs().max().item() < 1e-4 * refpc.abs().max().item()


def test_reproject_clamped_depth_clamp_branch(ext):
    """reproject_clamped (the correlation's input) where the depth clamp 1 / max(Z, 0.1) acts: Z in {-1, 0, 0.05, just
    below and above 0.1, 0.2} (frame 1 is frame 0 moved by -1 along z, so Z = 1 - d exactly in fp32), edges with
    ii = jj, and a frame whose quaternion is 1e-3 off unit length; against oracle/ba.py's transform within a bar that
    scales with the magnitudes: out = f X / max(Z, 0.1) + c with X, Z from fp32 rotations of |p| + |d| |t|"""
    P = 3
    d_just = [float(torch.tensor(0.9, dtype=torch.float32)), float(torch.nextafter(torch.tensor(0.9), torch.tensor(1.0)))]
    depths = torch.tensor([2.0, 1.0, 0.95] + d_just + [0.8, 0.5])
    q = torch.tensor([0.1, 0.2, 0.05, 0.97])
    q = q / q.norm() * (1 + 1e-3)
    poses = torch.tensor([[0, 0, 0, 0, 0, 0, 1.0], [0, 0, -1.0, 0, 0, 0, 1.0], [0.3, -0.2, -0.9] + q.tolist()])
    intr = torch.tensor([[320.0, 300.0, 320.0, 240.0]]).repeat(3, 1)
    g = torch.Generator().manual_seed(7)
    N = depths.numel()
    patches = torch.zeros(N, 3, P, P)
    patches[:, 0] = 320 + 60 * torch.randn(N, P, P, generator=g)
    patches[:, 1] = 240 + 60 * torch.randn(N, P, P, generator=g)
    patches[:, 2] = depths[:, None, None]
    pairs = [(0, 1), (1, 1), (0, 0), (0, 2), (2, 2), (2, 1), (1, 0)]
    ii = torch.tensor([a for a, _ in pairs for _ in range(N)])
    jj = torch.tensor([b for _, b in pairs for _ in range(N)])
    kk = torch.arange(N).repeat(len(pairs))
    out = ext[3].reproject_clamped(poses.to(DEV)[None], patches.to(DEV)[None], intr.to(DEV)[None], ii.to(DEV), jj.to(DEV),
                                   kk.to(DEV))[0].cpu().double().permute(0, 2, 3, 1)           # [E, P, P, 2]
    p64, x64, k64 = poses.double()[None], patches.double()[None], intr.double()[None]
    ref = OB.transform(p64, x64, k64, ii, jj, kk)[0]
    X0 = OB.iproj(x64[:, kk], k64[:, ii])
    X1 = OL.se3_act4(OL.se3_mul(p64[:, jj], OL.se3_inv(p64[:, ii]))[:, :, None, None], X0)[0]
    Z = X1[..., 2]
    assert bool((Z < 0.1).any() & (Z > 0.1).any() & (Z <= 0).any() & ((Z - 0.1).abs() < 1e-7).any())
    Zc = Z.clamp(min=0.1)
    mag = X0[0, ..., :3].norm(dim=-1) + x64[0, kk, 2].abs() * (p64[0, ii, :3].norm(dim=-1) + p64[0, jj, :3].norm(dim=-1))[:, None, None]
    f, c = k64[0, jj, :2][:, None, None], k64[0, jj, 2:][:, None, None]
    XY = X1[..., :2].abs()
    bar = 16 * 2.0 ** -24 * (f * (mag[..., None] + XY * mag[..., None] / Zc[..., None] + XY) / Zc[..., None] +
                             f * XY / Zc[..., None] + c.abs())
    err = (out - ref).abs()
    assert bool((err <= bar).all()), float((err / bar).max())
