"""lietorch_backends on the device vs the CPU oracle (which is pinned by the reference's own tests)."""
import pytest
import torch

from oracle import lie as OL

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rand(gid, n, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    G = OL.GROUPS[gid]
    a = torch.randn(n, G.K, generator=g, dtype=torch.float64)
    if gid in (2, 4):
        a *= 0.5              # scaled groups: Sim3's Jacobians are truncated series (sim3.h:169-191), meant for small tangents
    X = G.exp(0.7 * torch.randn(n, G.K, generator=g, dtype=torch.float64))
    Y = G.exp(0.7 * torch.randn(n, G.K, generator=g, dtype=torch.float64))
    if gid == 3:
        X[:, :3] *= 3
    p3 = torch.randn(n, 3, generator=g, dtype=torch.float64)
    p4 = torch.randn(n, 4, generator=g, dtype=torch.float64)
    return [t.to(dtype) for t in (a, X, Y, p3, p4)]


@pytest.mark.parametrize("gid", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-12), (torch.float32, 2e-5)])
def test_forward_and_backward_ops(ext, gid, dtype, tol):
    L = ext[2]
    G = OL.GROUPS[gid]
    if gid in (2, 4) and dtype == torch.float64:
        # the oracle keeps lietorch's closed forms for W(phi, sigma), which lose ~ulp / |sigma| in double at small random
        # sigma; tests/test_lie_edges_gpu.py holds these kernels to 1e-12 against the cancellation-free reference
        tol = 1e-10
    n = 1000
    a, X, Y, p3, p4 = _rand(gid, n, dtype, 11)
    ad, Xd, Yd, p3d, p4d = [t.to(DEV) for t in (a, X, Y, p3, p4)]
    g = torch.Generator().manual_seed(12)
    gN = torch.randn(n, G.N, generator=g, dtype=torch.float64).to(dtype)
    gK = torch.randn(n, G.K, generator=g, dtype=torch.float64).to(dtype)
    g3 = torch.randn(n, 3, generator=g, dtype=torch.float64).to(dtype)
    g4 = torch.randn(n, 4, generator=g, dtype=torch.float64).to(dtype)
    a64, X64, Y64, p364, p464 = [t.double() for t in (a, X, Y, p3, p4)]

    def close(dev, ref, what):
        err = (dev.cpu().double() - ref).abs().max().item()
        assert err <= tol * max(1.0, ref.abs().max().item()), (what, err)

    close(L.expm(gid, ad), G.exp(a64), "exp")
    close(L.logm(gid, Xd), G.log(X64), "log")
    close(L.inv(gid, Xd), G.inv(X64), "inv")
    close(L.mul(gid, Xd, Yd), G.mul(X64, Y64), "mul")
    close(L.adj(gid, Xd, ad), G.adj(X64, a64), "adj")
    close(L.adjT(gid, Xd, ad), G.adjT(X64, a64), "adjT")
    close(L.act(gid, Xd, p3d), G.act(X64, p364), "act")
    close(L.act4(gid, Xd, p4d), G.act4(X64, p464), "act4")
    close(L.as_matrix(gid, Xd), G.matrix(X64), "as_matrix")
    close(L.projector(gid, Xd), G.projector(X64), "projector")
    close(L.Jinv(gid, Xd, ad), OL.jinv(gid, X64, a64), "Jinv")
    # backward operators (lietorch_gpu.cu:32-256)
    close(L.expm_backward(gid, gN.to(DEV), ad)[0], OL.expm_backward(gid, gN.double(), a64), "exp_b")
    close(L.logm_backward(gid, gK.to(DEV), Xd)[0], OL.logm_backward(gid, gK.double(), X64), "log_b")
    close(L.inv_backward(gid, gN.to(DEV), Xd)[0], OL.inv_backward(gid, gN.double(), X64), "inv_b")
    for dev, ref, nm in zip(L.mul_backward(gid, gN.to(DEV), Xd, Yd), OL.mul_backward(gid, gN.double(), X64, Y64), ("mul_bX", "mul_bY")):
        close(dev, ref, nm)
    for dev, ref, nm in zip(L.adj_backward(gid, gK.to(DEV), Xd, ad), OL.adj_backward(gid, gK.double(), X64, a64), ("adj_bX", "adj_ba")):
        close(dev, ref, nm)
    for dev, ref, nm in zip(L.adjT_backward(gid, gK.to(DEV), Xd, ad), OL.adjT_backward(gid, gK.double(), X64, a64), ("adjT_bX", "adjT_ba")):
        close(dev, ref, nm)
    for dev, ref, nm in zip(L.act_backward(gid, g3.to(DEV), Xd, p3d), OL.act_backward(gid, g3.double(), X64, p364), ("act_bX", "act_bp")):
        close(dev, ref, nm)
    for dev, ref, nm in zip(L.act4_backward(gid, g4.to(DEV), Xd, p4d), OL.act4_backward(gid, g4.double(), X64, p464), ("act4_bX", "act4_bp")):
        close(dev, ref, nm)


@pytest.mark.parametrize("gid", [1, 2, 3, 4])
def test_small_angle_and_identity(ext, gid):
    L = ext[2]
    G = OL.GROUPS[gid]
    a = torch.zeros(4, G.K, dtype=torch.float64)
    a[1] = 1e-9
    a[2, -1] = 1e-7
    a[3, 0] = 2.0
    X = L.expm(gid, a.to(DEV))
    loose = gid in (2, 4)     # W(phi, sigma) and its inverse sit between exp and log for the scaled groups
    assert (X.cpu() - G.exp(a)).abs().max().item() < (1e-12 if loose else 1e-14)
    assert (L.logm(gid, X).cpu() - a).abs().max().item() < (1e-10 if loose else 1e-12)


def test_reference_identities_through_host_mirror(ext):
    """the reference's forward known-answer tests (run_tests.py:16-52) on the device kernels"""
    from dpvo_b200.lietorch import SE3, SO3, RxSO3, Sim3
    torch.manual_seed(5)
    for Group in (SO3, RxSO3, SE3, Sim3):
        a = .2 * torch.randn(2, 3, 4, 5, Group.manifold_dim, device=DEV).double()
        assert torch.allclose(a, Group.exp(a).log(), atol=1e-8)
        X = Group.exp(.1 * torch.randn(2, 3, 4, 5, Group.manifold_dim, device=DEV).double())
        z = (X * X.inv()).log()
        assert torch.allclose(z, torch.zeros_like(z), atol=1e-8)
        X = Group.exp(torch.randn(2, 3, 4, 5, Group.manifold_dim, device=DEV).double())
        a = torch.randn(2, 3, 4, 5, Group.manifold_dim, device=DEV).double()
        c = ((X * Group.exp(a)) * (Group.exp(X.adj(a)) * X).inv()).log()
        assert torch.allclose(c, torch.zeros_like(c), atol=1e-8)
        X = Group.exp(torch.randn(1, Group.manifold_dim, device=DEV).double())
        p = torch.randn(1, 3, device=DEV).double()
        p2 = (X.matrix() @ torch.cat([p, torch.ones_like(p[..., :1])], -1)[..., None])[..., 0]
        assert torch.allclose(X.act(p), p2[..., :3], atol=1e-8)


def test_unsupported_groups_raise(ext):
    with pytest.raises(RuntimeError):
        ext[2].expm(7, torch.zeros(2, 7, device=DEV))          # no such group id
    with pytest.raises(RuntimeError):
        ext[2].expm(3, torch.zeros(2, 6))          # CPU tensor: no fallback
