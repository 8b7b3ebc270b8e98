"""Parity of cuda_corr (forward, backward, patchify) with the CPU oracle, through the shim -> C-ABI."""
import pytest
import torch

from oracle import corr as OC

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _case(seed, M, C=128, S1=40, S2=5, H=30, W=40, dtype=torch.float32, spread=1.0, margin=6.0, cl=False, P=3):
    g = torch.Generator().manual_seed(seed)
    f1 = torch.randn(1, S1, C, P, P, generator=g) / 4
    f2 = torch.randn(1, S2, C, H, W, generator=g) / 4
    cx = torch.rand(M, generator=g) * (W + 2 * margin) - margin
    cy = torch.rand(M, generator=g) * (H + 2 * margin) - margin
    offs = (torch.arange(P).float() - P // 2) * spread
    coords = torch.zeros(1, M, 2, P, P)
    coords[0, :, 0] = cx[:, None, None] + offs[None, None, :] + 0.05 * torch.randn(M, P, P, generator=g)
    coords[0, :, 1] = cy[:, None, None] + offs[None, :, None] + 0.05 * torch.randn(M, P, P, generator=g)
    ii = torch.randint(0, S1, (M,), generator=g)
    jj = torch.randint(0, S2, (M,), generator=g)
    f1, f2 = f1.to(dtype), f2.to(dtype)
    f1d, f2d = f1.to(DEV), f2.to(DEV)
    if cl:
        f1d = f1d.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
        f2d = f2d.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
    return f1, f2, coords, ii, jj, f1d, f2d


@pytest.mark.parametrize("cl", [False, True])
@pytest.mark.parametrize("spread", [1.0, 0.25, 2.7])
def test_corr_forward_fp32(ext, cl, spread):
    f1, f2, coords, ii, jj, f1d, f2d = _case(1, 300, spread=spread, cl=cl)
    ref, b = OC.corr_bar(f1, f2, coords, ii, jj, 3, OC.acc_generic(128))
    out, = ext[0].forward(f1d, f2d, coords.to(DEV), ii.to(DEV), jj.to(DEV), 3)
    assert out.shape == ref.shape
    assert bool(OC.within(out.cpu(), ref, b).all()), OC.bar_use(out.cpu(), ref, b).max().item()


def test_corr_forward_fp64(ext):
    f1, f2, coords, ii, jj, f1d, f2d = _case(2, 100, dtype=torch.float64)
    ref = OC.corr_forward(f1, f2, coords, ii, jj, 3)
    out, = ext[0].forward(f1d, f2d, coords.to(DEV), ii.to(DEV), jj.to(DEV), 3)
    assert (out.cpu() - ref).abs().max().item() <= 1e-12 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("cl", [False, True])
@pytest.mark.parametrize("spread", [1.0, 0.25, 2.7])
def test_corr_forward_fp16(ext, cl, spread):
    """cl=True, C=128 takes the mma.sync kernel; the rest the generic one.  Per element within the bar of
    oracle/corr.py (the kernel's fp32 accumulation and blend, then one fp16 rounding) -- the reference, which
    accumulates in fp16 (correlation_kernel.cu:121-131), is outside it (tests/test_corr_ref_cpu.py)."""
    f1, f2, coords, ii, jj, f1d, f2d = _case(3, 500, dtype=torch.half, spread=spread, cl=cl)
    ref, b = OC.corr_bar(f1, f2, coords, ii, jj, 3, OC.ACC_MMA if cl else OC.acc_generic(128))
    out, = ext[0].forward(f1d, f2d, coords.to(DEV), ii.to(DEV), jj.to(DEV), 3)
    assert bool(OC.within(out.cpu(), ref, b).all()), OC.bar_use(out.cpu(), ref, b).max().item()


def test_corr_forward_oob_is_zero(ext):
    """windows fully outside the map give exact zeros; partially outside match the oracle"""
    f1, f2, coords, ii, jj, f1d, f2d = _case(4, 64, dtype=torch.half, cl=True)
    coords[0, :16] += 1000.0
    coords[0, 16:32] -= 1000.0
    out, = ext[0].forward(f1d, f2d, coords.to(DEV), ii.to(DEV), jj.to(DEV), 3)
    assert float(out[0, :32].abs().max()) == 0.0
    ref, b = OC.corr_bar(f1, f2, coords, ii, jj, 3, OC.ACC_MMA)
    assert bool(OC.within(out.cpu(), ref, b).all())


def test_corr_forward_nonfinite_coords_do_not_crash(ext):
    f1, f2, coords, ii, jj, f1d, f2d = _case(5, 8, dtype=torch.half, cl=True)
    coords[0, 0] = float("nan")
    coords[0, 1] = float("inf")
    out, = ext[0].forward(f1d, f2d, coords.to(DEV), ii.to(DEV), jj.to(DEV), 3)
    torch.cuda.synchronize()
    assert torch.isfinite(out[0, 2:]).all()


def test_corr_empty(ext):
    f1, f2, coords, ii, jj, f1d, f2d = _case(6, 4)
    out, = ext[0].forward(f1d, f2d, coords[:, :0].to(DEV), ii[:0].to(DEV), jj[:0].to(DEV), 3)
    assert out.shape == (1, 0, 7, 7, 3, 3)


def _pyramid_inputs(dtype, M, seed=7, S1=50, S2=4, H=32, W=48, stretch_every=0, fx=2.7, fy=2.7):
    g = torch.Generator().manual_seed(seed)
    f1 = (torch.randn(1, S1, 3, 3, 128, generator=g) / 4).to(dtype).to(DEV).permute(0, 1, 4, 2, 3)
    l0 = (torch.randn(1, S2, H, W, 128, generator=g) / 4).to(dtype).to(DEV).permute(0, 1, 4, 2, 3)
    l1 = (torch.randn(1, S2, H // 4, W // 4, 128, generator=g) / 4).to(dtype).to(DEV).permute(0, 1, 4, 2, 3)
    coords = torch.zeros(1, M, 2, 3, 3)
    offs = torch.arange(3).float() - 1
    sx, sy = torch.ones(M), torch.ones(M)
    if stretch_every:
        sx[::stretch_every] = fx              # 2.7: the nine tap windows no longer fit any box of the wgmma kernel
        sy[::stretch_every] = fy
    coords[0, :, 0] = (torch.rand(M, generator=g) * (W + 8) - 4)[:, None, None] + offs[None, None, :] * sx[:, None, None]
    coords[0, :, 1] = (torch.rand(M, generator=g) * (H + 8) - 4)[:, None, None] + offs[None, :, None] * sy[:, None, None]
    ii = torch.randint(0, S1, (M,), generator=g).to(DEV)
    jj = torch.randint(0, S2, (M,), generator=g).to(DEV)
    return f1, l0, l1, coords.to(DEV), ii, jj


@pytest.mark.parametrize("dtype", [torch.half, torch.float32])
def test_corr_pyramid2_matches_two_calls(ext, dtype):
    """fused two-level entry == torch.stack of two single-level calls (dpvo.py:205-207)"""
    f1, l0, l1, coords, ii, jj = _pyramid_inputs(dtype, 400)
    a, = ext[0].forward(f1, l0, coords, ii, jj, 3)
    b, = ext[0].forward(f1, l1, coords / 4, ii, jj, 3)
    fused = ext[3].corr_pyramid2(f1, l0, l1, coords, ii, jj, 3, 4.0)
    ref = torch.stack([a, b], -1)
    if dtype == torch.float32:
        assert torch.equal(fused, ref)
    else:
        # fp16 features: level 0 of the fused call runs on wgmma (fp32 accumulation in another order than mma.sync):
        # both levels within the bar of the fp64 oracle
        for lev, (fm, c, n) in enumerate(((l0, coords, OC.ACC_WGMMA), (l1, OC.level_coords(coords, 4.0), OC.ACC_MMA))):
            want, b = OC.corr_bar(f1, fm, c, ii, jj, 3, n)
            assert bool(OC.within(fused[..., lev], want, b).all())


@pytest.mark.parametrize("M,stretch,pad,fx,fy", [(1, 0, 0, 1, 1), (149, 3, 896, 2.7, 2.7), (5000, 7, 896, 2.7, 2.7), (3000, 0, 0, 1, 1),
                                                 (3000, 2, 896, 1.4, 1.4), (3000, 2, 896, 1.9, 1.0), (3000, 3, 0, 0.6, 1.9),
                                                 (2000, 2, 0, 1.9, 1.9), (2000, 2, 0, 0.3, 0.3)])
def test_corr_tcgen05_vs_oracle(ext, M, stretch, pad, fx, fy):
    """wgmma/TMA kernel (every box shape 8..12 x 8..12 up to 128 pixels, the stretched-edge list finished by
    the mma.sync kernel, out-of-map boxes zero-filled by TMA, padded rows) against the fp64 restatement of
    correlation_kernel.cu:78-137"""
    f1, l0, l1, coords, ii, jj = _pyramid_inputs(torch.half, M, seed=11 + M, stretch_every=stretch, fx=fx, fy=fy)
    out = ext[3].corr_pyramid2(f1, l0, l1, coords, ii, jj, 3, 4.0, pad)
    if pad:
        assert out.shape == (1, M, pad)
        assert torch.count_nonzero(out[..., 882:]) == 0
        out = out[..., :882].reshape(1, M, 7, 7, 3, 3, 2)
    # level 0: wgmma, or the mma.sync list kernel for stretched edges (the larger bar); level 1: mma.sync order
    for lev, (fm, c, n) in enumerate(((l0, coords, OC.ACC_WGMMA), (l1, OC.level_coords(coords, 4.0), OC.ACC_MMA))):
        want, b = OC.corr_bar(f1, fm, c, ii, jj, 3, n)
        assert bool(OC.within(out[..., lev], want, b).all()), (lev, OC.bar_use(out[..., lev], want, b).max().item())


def test_corr_tcgen05_non_pow2_divisor(ext):
    """level-1 divisor that is not a power of two takes the true-division instantiation"""
    f1, l0, l1, coords, ii, jj = _pyramid_inputs(torch.half, 700, seed=5)
    out = ext[3].corr_pyramid2(f1, l0, l1, coords, ii, jj, 3, 3.0)
    want1, b = OC.corr_bar(f1, l1, OC.level_coords(coords, 3.0), ii, jj, 3, OC.ACC_MMA)
    assert bool(OC.within(out[..., 1], want1, b).all()), OC.bar_use(out[..., 1], want1, b).max().item()


def test_corr_tcgen05_far_outside(ext):
    """boxes entirely outside the map (also by millions of pixels) give exact zeros"""
    f1, l0, l1, coords, ii, jj = _pyramid_inputs(torch.half, 64)
    coords[0, ::2] += 3.0e6
    coords[0, 1::4] -= 5.0e8
    out = ext[3].corr_pyramid2(f1, l0, l1, coords, ii, jj, 3, 4.0)
    assert torch.count_nonzero(out[0, ::2]) == 0
    assert torch.count_nonzero(out[0, 1::4]) == 0
    assert torch.isfinite(out).all()


@pytest.mark.parametrize("cl", [False, True])
def test_corr_backward_fp32(ext, cl):
    f1, f2, coords, ii, jj, f1d, f2d = _case(8, 60, C=128, S1=20, S2=3, H=20, W=24, cl=cl)
    g = torch.Generator().manual_seed(9)
    grad = torch.randn(1, 60, 7, 7, 3, 3, generator=g)
    r1, r2, b1, b2 = OC.corr_backward_bar(f1, f2, coords, ii, jj, grad, 3)
    g1, g2 = ext[0].backward(f1d, f2d, coords.to(DEV), ii.to(DEV), jj.to(DEV), grad.to(DEV), 3)
    assert bool(OC.within(g1.cpu(), r1, b1).all()) and bool(OC.within(g2.cpu(), r2, b2).all())


@pytest.mark.parametrize("radius,C", [(0, 384), (1, 128), (0, 1), (1, 3)])
def test_patchify_forward_backward(ext, radius, C):
    g = torch.Generator().manual_seed(10 + radius)
    net = torch.randn(2, C, 30, 40, generator=g)
    coords = torch.stack([torch.rand(2, 96, generator=g) * 44 - 2, torch.rand(2, 96, generator=g) * 34 - 2], -1)
    ref = OC.patchify_raw(net, coords, radius)
    out, = ext[0].patchify_forward(net.to(DEV), coords.to(DEV), radius)
    assert torch.equal(out.cpu(), ref)          # pure gather: bit exact
    grad = torch.randn(ref.shape, generator=g)
    n = net.clone().requires_grad_(True)
    OC.patchify_raw(n, coords, radius).backward(grad)
    gout, = ext[0].patchify_backward(net.to(DEV), coords.to(DEV), grad.to(DEV), radius)
    assert (gout.cpu() - n.grad).abs().max().item() <= 1e-5


# ---------------------------------------------------------------- host wrappers (dpvo_b200/altcorr.py) with autograd
def test_altcorr_corr_autograd_with_dropout_matches_oracle(ext):
    """altcorr.corr forward + backward through torch autograd, including the edge dropout drawn with torch.rand on
    the CUDA generator inside backward (correlation.py:20-25): same seed -> same kept edges -> oracle gradient"""
    from dpvo_b200 import altcorr
    g = torch.Generator().manual_seed(171)
    M, S1, S2, H, W = 90, 20, 3, 18, 22
    f1 = torch.randn(1, S1, 128, 3, 3, generator=g) / 4
    f2 = torch.randn(1, S2, 128, H, W, generator=g) / 4
    coords = torch.zeros(1, M, 2, 3, 3)
    offs = torch.arange(3).float() - 1
    coords[0, :, 0] = (torch.rand(M, generator=g) * W)[:, None, None] + offs[None, None, :]
    coords[0, :, 1] = (torch.rand(M, generator=g) * H)[:, None, None] + offs[None, :, None]
    ii, jj = torch.randint(0, S1, (M,), generator=g), torch.randint(0, S2, (M,), generator=g)
    grad = torch.randn(1, M, 7, 7, 3, 3, generator=g)
    for dropout in (1, 0.5):
        a = f1.to(DEV).requires_grad_(True)
        b = f2.to(DEV).requires_grad_(True)
        out = altcorr.corr(a, b, coords.to(DEV), ii.to(DEV), jj.to(DEV), 3, dropout)
        torch.manual_seed(99)
        out.backward(grad.to(DEV))
        torch.manual_seed(99)
        keep = (torch.rand(M, device=DEV) < dropout).cpu() if dropout < 1 else torch.ones(M, dtype=torch.bool)
        ref, bar = OC.corr_bar(f1, f2, coords, ii, jj, 3, OC.acc_generic(128))
        assert bool(OC.within(out.detach().cpu(), ref, bar).all())
        r1, r2, b1, b2 = OC.corr_backward_bar(f1, f2, coords, ii, jj, grad * keep[None, :, None, None, None, None], 3)
        assert bool(OC.within(a.grad.cpu(), r1, b1).all()) and bool(OC.within(b.grad.cpu(), r2, b2).all())


def test_altcorr_patchify_bilinear_autograd_matches_oracle(ext):
    from dpvo_b200 import altcorr
    g = torch.Generator().manual_seed(172)
    net = torch.randn(2, 24, 20, 28, generator=g)
    coords = torch.stack([torch.rand(2, 30, generator=g) * 24 + 1.5, torch.rand(2, 30, generator=g) * 16 + 1.5], -1)
    x = net.to(DEV).requires_grad_(True)
    out = altcorr.patchify(x, coords.to(DEV), 1)
    grad = torch.randn(out.shape, generator=g)
    out.backward(grad.to(DEV))
    x64 = net.double().requires_grad_(True)
    ref = OC.patchify(x64, coords.double(), 1)
    ref.backward(grad.double())
    assert (out.detach().cpu().double() - ref.detach()).abs().max().item() < 1e-5
    assert (x.grad.cpu().double() - x64.grad).abs().max().item() < 1e-4
    raw = altcorr.patchify(net.to(DEV), coords.to(DEV), 1, mode="nearest")
    assert torch.equal(raw.cpu(), OC.patchify_raw(net, coords, 1))
