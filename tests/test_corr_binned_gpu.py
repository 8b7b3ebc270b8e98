"""The binned two-level correlation (corr_pyramid2 with its workspace: level 1 from one shared-memory region per bin,
level 0 on wgmma + TMA in bin order, stretched edges on the list kernel) against the mma.sync kernel (the same
correlation without the workspace, one level per call), full [E, 882] rows.

Level 1 uses the mma.sync kernel's k order, accumulation chains and blend, so it must be bit-identical.  Level 0 is
accumulated by wgmma in another order: it must stay, element by element, within the bar of oracle/corr.py against the
float64 restatement (computed on the device)."""
import pytest
import torch

from oracle import corr as OC

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _inputs(M, seed=3, S1=40, S2=4, H=120, W=160, centres=None, slots=None, stretch_every=0, stretch=2.7):
    g = torch.Generator().manual_seed(seed)
    f1 = (torch.randn(1, S1, 3, 3, 128, generator=g) / 4).half().to(DEV).permute(0, 1, 4, 2, 3)
    l0 = (torch.randn(1, S2, H, W, 128, generator=g) / 4).half().to(DEV).permute(0, 1, 4, 2, 3)
    l1 = (torch.randn(1, S2, H // 4, W // 4, 128, generator=g) / 4).half().to(DEV).permute(0, 1, 4, 2, 3)
    if centres is None:
        centres = torch.stack([torch.rand(M, generator=g) * (W + 8) - 4, torch.rand(M, generator=g) * (H + 8) - 4], 1)
    offs = torch.arange(3).float() - 1
    s = torch.ones(M)
    if stretch_every:
        s[::stretch_every] = stretch
    coords = torch.zeros(1, M, 2, 3, 3)
    coords[0, :, 0] = centres[:, 0, None, None] + offs[None, None, :] * s[:, None, None] + 0.1 * torch.randn(M, 3, 3, generator=g)
    coords[0, :, 1] = centres[:, 1, None, None] + offs[None, :, None] * s[:, None, None] + 0.1 * torch.randn(M, 3, 3, generator=g)
    ii = torch.randint(0, S1, (M,), generator=g)
    jj = torch.randint(0, S2, (M,), generator=g) if slots is None else slots[torch.randint(0, len(slots), (M,), generator=g)]
    return f1, l0, l1, coords.to(DEV), ii.to(DEV), jj.to(DEV)


def _check(ext, f1, l0, l1, coords, ii, jj, div=4.0, out=None):
    got = ext[3].corr_pyramid2(f1, l0, l1, coords, ii, jj, 3, div, 896 if out is not None else 0, out)
    M = coords.shape[1]
    got = got.reshape(1, M, -1)[..., :882].reshape(1, M, 7, 7, 3, 3, 2)
    # the level-1 coordinates divided on the CPU (IEEE division, as the kernels; a CUDA tensor divided by a scalar is
    # multiplied by its reciprocal, which differs in the last bit for divisors that are not powers of two)
    want1, = ext[0].forward(f1, l1, (coords.cpu() / div).to(DEV), ii, jj, 3)
    assert torch.equal(got[..., 1], want1), float((got[..., 1].float() - want1.float()).abs().max())
    # level 0: wgmma, or the mma.sync list kernel for stretched edges (the larger bar of the two)
    ref, b = OC.corr_bar(f1, l0, coords, ii, jj, 3, OC.ACC_WGMMA)
    assert bool(OC.within(got[..., 0], ref, b).all()), OC.bar_use(got[..., 0], ref, b).max().item()
    return got


def test_binned_bench_graph(ext):
    """the bench state: E = 47,712 edges of the default config reprojected into a 36-slot ring"""
    from dpvo_b200 import projective_ops as pops, synthetic
    from dpvo_b200.runner import UpdateRunner
    st = synthetic.make_state("default", 36, device=DEV, seed=1234)
    run = UpdateRunner(st)
    coords = pops.transform_fused(st.poses.view(1, -1, 7), st.patches.view(1, -1, 3, 3, 3), st.intrinsics.view(1, -1, 4),
                                  st.ii, st.jj, st.kk)
    _check(ext, st.gmap, st.fmap1, st.fmap2, coords, run.kk_ring, run.jj_ring,
           out=torch.zeros(1, coords.shape[1], 896, dtype=torch.half, device=DEV))


def test_binned_tile_and_band_edges(ext):
    """box origins on every residue around the 7-pixel level-1 tile boundaries, on the whole frame"""
    H, W = 120, 160
    ys, xs = torch.meshgrid(torch.arange(-6.0, H + 6, 1.25), torch.arange(-6.0, W + 6, 1.25), indexing="ij")
    centres = torch.stack([xs.flatten(), ys.flatten()], 1)
    _check(ext, *_inputs(centres.shape[0], seed=4, H=H, W=W, centres=centres))


@pytest.mark.parametrize("margin", [12.0, 60.0, 3.0e6])
def test_binned_outside_the_frame(ext, margin):
    """boxes partly or entirely outside the frame, also by millions of pixels"""
    M, H, W = 4000, 120, 160
    g = torch.Generator().manual_seed(5)
    centres = torch.stack([torch.rand(M, generator=g) * (W + 2 * margin) - margin,
                           torch.rand(M, generator=g) * (H + 2 * margin) - margin], 1)
    got = _check(ext, *_inputs(M, seed=6, H=H, W=W, centres=centres))
    far = ((centres[:, 0] < -20) | (centres[:, 0] > W + 20) | (centres[:, 1] < -20) | (centres[:, 1] > H + 20)).to(DEV)
    assert torch.count_nonzero(got[0, far]) == 0


def test_binned_one_bin_holds_every_edge(ext):
    """3,000 edges at one spot of one frame: one bin far beyond the edges one CTA takes at a time"""
    M = 3000
    centres = torch.tensor([[57.3, 41.8]]).repeat(M, 1)
    _check(ext, *_inputs(M, seed=7, centres=centres, slots=torch.tensor([2])))


def test_binned_frames_without_edges(ext):
    """a six-slot ring whose edges all land in slots 1 and 4"""
    _check(ext, *_inputs(2500, seed=8, S2=6, slots=torch.tensor([1, 4])))


def test_binned_single_edge(ext):
    _check(ext, *_inputs(1, seed=9))


@pytest.mark.parametrize("every,stretch", [(3, 2.7), (2, 1.4), (5, 0.3)])
def test_binned_stretched_edges_mixed_in(ext, every, stretch):
    """edges whose windows fit no box (list kernel) and shrunk ones, between ordinary edges"""
    _check(ext, *_inputs(3000, seed=10 + every, stretch_every=every, stretch=stretch))


def test_binned_non_pow2_divisor(ext):
    _check(ext, *_inputs(2000, seed=13), div=3.0)


def test_binned_second_call_on_the_same_buffers(ext):
    """the bin counters are reset by every call: a second call with other edges on the same output buffer"""
    out = torch.zeros(1, 3000, 896, dtype=torch.half, device=DEV)
    a = _inputs(3000, seed=14)
    b = _inputs(3000, seed=15, slots=torch.tensor([0]))
    first = _check(ext, *a, out=out).clone()
    _check(ext, *b, out=out)
    again = _check(ext, *a, out=out)
    assert torch.equal(first, again)
