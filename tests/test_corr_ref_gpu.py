"""Every correlation path element by element against the float64 restatement, within the per-element bar of
oracle/corr.py (corr_bar: the kernel's fp32 accumulation and blend; corr_interval: one rounding to the output dtype),
at the box shapes, bins, frame edges and coordinates where the kernels switch paths:
  * corr_fwd_tc (level 0 of the binned corr_pyramid2): each of the 22 TMA box shapes inside the frame, across each
    border and corner and fully outside; 12x11 and 13x8, which go to the list kernel;
  * corr_fwd_l1_tiles (level 1): box origins on every residue of the 7-pixel tiles and in the apron, bins of 47..97
    edges around CB_ITEM = 48, the level-1 frames of the three encoder image sizes and a frame smaller than a box; still
    bit-equal to the mma.sync kernel;
  * corr_fwd_mma: union boxes of 10 (one pass) and 11 (nine passes), whole-call pyramid2 with 16-byte and unaligned
    output rows, the fallback when the bins of a large ring exceed the workspace;
  * corr_fwd_generic: fp32 / fp16 / bf16 (fp64 to 1e-12), channels-first and -last, C in {1, 3, 64, 128}, P 1..3, R 0..4;
  * coordinates: integers, (-1, 0) down to -1e-8 (fx rounds to 1), exactly W - 1 / H - 1, 2^20..2^23, divisors 3, 5, 6;
  * the bench state (E = 47,712 through altcorr.corr_pyramid as UpdateRunner.step calls it), the oracle on the device;
  * corr_backward and patchify_backward in fp32.
The largest fraction of its bar each path uses is printed by test_bar_use_report (run with -s)."""
import pytest
import torch

from oracle import corr as OC

pytestmark = pytest.mark.gpu
DEV = "cuda"
_USE = {}


def _expect(name, out, ref, b):
    """out within its bar everywhere; record the largest fraction of the bar used"""
    ref, b = ref.to(DEV), b.to(DEV)
    ok = OC.within(out, ref, b)
    use = OC.bar_use(out, ref, b).max().item()
    _USE[name] = max(_USE.get(name, 0.0), use)
    assert bool(ok.all()), "%s: %d of %d outside the bar (%.3g of it used)" % (name, int((~ok).sum()), ok.numel(), use)


def _ring(S1, S2, H, W, seed, H1=None, W1=None):
    """channels-last fp16 patch features [1,S1,128,3,3] and the two levels of a feature ring, [1,S2,128,H,W] and
    [1,S2,128,H1,W1] (a quarter of H, W unless given)"""
    g = torch.Generator().manual_seed(seed)
    f1 = (torch.randn(1, S1, 3, 3, 128, generator=g) / 4).half().to(DEV).permute(0, 1, 4, 2, 3)
    l0 = (torch.randn(1, S2, H, W, 128, generator=g) / 4).half().to(DEV).permute(0, 1, 4, 2, 3)
    l1 = (torch.randn(1, S2, H1 or H // 4, W1 or W // 4, 128, generator=g) / 4).half().to(DEV).permute(0, 1, 4, 2, 3)
    return f1, l0, l1


def _pyramid(ext, name, f1, l0, l1, coords, ii, jj, div=4.0, pad=0, n_acc0=OC.ACC_WGMMA, bit_equal=True):
    """corr_pyramid2 against the bar on both levels (level 0: wgmma or the list kernel, the larger bar of the two;
    level 1: mma.sync order), and level 1 bit-equal to the mma.sync kernel"""
    M = coords.shape[1]
    out = ext[3].corr_pyramid2(f1, l0, l1, coords, ii, jj, 3, div, pad)
    out = out.reshape(1, M, -1)[..., :882].reshape(1, M, 7, 7, 3, 3, 2)
    c1 = OC.level_coords(coords, div)
    if bit_equal:
        want1, = ext[0].forward(f1, l1, c1, ii, jj, 3)
        assert torch.equal(out[..., 1], want1), name
    ref, b = OC.corr_bar(f1, l0, coords, ii, jj, 3, max(n_acc0, OC.ACC_MMA))
    _expect(name + " level 0", out[..., 0], ref, b)
    ref, b = OC.corr_bar(f1, l1, c1, ii, jj, 3, OC.ACC_MMA)
    _expect(name + " level 1", out[..., 1], ref, b)
    return out


def _edges(origins, spreads, g, frac=None):
    """coords [1, M, 2, 3, 3] whose nine anchors floor(x) - 3 span exactly the given box: origin (bx, by), anchor spread
    (sx, sy) per edge, so the box is (8 + sx) x (8 + sy); fractions random (or the given one)"""
    M = origins.shape[0]
    steps = torch.stack([torch.zeros_like(spreads), spreads // 2, spreads], -1).float()      # [M, 2 (x, y), 3]
    fr = torch.rand(M, 2, 3, 3, generator=g) if frac is None else torch.full((M, 2, 3, 3), frac)
    coords = torch.zeros(1, M, 2, 3, 3)
    coords[0, :, 0] = origins[:, 0, None, None] + 3 + steps[:, 0, None, :] + fr[:, 0]     # columns spread in x
    coords[0, :, 1] = origins[:, 1, None, None] + 3 + steps[:, 1, :, None] + fr[:, 1]     # rows spread in y
    return coords


def _placements(bw, bh, H, W):
    """box origins inside, across each border and each corner, and fully outside the H x W frame"""
    xs = {"in": W // 2 - bw // 2, "lo": -(bw // 2), "hi": W - bw // 2}
    ys = {"in": H // 2 - bh // 2, "lo": -(bh // 2), "hi": H - bh // 2}
    pl = [(xs[a], ys[c]) for a in ("in", "lo", "hi") for c in ("in", "lo", "hi")]
    return pl + [(W + 3, H // 2), (-bw - 2, -bh - 5)]


BOXES = [(bw, bh) for bw in range(8, 13) for bh in range(8, 13) if bw * bh <= 128]


def test_there_are_22_box_shapes():
    assert len(BOXES) == 22


def _box_case(shapes, H, W, reps, seed):
    g = torch.Generator().manual_seed(seed)
    o, s = [], []
    for bw, bh in shapes:
        for bx, by in _placements(bw, bh, H, W):
            for r in range(reps):
                o.append((bx + r % 2, by - r % 3)); s.append((bw - 8, bh - 8))
    return _edges(torch.tensor(o), torch.tensor(s), g)


@pytest.mark.parametrize("shapes", [BOXES, [(12, 11), (13, 8), (8, 13)]], ids=["tma_boxes", "list_kernel"])
def test_level0_box_shapes_at_every_border(ext, shapes):
    H, W, S1, S2 = 40, 48, 30, 3
    f1, l0, l1 = _ring(S1, S2, H, W, seed=21)
    coords = _box_case(shapes, H, W, 4, seed=22)
    M = coords.shape[1]
    g = torch.Generator().manual_seed(23)
    ii, jj = torch.randint(0, S1, (M,), generator=g).to(DEV), torch.randint(0, S2, (M,), generator=g).to(DEV)
    out = _pyramid(ext, "corr_fwd_tc boxes" if shapes is BOXES else "list kernel boxes", f1, l0, l1, coords.to(DEV), ii, jj)
    n_place = len(_placements(8, 8, H, W))
    far = torch.zeros(M, dtype=torch.bool)
    for k in range(len(shapes)):
        far[(k * n_place + n_place - 2) * 4:(k * n_place + n_place) * 4] = True
    assert torch.count_nonzero(out[0, far.to(DEV), ..., 0]) == 0


@pytest.mark.parametrize("H1,W1", [(30, 40), (30, 47), (15, 20), (5, 6)])
def test_level1_tile_residues_and_frame_sizes(ext, H1, W1):
    """box origins on every residue of the 7-pixel level-1 tiles and in the 9-pixel apron, on the level-1 frames of
    480x640, 480x752 and 250x330 images and one smaller than a box"""
    f1, l0, l1 = _ring(20, 2, 4 * H1, 4 * W1, seed=31 + W1, H1=H1, W1=W1)
    ys, xs = torch.meshgrid(torch.arange(-10.0, H1 + 3, 0.55), torch.arange(-10.0, W1 + 3, 0.55), indexing="ij")
    centres = torch.stack([xs.flatten(), ys.flatten()], 1) * 4
    M = centres.shape[0]
    g = torch.Generator().manual_seed(33)
    offs = torch.arange(3).float() - 1
    coords = torch.zeros(1, M, 2, 3, 3)
    coords[0, :, 0] = centres[:, 0, None, None] + offs[None, None, :] + 0.1 * torch.randn(M, 3, 3, generator=g)
    coords[0, :, 1] = centres[:, 1, None, None] + offs[None, :, None] + 0.1 * torch.randn(M, 3, 3, generator=g)
    ii, jj = torch.randint(0, 20, (M,), generator=g).to(DEV), torch.randint(0, 2, (M,), generator=g).to(DEV)
    _pyramid(ext, "corr_fwd_l1_tiles frames", f1, l0, l1, coords.to(DEV), ii, jj)


def test_level1_bins_around_the_work_item_size(ext):
    """one bin each of 47, 48, 49, 96 and 97 edges (CB_ITEM = 48 per work item), in five frames"""
    counts = [47, 48, 49, 96, 97]
    f1, l0, l1 = _ring(40, len(counts), 120, 160, seed=41)
    g = torch.Generator().manual_seed(42)
    M = sum(counts)
    centre = torch.tensor([57.3, 41.8]) + 0.2 * torch.rand(M, 2, generator=g)     # level 1: floor fixed, one tile
    offs = torch.arange(3).float() - 1
    coords = torch.zeros(1, M, 2, 3, 3)
    coords[0, :, 0] = centre[:, 0, None, None] + offs[None, None, :]
    coords[0, :, 1] = centre[:, 1, None, None] + offs[None, :, None]
    jj = torch.cat([torch.full((n,), k) for k, n in enumerate(counts)])
    perm = torch.randperm(M, generator=g)
    ii = torch.randint(0, 40, (M,), generator=g)
    _pyramid(ext, "corr_fwd_l1_tiles bins", f1, l0, l1, coords[:, perm].to(DEV), ii.to(DEV), jj[perm].to(DEV))


def _forward(ext, name, f1, f2, coords, ii, jj, R, n_acc):
    out, = ext[0].forward(f1, f2, coords, ii, jj, R)
    ref, b = OC.corr_bar(f1, f2, coords, ii, jj, R, n_acc)
    _expect(name, out, ref, b)
    return out


def test_mma_union_boxes_of_10_and_11(ext):
    """corr_fwd_mma: union boxes of exactly 10 (one pass) and 11 pixels per side (nine per-pixel passes)"""
    H, W = 30, 40
    f1, l0, _ = _ring(20, 3, H, W, seed=51)
    g = torch.Generator().manual_seed(52)
    shapes = [(10, 10), (10, 8), (8, 10), (11, 8), (8, 11), (11, 11), (11, 10)]
    coords = _box_case(shapes, H, W, 3, seed=53)
    M = coords.shape[1]
    ii, jj = torch.randint(0, 20, (M,), generator=g).to(DEV), torch.randint(0, 3, (M,), generator=g).to(DEV)
    _forward(ext, "corr_fwd_mma union boxes", f1, l0, coords.to(DEV), ii, jj, 3, OC.ACC_MMA)


def _padded_slots(f1):
    """the same patch features with 1160-element slots: mma.sync-eligible, but not the layout of the binned path"""
    S1 = f1.shape[1]
    buf = torch.zeros(1, S1, 1160, dtype=f1.dtype, device=DEV)
    buf[..., :1152] = f1.permute(0, 1, 3, 4, 2).reshape(1, S1, 1152)
    return buf.as_strided((1, S1, 128, 3, 3), (S1 * 1160, 1160, 1, 384, 128))


@pytest.mark.parametrize("pad", [0, 896])
def test_mma_whole_call_rows(ext, pad):
    """corr_pyramid2 on the mma.sync kernel for the whole call: output rows of 882 halves (not 16-byte aligned) and of
    896 (16-byte stores)"""
    f1, l0, l1 = _ring(30, 4, 32, 48, seed=61)
    g = torch.Generator().manual_seed(62)
    M = 700
    coords = torch.zeros(1, M, 2, 3, 3)
    offs = torch.arange(3).float() - 1
    s = torch.where(torch.arange(M) % 5 == 0, 2.7, 1.0)
    coords[0, :, 0] = (torch.rand(M, generator=g) * 56 - 4)[:, None, None] + offs[None, None, :] * s[:, None, None]
    coords[0, :, 1] = (torch.rand(M, generator=g) * 40 - 4)[:, None, None] + offs[None, :, None] * s[:, None, None]
    ii, jj = torch.randint(0, 30, (M,), generator=g).to(DEV), torch.randint(0, 4, (M,), generator=g).to(DEV)
    _pyramid(ext, "corr_fwd_mma whole call", _padded_slots(f1), l0, l1, coords.to(DEV), ii, jj, pad=pad, n_acc0=OC.ACC_MMA)


def test_mma_fallback_when_the_bins_exceed_the_workspace(ext):
    """300 ring slots and 20 edges: S2 * nty * ntx > 2 M + 4096 bins, so the whole call runs on the mma.sync kernel"""
    f1, l0, l1 = _ring(10, 300, 16, 24, seed=71, H1=30, W1=40)     # level 1 of 30 x 40: 42 tiles per slot
    g = torch.Generator().manual_seed(73)
    M = 20
    coords = torch.zeros(1, M, 2, 3, 3)
    offs = torch.arange(3).float() - 1
    coords[0, :, 0] = (torch.rand(M, generator=g) * 24)[:, None, None] + offs[None, None, :]
    coords[0, :, 1] = (torch.rand(M, generator=g) * 16)[:, None, None] + offs[None, :, None]
    ii, jj = torch.randint(0, 10, (M,), generator=g).to(DEV), torch.randint(0, 300, (M,), generator=g).to(DEV)
    assert 300 * ((30 + 15) // 7) * ((40 + 15) // 7) > 2 * M + 4096
    _pyramid(ext, "corr_fwd_mma fallback", f1, l0, l1, coords.to(DEV), ii, jj, n_acc0=OC.ACC_MMA)


@pytest.mark.parametrize("cl", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16, torch.bfloat16])
def test_generic_kernel(ext, dtype, cl):
    """every dtype and layout, C in {1, 3, 64, 128}, patch sizes 1..3 and radii 0..4 (fp16 / channels-last / C = 128 /
    P = 3 / R = 3 is the mma.sync kernel)"""
    g = torch.Generator().manual_seed(81)
    H, W, S1, S2, M = 14, 17, 6, 2, 24
    for C in (1, 3, 64, 128):
        f2 = torch.randn(1, S2, C, H, W, generator=g) / 4
        for P in (1, 2, 3):
            f1 = torch.randn(1, S1, C, P, P, generator=g) / 4
            coords = torch.zeros(1, M, 2, P, P)
            offs = torch.arange(P).float() - P // 2
            coords[0, :, 0] = (torch.rand(M, generator=g) * (W + 10) - 5)[:, None, None] + offs[None, None, :] + 0.1 * torch.randn(M, P, P, generator=g)
            coords[0, :, 1] = (torch.rand(M, generator=g) * (H + 10) - 5)[:, None, None] + offs[None, :, None] + 0.1 * torch.randn(M, P, P, generator=g)
            ii, jj = torch.randint(0, S1, (M,), generator=g).to(DEV), torch.randint(0, S2, (M,), generator=g).to(DEV)
            a, b = f1.to(dtype).to(DEV), f2.to(dtype).to(DEV)
            if cl:
                a = a.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
                b = b.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
            for R in range(5):
                if dtype == torch.float64:
                    out, = ext[0].forward(a, b, coords.to(DEV), ii, jj, R)
                    ref = OC.corr_forward(a.double(), b.double(), coords.to(DEV), ii, jj, R)
                    assert (out - ref).abs().max().item() <= 1e-12 * max(1.0, ref.abs().max().item())
                    continue
                mma = dtype == torch.float16 and cl and C == 128 and P == 3 and R == 3
                _forward(ext, "corr_fwd_mma" if mma else "corr_fwd_generic %s" % str(dtype)[6:], a, b, coords.to(DEV),
                         ii, jj, R, OC.ACC_MMA if mma else OC.acc_generic(C))


def _special_coords(H, W, g):
    """edges whose nine pixels sit on integers, in (-1, 0) (down to -1e-8, where x - floor(x) rounds to 1), on W - 1 and
    H - 1 exactly, and at magnitudes 2^20 .. 2^23 of both signs"""
    vals = [torch.arange(-3.0, W + 3), torch.tensor([-1e-8, -1e-7, -0.5, -0.999, -2.0 ** -20, -1e-30]),
            torch.tensor([W - 1.0, H - 1.0, W - 1.0 - 2.0 ** -19, H - 1.0 + 2.0 ** -19, 0.0])]
    big = torch.tensor([2.0 ** 20, 2.0 ** 21 + 0.5, 2.0 ** 22 + 0.25, 2.0 ** 23, 2.0 ** 23 - 1.5])
    pool = torch.cat(vals)
    rows = []
    for k in range(160):
        x = pool[torch.randint(0, len(pool), (3, 3), generator=g)]
        y = pool[torch.randint(0, len(pool), (3, 3), generator=g)].clamp(max=H + 2)
        if k % 4 == 1:                                  # a compact patch around a special anchor
            x = x[0, 0] + (torch.arange(3).float() - 1)[None, :].expand(3, 3)
            y = y[0, 0] + (torch.arange(3).float() - 1)[:, None].expand(3, 3)
        rows.append(torch.stack([x, y]))
    for k in range(10):
        s = 1.0 if k % 2 else -1.0
        rows.append(torch.stack([s * big[k % 5] + torch.arange(3.0)[None, :].expand(3, 3),
                                 -s * big[(k + 2) % 5] + torch.arange(3.0)[:, None].expand(3, 3)]))
    return torch.stack(rows)[None].float()


def test_special_coordinates_on_every_path(ext):
    H, W, S1, S2 = 32, 48, 10, 2
    g = torch.Generator().manual_seed(91)
    f1, l0, l1 = _ring(S1, S2, H, W, seed=92)
    coords = _special_coords(H, W, g).to(DEV)
    M = coords.shape[1]
    ii, jj = torch.randint(0, S1, (M,), generator=g).to(DEV), torch.randint(0, S2, (M,), generator=g).to(DEV)
    assert (coords - torch.floor(coords) == 1.0).any()
    _forward(ext, "corr_fwd_mma special coords", f1, l0, coords, ii, jj, 3, OC.ACC_MMA)
    _forward(ext, "corr_fwd_generic special coords", f1.float(), l0.float(), coords, ii, jj, 3, OC.acc_generic(128))
    _pyramid(ext, "binned special coords", f1, l0, l1, coords, ii, jj)
    for div in (3.0, 5.0, 6.0):
        _pyramid(ext, "binned divisor", f1, l0, l1, coords, ii, jj, div=div)
        _pyramid(ext, "corr_fwd_mma whole call divisor", _padded_slots(f1), l0, l1, coords, ii, jj, div=div, n_acc0=OC.ACC_MMA)


def test_non_pow2_divisors_on_random_edges(ext):
    f1, l0, l1 = _ring(40, 4, 120, 160, seed=95)
    g = torch.Generator().manual_seed(96)
    M = 2000
    offs = torch.arange(3).float() - 1
    coords = torch.zeros(1, M, 2, 3, 3)
    coords[0, :, 0] = (torch.rand(M, generator=g) * 168 - 4)[:, None, None] + offs[None, None, :] + 0.1 * torch.randn(M, 3, 3, generator=g)
    coords[0, :, 1] = (torch.rand(M, generator=g) * 128 - 4)[:, None, None] + offs[None, :, None] + 0.1 * torch.randn(M, 3, 3, generator=g)
    ii, jj = torch.randint(0, 40, (M,), generator=g).to(DEV), torch.randint(0, 4, (M,), generator=g).to(DEV)
    for div in (3.0, 5.0, 6.0):
        _pyramid(ext, "binned divisor", f1, l0, l1, coords.to(DEV), ii, jj, div=div)
        _pyramid(ext, "corr_fwd_mma whole call divisor", _padded_slots(f1), l0, l1, coords.to(DEV), ii, jj, div=div, n_acc0=OC.ACC_MMA)


def test_bench_state(ext):
    """the bench's correlation: E = 47,712 edges of the default config in a 36-slot ring, through altcorr.corr_pyramid
    into the padded [E, 896] buffer as UpdateRunner.step calls it; the float64 oracle runs on the device"""
    from dpvo_b200 import altcorr, projective_ops as pops, synthetic
    from dpvo_b200.runner import UpdateRunner
    st = synthetic.make_state("default", 36, device=DEV, seed=1234)
    run = UpdateRunner(st)
    coords = pops.transform_fused(st.poses.view(1, -1, 7), st.patches.view(1, -1, 3, 3, 3), st.intrinsics.view(1, -1, 4),
                                  st.ii, st.jj, st.kk)
    E = coords.shape[1]
    assert E == 47712
    buf = torch.zeros(1, E, 896, dtype=torch.half, device=DEV)
    out = altcorr.corr_pyramid(st.gmap, (st.fmap1, st.fmap2), coords, run.kk_ring, run.jj_ring, 3, 4.0, 896, buf)
    assert torch.count_nonzero(out[..., 882:]) == 0
    out = out[..., :882].reshape(1, E, 7, 7, 3, 3, 2)
    for lev, (fmap, c, n) in enumerate(((st.fmap1, coords, OC.ACC_WGMMA), (st.fmap2, OC.level_coords(coords, 4.0), OC.ACC_MMA))):
        ref, b = OC.corr_bar(st.gmap, fmap, c, run.kk_ring, run.jj_ring, 3, n)
        _expect("bench state level %d" % lev, out[..., lev], ref, b)


@pytest.mark.parametrize("cl", [False, True])
def test_backward_fp32(ext, cl):
    g = torch.Generator().manual_seed(101)
    M, S1, S2, H, W = 80, 20, 3, 20, 24
    f1 = (torch.randn(1, S1, 128, 3, 3, generator=g) / 4).to(DEV)
    f2 = (torch.randn(1, S2, 128, H, W, generator=g) / 4).to(DEV)
    if cl:
        f1 = f1.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
        f2 = f2.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
    s = torch.where(torch.arange(M) % 4 == 0, 2.5, 1.0)            # some nine-pass (stretched) edges
    offs = torch.arange(3).float() - 1
    coords = torch.zeros(1, M, 2, 3, 3)
    coords[0, :, 0] = (torch.rand(M, generator=g) * (W + 8) - 4)[:, None, None] + offs[None, None, :] * s[:, None, None]
    coords[0, :, 1] = (torch.rand(M, generator=g) * (H + 8) - 4)[:, None, None] + offs[None, :, None] * s[:, None, None]
    coords = coords.to(DEV)
    ii, jj = torch.randint(0, S1, (M,), generator=g).to(DEV), torch.randint(0, S2, (M,), generator=g).to(DEV)
    grad = torch.randn(1, M, 7, 7, 3, 3, generator=g).to(DEV)
    g1, g2 = ext[0].backward(f1, f2, coords, ii, jj, grad, 3)
    r1, r2, b1, b2 = OC.corr_backward_bar(f1, f2, coords, ii, jj, grad, 3)
    _expect("corr_bwd_generic fmap1", g1, r1, b1)
    _expect("corr_bwd_generic fmap2", g2, r2, b2)


@pytest.mark.parametrize("radius,C", [(0, 384), (1, 128), (3, 3)])
def test_patchify_backward_fp32(ext, radius, C):
    g = torch.Generator().manual_seed(110 + radius)
    net = torch.randn(2, C, 30, 40, generator=g).to(DEV)
    coords = torch.stack([torch.rand(2, 300, generator=g) * 44 - 2, torch.rand(2, 300, generator=g) * 34 - 2], -1).to(DEV)
    D = 2 * radius + 2
    grad = torch.randn(2, 300, C, D, D, generator=g).to(DEV)
    out, = ext[0].patchify_backward(net, coords, grad, radius)
    ref, b = OC.patchify_backward_bar(net, coords, grad, radius)
    _expect("patchify_backward", out, ref, b)


def test_bar_use_report():
    """the largest fraction of its bar each path used in this session (printed with -s)"""
    print()
    for k in sorted(_USE):
        print("  bar use %-40s %.3g" % (k, _USE[k]))
