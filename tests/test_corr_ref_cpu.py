"""The correlation's error bar (oracle/corr.py: corr_bar, corr_interval) pinned on the CPU.

Without rounding the float64 restatement is corr_grid_sample and the reference kernel's fixture.  The bar accepts a
float32 emulation of each kernel's arithmetic -- corr_fwd_mma's two k16 chains and their join, corr_fwd_tc's eight
sequential k16 steps, corr_fwd_generic's per-channel FMAs, the fp32 blend, one rounding to fp16 -- and rejects
kernel-shaped mutations of it in every value regime where the mutation changes the output, apart from the cases listed
in BELOW with their reasons."""
import functools
import os

import numpy as np
import pytest
import torch

from oracle import corr as OC

GOLD = os.path.join(os.path.dirname(__file__), "golden")
R, P, C = 3, 3, 128
D = 2 * R + 2


def _rn32(x):
    return x.float().double()


def _rn16(x):
    return OC.round_to(x, torch.float16)


def _case(regime, seed=0, M=48, S1=6, S2=2, H=20, W=24):
    """fp16 features and fp32 coordinates; boxes inside, across the borders (negative coordinates) and outside"""
    g = torch.Generator().manual_seed(seed)
    f1 = torch.randn(1, S1, C, P, P, generator=g) / 4
    f2 = torch.randn(1, S2, C, H, W, generator=g) / 4
    if regime == "cancelling":
        # per-channel offsets (equal within channel pairs) against patch features of opposite sign in each pair: every
        # dot product cancels, S is ~500x the output
        off = (4 + 8 * torch.rand(C // 2, generator=g)).repeat_interleave(2) * torch.sign(torch.randn(C, generator=g))
        f2 = off[None, None, :, None, None] + 0.05 * torch.randn(1, S2, C, H, W, generator=g)
        a = torch.randn(1, S1, C // 2, P, P, generator=g) / 4
        f1 = torch.stack([a, -a], 3).reshape(1, S1, C, P, P) * torch.sign(off)[None, None, :, None, None]
    elif regime == "fp16max":
        f1, f2 = f1 * 110, f2 * 110                     # outputs up to ~5e4, below 65504
    elif regime == "subnormal":
        f1, f2 = f1 / 300, f2 / 300                     # outputs below 2^-14
    f1, f2 = f1.half(), f2.half()
    cx = torch.rand(M, generator=g) * (W + 8) - 4
    cy = torch.rand(M, generator=g) * (H + 8) - 4
    offs = torch.arange(P).float() - P // 2
    coords = torch.zeros(1, M, 2, P, P)
    coords[0, :, 0] = cx[:, None, None] + offs[None, None, :] + 0.1 * torch.randn(M, P, P, generator=g)
    coords[0, :, 1] = cy[:, None, None] + offs[None, :, None] + 0.1 * torch.randn(M, P, P, generator=g)
    coords[0, :4] = torch.round(coords[0, :4])          # integer coordinates
    ii = torch.randint(0, S1, (M,), generator=g)
    jj = torch.randint(0, S2, (M,), generator=g)
    return f1, f2, coords, ii, jj


def _frac(x, m):
    if m == "frac_from_fp16_coords":
        x = x.half().float()
    if m == "trunc_floor":
        return torch.trunc(x), x - torch.trunc(x)
    return torch.floor(x), x - torch.floor(x)


def emulate(f1, f2, coords, ii, jj, order="mma", m=None, div=1.0, out_dtype=torch.float16):
    """float32 emulation of one correlation kernel (order: mma, wgmma, generic) with mutation m, as float64"""
    H, W = f2.shape[3], f2.shape[4]
    M = coords.shape[1]
    c = coords[0].float()
    if div != 1.0:
        c = c * torch.tensor(1.0 / div, dtype=torch.float32) if m == "recip_div" else OC.level_coords(c, div)
    fl_x, fx = _frac(c[:, 0], m)                        # [M, P, P]
    fl_y, fy = _frac(c[:, 1], m)
    taps = torch.arange(D) - R
    yy = (fl_y.long()[:, None, None] + taps[None, :, None, None, None]).expand(M, D, D, P, P)
    xx = (fl_x.long()[:, None, None] + taps[None, None, :, None, None]).expand(M, D, D, P, P)
    inb = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
    lin = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).reshape(M, 1, -1).expand(M, C, -1)
    win = torch.gather(f2[0, jj].double().reshape(M, C, H * W), 2, lin).reshape(M, C, D, D, P, P)
    if m != "clamp_oob":
        win = torch.where(inb[:, None], win, torch.zeros((), dtype=torch.float64))
    prod = win * f1[0, ii].double()[:, :, None, None]   # exact
    if m == "acc_fp16":                                 # the reference's fp16 kernel: s += f1 * f2 in half
        acc = torch.zeros(M, D, D, P, P, dtype=torch.float64)
        for k in range(C):
            acc = _rn16(acc + _rn16(prod[:, k]))
        raw = acc
    elif order == "generic":
        acc = torch.zeros(M, D, D, P, P, dtype=torch.float64)
        for k in range(C):
            acc = _rn32(acc + prod[:, k])
        raw = acc
    elif order == "wgmma":
        acc = torch.zeros(M, D, D, P, P, dtype=torch.float64)
        for k in range(C // 16):
            acc = _rn32(acc + prod[:, 16 * k:16 * k + 16].sum(1))
        raw = acc
    else:
        # k step (kb, h) of chain h: channels 32 kb + 8 t + 4 h + {0..3}, t = 0..3
        ch = [torch.tensor([32 * kb + 8 * t + 4 * h + j for t in range(4) for j in range(4)]) for kb in range(4) for h in range(2)]
        acc = [torch.zeros(M, D, D, P, P, dtype=torch.float64) for _ in range(2)]
        for s, idx in enumerate(ch):
            acc[s % 2] = _rn32(acc[s % 2] + prod[:, idx].sum(1))
        raw = _rn32(acc[0] + acc[1])
    if m == "taps_fp16":
        raw = _rn16(raw)
    fx, fy = fx.double()[:, None, None], fy.double()[:, None, None]
    ox, oy = _rn32(1 - fx), _rn32(1 - fy)
    w = [_rn32(ox * oy), _rn32(fx * oy), _rn32(ox * fy), _rn32(fx * fy)]
    if m == "corner_swap":
        w[1] = _rn32(ox * oy)
    if m == "weights_fp16":
        w = [_rn16(v) for v in w]
    r = [raw[:, 0:D - 1, 0:D - 1], raw[:, 0:D - 1, 1:D], raw[:, 1:D, 0:D - 1], raw[:, 1:D, 1:D]]
    v = _rn32(w[0] * r[0])
    for k in range(1, 4):
        v = _rn32(w[k] * r[k] + v)                      # fused multiply-add
    out = v.permute(0, 2, 1, 3, 4) if m != "xy_swap" else v
    if out_dtype == torch.float16:
        out = _rn16(out)
    return out[None]


def _bar(f1, f2, coords, ii, jj, order, div=1.0):
    n_acc = {"mma": OC.ACC_MMA, "wgmma": OC.ACC_WGMMA, "generic": OC.acc_generic(C)}[order]
    return OC.corr_bar(f1, f2, OC.level_coords(coords, div), ii, jj, R, n_acc)


def _inside(out, ref, b, dtype=torch.float16):
    lo, hi = OC.corr_interval(ref, b, dtype)
    return bool(((out >= lo) & (out <= hi)).all())


REGIMES = ["nominal", "cancelling", "fp16max", "subnormal"]
_USED = {}


@pytest.mark.parametrize("regime", REGIMES)
def test_regimes_reach_their_ranges(regime):
    f1, f2, coords, ii, jj = _case(regime)
    ref, b = _bar(f1, f2, coords, ii, jj, "mma")
    S = b / OC.gamma(OC.ACC_MMA + OC.BLEND)
    top = ref.abs().max().item()
    if regime == "fp16max":
        assert 2e4 < top < 65504
    if regime == "subnormal":
        assert 0 < top < 2.0 ** -14
    if regime == "cancelling":
        live = ref.abs() > 0
        assert (S[live] / ref.abs()[live]).median().item() > 100


@pytest.mark.parametrize("order", ["mma", "wgmma", "generic"])
@pytest.mark.parametrize("regime", REGIMES)
def test_bar_accepts_the_kernel_arithmetic(order, regime):
    for seed in range(2):
        f1, f2, coords, ii, jj = _case(regime, seed)
        ref, b = _bar(f1, f2, coords, ii, jj, order)
        out = emulate(f1, f2, coords, ii, jj, order)
        lo, hi = OC.corr_interval(ref, b, torch.float16)
        assert bool(((out >= lo) & (out <= hi)).all()), "%s %s seed %d" % (order, regime, seed)
        use = OC.bar_use(out.half(), ref, b)
        assert bool((use <= 1).all())
        _USED[(order, regime)] = max(_USED.get((order, regime), 0.0), use.max().item())
        if order == "generic":                          # the fp32 outputs of the generic kernel, without the bracket
            out32 = emulate(f1, f2, coords, ii, jj, order, out_dtype=torch.float32)
            assert _inside(out32, ref, b, torch.float32)


def test_bar_use_is_reported():
    """the largest fraction of the bar the emulation uses, per kernel order and regime: 0 is a correctly rounded
    output; the fp32 arithmetic moves some outputs across an fp16 rounding boundary"""
    print()
    for k, v in sorted(_USED.items()):
        print("  %-8s %-11s %.3g" % (k[0], k[1], v))


MUTATIONS = ["taps_fp16", "acc_fp16", "weights_fp16", "frac_from_fp16_coords", "corner_swap", "trunc_floor", "clamp_oob",
             "xy_swap", "recip_div"]
# Mutations the bar cannot see in a regime although they change some output bits, with the reason:
#   * taps_fp16 / weights_fp16 in the cancelling regime: the bar there is gamma(12) S ~ 700 ulps of fp32 at the scale
#     of S, wider than the relative 2^-12 of one fp16 rounding of a tap or a weight at the (500x smaller) scale of the
#     output; the kernels' own fp32 accumulation of the large cancelling terms moves outputs by as much
#   * recip_div in the cancelling and subnormal regimes: x * RN(1 / 3) differs from x / 3 by at most one fp32 ulp of
#     the level-1 coordinate, which moves fx by ~2^-24 |x| / 3 and the output by ~1e-6 of the taps' spread: inside the
#     bar's wide accumulation term when the taps cancel, and below half an fp16 ulp of a subnormal output.  (In the
#     other two regimes a few outputs leave the bar; on the GPU the bit-equality of level 1 with the mma.sync kernel
#     also catches a reciprocal)
BELOW = {("taps_fp16", "cancelling"), ("weights_fp16", "cancelling"), ("recip_div", "cancelling"), ("recip_div", "subnormal")}


@functools.lru_cache(maxsize=None)
def _mutated(m, regime):
    f1, f2, coords, ii, jj = _case(regime)
    div = 3.0 if m == "recip_div" else 1.0
    if m == "recip_div":                               # coordinates where x / 3 and x * RN(1 / 3) differ in fp32
        coords = coords * 3.0 + 0.37
    ref, b = _bar(f1, f2, coords, ii, jj, "mma", div)
    base = emulate(f1, f2, coords, ii, jj, "mma", div=div)
    got = emulate(f1, f2, coords, ii, jj, "mma", m, div=div)
    return base, got, ref, b


MCASES = [pytest.param(m, r, marks=[pytest.mark.xfail(strict=True, reason="listed in BELOW")] if (m, r) in BELOW else [])
          for m in MUTATIONS for r in REGIMES]


@pytest.mark.parametrize("mutation,regime", MCASES)
def test_bar_rejects_mutations(mutation, regime):
    base, got, ref, b = _mutated(mutation, regime)
    if torch.equal(base, got):
        pytest.skip("the mutation does not change the output in this regime")
    assert not _inside(got, ref, b), "the bar accepts %s in the %s regime" % (mutation, regime)


def test_every_mutation_is_rejected_somewhere():
    caught = set()
    for m in MUTATIONS:
        for r in REGIMES:
            base, got, ref, b = _mutated(m, r)
            if not torch.equal(base, got) and not _inside(got, ref, b):
                caught.add(m)
    assert caught == set(MUTATIONS)


# ----------------------------------------------------------------------------------------------- pin
def test_restatement_is_grid_sample_and_the_reference_fixture():
    """without rounding (float64 coordinates: exact fractions), corr_bar's ref is corr_grid_sample to 1e-12, on a case
    of this file and on the reference kernel's fixture; the fixture's fp32 outputs lie inside the bar of a sequential
    fp32 accumulation over its 128 channels (with the fixture's fp32 coordinates, as the kernel took them)"""
    d = torch.load(os.path.join(GOLD, "corr_ref_fp32.pt"))
    for f1, f2, coords, ii, jj in (_case("nominal"), (d["fmap1"], d["fmap2"], d["coords"], d["ii"], d["jj"])):
        ref, _ = OC.corr_bar(f1, f2, coords.double(), ii, jj, R, OC.ACC_MMA)
        gs = OC.corr_grid_sample(f1.double(), f2.double(), coords.double(), ii, jj, R)
        assert (ref - gs).abs().max().item() <= 1e-12 * ref.abs().max().item()
    ref, b = OC.corr_bar(d["fmap1"], d["fmap2"], d["coords"], d["ii"], d["jj"], d["radius"], OC.acc_generic(128))
    assert _inside(d["out"], ref, b, torch.float32), OC.bar_use(d["out"], ref, b).max().item()


def test_reference_fp16_kernel_is_outside_the_bar():
    """the reference's fp16 kernel accumulates in fp16 (correlation_kernel.cu:121-131): its outputs leave the bar"""
    f1, f2, coords, ii, jj = _case("nominal")
    ref, b = _bar(f1, f2, coords, ii, jj, "mma")
    got = emulate(f1, f2, coords, ii, jj, "mma", "acc_fp16")
    assert (~OC.within(got.half(), ref, b)).sum().item() > ref.numel() // 10


def test_round_to_is_one_rounding():
    """round_to equals numpy's float64 -> float16 conversion (one rounding), also at and next to the half-way points
    where torch's CPU cast, which rounds through float32, can differ; bf16 agrees with torch on float32 inputs"""
    g = torch.Generator().manual_seed(0)
    h = torch.randn(20000, generator=g).half().double()
    ulp = torch.pow(2.0, (torch.frexp(h)[1] - 11).clamp(min=-24).double())
    x = torch.cat([torch.randn(20000, generator=g, dtype=torch.float64) * 10.0 ** torch.randint(-9, 5, (20000,), generator=g),
                   h + ulp / 2, h - ulp / 2, h + ulp / 2 * (1 + 2.0 ** -30), h + ulp / 2 * (1 - 2.0 ** -30),
                   torch.tensor([65504.0, 65519.99, 65520.0, -7e4, 0.0, 2.0 ** -25, 3 * 2.0 ** -26])])
    with np.errstate(over="ignore"):
        want = torch.from_numpy(x.numpy().astype(np.float16).astype(np.float64))
    assert torch.equal(OC.round_to(x, torch.float16), want)
    y = torch.randn(20000, generator=g).double()
    assert torch.equal(OC.round_to(y, torch.bfloat16), y.float().bfloat16().double())


def test_bar_use_measures_the_rounding_cell():
    """bar_use is 0 for correctly rounded outputs and just above 1 one fp16 ulp away with a tiny bar"""
    ref = torch.tensor([1.0 + 2.0 ** -12, 0.0, -3.0, 2.0 ** -20], dtype=torch.float64)
    b = torch.full_like(ref, 1e-9)
    out = OC.round_to(ref, torch.float16).half()
    assert OC.bar_use(out, ref, b).max().item() == 0
    off = (out.view(torch.int16) + 1).view(torch.float16)
    assert (OC.bar_use(off, ref, b) > 1).all()
    assert not OC.within(off, ref, b).any() and OC.within(out, ref, b).all()
