"""The error bar of oracle/softagg.py is tight enough to matter: on small versions of the group layouts of
test_softagg_ref_gpu.py it accepts the fp64 SoftAgg computed from fp16-rounded and one-ulp-perturbed F and G, and it
rejects the fp64 result of each of the mistakes a fused SoftAgg kernel could make -- a group edge one row off at a tile
edge, a tile's partial result left out of the merge, g channel slices interleaved wrongly, f and g exchanged.  Also pins
the restatement to the SoftAgg of oracle/update.py."""
import numpy as np
import pytest
import torch

from oracle import softagg as OS, update as OU

DIM = 384
E = 64 * 5
LAYOUTS = ["one-65", "one-320", "aligned", "shifted", "size63", "size65", "size128", "size129", "edges1", "alt1_127", "ragged"]
REGIMES = ["nominal", "peaked", "flat", "largeF"]


def _case(layout, regime):
    """(x16 [E, 384], Wf, bf, Wg, bg, group_of, order): rows dealt to the groups by a fixed permutation; `order` lists
    the rows in sorted group order, as the grouping kernel does"""
    kind, _, rows = layout.partition("-")
    n = int(rows) if rows else E
    sizes = OS.group_sizes(kind, n, seed=3)
    g = torch.Generator().manual_seed(n + len(sizes) + REGIMES.index(regime))
    order = torch.randperm(n, generator=g)
    group_of = torch.empty(n, dtype=torch.long)
    group_of[order] = torch.repeat_interleave(torch.arange(len(sizes)), torch.as_tensor(sizes))
    x = (torch.randn(n, DIM, generator=g) * 0.5).half()
    lim = DIM ** -0.5                                         # nn.Linear's initialisation
    Wf, Wg = [(torch.rand(DIM, DIM, generator=g) * 2 - 1) * lim for _ in range(2)]
    bf, bg = [(torch.rand(DIM, generator=g) * 2 - 1) * lim for _ in range(2)]
    if regime == "peaked":
        Wg, bg = Wg * 8, bg * 8
    elif regime == "flat":
        Wg, bg = torch.zeros_like(Wg), torch.full_like(bg, 0.75)
    elif regime == "largeF":
        s = 3.0e4 / OS.layer(x, Wf, bf).abs().max().item()
        Wf, bf = Wf * s, bf * s
    return x, Wf.half(), bf, Wg.half(), bg, group_of, order


def _rejects(y, ref, B):
    return bool(((y - ref).abs() > B).any())


def _row_moved_back(group_of, order):
    """the row at sorted position 64 t (the first such t that starts a group) moved into the previous group"""
    gs = group_of[order]
    for p in range(64, gs.numel(), 64):
        if gs[p] != gs[p - 1]:
            out = group_of.clone()
            out[order[p]] = gs[p - 1]
            return out
    return None


def _tile_left_out(group_of, order):
    """the rows of the first tile of the first group that crosses a tile edge given a group of their own (index G): the
    group's result is then what a merge without that tile's partial (m, z, a) would give"""
    gs = group_of[order]
    for p in range(64, gs.numel(), 64):
        if gs[p] == gs[p - 1]:
            out = group_of.clone()
            seg = order[p - 64:p][gs[p - 64:p] == gs[p]]
            out[seg] = int(group_of.max()) + 1
            return out
    return None


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("layout", LAYOUTS)
def test_bar_accepts_fp16_rounding_and_one_ulp(layout, regime):
    x, Wf, bf, Wg, bg, group_of, order = _case(layout, regime)
    ref, F, G = OS.reference(x, Wf, bf, Wg, bg, group_of)
    assert G.abs().max() < 64
    B = OS.bar(F, G, OS.magnitude(x, Wf, bf), OS.magnitude(x, Wg, bg), group_of, ref)
    # F and G rounded to fp16 once, y rounded to fp16
    F16, G16 = F.half().double(), G.half().double()
    assert not _rejects(OS.aggregate(F16, G16, group_of).half().double(), ref, B)
    # the kernels' rounding points: the layer accumulated in fp32, then rounded to fp16
    F32, G32 = [(x.float() @ W.float().t() + b.float()).half().double() for W, b in ((Wf, bf), (Wg, bg))]
    assert not _rejects(OS.aggregate(F32, G32, group_of).half().double(), ref, B)
    # F and G one ulp away from their exact values: random directions, and the direction that moves y the most
    g = torch.Generator().manual_seed(7)
    worst = torch.sign(F - ref[group_of])
    for sf, sg in [[torch.randint(-1, 2, F.shape, generator=g).double() for _ in range(2)] for _ in range(2)] + [(1, worst)]:
        Fp, Gp = F + sf * OS.ulp16(F), G + sg * OS.ulp16(G)
        assert not _rejects(OS.aggregate(Fp, Gp, group_of).half().double(), ref, B)
        # softagg_reduce's bar: exact fp16 inputs, the result rounded once
        F16p, G16p = Fp.half().double(), Gp.half().double()
        r16 = OS.aggregate(F16p, G16p, group_of)
        assert not _rejects(r16.half().double(), r16, OS.bar_input16(F16p, G16p, group_of, r16))


def test_bar_is_not_loose():
    """the worst-direction one-ulp perturbation uses most of the bar somewhere: a bar several times too wide fails here"""
    worst_ratio = 0.0
    for layout in LAYOUTS:
        x, Wf, bf, Wg, bg, group_of, _ = _case(layout, "nominal")
        ref, F, G = OS.reference(x, Wf, bf, Wg, bg, group_of)
        B = OS.bar(F, G, OS.magnitude(x, Wf, bf), OS.magnitude(x, Wg, bg), group_of, ref)
        y = OS.aggregate(F + OS.ulp16(F), G + torch.sign(F - ref[group_of]) * OS.ulp16(G), group_of)
        worst_ratio = max(worst_ratio, ((y - ref).abs() / B).max().item())
    assert 0.5 < worst_ratio <= 1.0, worst_ratio


MUTATIONS = {
    "row_at_64t_in_previous_group": _row_moved_back,
    "tile_partial_left_out": _tile_left_out,
    "g_slices_swapped": None,
    "f_g_swapped": None,
}
# a mutation runs where it means something: a group edge at a row 64 t, a group across a tile edge, g not constant
CASES = [(lay, reg, mut) for lay in LAYOUTS for reg in REGIMES for mut, where in MUTATIONS.items()
         if (where is None or where(*_case(lay, reg)[5:]) is not None) and not (mut == "g_slices_swapped" and reg == "flat")]


def test_every_mutation_applies_to_its_layouts():
    runs = {mut: {lay for lay, _, m in CASES if m == mut} for mut in MUTATIONS}
    assert {"aligned", "size128", "edges1", "alt1_127"} <= runs["row_at_64t_in_previous_group"]
    assert {"one-65", "one-320", "shifted", "size63", "size65", "size128", "size129", "alt1_127"} <= runs["tile_partial_left_out"]
    assert runs["g_slices_swapped"] == runs["f_g_swapped"] == set(LAYOUTS)


@pytest.mark.parametrize("layout,regime,mutation", CASES)
def test_bar_rejects_mutations(layout, regime, mutation):
    x, Wf, bf, Wg, bg, group_of, order = _case(layout, regime)
    ref, F, G = OS.reference(x, Wf, bf, Wg, bg, group_of)
    n = ref.shape[0]
    B = OS.bar(F, G, OS.magnitude(x, Wf, bf), OS.magnitude(x, Wg, bg), group_of, ref)
    if mutation == "row_at_64t_in_previous_group":
        y = OS.aggregate(F, G, _row_moved_back(group_of, order), n)
    elif mutation == "tile_partial_left_out":
        y = OS.aggregate(F, G, _tile_left_out(group_of, order), n + 1)[:n]
    elif mutation == "g_slices_swapped":
        p = torch.arange(DIM)
        p[:96], p[96:192] = torch.arange(96, 192), torch.arange(96)
        y = OS.aggregate(F, G[:, p], group_of, n)
    else:
        y = OS.aggregate(G, F, group_of, n)
    assert _rejects(y.half().double(), ref, B)


def test_reference_is_the_oracle_softagg():
    """reference() is oracle/update.py's SoftAgg (f, g and the scatter softmax; h the identity) in fp64"""
    x, Wf, bf, Wg, bg, group_of, _ = _case("ragged", "nominal")
    key = group_of * 7 + 3                                    # any key with the same order of groups
    m = OU.SoftAgg(DIM, expand=False).double()
    with torch.no_grad():
        for lin, W, b in ((m.f, Wf, bf), (m.g, Wg, bg), (m.h, torch.eye(DIM), torch.zeros(DIM))):
            lin.weight.copy_(W.double())
            lin.bias.copy_(b.double())
        want = m(x.double()[None], key)[0]
    ref, _, _ = OS.reference(x, Wf, bf, Wg, bg, group_of)
    assert (ref - want).abs().max().item() <= 1e-12 * want.abs().max().item()


def test_ulp16_is_the_fp16_spacing():
    v = np.concatenate([np.float16(2.0) ** np.arange(-24, 16, dtype=np.float16),
                        np.random.default_rng(0).standard_normal(1000).astype(np.float16) * 100])
    v = v[v != 0]
    want = np.spacing(np.abs(v)).astype(np.float64)
    got = OS.ulp16(torch.from_numpy(v.astype(np.float64))).numpy()
    assert np.array_equal(got, want)
