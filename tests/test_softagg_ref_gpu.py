"""The SoftAgg kernels against the float64 SoftAgg of oracle/softagg.py, element by element within its error bar.

Every case runs dpvo_softagg_fused (the f|g layer fused with the segment softmax, `fgi_*` weights), linear_f16 +
dpvo_softagg_reduce (`fg_*` weights) and the fp64 reference built from the module's own agg.f / agg.g parameters (so a
mistake in Update.pack() shows), on the same rows and grouping.  The layouts are the ones where the fused kernel's 64-row
tile logic changes -- group edges on, and one row either side of, tile edges; groups spanning hundreds of tiles; CTAs with
1, 2 and 3 tiles of the persistent grid; the parked-slot groups of a DevicePatchGraph store -- and the value regimes push
the softmax to flat, peaked and one-hot and F close to the fp16 range.  A workspace full of NaN must give the same bits
as a zeroed one.  The last tests follow one update's aggregation stage through h and residual_sum16."""
import copy

import pytest
import torch

from oracle import softagg as OS
from dpvo_b200 import synthetic
from dpvo_b200.net import Update, EdgeGroups, DIM
from dpvo_b200.patchgraph import DevicePatchGraph

pytestmark = pytest.mark.gpu
DEV = "cuda"

# tile counts a s + b, s = SMs / 4 the CTAs per channel slice of the persistent grid (min(tiles, s) per slice): s - 1 and
# s tiles give every CTA one tile, s + 1 and 2 s + 1 give one CTA a tile more than the rest, 2 s and 3 s give every CTA
# 2 and 3 tiles, which its two consumer warpgroups take alternately
TILES = {"s-1": (1, -1), "s": (1, 0), "s+1": (1, 1), "2s": (2, 0), "2s+1": (2, 1), "3s": (3, 0)}
LAYOUTS = (["one-E%d" % e for e in (1, 63, 64, 65, 47712)]
           + ["aligned-" + t for t in TILES] + ["shifted-" + t for t in TILES]
           + ["size%d-%s" % (k, t) for k in (63, 65, 128, 129) for t in ("s", "2s+1")]
           + ["edges1-2s+1", "alt1_127-3s", "ragged-G", "ragged-G+77", "ragged-E"]
           + ["state_%s-%s" % (c, nm) for c in ("default", "fast") for nm in ("kk", "ij")]
           + ["store%d-%s" % (b, nm) for b in (1, 3) for nm in ("kk", "ij")])
REGIMES = ["nominal", "peaked", "flat", "largeF", "onehot"]
ONEHOT_COEF = (64.0, -64.0, 32.0)          # G = coef s + bias for an integer row score s in [-310, 310]: per channel the
ONEHOT_BIAS = (0.0, 0.0, -1.0e4)           # argmax is the top score, the bottom one, and the top one with all G < 0


def _tiles(spec):
    a, b = TILES[spec]
    return a * (torch.cuda.get_device_properties(0).multi_processor_count // 4) + b


def _key_index(key):
    """groups numbered by sorted key, as the grouping kernel numbers them"""
    return torch.unique(key, return_inverse=True)[1]


class _Layout:
    pass


_LAYOUTS = {}


def _layout(name):
    """grouping, group bound, reference group index, parked rows and the aggregation (kk / ij) of a layout"""
    if name in _LAYOUTS:
        return _LAYOUTS[name]
    L = _Layout()
    kind, arg = name.split("-", 1)
    L.nm, L.parked, L.max_groups = "ij", None, None
    if kind.startswith("state_"):
        st = synthetic.make_state(kind[6:], 36 if kind == "state_default" else 14, device=DEV, features=False)
        M = st.cfg["M"]
        # the bounds UpdateRunner sizes the per-group buffers with: padding rows past the group count
        bounds = (int((st.kk // M).unique().numel()) * M, int(torch.unique(st.ii * 100000 + st.jj).numel()))
        gk, gp = EdgeGroups.pair((st.kk, None, st.jj), (st.ii, st.jj, None), *bounds)
        L.nm = arg
        L.grp, L.max_groups = (gk, bounds[0]) if arg == "kk" else (gp, bounds[1])
        L.idx = _key_index(st.kk if arg == "kk" else st.ii * 12345 + st.jj)
    elif kind.startswith("store"):
        # a DevicePatchGraph store with parked slots: all of a stream's parked slots share kk = dummy_patch and
        # ii = jj = dummy_frame, one kk group and one ij group of ~1,000 rows per stream; their state rows are zero
        B, cfg, F = int(kind[5:]), synthetic.CONFIGS["fast"], 64
        M = cfg["M"]
        edges = [synthetic.replay_edges(n, M, cfg["lifetime"], cfg["removal"]) for n in (14, 12, 10)[:B]]
        cap = max(e[0].numel() for e in edges) + 1000
        dummies = [b * F + F - 1 for b in range(B)]
        if B == 1:
            store = DevicePatchGraph(cap, M, dummies[0], DEV)
            graphs = [store]
        else:
            store, graphs = DevicePatchGraph.stacked(B, cap, M, dummies, DEV)
        for b, (ii, jj, kk) in enumerate(edges):
            graphs[b].append(ii.to(DEV) + b * F, jj.to(DEV) + b * F, kk.to(DEV) + b * F * M)
        ii, jj, kk = store.ii, store.jj, store.kk
        L.parked = ~store.active.bool()
        assert int(L.parked.sum()) >= 1000 * B
        gk, gp = EdgeGroups.pair((kk, None, jj), (ii, jj, None))
        L.nm = arg
        L.grp = gk if arg == "kk" else gp
        L.idx = _key_index(kk if arg == "kk" else ii * 12345 + jj)
    else:
        E = int(arg[1:]) if kind == "one" else 64 * _tiles("2s+1" if kind == "ragged" else arg)
        sizes = OS.group_sizes(kind, E, seed=11)
        # a fixed permutation deals the rows to the groups, so `order` is not the identity
        key = torch.repeat_interleave(torch.arange(len(sizes)), torch.as_tensor(sizes))
        key = key[torch.randperm(E, generator=torch.Generator().manual_seed(E + len(sizes)))].to(DEV)
        G = len(sizes)
        if kind == "ragged":
            L.max_groups = {"G": G, "G+77": G + 77, "E": E}[arg]
        L.grp = EdgeGroups(key, max_groups=L.max_groups or G)
        L.idx = _key_index(key)
    L.max_groups = L.grp.max_groups
    L.E = L.idx.numel()
    L.G = int(L.grp.n.item())
    assert L.G == int(L.idx.max()) + 1
    _LAYOUTS[name] = L
    return L


@pytest.fixture(scope="module")
def base():
    torch.manual_seed(5)
    return Update().to(DEV).eval()


def _inputs(L, base, regime, seed):
    """x [1, E, 384] fp16 and the module of the regime (a copy of `base` with the aggregation's f / g changed)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(L.E, DIM, generator=g, device=DEV) * 0.5
    if L.parked is not None:
        x[L.parked] = 0                               # parked slots: zero state rows, identical F and G (ties)
    m = copy.deepcopy(base)
    agg = getattr(m, "agg_" + L.nm)
    with torch.no_grad():
        if regime == "peaked":                        # a few rows of each group carry almost all the weight
            agg.g.weight.mul_(8)
            agg.g.bias.mul_(8)
        elif regime == "flat":                        # equal weights: y is the mean of F
            agg.g.weight.zero_()
            agg.g.bias.fill_(0.75)
        elif regime == "largeF":                      # |F| up to 3e4, below the fp16 maximum 65504
            F = x.half().float() @ agg.f.weight.half().float().t() + agg.f.bias
            s = 3.0e4 / F.abs().max().item()
            agg.f.weight.mul_(s)
            agg.f.bias.mul_(s)
        elif regime == "onehot":
            # column 0 of x is an integer score per row; the first row of each group (sorted order) gets 310, the last
            # -310, the others [-300, 300], so per channel the top G exceeds the next by >= 320
            s = torch.randint(-300, 301, (L.E,), generator=g, device=DEV).float()
            gs = L.grp.group_start[:L.G + 1].long()
            first, last = L.grp.order[gs[:-1]].long(), L.grp.order[gs[1:] - 1].long()
            s[last] = -310
            s[first] = 310                            # a 1-row group keeps 310
            x[:, 0] = s
            c = torch.tensor(ONEHOT_COEF, device=DEV).repeat(DIM // 3)
            agg.g.weight.zero_()
            agg.g.weight[:, 0] = c
            agg.g.bias.copy_(torch.tensor(ONEHOT_BIAS, device=DEV).repeat(DIM // 3))
    return x.half()[None], m, agg


def _within(y, ref, B, L, what):
    """|y - ref| <= B per element, with the worst element described on failure"""
    y = y.double()
    assert torch.isfinite(y).all(), what + ": non-finite output"
    ratio = (y - ref).abs() / B
    worst = ratio.max().item()
    if worst > 1.0:
        g, c = divmod(int(ratio.argmax()), ratio.shape[1])
        n = int((L.idx == g).sum())
        raise AssertionError("%s: |y - ref| = %.3g > bar %.3g (x%.2f) at group %d (%d rows), channel %d: y %.6g, ref %.6g; "
                             "%d elements over" % (what, abs(y[g, c] - ref[g, c]).item(), B[g, c].item(), worst, g, n, c,
                                                   y[g, c].item(), ref[g, c].item(), int((ratio > 1).sum())))
    return worst


def _bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("layout", LAYOUTS)
def test_softagg_vs_fp64(ext, base, layout, regime):
    ex = ext[3]
    L = _layout(layout)
    x, m, agg = _inputs(L, base, regime, seed=LAYOUTS.index(layout) * 7 + REGIMES.index(regime))
    P = m.packed()
    grp, mg, G = L.grp, L.max_groups, L.G

    def fused(ws=None):
        return ex.softagg_fused(x, grp.order, grp.group_of, grp.group_start, grp.n, mg, *P["fgi_" + L.nm], ws)

    # workspace: records the launch did not write are never read, and nothing past the required size is written
    wsb = ex.softagg_fused_workspace_bytes(L.E)
    y = fused()
    y_zero = fused(torch.zeros(wsb + 4096, dtype=torch.uint8, device=DEV))
    nan_ws = torch.full(((wsb + 4096) // 4,), float("nan"), device=DEV).view(torch.uint8)
    tail = nan_ws[wsb:].clone()
    y_nan = fused(nan_ws)
    assert y.shape == (1, mg, DIM)
    assert torch.equal(_bits(y), _bits(y_zero)), "two launches differ"
    assert torch.equal(_bits(y), _bits(y_nan)), "the result depends on stale workspace contents"
    assert torch.equal(nan_ws[wsb:], tail), "written past the required workspace"

    fg = ex.linear_f16(x, *P["fg_" + L.nm], 0)
    y2 = ex.softagg_reduce(fg, grp.order, grp.group_start, grp.n, mg)
    for t, nm in ((y, "fused"), (y2, "reduce")):
        assert (_bits(t[0, G:]) == 0).all(), nm + ": rows G..max_groups-1 must be +0"
    # the two forms round F and G alike (1-row groups agree bit for bit) and differ in the order of the fp32 sums: within
    # 2 fp16 ulps, except where the group's sum cancels (|y| < sum w |F| / 8).  There the order alone moves y by more
    # than 2 of its own ulps (79 at y = 3e-3, sum w |F| = 6e3 in the large-F regime), and the bar's sum term is added
    F16, G16 = fg[0, :, :DIM].double(), fg[0, :, DIM:].double()
    ref16 = OS.aggregate(F16, G16, L.idx, G)
    mag16 = OS.aggregate(F16.abs(), G16, L.idx, G)
    rows = torch.bincount(L.idx, minlength=G).double()[:, None]
    cancels = ref16.abs() < mag16 / 8
    _within(y[0, :G], y2[0, :G].double(), 2 * OS.ulp16(ref16) + torch.where(cancels, rows * OS.U22 * mag16, 0.0), L,
            "fused vs linear_f16 + reduce")

    ref, F, Gl = OS.reference(x, agg.f.weight, agg.f.bias, agg.g.weight, agg.g.bias, L.idx, G)
    SF, SG = OS.magnitude(x, agg.f.weight, agg.f.bias), OS.magnitude(x, agg.g.weight, agg.g.bias)
    if regime == "onehot":
        # the first-order bar does not hold here; every group's top G is separated from the next by more than
        # 20 + 2 ulp16(G), so no rounding moves the argmax and y is the argmax row's fp16 F, within one ulp of F and of y
        # and the layer's fp32 accumulation error (the bar's ACC term: x[:, 0] = +-310 makes some of these F cancel)
        top = OS.scatter_max(Gl[None], L.idx, dim=1, dim_size=G)[0][0]
        at_top = Gl == top[L.idx]
        assert (OS.scatter_sum(at_top.double()[None], L.idx, dim=1, dim_size=G)[0] == 1).all()
        second = OS.scatter_max(torch.where(at_top, -torch.inf, Gl)[None], L.idx, dim=1, dim_size=G)[0][0]
        sizes = torch.bincount(L.idx, minlength=G)
        gap = (top - second)[sizes > 1]
        assert (gap > 20 + 2 * OS.ulp16(top[sizes > 1])).all() and Gl.abs().max() <= 2.0e4
        assert (Gl.view(-1, 3)[:, 2] < 0).all()
        f_top = ref.half().double()                 # = fp16(F) of the argmax row: all other weights are < e^-320
        acc_top = OS.ACC * OS.aggregate(SF, Gl, L.idx, G)
        for t, nm in ((y, "fused"), (y2, "reduce")):
            _within(t[0, :G], f_top, OS.ulp16(f_top) + OS.ulp16(t[0, :G].double()) + acc_top, L, nm + " one-hot")
        return
    assert Gl.abs().max() < 64, "the first-order bar needs |G| < 64"
    B = OS.bar(F, Gl, SF, SG, L.idx, ref, G)
    _within(y[0, :G], ref, B, L, "fused")
    _within(y2[0, :G], ref, B, L, "linear_f16 + reduce")
    # both forms against the fp64 aggregation of linear_f16's fp16 F and G: softagg_reduce's exact inputs, and the values
    # the fused kernel rounds its own layer output to
    B16 = OS.bar_input16(F16, G16, L.idx, ref16, G)
    _within(y2[0, :G], ref16, B16, L, "reduce on its fp16 inputs")
    _within(y[0, :G], ref16, B16, L, "fused on linear_f16's fp16 F and G")


def _gemm_ok(y, x16, lin):
    """linear_f16's bar (tests/test_gemm_gpu.py): 2e-3 of max(1, |ref|) against the layer on the device's own input"""
    ref = x16.reshape(-1, DIM).double() @ lin.weight.half().double().t() + lin.bias.float().double()
    err = (y.reshape(-1, DIM).double() - ref).abs().max().item()
    assert err <= 2e-3 * max(1.0, ref.abs().max().item()), err


def test_aggregation_stage_of_an_update(ext, base):
    """agg_kk -> h_kk -> residual_sum16 -> agg_ij -> h_ij as Update._forward_chains runs them on the bench state
    (E = 47,712, the runner's group bounds), each stage against fp64 on the device's own input to that stage"""
    ex = ext[3]
    L_kk, L_ij = _layout("state_default-kk"), _layout("state_default-ij")
    P = base.packed()
    g = torch.Generator(device=DEV).manual_seed(31)
    E = L_kk.E
    net32 = torch.randn(1, E, DIM, generator=g, device=DEV)
    inp16 = torch.randn(E, DIM, generator=g, device=DEV).half()
    corr = (torch.randn(1, E, 896, generator=g, device=DEV) * 0.5).half()
    gk, gp = L_kk.grp, L_ij.grp
    n16 = ex.update_corr_norm(corr, P["A_W0"], P["A_W25"], P["A_p"], net32, inp16, None)
    ix, jx = ex.neighbors_from_groups(gk.order, gk.group_of)
    n16b = ex.update_neighbor_mlp(n16, ix, P["C1_W"], P["C1_p"], net32)
    n16 = ex.update_neighbor_mlp(n16b, jx, P["C2_W"], P["C2_p"], net32, n16)
    for L, grp, agg, nm in ((L_kk, gk, base.agg_kk, "kk"), (L_ij, gp, base.agg_ij, "ij")):
        y = ex.softagg_fused(n16, grp.order, grp.group_of, grp.group_start, grp.n, grp.max_groups, *P["fgi_" + nm])
        ref, F, Gl = OS.reference(n16, agg.f.weight, agg.f.bias, agg.g.weight, agg.g.bias, L.idx, L.G)
        B = OS.bar(F, Gl, OS.magnitude(n16, agg.f.weight, agg.f.bias), OS.magnitude(n16, agg.g.weight, agg.g.bias), L.idx, ref, L.G)
        _within(y[0, :L.G], ref, B, L, "agg_" + nm)
        h = ex.linear_f16(y, *P["h_" + nm], 0)
        assert h.shape == (1, grp.max_groups, DIM)
        _gemm_ok(h, y, agg.h)
        if nm == "kk":
            h_kk = h.reshape(-1, DIM)
            n16 = ex.residual_sum16(net32, h_kk, gk.group_of)
            assert torch.equal(n16, (net32 + h_kk.float()[gk.group_of.long()]).half())


@pytest.mark.parametrize("E", [1, 77, 47712])
def test_residual_sum16(ext, E):
    """fp16(net + u[group_of]) bit for bit, with fp16 and fp32 u and without a grouping; net itself is not written"""
    g = torch.Generator(device=DEV).manual_seed(E)
    net = torch.randn(1, E, DIM, generator=g, device=DEV) * 4
    n_u = max(1, E // 20)
    gof = torch.randint(0, n_u, (E,), generator=g, device=DEV, dtype=torch.int32)
    net0 = net.clone()
    for u in (torch.randn(n_u, DIM, generator=g, device=DEV).half(), torch.randn(n_u, DIM, generator=g, device=DEV) * 1e3):
        out = ext[3].residual_sum16(net, u, gof)
        assert out.dtype == torch.half and out.shape == net.shape
        assert torch.equal(out, (net + u.float()[gof.long()]).half())
    u = torch.randn(1, E, DIM, generator=g, device=DEV).half()
    assert torch.equal(ext[3].residual_sum16(net, u), (net + u.float()).half())
    assert torch.equal(net, net0)
