"""ORACLE (test infrastructure -- never imported by the product path).

The SoftAgg aggregation of the reference (blocks.py:31-48, without the h layer) in float64, and the per-element error
bar of the fp16 kernels that compute it (dpvo_softagg_fused, linear_f16 + dpvo_softagg_reduce):

    F = x Wf^T + bf,  G = x Wg^T + bg,  y[g, c] = sum_{i in g} softmax_g(G[:, c])_i F[i, c]

with scatter_softmax / scatter_sum from oracle/update.py, the restatement pinned to the reference.  Works on any device;
on CUDA the layer of E = 47,712 rows is ~30 GFLOP of fp64.

Group index: `group_of[i]` in [0, n_groups) for every row i, groups numbered in the kernels' order (sorted key).
"""
import torch

from .update import scatter_max, scatter_softmax, scatter_sum

U22, U20 = 2.0 ** -22, 2.0 ** -20
# fp32 accumulation of a K = 384 fp16 dot product on the tensor cores: one rounding of the accumulator per k16 MMA step
# (24 steps) and one for the bias, each at most one fp32 ulp (2^-23, truncation included) of a partial sum whose size is
# at most sum_k |x_k W_k| + |b|.  This is a model of the accumulator, not a documented or separately measured property:
# tensor cores that align the products of a step to the largest one and truncate could lose up to about k ulps of the
# largest product per step.  A model that is too optimistic makes the tests fail rather than pass a wrong kernel; on an
# H100 the kernels stay within the bar built on it
ACC = (384 // 16 + 1) * 2.0 ** -23


def ulp16(v):
    """the fp16 spacing at |v|: 2^(floor(log2 |v|) - 10) for normal values, 2^-24 in the subnormal range"""
    a = v.abs()
    _, e = torch.frexp(a)                              # a = m 2^e, m in [0.5, 1)
    return torch.where(a < 2.0 ** -14, torch.full_like(a, 2.0 ** -24), torch.ldexp(torch.ones_like(a), e - 11))


def layer(x16, W, b):
    """x W^T + b exactly (fp64) from the fp16 operands: x and W as fp16, b as fp32 -- the values the kernels read"""
    return x16.reshape(-1, x16.shape[-1]).half().double() @ W.half().double().t() + b.float().double()


def magnitude(x16, W, b):
    """sum_k |x_k W_k| + |b| per row and output channel (fp64): the size of the partial sums of the layer"""
    return x16.reshape(-1, x16.shape[-1]).half().double().abs() @ W.half().double().abs().t() + b.float().double().abs()


def aggregate(F, G, group_of, n_groups=None):
    """y [n_groups, C] = scatter_sum(F * scatter_softmax(G)) over rows of [E, C] fp64 F, G"""
    idx = group_of.long()
    n = int(idx.max().item()) + 1 if n_groups is None else int(n_groups)
    w = scatter_softmax(G[None], idx, dim=1)
    return scatter_sum(F[None] * w, idx, dim=1, dim_size=n)[0]


def reference(x16, Wf, bf, Wg, bg, group_of, n_groups=None):
    """the SoftAgg aggregation (no h) in fp64: returns (y [n_groups, C], F [E, C], G [E, C])"""
    F, G = layer(x16, Wf, bf), layer(x16, Wg, bg)
    return aggregate(F, G, group_of, n_groups), F, G


def _bar(F, G, group_of, y, n_groups, input16, SF=None, SG=None):
    idx = group_of.long()
    n = int(idx.max().item()) + 1 if n_groups is None else int(n_groups)
    if y is None:
        y = aggregate(F, G, idx, n)
    w = scatter_softmax(G[None], idx, dim=1)[0]
    top = scatter_max(G[None], idx, dim=1, dim_size=n)[0][0]
    rows = torch.bincount(idx, minlength=n).to(F.dtype)[:, None]
    dG = (G.abs() + top[idx].abs()) * U22 + U20                   # exp2f argument g log2e - m log2e, and exp2f itself
    dF = torch.zeros_like(F)
    if not input16:
        dF = ulp16(F) + ACC * SF                                  # fp32 accumulation + one fp16 rounding of F
        dG = dG + ulp16(G) + ACC * SG                             # ... and of G
    per_row = w * (dF + (F - y[idx]).abs() * dG)
    sums = scatter_sum(per_row[None], idx, dim=1, dim_size=n)[0]
    mag = scatter_sum((w * F.abs())[None], idx, dim=1, dim_size=n)[0]
    return ulp16(y) + sums + rows * U22 * mag


def bar(F, G, SF, SG, group_of, y=None, n_groups=None):
    """Per-element bound on |y_kernel - y| for the fp16 kernels that compute F and G themselves (softagg_fused,
    linear_f16 + softagg_reduce), from the fp64 F, G of `reference`, their result y and the magnitudes SF, SG
    (`magnitude`) of the two layers:

        B = ulp16(y) + sum_i w_i [ dF_i + |F_i - y| (dG_i + (|G_i| + |max G|) 2^-22 + 2^-20) ] + n 2^-22 sum_i w_i |F_i|
        dF_i = ulp16(F_i) + ACC SF_i,  dG_i = ulp16(G_i) + ACC SG_i,  ACC = 25 2^-23

    w_i are the fp64 softmax weights of the group, n its size.  The terms:
      - ulp16(F_i), ulp16(G_i): F and G are rounded to fp16 once; the kernel's fp32 accumulation of the layer can move
        the value across a rounding boundary, so the bound takes a whole ulp, not half.  dy/dF_i = w_i and
        dy/dG_i = w_i (F_i - y) (the shift by the group maximum cancels in the ratio);
      - ACC SF_i, ACC SG_i: the fp32 accumulation error itself (ACC rests on the accumulator model described at its
        definition), which the whole ulp does not cover where the dot product cancels (|F| much smaller than
        sum_k |x_k W_k|).  There a 1-row group, whose y is its own fp16 F, is off by more than ulp16(F) + ulp16(y).
        Elsewhere the term adds ~5% to the bar;
      - (|G_i| + |max G|) 2^-22 + 2^-20: the relative error of the weight exp2f(g log2e - m log2e).  The two fp32
        products round at 2^-24 of their size, an argument error d changes the weight by d ln 2, so the weight's error
        is below (|G_i| + |max G|) 2^-24 (log2e ln 2 = 1); the bound takes 4x that.  2^-20 covers exp2f's own error,
        the rounding of the difference and the second exp2f of the combine step;
      - n 2^-22 sum w |F|: the fp32 running sums z and a over up to n rows (2^-24 each, x 4 for both sums and the
        division);
      - ulp16(y): the final fp16 rounding of a / z.
    The bound is first order in these perturbations: it holds while they are small, so inputs keep |G| < 64 (ulp16(G)
    <= 2^-5).  No safety factor is applied."""
    return _bar(F, G, group_of, y, n_groups, False, SF, SG)


def bar_input16(F16, G16, group_of, y=None, n_groups=None):
    """`bar` for softagg_reduce, whose F and G are its exact fp16 inputs: the same bound without the dF_i and dG_i
    terms (accumulation and rounding of the layer).  F16, G16 are those inputs as fp64 and y the fp64 aggregation of them."""
    return _bar(F16.double(), G16.double(), group_of, y, n_groups, True)


def group_sizes(kind, rows, seed=0):
    """Group sizes, in sorted order, of the layouts at which dpvo_softagg_fused's 64-row tile logic changes, over `rows`
    rows (a multiple of 64 except for "one"):
        one        one group of every row
        aligned    groups of 64, each exactly one tile (no crossing group)
        shifted    the same moved by one row: 1, 64, ..., 64, 63 -- every group crosses a tile edge
        size<k>    groups of k rows (63, 65, 128, 129: one row short of / past one and two tiles), the last one shorter
        edges1     1-row groups at rows 64 t - 1 and 64 t, the last row of a tile and the first of the next
        alt1_127   1-row groups alternating with 127-row groups
        ragged     random sizes in [1, 150]"""
    if kind == "one":
        return [rows]
    if kind == "aligned":
        return [64] * (rows // 64)
    if kind == "shifted":
        return [1] + [64] * (rows // 64 - 1) + [63]
    if kind.startswith("size"):
        k = int(kind[4:])
        return [k] * (rows // k) + ([rows % k] if rows % k else [])
    if kind == "edges1":
        starts = sorted({0} | {s for t in range(1, rows // 64) for s in (64 * t - 1, 64 * t, 64 * t + 1)})
        return [b - a for a, b in zip(starts, starts[1:] + [rows])]
    if kind == "alt1_127":
        sizes = []
        while sum(sizes) < rows:
            sizes.append(1 if len(sizes) % 2 == 0 else min(127, rows - sum(sizes)))
        return sizes
    if kind == "ragged":
        g = torch.Generator().manual_seed(seed)
        sizes = []
        while sum(sizes) < rows:
            sizes.append(min(int(torch.randint(1, 151, (1,), generator=g)), rows - sum(sizes)))
        return sizes
    raise ValueError(kind)
