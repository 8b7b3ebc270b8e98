"""The error bar of oracle/chain.py is tight enough to matter.  On 128-row versions of the value regimes of
test_chain_ref_gpu.py it accepts a float32 emulation of each chain (the kernels' rounding points, fp32 GEMMs of the fp16
operands, the LayerNorm in the kernels' reduction order) with and without random one-ulp flips at every fp16 rounding
point, and it rejects each mistake a chain kernel could make wherever the mistake applies: the former one-pass
LayerNorm variance, LayerNorm eps 1e-5, gru.0 / gru.2 parameters exchanged, a bias shifted by one column in one column
half, the two column halves of a layer exchanged, a weight k-block taken from the wrong layer, the d / w head rows
exchanged, the centre pixel off by one, a masked neighbour read as row 0, hkk added twice.  Also pins the restatement
without its rounding points to oracle/update.py's Update in float64."""
import copy

import pytest
import torch

from oracle import chain as OC, update as OU

DEV = "cpu"
E = 128
DIM = OC.DIM
A_REGIMES = ["nominal", "offset30/0.1", "offset100/1", "offset300/1", "innerbias300", "innerbias1000", "constant", "large", "deadrelu"]
C_REGIMES = ["nominal", "offset100/1", "large", "deadrelu"]
G_REGIMES = ["nominal", "offset30/0.1", "offset100/1", "offset300/1", "innerbias300", "innerbias1000", "constant", "large", "deadrelu", "satgate", "satlogit"]
CASES = [("A", r) for r in A_REGIMES] + [("C", r) for r in C_REGIMES] + [("G", r) for r in G_REGIMES]
_BASE = []


def _base():
    if not _BASE:
        _BASE.append(OC.module(3, OU.Update, DEV))
    return _BASE[0]


def _case(chain, regime):
    return {"A": OC.case_a, "C": OC.case_c, "G": OC.case_g}[chain](_base(), E, DEV, regime)


def _outputs(chain, case, ar=None, params=None):
    """[(value, bar)] of the chain's outputs (state; G: also delta and weight); the reference's bars capped by the
    max-norm tolerance, as the GPU test holds the kernels"""
    upd = case[0]
    P = params or OC.Params(upd)
    if chain == "A":
        outs = [OC.chain_a(P, *case[1:], ar=ar)]
    elif chain == "C":
        outs = [OC.chain_c(P, *case[1:], ar=ar)]
    else:
        outs = list(OC.chain_g(P, *case[1:], ar=ar))
    return outs if ar is not None else OC.outputs_capped(chain, outs, case[6] if chain == "G" else None)


def _ratio(chain, case, got):
    """largest |got - ref| / bar over the outputs"""
    return max(((g.double() - r).abs() / b).max().item() for (g, _), (r, b) in zip(got, _outputs(chain, case)))


_USED = {}


@pytest.mark.parametrize("chain,regime", CASES)
def test_bar_accepts_the_kernel_arithmetic(chain, regime):
    case = _case(chain, regime)
    worst = _ratio(chain, case, _outputs(chain, case, OC.Arith(emulate=True)))
    for seed in range(2):
        worst = max(worst, _ratio(chain, case, _outputs(chain, case, OC.Arith(flip=torch.Generator().manual_seed(seed)))))
    _USED[(chain, regime)] = worst
    assert worst <= 1.0, "%s %s: %.3g of the bar" % (chain, regime, worst)


def test_bar_use_is_reported():
    """the largest fraction of the bar the emulation uses, per chain (the bar is a worst case over signs: the |W| e
    propagation through 384-wide layers makes random rounding errors use a small part of it)"""
    if len(_USED) < len(CASES):
        for chain, regime in CASES:
            if (chain, regime) not in _USED:
                test_bar_accepts_the_kernel_arithmetic(chain, regime)
    for chain in "ACG":
        k, v = max(((k, v) for k, v in _USED.items() if k[0] == chain), key=lambda kv: kv[1])
        print("chain %s: largest fraction of the bar used %.3g (%s)" % (chain, v, k[1]))
    assert max(_USED.values()) > 0.05


# ----------------------------------------------------------------------------------------------- mutations
def _swap_halves(lin):
    p = torch.cat([torch.arange(192, 384), torch.arange(192)])
    lin.weight.copy_(lin.weight[p])
    lin.bias.copy_(lin.bias[p])


def _shift_bias(b):
    b[:192] = torch.roll(b[:192].clone(), 1)


def _wrong_kblock(dst, src):
    dst.weight[:, 64:128] = src.weight[:, 64:128]


def _last_layers(upd, chain):
    """(the chain's output-side dense layer, another dense layer of the chain, the bias vector a shift shows in)"""
    if chain == "A":
        return upd.corr[5], upd.corr[2], upd.norm.bias
    if chain == "C":
        return upd.c1[2], upd.c1[0], upd.c1[2].bias
    return upd.gru[3].res[2], upd.gru[3].res[0], upd.gru[2].bias


def _mutated(chain, mutation, case):
    """the chain's outputs under the mutation, computed at the kernels' rounding points (None: does not apply)"""
    upd = copy.deepcopy(case[0])
    args = list(case)
    args[0] = upd
    ar = None
    with torch.no_grad():
        if mutation == "one_pass_variance":
            ar = OC.Arith(emulate=True, one_pass=True)
        elif mutation == "eps_1e-5":
            ar = OC.Arith(emulate=True, eps=1e-5)
        elif mutation == "gru_ln_params_swapped":
            if chain != "G":
                return None
            for nm in ("weight", "bias"):
                a, b = getattr(upd.gru[0], nm), getattr(upd.gru[2], nm)
                t = a.clone()
                a.copy_(b)
                b.copy_(t)
        elif mutation == "bias_shifted":
            _shift_bias(_last_layers(upd, chain)[2])
        elif mutation == "halves_swapped":
            _swap_halves(_last_layers(upd, chain)[0])
        elif mutation == "kblock_from_wrong_layer":
            out, other, _ = _last_layers(upd, chain)
            _wrong_kblock(out, other)
        elif mutation == "heads_swapped":
            if chain != "G":
                return None
            for nm in ("weight", "bias"):
                a, b = getattr(upd.d[1], nm), getattr(upd.w[1], nm)
                t = a.clone()
                a.copy_(b)
                b.copy_(t)
        elif mutation == "centre_off_by_one":
            if chain != "G" or args[6] is None:
                return None
            cd = args[6]
            pp = cd.shape[-1]
            args[6] = torch.roll(cd.reshape(-1, 2, pp * pp), -1, dims=2).reshape(cd.shape)
        elif mutation == "masked_read_as_row0":
            if chain != "C" or not (args[3] < 0).any():
                return None
            args[3] = args[3].clamp(min=0)
        elif mutation == "hkk_twice":
            if chain != "G" or args[4] is None:
                return None
            args[4] = (args[4].float() * 2).half()
        else:
            raise ValueError(mutation)
    if ar is not None and chain == "C":
        return None                                                  # no LayerNorm in chain C
    return _outputs(chain, args, ar=ar or OC.Arith(bars=False), params=OC.Params(upd))


MUTATIONS = ["one_pass_variance", "eps_1e-5", "gru_ln_params_swapped", "bias_shifted", "halves_swapped", "kblock_from_wrong_layer",
             "heads_swapped", "centre_off_by_one", "masked_read_as_row0", "hkk_twice"]
# where the LayerNorm arithmetic mutations apply: the one-pass variance cancels where a row's mean dominates its spread
# (at m / s = 100 its error exceeds the bar only in the worst of many rows, more than these 128 have); eps matters where
# the variance is not large against it
APPLIES = {"one_pass_variance": {"offset30/0.1", "offset300/1", "innerbias300", "innerbias1000"},
           "eps_1e-5": {"offset30/0.1", "constant"}}


ONLY = {"gru_ln_params_swapped": "G", "heads_swapped": "G", "centre_off_by_one": "G", "hkk_twice": "G",
        "masked_read_as_row0": "C", "one_pass_variance": "AG", "eps_1e-5": "AG"}


def _applies(chain, regime, mutation):
    if mutation in APPLIES and regime not in APPLIES[mutation]:
        return False
    return chain in ONLY.get(mutation, "ACG")


# no effect to see: corr.5's weight is zero in A's constant regime, and so is eps's on rows of one value (gru.0's output
# on them is beta whatever eps is), and G's has no hkk rows; a masked neighbour and row 0 are both zero rows in C's dead-ReLU regime; the second
# block's res.2 (the layer the column-half and k-block mutations change) is behind a closed gate in G's offset and
# inner-bias regimes (in the offset regimes both gates are closed), and its input is zero in G's dead-ReLU regime
NO_EFFECT = ({("A", "constant", "eps_1e-5"), ("A", "constant", "halves_swapped"), ("A", "constant", "kblock_from_wrong_layer"),
              ("C", "deadrelu", "masked_read_as_row0"), ("G", "constant", "eps_1e-5"), ("G", "constant", "hkk_twice"), ("G", "deadrelu", "kblock_from_wrong_layer")}
             | {("G", r, m) for r in ("offset30/0.1", "offset100/1", "offset300/1", "innerbias300", "innerbias1000")
                for m in ("halves_swapped", "kblock_from_wrong_layer")})
# Smaller than the bar, for reasons in the arithmetic, not in the bar's construction: in G's state-offset regimes gru.0's
# output reaches net only through gru.2, which removes its mean and most of its scale again, so a doubled hkk row (its
# rows are 1e-3 of the spread there) and, at a row mean of 30, gru.0's one-pass variance move net by less than the
# kernels' own fp32 LayerNorm arithmetic.  The one-pass variance is rejected for G at a row mean of 300 and in the
# inner-bias regimes, where gru.2 sees the offset; both LayerNorms of chain G run the same code
BELOW = {("G", "offset30/0.1", "one_pass_variance")} | {("G", r, "hkk_twice") for r in ("offset30/0.1", "offset100/1", "offset300/1")}
MCASES = [pytest.param(c, r, m, marks=[pytest.mark.xfail(strict=True, reason="the mutation moves the outputs by less than the bar here")]
                       if (c, r, m) in BELOW else [])
          for c, r in CASES for m in MUTATIONS if _applies(c, r, m) and (c, r, m) not in NO_EFFECT]


@pytest.mark.parametrize("chain,regime,mutation", MCASES)
def test_bar_rejects_mutations(chain, regime, mutation):
    case = _case(chain, regime)
    got = _mutated(chain, mutation, case)
    if got is None:
        pytest.skip("%s does not apply to chain %s" % (mutation, chain))
    ref = _outputs(chain, case)
    assert any(((g.double() - r).abs() > b).any() for (g, _), (r, b) in zip(got, ref)), \
        "%s %s: the bar accepts %s" % (chain, regime, mutation)


def test_every_mutation_is_rejected_somewhere():
    caught = {p.values[2] for p in MCASES if not p.marks and _mutated(p.values[0], p.values[2], _case(*p.values[:2])) is not None}
    assert caught == set(MUTATIONS)


# ----------------------------------------------------------------------------------------------- pin
def test_restatement_is_the_update_module():
    """without its rounding points the restatement is oracle/update.py's Update, submodule by submodule, in float64"""
    upd = copy.deepcopy(_base()).double()
    P = OC.Params(upd, rounding=False)
    ar = OC.Arith(rounding=False, bars=False)
    _, corr, net, inp, idx = OC.case_a(upd, E, DEV)
    got, _ = OC.chain_a(P, corr[:, :882], net, inp, idx, ar=ar)
    with torch.no_grad():
        want = upd.norm(net.double() + inp.double()[idx] + upd.corr(corr[:, :882].double()))
    assert (got - want).abs().max().item() <= 1e-12 * want.abs().max().item()
    _, _, x16, ix, net = OC.case_c(upd, E, DEV)
    for which in ("c1", "c2"):
        got, _ = OC.chain_c(P, which, x16, ix, net, ar=ar)
        with torch.no_grad():
            want = net.double() + getattr(upd, which)((ix >= 0).double()[:, None] * x16.double()[ix.clamp(min=0)])
        assert (got - want).abs().max().item() <= 1e-12 * want.abs().max().item()
    _, net, hij, gof, hkk, gkk, _ = OC.case_g(upd, E, DEV)
    (x, _), (d, _), (w, _) = OC.chain_g(P, net, hij, gof, hkk, gkk, None, ar=ar)
    with torch.no_grad():
        want = upd.gru(net.double() + hkk.double()[gkk.long()] + hij.double()[gof.long()])
        for got, ref in ((x, want), (d, upd.d(want)), (w, upd.w(want))):
            assert (got - ref).abs().max().item() <= 1e-12 * max(ref.abs().max().item(), 1.0)


def test_ln_emulation_is_layer_norm():
    """the float32 LayerNorm in the kernels' reduction order is nn.LayerNorm to fp32 accuracy (which at a row mean m and
    spread s is a few ulps of m / s: x - mean rounds at the scale of m), and the one-pass form is far worse there"""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(200, DIM, generator=g, dtype=torch.float64)
    gam, bet = torch.rand(DIM, generator=g, dtype=torch.float64) + 0.5, torch.randn(DIM, generator=g, dtype=torch.float64)
    for m, s in ((0, 1), (300, 1), (30, 0.1)):
        xs = (m + s * x).float().double()
        want = torch.nn.functional.layer_norm(xs, (DIM,), gam, bet, eps=OC.EPS)
        err = (OC.ln_emulated(xs, gam, bet) - want).abs().max().item()
        tol = 2e-6 * (1 + m / s)
        assert err < tol, (m, s, err)
        if m:
            assert (OC.ln_emulated(xs, gam, bet, one_pass=True) - want).abs().max().item() > 10 * tol


@pytest.mark.parametrize("chain,regime", CASES)
def test_bar_rejects_outputs_that_ignore_the_inputs(chain, regime):
    """a kernel that writes a zero state, or (G) weight 0.5 everywhere, or delta = the centre pixel without the d head,
    fails the bar"""
    case = _case(chain, regime)
    outs = _outputs(chain, case)
    (ref, bar) = outs[0]
    assert ((ref.abs() > bar)).any(), "%s %s: a zero state passes" % (chain, regime)
    if chain == "G":
        (d, bd), (w, bw) = outs[1], outs[2]
        assert ((w - 0.5).abs() > bw).any(), "%s: weight 0.5 passes" % regime
        assert ((d - OC.centre(case[6]).double()).abs() > bd).any(), "%s: delta = centre passes" % regime
