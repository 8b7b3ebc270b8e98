"""The fused layer chains (csrc/chain.cu) against the float64 restatement of oracle/chain.py, element by element within
its error bar: the fp32 state, the fp16 state copy (which must also be the rounded fp32 state, bit for bit), delta and
weight.

The restatement is built from the Update module's own submodules and the kernels are fed Update.pack()'s blocks, with
every parameter random (LayerNorm gamma away from 1, beta away from 0), so a packing mistake shows.  Edge counts cover
the cluster walk of the persistent grid: c = SMs / 2 clusters per wave, read at run time; an odd tile count leaves the
second CTA of the last cluster without a tile, and 64 * 2c +- 1 rows end a wave one tile early or late.  The value
regimes push the four LayerNorms to rows whose mean dominates their spread, to zero variance, the fp16 rounding points
close to the fp16 range, ReLUs dead, gates and weight logits saturated.  Outputs are views of larger sentinel-filled
buffers; nothing past row E may change."""
import pytest
import torch

from oracle import chain as OC
from dpvo_b200.net import Update, DIM

pytestmark = pytest.mark.gpu
DEV = "cuda"
PAD = 70                                          # sentinel rows past the end of every output
SENT32, SENT16 = -12345.0, -1234.0


def _ext():
    import dpvo_b200
    return dpvo_b200.extensions()[3]


def _c():
    return torch.cuda.get_device_properties(0).multi_processor_count // 2


# edge counts by name; c = SMs / 2, the clusters of one wave.  8448, 8453 and 18949 are the sizes of the former
# test_chain_gpu.py (132 * 64, 132 * 64 + 5, 148 * 128 + 5)
SIZES = {"64*2c-1": lambda c: 64 * 2 * c - 1, "64*2c": lambda c: 64 * 2 * c, "64*2c+1": lambda c: 64 * 2 * c + 1,
         "64*(2c+1)": lambda c: 64 * (2 * c + 1), "64*4c+5": lambda c: 64 * 4 * c + 5}
E_SPECS = ["1", "63", "64", "65", "127", "128", "129", "191", "77", "1000", *SIZES, "8448", "8453", "18949", "14496", "47712"]


def _E(spec):
    return SIZES[spec](_c()) if spec in SIZES else int(spec)


@pytest.fixture(scope="module")
def base():
    return OC.module(3, Update, DEV)


def _within(got, ref, bar, what):
    got = got.double().reshape(ref.shape)
    err = (got - ref).abs()
    bad = ~(err <= bar)
    if bad.any():
        i = int(bad.reshape(-1).nonzero()[0])
        ratio = (err / bar).reshape(-1)
        raise AssertionError("%s: %d of %d elements outside the bar (first at row %d col %d: got %.9g ref %.9g bar %.3g); worst err/bar %.3g"
                             % (what, int(bad.sum()), bad.numel(), i // ref.shape[-1], i % ref.shape[-1], got.reshape(-1)[i].item(),
                                ref.reshape(-1)[i].item(), bar.reshape(-1)[i].item(), ratio[torch.isfinite(ratio)].max().item()))


def _sentinel(E, cols, dtype, value):
    return torch.full((E + PAD, cols), value, dtype=dtype, device=DEV)


def _untouched(buf, E, value, what):
    assert torch.equal(buf[E:], torch.full_like(buf[E:], value)), "%s: rows past E = %d were written" % (what, E)


# ------------------------------------------------------------------------------------------------------- chain A
def _run_a(upd, corr, net, inp, idx):
    ex, P = _ext(), upd.pack()
    E = net.shape[0]
    n32, n16 = _sentinel(E, DIM, torch.float32, SENT32), _sentinel(E, DIM, torch.half, SENT16)
    n32[:E] = net
    ex.update_corr_norm(corr, P["A_W0"], P["A_W25"], P["A_p"], n32[:E], inp, idx, n16[:E])
    torch.cuda.synchronize()
    _untouched(n32, E, SENT32, "net32")
    _untouched(n16, E, SENT16, "net16")
    return n32[:E], n16[:E]


def _check_a(upd, corr, net, inp, idx):
    n32, n16 = _run_a(upd, corr, net, inp, idx)
    (ref, bar), = OC.outputs_capped("A", [OC.chain_a(OC.Params(upd, device=DEV), corr, net, inp, idx)])
    _within(n32, ref, bar, "chain A state")
    assert torch.equal(n16, n32.half()), "chain A: the fp16 copy is not the rounded fp32 state"
    _within(n16, ref, bar + OC.ulp16(ref.abs() + bar), "chain A fp16 state")
    return n32, n16


@pytest.mark.parametrize("E", E_SPECS)
def test_corr_norm_layouts(base, E):
    _check_a(*OC.case_a(base, _E(E), DEV))


A_REGIMES = ["offset30/0.1", "offset100/1", "offset300/1", "innerbias300", "innerbias1000", "constant", "large", "deadrelu"]


@pytest.mark.parametrize("E", ["1000", "64*2c+1"])
@pytest.mark.parametrize("regime", A_REGIMES)
def test_corr_norm_regimes(base, regime, E):
    _check_a(*OC.case_a(base, _E(E), DEV, regime))


@pytest.mark.parametrize("regime", ["nominal", "offset100/1"])
def test_corr_norm_regimes_large_E(base, regime):
    _check_a(*OC.case_a(base, 47712, DEV, regime))


@pytest.mark.parametrize("E", ["77", "64*2c+1"])
def test_corr_norm_operands(base, E):
    """no context index (one inp row per edge); a correlation buffer of row stride 1024 whose pad columns 882..895
    hold finite garbage gives the bits of the zero-padded rows (the pad weights are zero)"""
    E = _E(E)
    _check_a(*OC.case_a(base, E, DEV, variant="none"))
    upd, corr, net, inp, idx = OC.case_a(base, E, DEV, variant="stride")
    got = _check_a(upd, corr, net, inp, idx)
    clean = corr.clone()
    clean[:, 882:] = 0
    want = _run_a(upd, clean, net, inp, idx)
    assert all(torch.equal(a, b) for a, b in zip(got, want)), "chain A: garbage in the pad columns changed the result"


def test_corr_norm_packing_matters(base):
    """the check can see a packing mistake: corr.3's and norm's gamma exchanged in A_p fail it"""
    upd, corr, net, inp, idx = OC.case_a(base, 1000, DEV)
    P = dict(upd.pack())
    p = P["A_p"].reshape(7, DIM).clone()
    p[[2, 5]] = p[[5, 2]]
    ex = _ext()
    n32 = net.clone()
    ex.update_corr_norm(corr, P["A_W0"], P["A_W25"], p.reshape(-1).contiguous(), n32, inp, idx)
    (ref, bar), = OC.outputs_capped("A", [OC.chain_a(OC.Params(upd, device=DEV), corr, net, inp, idx)])
    with pytest.raises(AssertionError):
        _within(n32, ref, bar, "chain A with swapped gammas")


# ------------------------------------------------------------------------------------------------------- chain C
def _check_c(upd, which, x16, idx, net):
    ex, P = _ext(), upd.pack()
    E = net.shape[0]
    n32, n16 = _sentinel(E, DIM, torch.float32, SENT32), _sentinel(E, DIM, torch.half, SENT16)
    n32[:E] = net
    key = which.upper()
    ex.update_neighbor_mlp(x16, idx, P[key + "_W"], P[key + "_p"], n32[:E], n16[:E])
    torch.cuda.synchronize()
    _untouched(n32, E, SENT32, "net32")
    _untouched(n16, E, SENT16, "net16")
    (ref, bar), = OC.outputs_capped("C", [OC.chain_c(OC.Params(upd, device=DEV), which, x16, idx, net)])
    _within(n32[:E], ref, bar, "chain C state")
    assert torch.equal(n16[:E], n32[:E].half()), "chain C: the fp16 copy is not the rounded fp32 state"
    _within(n16[:E], ref, bar + OC.ulp16(ref.abs() + bar), "chain C fp16 state")


@pytest.mark.parametrize("E", E_SPECS)
def test_neighbor_mlp_layouts(base, E):
    _check_c(*OC.case_c(base, _E(E), DEV))


@pytest.mark.parametrize("which", ["c1", "c2"])
@pytest.mark.parametrize("regime", ["offset100/1", "large", "deadrelu"])
def test_neighbor_mlp_regimes(base, regime, which):
    _check_c(*OC.case_c(base, _E("64*2c+1"), DEV, regime, which=which))


@pytest.mark.parametrize("variant", ["all_masked", "none_masked", "self", "row0", "rowlast"])
def test_neighbor_mlp_indices(base, variant):
    _check_c(*OC.case_c(base, _E("64*2c+1"), DEV, variant=variant))


# ------------------------------------------------------------------------------------------------------- chain G
def _run_g(upd, net, hij, gof, hkk, gkk, cd, ws=None):
    ex, P = _ext(), upd.pack()
    E = net.shape[0]
    n32, dl, wt = _sentinel(E, DIM, torch.float32, SENT32), _sentinel(E, 2, torch.float32, SENT32), _sentinel(E, 2, torch.float32, SENT32)
    n32[:E] = net
    ex.update_gru_heads(n32[:E], hij, gof, P["G_W6"], P["G_p"], cd, ws, hkk, gkk, dl[:E], wt[:E])
    torch.cuda.synchronize()
    for buf, nm in ((n32, "net32"), (dl, "delta"), (wt, "weight")):
        _untouched(buf, E, SENT32, nm)
    return n32[:E], dl[:E], wt[:E]


def _check_g(upd, net, hij, gof, hkk, gkk, cd):
    n32, dl, wt = _run_g(upd, net, hij, gof, hkk, gkk, cd)
    (ref, bar), (rd, bd), (rw, bw) = OC.outputs_capped("G", OC.chain_g(OC.Params(upd, device=DEV), net, hij, gof, hkk, gkk, cd), cd)
    _within(n32, ref, bar, "chain G state")
    _within(dl, rd, bd, "chain G delta")
    _within(wt, rw, bw, "chain G weight")


@pytest.mark.parametrize("E", E_SPECS)
def test_gru_heads_layouts(base, E):
    _check_g(*OC.case_g(base, _E(E), DEV))


G_REGIMES = ["offset30/0.1", "offset100/1", "offset300/1", "innerbias300", "innerbias1000", "constant", "large", "deadrelu", "satgate", "satlogit"]


@pytest.mark.parametrize("E", ["1000", "64*2c+1"])
@pytest.mark.parametrize("regime", G_REGIMES)
def test_gru_heads_regimes(base, regime, E):
    _check_g(*OC.case_g(base, _E(E), DEV, regime))


@pytest.mark.parametrize("regime", ["nominal", "offset100/1"])
def test_gru_heads_regimes_large_E(base, regime):
    _check_g(*OC.case_g(base, 47712, DEV, regime))


@pytest.mark.parametrize("groups,gid,P,coords", [("none", "random", 3, True), ("hij", "random", 3, True), ("hkk", "random", 3, True),
                                                 ("both", "zero", 3, True), ("both", "max", 3, True), ("both", "random", 1, True),
                                                 ("both", "random", 3, False)])
@pytest.mark.parametrize("E", ["77", "64*2c+1"])
def test_gru_heads_operands(base, E, groups, gid, P, coords):
    _check_g(*OC.case_g(base, _E(E), DEV, groups=groups, gid=gid, P=P, coords=coords))


@pytest.mark.parametrize("E", ["1000", "47712"])
def test_gru_heads_workspace_contents_do_not_matter(base, E):
    """a NaN-filled workspace gives the bits of a zeroed one: every scratch value is written before it is read"""
    case = OC.case_g(base, _E(E), DEV)
    nbytes = _ext().update_gru_workspace_bytes()
    zero = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    nan = torch.full((nbytes // 4,), float("nan"), device=DEV).view(torch.uint8)
    a, b = _run_g(*case, ws=zero), _run_g(*case, ws=nan)
    assert all(torch.equal(x, y) for x, y in zip(a, b)), "chain G: the workspace's prior contents changed the result"
