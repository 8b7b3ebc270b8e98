"""The fused layer chains (csrc/chain.cu) run their tiles in CTA clusters that share every weight k-block. Each chain is
row-local, so row i of a launch must not depend on how many rows the launch has, nor on which CTA of a cluster took its
tile, nor on whether the other tiles of its group exist: compared bit for bit, which also catches a CTA's share of a
weight k-block landing in the wrong place."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DIM = 384
E_FULL = 47712
# one row (a group whose other tiles are past the end), one tile, a tile and one row, three tiles (a group with one
# tile past the end when the cluster has two CTAs), more groups than clusters fit on the device
PREFIXES = [1, 64, 65, 3 * 64, 132 * 64 + 5]


def _ext():
    import dpvo_b200
    return dpvo_b200.extensions()[3]


def _rand_w(n, k, gen):
    return (torch.randn(n, k, generator=gen, device="cuda") / k ** 0.5).half()


def _corr_norm(E):
    """returns run(k): the chain on the first k rows, and its outputs"""
    ex, g = _ext(), torch.Generator(device="cuda").manual_seed(11)
    corr = torch.zeros(E, 896, device="cuda", dtype=torch.half)
    corr[:, :882] = (torch.randn(E, 882, generator=g, device="cuda") * 2).half()
    W0 = torch.zeros(DIM, 896, device="cuda", dtype=torch.half)
    W0[:, :882] = _rand_w(DIM, 882, g)
    W25 = _rand_w(2 * DIM, DIM, g)
    p = torch.randn(7, DIM, generator=g, device="cuda") * 0.3
    p[2] += 1.0
    p[5] += 1.0
    p = p.reshape(-1).contiguous()
    net = torch.randn(E, DIM, generator=g, device="cuda")
    inp = torch.randn(E // 20, DIM, generator=g, device="cuda").half()
    idx = torch.randint(0, E // 20, (E,), generator=g, device="cuda")

    def run(k):
        net32 = net[:k].clone()
        n16 = ex.update_corr_norm(corr[:k], W0, W25, p, net32, inp, idx[:k])
        return net32, n16.reshape(k, DIM)
    return run


def _neighbor_mlp(E):
    ex, g = _ext(), torch.Generator(device="cuda").manual_seed(12)
    x16 = torch.randn(E, DIM, generator=g, device="cuda").half()
    # row i gathers from a row <= i (or nothing), so the first k rows of the launch gather from the first k source rows
    idx = (torch.rand(E, generator=g, device="cuda") * (torch.arange(E, device="cuda") + 2)).long() - 1
    idx[::7] = -1
    Wab = _rand_w(2 * DIM, DIM, g)
    p = (torch.randn(2, DIM, generator=g, device="cuda") * 0.3).reshape(-1).contiguous()
    net = torch.randn(E, DIM, generator=g, device="cuda")

    def run(k):
        net32 = net[:k].clone()
        n16 = ex.update_neighbor_mlp(x16[:k], idx[:k], Wab, p, net32)
        return net32, n16.reshape(k, DIM)
    return run


def _gru_heads(E):
    ex, g = _ext(), torch.Generator(device="cuda").manual_seed(13)
    W6 = _rand_w(6 * DIM, DIM, g)
    vec = torch.randn(10, DIM, generator=g, device="cuda") * 0.3
    vec[0] += 1.0
    vec[5] += 1.0
    W4 = torch.randn(4, DIM, generator=g, device="cuda") / DIM ** 0.5
    b4 = torch.randn(4, generator=g, device="cuda") * 0.1
    params = torch.cat([vec.reshape(-1), W4.reshape(-1), b4]).contiguous()
    net = torch.randn(E, DIM, generator=g, device="cuda")
    hij = torch.randn(E // 90, DIM, generator=g, device="cuda").half()
    gof = torch.randint(0, E // 90, (E,), generator=g, device="cuda", dtype=torch.int32)
    hkk = torch.randn(E // 22, DIM, generator=g, device="cuda").half()
    gkk = torch.randint(0, E // 22, (E,), generator=g, device="cuda", dtype=torch.int32)
    coords = torch.randn(E, 2, 3, 3, generator=g, device="cuda") * 50

    def run(k):
        net32 = net[:k].clone()
        delta, weight = ex.update_gru_heads(net32, hij, gof[:k], W6, params, coords[:k], None, hkk, gkk[:k])
        return net32, delta.reshape(k, 2), weight.reshape(k, 2)
    return run


CHAINS = {"corr_norm": _corr_norm, "neighbor_mlp": _neighbor_mlp, "gru_heads": _gru_heads}


@pytest.mark.parametrize("chain", list(CHAINS))
def test_chain_rows_do_not_depend_on_the_launch_size(chain):
    run = CHAINS[chain](E_FULL)
    full = run(E_FULL)
    torch.cuda.synchronize()
    for k in PREFIXES:
        part = run(k)
        torch.cuda.synchronize()
        for i, (a, b) in enumerate(zip(part, full)):
            assert torch.equal(a, b[:k]), "%s: output %d of a %d-row launch differs from the first %d rows of the %d-row launch" % (chain, i, k, k, E_FULL)


@pytest.mark.parametrize("chain", list(CHAINS))
def test_chain_reruns_are_bit_identical(chain):
    run = CHAINS[chain](E_FULL)
    first = run(E_FULL)
    second = run(E_FULL)
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(first, second)):
        assert torch.equal(a, b), "%s: output %d differs between two launches on the same inputs" % (chain, i)
