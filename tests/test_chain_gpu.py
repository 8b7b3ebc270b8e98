"""Fused layer chains of the update operator (csrc/chain.cu) against a float64 restatement of the same layers with the
same fp16 rounding points (operands of every dense layer are fp16, as under the reference's autocast, dpvo.py:332).
Reference arithmetic: dpvo/net.py:74-92, dpvo/blocks.py:15-29."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DIM = 384


def _ext():
    import dpvo_b200
    return dpvo_b200.extensions()[3]


def _ln(x, g, b):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-3) * g + b


def _h(x):      # the fp16 rounding point of a GEMM operand
    return x.half().double()


def _rand_w(n, k, gen):
    return (torch.randn(n, k, generator=gen, device="cuda") / k ** 0.5).half()


def _close(a, b, tol, what):
    err = (a.double() - b.double()).abs().max().item()
    ref = b.double().abs().max().item()
    assert err <= tol * max(ref, 1.0), "%s: max err %.3g (ref scale %.3g)" % (what, err, ref)


@pytest.mark.parametrize("E", [47712, 128, 77, 1000, 148 * 128 + 5, 132 * 64, 132 * 64 + 5])
def test_corr_norm_chain(E):
    ex = _ext()
    g = torch.Generator(device="cuda").manual_seed(E)
    corr = torch.zeros(E, 896, device="cuda", dtype=torch.half)
    corr[:, :882] = (torch.randn(E, 882, generator=g, device="cuda") * 2).half()
    W0 = torch.zeros(DIM, 896, device="cuda", dtype=torch.half)
    W0[:, :882] = _rand_w(DIM, 882, g)
    W2, W5 = _rand_w(DIM, DIM, g), _rand_w(DIM, DIM, g)
    p = torch.randn(7, DIM, generator=g, device="cuda") * 0.3
    p[2] += 1.0
    p[5] += 1.0
    net = torch.randn(E, DIM, generator=g, device="cuda")
    n_ctx = max(1, E // 20)
    inp = torch.randn(n_ctx, DIM, generator=g, device="cuda").half()
    idx = torch.randint(0, n_ctx, (E,), generator=g, device="cuda")
    pd = p.double()
    h = _h(torch.relu(corr.double() @ W0.double().T + pd[0]))
    h = _h(torch.relu(_ln(h @ W2.double().T + pd[1], pd[2], pd[3])))
    h = h @ W5.double().T + pd[4]
    ref = _ln(net.double() + inp[idx].double() + h, pd[5], pd[6])
    net32 = net.clone()
    n16 = ex.update_corr_norm(corr, W0, torch.cat([W2, W5], 0).contiguous(), p.reshape(-1).contiguous(), net32, inp, idx)
    torch.cuda.synchronize()
    _close(net32, ref, 2e-3, "state")
    _close(n16.reshape(E, DIM), ref, 3e-3, "fp16 copy")
    assert torch.equal(n16.reshape(E, DIM), net32.half()), "the fp16 copy is the rounded fp32 state"


@pytest.mark.parametrize("E", [47712, 128, 77, 1000, 148 * 128 + 5, 132 * 64, 132 * 64 + 5])
def test_neighbor_mlp_chain(E):
    ex = _ext()
    g = torch.Generator(device="cuda").manual_seed(E + 1)
    x16 = torch.randn(E, DIM, generator=g, device="cuda").half()
    idx = torch.randint(-1, E, (E,), generator=g, device="cuda")
    idx[::7] = -1
    Wa, Wb = _rand_w(DIM, DIM, g), _rand_w(DIM, DIM, g)
    p = torch.randn(2, DIM, generator=g, device="cuda") * 0.3
    net = torch.randn(E, DIM, generator=g, device="cuda")
    gathered = torch.where((idx >= 0)[:, None], x16[idx.clamp(min=0)].double(), torch.zeros((), dtype=torch.double, device="cuda"))
    h = _h(torch.relu(gathered @ Wa.double().T + p[0].double()))
    ref = net.double() + h @ Wb.double().T + p[1].double()
    net32 = net.clone()
    n16 = ex.update_neighbor_mlp(x16, idx, torch.cat([Wa, Wb], 0).contiguous(), p.reshape(-1).contiguous(), net32)
    torch.cuda.synchronize()
    _close(net32, ref, 2e-3, "state")
    assert torch.equal(n16.reshape(E, DIM), net32.half())


@pytest.mark.parametrize("E", [47712, 128, 77, 1000, 148 * 128 + 5, 132 * 64, 132 * 64 + 5])
@pytest.mark.parametrize("with_groups", [True, False])
def test_gru_heads_chain(E, with_groups):
    ex = _ext()
    g = torch.Generator(device="cuda").manual_seed(E + 2)
    W = [_rand_w(DIM, DIM, g) for _ in range(6)]
    vec = torch.randn(10, DIM, generator=g, device="cuda") * 0.3
    vec[0] += 1.0
    vec[5] += 1.0
    W4 = torch.randn(4, DIM, generator=g, device="cuda") / DIM ** 0.5
    b4 = torch.randn(4, generator=g, device="cuda") * 0.1
    params = torch.cat([vec.reshape(-1), W4.reshape(-1), b4]).contiguous()
    net = torch.randn(E, DIM, generator=g, device="cuda")
    G = max(1, E // 90)
    hij = torch.randn(G, DIM, generator=g, device="cuda").half()
    gof = torch.randint(0, G, (E,), generator=g, device="cuda", dtype=torch.int32)
    coords = torch.randn(E, 2, 3, 3, generator=g, device="cuda") * 50
    v = vec.double()
    G2 = max(1, E // 22)
    hkk = torch.randn(G2, DIM, generator=g, device="cuda").half()
    gkk = torch.randint(0, G2, (E,), generator=g, device="cuda", dtype=torch.int32)
    x = net.double() + ((hkk[gkk.long()].double() + hij[gof.long()].double()) if with_groups else 0)
    x = _ln(x, v[0], v[1])
    for blk in range(2):
        Wg, Wa, Wb = (w.double() for w in W[3 * blk:3 * blk + 3])
        bg, ba, bb = v[2 + 5 * blk], v[3 + 5 * blk], v[4 + 5 * blk]
        gate = _h(torch.sigmoid(_h(x) @ Wg.T + bg))
        r1 = _h(torch.relu(_h(x) @ Wa.T + ba))
        x = x + gate * (r1 @ Wb.T + bb)
        if blk == 0:
            x = _ln(x, v[5], v[6])
    hd = torch.relu(x) @ W4.double().T + b4.double()
    ref_delta = hd[:, :2] + coords[:, :, 1, 1].double()
    ref_weight = torch.sigmoid(hd[:, 2:])
    net32 = net.clone()
    delta, weight = ex.update_gru_heads(net32, hij if with_groups else None, gof if with_groups else None, torch.cat(W, 0).contiguous(),
                                        params, coords, None, hkk if with_groups else None, gkk if with_groups else None)
    torch.cuda.synchronize()
    _close(net32, x, 3e-3, "state")
    _close(delta.reshape(E, 2) - coords[:, :, 1, 1], ref_delta - coords[:, :, 1, 1].double(), 3e-3, "delta")
    _close(weight.reshape(E, 2), ref_weight, 3e-3, "weight")
