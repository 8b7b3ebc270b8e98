"""Pins oracle/lie_series.py, the cancellation-free fp64 reference of the Lie group operators: to oracle/lie.py on O(1)
inputs, where lietorch's closed forms are accurate, which fixes every layout, sign and ordering convention; and to
30-digit mpmath at points of the small-angle band, where the closed forms are not."""
import math

import mpmath
import pytest
import torch

from oracle import lie as OL
from oracle import lie_series as LS

D = torch.float64


def _o1_inputs(gid, op, n, g):
    """inputs of lietorch_backends.<op>(gid, ...) at O(1) angles and scales"""
    N, K = LS.DIMS[gid]
    G = OL.GROUPS[gid]
    X = G.exp(0.7 * torch.randn(n, K, generator=g, dtype=D))
    Y = G.exp(0.7 * torch.randn(n, K, generator=g, dtype=D))
    X[:, 3] *= -1 if gid == 1 else 1                      # a negated quaternion must give the same results
    a = 0.5 * torch.randn(n, K, generator=g, dtype=D)
    p3, p4 = torch.randn(n, 3, generator=g, dtype=D), torch.randn(n, 4, generator=g, dtype=D)
    gN, gK = torch.randn(n, N, generator=g, dtype=D), torch.randn(n, K, generator=g, dtype=D)
    g3, g4 = torch.randn(n, 3, generator=g, dtype=D), torch.randn(n, 4, generator=g, dtype=D)
    return {"expm": [a], "expm_backward": [gN, a], "logm": [X], "logm_backward": [gK, X], "inv": [X], "inv_backward": [gN, X],
            "mul": [X, Y], "mul_backward": [gN, X, Y], "adj": [X, a], "adj_backward": [gK, X, a], "adjT": [X, a],
            "adjT_backward": [gK, X, a], "act": [X, p3], "act_backward": [g3, X, p3], "act4": [X, p4],
            "act4_backward": [g4, X, p4], "as_matrix": [X], "projector": [X], "Jinv": [X, a]}[op]


def _oracle(gid, op, ins):
    G = OL.GROUPS[gid]
    fwd = {"expm": G.exp, "logm": G.log, "inv": G.inv, "mul": G.mul, "adj": G.adj, "adjT": G.adjT, "act": G.act,
           "act4": G.act4, "as_matrix": lambda X: G.matrix(X).reshape(-1, 16),
           "projector": lambda X: G.projector(X).reshape(X.shape[0], -1), "Jinv": lambda X, a: OL.jinv(gid, X, a)}
    if op in fwd:
        return [fwd[op](*ins)]
    out = getattr(OL, op)(gid, *ins)
    return list(out) if isinstance(out, tuple) else [out]


@pytest.mark.parametrize("gid", [1, 2, 3, 4])
@pytest.mark.parametrize("op", LS.OPS)
def test_series_reference_matches_the_oracle_at_order_one(gid, op):
    g = torch.Generator().manual_seed(7 + gid)
    ins = _o1_inputs(gid, op, 200, g)
    got, ref = LS.op(op, gid, *ins), _oracle(gid, op, ins)
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        assert a.shape == b.shape, (op, a.shape, b.shape)
        err = ((a - b).abs().amax(-1) / b.abs().amax(-1).clamp_min(1.0)).max().item()
        assert err <= 1e-12, (op, err)


# ---- 30-digit spot checks in the band where lietorch's closed forms cancel ------------------------------------------
mpmath.mp.dps = 30


def _mp_hat(p):
    return mpmath.matrix([[0, -p[2], p[1]], [p[2], 0, -p[0]], [-p[1], p[0], 0]])


def _mp_series_block(A):
    """sum_k A^k/(k+1)! of an mpmath matrix, by its (absolutely convergent) series"""
    n = A.rows
    S, P, k = mpmath.eye(n), mpmath.eye(n), 1
    while True:
        P = P * A / (k + 1)
        S += P
        k += 1
        if mpmath.mnorm(P, 1) < mpmath.mpf(10) ** -40:
            return S


def _mp_to_torch(M):
    return torch.tensor([[float(M[i, j]) for j in range(M.cols)] for i in range(M.rows)], dtype=D)


TAU = (0.3, -0.8, 0.5)


@pytest.mark.parametrize("theta", [3e-6, 1e-4, 3e-4, 3e-2, 0.3])
def test_se3_exp_and_left_jacobian_against_mpmath(theta):
    d = [mpmath.mpf(x) for x in (0.36, -0.48, 0.8)]                   # a unit direction
    phi = [theta * x for x in d]
    a = torch.tensor([TAU + tuple(float(x) for x in phi)], dtype=D)
    Phi = _mp_hat(phi)
    V = _mp_series_block(Phi)
    t_ref = torch.tensor([float(x) for x in V * mpmath.matrix(list(TAU))], dtype=D)
    assert (LS.exp(3, a)[0, :3] - t_ref).abs().max().item() <= 1e-15
    # the 6x6 left Jacobian [[J, Q], [0, J]] from the series of ad
    ad = mpmath.zeros(6, 6)
    Tau = _mp_hat([mpmath.mpf(x) for x in TAU])
    for i in range(3):
        for j in range(3):
            ad[i, j] = Phi[i, j]
            ad[3 + i, 3 + j] = Phi[i, j]
            ad[i, 3 + j] = Tau[i, j]
    J_ref = _mp_to_torch(_mp_series_block(ad))
    assert (LS.left_jacobian(3, a)[0] - J_ref).abs().max().item() <= 1e-15
    Ji_ref = _mp_to_torch(_mp_series_block(ad) ** -1)
    assert (LS.left_jacobian_inverse(3, a)[0] - Ji_ref).abs().max().item() <= 1e-15


@pytest.mark.parametrize("sigma,theta", [(1e-5, 1e-3), (1e-4, 0.0), (-1e-3, 3e-2), (2.0, 1e-6), (-2.0, 0.3)])
def test_sim3_exp_and_log_against_mpmath(sigma, theta):
    d = [mpmath.mpf(x) for x in (0.0, 0.6, -0.8)]
    phi = [theta * x for x in d]
    a = torch.tensor([TAU + tuple(float(x) for x in phi) + (sigma,)], dtype=D)
    W = _mp_series_block(_mp_hat(phi) + mpmath.mpf(sigma) * mpmath.eye(3))
    t_ref = torch.tensor([float(x) for x in W * mpmath.matrix(list(TAU))], dtype=D)
    X = LS.exp(4, a)
    assert (X[0, :3] - t_ref).abs().max().item() <= 1e-15 * max(1.0, t_ref.abs().max().item())
    assert abs(X[0, 7].item() - float(mpmath.exp(sigma))) <= 1e-15 * math.exp(abs(sigma))
    assert (LS.log(4, X)[0] - a[0]).abs().max().item() <= 1e-15
