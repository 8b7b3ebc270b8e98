"""ORACLE (test infrastructure): the edge sweep of the Lie group operators, shared by tests/test_lie_edges_host_cpu.py
(the operators run on the host) and tests/test_lie_edges_gpu.py (the same operators in the CUDA kernels).

Inputs probe the places where the closed forms of lietorch cancel or branch: rotation angles at 0, on both sides of
the 1e-6 Taylor switch, log-spaced through the band up to 0.3 rad, at O(1) and just short of pi, along random and
axis-aligned directions; scales sigma of both signs at the same magnitudes and +-2; translations of size 1e-3, 1 and
1e3.  Group elements are exp() of those tangents, plus the same element with its quaternion negated or multiplied by
1e-3 or 1e3 -- the operators normalise on load, so these must give the element's results.  The reference is
oracle/lie_series.py on the inputs as rounded to the tested dtype.
"""
import math

import torch

from oracle import lie_series as LS

D = torch.float64
SWITCH = 1e-6
THETAS = ([0.0, 1e-9, SWITCH * (1 - 2.0 ** -20), SWITCH, SWITCH * (1 + 2.0 ** -20)]
          + torch.logspace(math.log10(1e-6), math.log10(0.3), 24, dtype=D).tolist()
          + [0.5, 1.0, 2.0, 3.0, math.pi - 1e-3, math.pi - 1e-5])
SIGMAS = sorted({s * m for m in THETAS for s in (1.0, -1.0)} | {2.0, -2.0})
TRANSLATIONS = [1e-3, 1.0, 1e3]
NEAR_PI = math.pi - 2e-3          # rows whose angle exceeds this are checked through exp(log X) = X
# Bars relative to max(1, |reference|) of each output row, for every group and operator but the ones in OP_TOL.
TOL = {torch.float32: 2e-5, torch.float64: 1e-12}
# act4_backward's dp[3] = grad[:3] . t + grad[3] sums terms of size |grad| |t| (|t| up to 1e3 here) to an O(1) result:
# rounding the inputs' products costs ~ulp |grad| |t|, 3.8e-5 of max(1, |ref|) at worst in float, whatever the kernel.
OP_TOL = {("act4_backward", torch.float32): 1e-4}


def _directions(g, n_random):
    axes = torch.eye(3, dtype=D)
    rnd = torch.randn(n_random, 3, generator=g, dtype=D)
    return torch.cat([axes, rnd / rnd.norm(dim=-1, keepdim=True)])


def tangents(gid):
    """[n, K] tangents of the sweep"""
    g = torch.Generator().manual_seed(1000 + gid)
    th = torch.tensor(THETAS, dtype=D)
    if gid in (1, 3):                                   # every angle along 3 axes and 2 random directions
        dirs = _directions(g, 2)
        phi = (th[:, None, None] * dirs[None]).reshape(-1, 3)
        sig = None
    else:                                               # every angle x every scale, one axis and one random direction
        dirs = _directions(g, 1)
        n_t = len(THETAS)
        sel = torch.stack([dirs[torch.arange(n_t) % 3], dirs[torch.full((n_t,), 3)]], 1)     # [n_t, 2, 3]
        phi0 = (th[:, None, None] * sel).reshape(-1, 3)
        sg = torch.tensor(SIGMAS, dtype=D)
        phi = phi0.repeat_interleave(len(sg), 0)
        sig = sg.repeat(phi0.shape[0])[:, None]
    if gid in (3, 4):                                   # every rotation(-scale) with each translation size
        m = torch.tensor(TRANSLATIONS, dtype=D)
        u = torch.randn(phi.shape[0] * len(m), 3, generator=g, dtype=D)
        tau = u / u.norm(dim=-1, keepdim=True) * m.repeat(phi.shape[0])[:, None]
        phi = phi.repeat_interleave(len(m), 0)
        sig = sig.repeat_interleave(len(m), 0) if sig is not None else None
        parts = [tau, phi] + ([sig] if sig is not None else [])
    else:
        parts = [phi] + ([sig] if sig is not None else [])
    return torch.cat(parts, -1)


def _quat_slice(gid):
    return slice(0, 4) if gid in (1, 2) else slice(3, 7)


def elements(gid):
    """[4n, N]: exp of every sweep tangent, then the same elements with the quaternion negated, x1e-3 and x1e3"""
    X = LS.exp(gid, tangents(gid))
    out = [X]
    for f in (-1.0, 1e-3, 1e3):
        Y = X.clone()
        Y[:, _quat_slice(gid)] *= f
        out.append(Y)
    return torch.cat(out)


def inputs(gid, op, dtype):
    """inputs of lietorch_backends.<op>(gid, ...), rounded to `dtype`"""
    N, K = LS.DIMS[gid]
    g = torch.Generator().manual_seed(2000 + gid)
    if op in ("expm", "expm_backward"):
        a = tangents(gid)
        n = a.shape[0]
        ins = [a] if op == "expm" else [torch.randn(n, N, generator=g, dtype=D), a]
        return [t.to(dtype) for t in ins]
    X = elements(gid)
    n = X.shape[0]
    a = tangents(gid).repeat(4, 1).roll(7, 0)
    gN, gK = torch.randn(n, N, generator=g, dtype=D), torch.randn(n, K, generator=g, dtype=D)
    g3, g4 = torch.randn(n, 3, generator=g, dtype=D), torch.randn(n, 4, generator=g, dtype=D)
    p3, p4 = torch.randn(n, 3, generator=g, dtype=D), torch.randn(n, 4, generator=g, dtype=D)
    ins = {"logm": [X], "logm_backward": [gK, X], "inv": [X], "inv_backward": [gN, X], "mul": [X, X.roll(1, 0)],
           "mul_backward": [gN, X, X.roll(1, 0)], "adj": [X, a], "adj_backward": [gK, X, a], "adjT": [X, a],
           "adjT_backward": [gK, X, a], "act": [X, p3], "act_backward": [g3, X, p3], "act4": [X, p4],
           "act4_backward": [g4, X, p4], "as_matrix": [X], "projector": [X], "Jinv": [X, a]}[op]
    return [t.to(dtype) for t in ins]


def near_pi(gid, X):
    """rows of an element batch whose rotation angle exceeds NEAR_PI"""
    q = LS.split(gid, X)[1]
    return 2.0 * torch.atan2(q[:, :3].norm(dim=-1), q[:, 3].abs()) > NEAR_PI


def reference(gid, op, ins):
    """lie_series on the inputs as given (already rounded to the tested dtype)"""
    return LS.op(op, gid, *[t.to(D) for t in ins])


def row_errors(gid, op, ins, got, ref):
    """per-output [n] errors relative to max(1, |reference row|); logm rows near pi compare exp(log X) with X"""
    errs = []
    for k, (o, r) in enumerate(zip(got, ref)):
        o = o.to(D).reshape(r.shape)
        e = (o - r).abs().amax(-1) / r.abs().amax(-1).clamp_min(1.0)
        if op == "logm":
            X = ins[0].to(D)
            pi = near_pi(gid, X)
            if pi.any():
                Tr = LS.rep(gid, X[pi]).flatten(1)
                To = LS.rep(gid, LS.exp(gid, o[pi])).flatten(1)
                e[pi] = (To - Tr).abs().amax(-1) / Tr.abs().amax(-1).clamp_min(1.0)
        errs.append(e)
    return errs


def check(gid, op, dtype, ins, got, ref):
    """asserts the bar on the outputs `got` against `ref` = reference(gid, op, ins); returns the worst relative error"""
    assert len(got) == len(ref)
    worst, tol = 0.0, OP_TOL.get((op, dtype), TOL[dtype])
    for k, e in enumerate(row_errors(gid, op, ins, got, ref)):
        i = int(e.argmax())
        worst = max(worst, e[i].item())
        assert e[i].item() <= tol, "%s out%d row %d: rel err %.3g > %.1g, inputs %s" % (
            op, k, i, e[i].item(), tol, [t[i].tolist() for t in ins])
    return worst
