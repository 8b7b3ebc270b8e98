"""ORACLE fixtures (test infrastructure): run the reference's own Python code once on the CPU and store what the CPU
tests compare the oracle against, in tests/golden/reference_cpu.pt, so that those comparisons need no checkout of the
reference when they run.

    python oracle/make_golden_reference.py      (needs the reference tree, see oracle/refimport.py)

Stored, all float64:
  lie/<group>     the reference's lietorch classes (dpvo/lietorch/groups.py, group_ops.py, unmodified) with the oracle
                  as the native backend, as dpvo/lietorch/run_tests.py runs them: exp / log / inv / mul / adj / adjT /
                  act / matrix on seeded inputs, and the gradients of two scalar losses through exp, mul, log and act;
                  plus the list of run_tests.py checks that passed
  ba_transform    dpvo/projective_ops.py:transform (with Jacobians) and dpvo/ba.py:BA on tests/test_oracle_cpu.py's
                  _ba_problem(seed=5)
  update_live     dpvo/net.py:Update on small_graph(5, 4, 6, 9) with the weights of oracle.update.Update seeded 7
  train_ba/<so>   two dpvo/ba.py:BA iterations on tests/test_train_cpu.py's _problem(3): poses, patches and the
                  gradients of a seeded linear loss w.r.t. target, weight and patches (structure_only False / True)
"""
import importlib.util
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_cpu.pt")
LIE_GROUPS = ("SO3", "RxSO3", "SE3", "Sim3")


def _test_module(name):
    spec = importlib.util.spec_from_file_location("_golden_" + name, os.path.join(ROOT, "tests", name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def lie_inputs(K, seed):
    """seeded fp64 inputs of one group (CPU generator: identical on every host)"""
    g = torch.Generator().manual_seed(seed)
    a = 0.2 * torch.randn(2, 3, K, generator=g, dtype=torch.float64)
    b = 0.2 * torch.randn(2, 3, K, generator=g, dtype=torch.float64)
    p = torch.randn(2, 3, 3, generator=g, dtype=torch.float64)
    c = torch.randn(2, 3, K, generator=g, dtype=torch.float64)
    w = torch.randn(2, 3, 3, generator=g, dtype=torch.float64)
    return a, b, p, c, w


def lie_case(G, K, seed):
    a, b, p, c, w = lie_inputs(K, seed)
    X, Y = G.exp(a), G.exp(b)
    out = dict(exp=X.data, log=X.log(), inv=X.inv().data, mul=(X * Y).data, adj=X.adj(b), adjT=X.adjT(b),
               act=X.act(p), matrix=X.matrix())
    a1, b1 = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ((G.exp(a1) * G.exp(b1)).log() * c).sum().backward()
    a2, p2 = a.clone().requires_grad_(True), p.clone().requires_grad_(True)
    (G.exp(a2).act(p2) * w).sum().backward()
    out.update(grad_mullog_a=a1.grad, grad_mullog_b=b1.grad, grad_act_a=a2.grad, grad_act_p=p2.grad)
    return {k: v.detach().clone() for k, v in out.items()}


def make_lie():
    from oracle import pin_lie
    res = {"run_tests_passed": [list(x) for x in pin_lie.run(groups=LIE_GROUPS)]}
    saved = list(sys.path)
    sys.path[:0] = [os.path.join(ROOT, "oracle", "shims"), os.path.join(pin_lie.REF, "lietorch"), pin_lie.REF]
    for m in ("lietorch", "lietorch_backends"):
        sys.modules.pop(m, None)
    try:
        import lietorch as ref_lt
        for i, name in enumerate(LIE_GROUPS):
            G = getattr(ref_lt, name)
            res[name] = lie_case(G, G.manifold_dim, 100 + i)
    finally:
        sys.path[:] = saved
        for m in ("lietorch", "lietorch_backends"):
            sys.modules.pop(m, None)
    return res


def make_ba_transform():
    t = _test_module("test_oracle_cpu")
    poses, patches, intr, target, weight, ii, jj, kk, n = t._ba_problem(seed=5)
    with refimport.reference_modules():
        import dpvo.ba as RBA
        import dpvo.projective_ops as RP
        from dpvo.lietorch import SE3
        c, v, (Ji, Jj, Jz) = RP.transform(SE3(poses[None]), patches[None], intr[None], ii, jj, kk, jacobian=True)
        Gs, pt = RBA.BA(SE3(poses[None].clone()), patches[None].clone(), intr[None], target[None], weight[None], 1e-4,
                        ii, jj, kk, [-64, -64, 160 + 64, 120 + 64], ep=10.0, fixedp=1)
        return dict(coords=c.clone(), valid=v.clone(), Ji=Ji.clone(), Jj=Jj.clone(), Jz=Jz.clone(), poses=Gs.data.clone(), patches=pt.clone())


def make_update_live():
    from oracle import update as OU
    from oracle.make_golden_update import make_inputs, small_graph
    ii, jj, kk = small_graph(5, 4, 6, 9)
    net, inp, corr, _ = make_inputs(ii.numel(), 123)
    torch.manual_seed(7)
    mine = OU.Update(3).eval()
    with refimport.reference_modules():
        import dpvo.net as RN
        theirs = RN.Update(3).eval()
        theirs.load_state_dict(mine.state_dict())
        with torch.no_grad():
            rn, (rd, rw, _) = theirs(net, inp, corr, None, ii, jj, kk)
    return dict(net=rn.clone(), delta=rd.clone(), weight=rw.clone())


def make_train_ba():
    t = _test_module("test_train_cpu")
    out = {}
    with refimport.reference_modules():
        import dpvo.ba as RB
        from dpvo.lietorch import SE3 as RSE3
        for so in (False, True):
            out[str(so)] = dict(zip(t.BA_OUTPUTS, t.run_ba(RB.BA, RSE3, structure_only=so)))
    return out


def main():
    if not refimport.available():
        raise SystemExit("the reference tree is not present; see oracle/refimport.py")
    torch.set_num_threads(1)
    d = dict(lie=make_lie(), ba_transform=make_ba_transform(), update_live=make_update_live(), train_ba=make_train_ba(),
             source="princeton-vl/DPVO Python (dpvo/lietorch, dpvo/projective_ops.py, dpvo/ba.py, dpvo/net.py), unmodified, "
                    "fp64 / fp32 CPU, torch %s" % torch.__version__)
    torch.save(d, OUT)
    print("wrote %s: %.1f KB" % (OUT, os.path.getsize(OUT) / 1e3))


if __name__ == "__main__":
    main()
