"""ORACLE fixture (test infrastructure): run the reference's own keyframe motion test once on the CPU and store it in
tests/golden/keyframe_ref.pt, so that tests/test_keyframe_cpu.py holds oracle/keyframe.py to the reference without a
checkout of it.

    python oracle/make_golden_keyframe.py      (needs the reference tree, see oracle/refimport.py)

For each case it stores the poses, patches and intrinsics of the frames the test reads, the (i, j) and (j, i) edge sets
of DPVO.keyframe (i = n - KI - 1, j = n - KI + 1, from the steady-state edges of dpvo_b200.synthetic.replay_edges), and
what the reference computes from them: dpvo/projective_ops.py:flow_mag (beta = 0.5) of every pixel, motionmag's
flow.mean().item() of each set, m = the sum of the two and the decision m / 2 < KEYFRAME_THRESH (dpvo/dpvo.py:257-272).
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402
from dpvo_b200 import synthetic  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "keyframe_ref.pt")
KI, THRESH = 4, 15.0


def _states():
    """(name, poses, patches, intrinsics, M, lifetime, removal, n) of every case"""
    sg = synthetic.make_stop_go_state("fast", 30, total=30, device="cpu", features=False, seed=21)
    for n in (9, 12, 13, 20, 27):                   # stopped, stopped, moving, moving, stopped / moving boundary
        yield "stopgo_n%d" % n, sg.extras["trajectory"], sg.extras["patches"], sg.intrinsics[:30], sg.cfg, n
    for seed, cfgname in ((5, "fast"), (6, "default")):
        st = synthetic.make_state(cfgname, 24, device="cpu", features=False, seed=seed, buffer=26, noise=0.05)
        g = torch.Generator().manual_seed(seed)
        P = st.poses[:24].clone()
        P[:, :3] += 0.2 * torch.randn(24, 3, generator=g)              # random poses: rotations and translations
        q = torch.randn(24, 4, generator=g) * 0.05
        q[:, 3] += 1.0
        P[:, 3:] = q / q.norm(dim=1, keepdim=True)
        yield "random_%s" % cfgname, P, st.patches[:24 * st.cfg["M"]], st.intrinsics[:24], st.cfg, 24
    yield "empty_n4", sg.extras["trajectory"], sg.extras["patches"], sg.intrinsics[:30], sg.cfg, 4   # n < KI + 2: no edge


def main():
    out = dict(ki=KI, thresh=THRESH, cases={})
    with refimport.reference_modules():
        from dpvo import projective_ops as pops
        from dpvo.lietorch import SE3
        for name, poses, patches, intr, cfg, n in _states():
            M = cfg["M"]
            ii, jj, kk = synthetic.replay_edges(n, M, cfg["lifetime"], cfg["removal"])
            i, j = n - KI - 1, n - KI + 1
            case = dict(M=M, n=n, poses=poses[:n].clone(), patches=patches[:n * M].clone(), intrinsics=intr[:n].clone(), sets=[])
            means = []
            for a, b in ((i, j), (j, i)):
                sel = (ii == a) & (jj == b)
                e = (ii[sel], jj[sel], kk[sel])
                if sel.any():
                    flow, _ = pops.flow_mag(SE3(poses[None, :n]), patches[None, :n * M], intr[None, :n], *e, beta=0.5)
                else:                   # flow_mag of no edge is an empty tensor (the CPU lietorch cannot shape one)
                    flow = torch.zeros(1, 0, 3, 3)
                means.append(flow.mean().item())
                case["sets"].append(dict(ii=e[0], jj=e[1], kk=e[2], flow=flow[0].reshape(-1, 9).clone(), mean=means[-1]))
            m = means[0] + means[1]
            case["m"], case["removed"] = m, bool(m / 2 < THRESH)
            out["cases"][name] = case
            print(name, "edges", [s["ii"].numel() for s in case["sets"]], "m/2 %.4f" % (m / 2), "removed", case["removed"])
    torch.save(out, OUT)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
