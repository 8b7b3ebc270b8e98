"""ORACLE fixture (test infrastructure): run the reference's own loop-candidate scoring and selection once on the CPU
and store it in tests/golden/loop_ref.pt, so that tests/test_loop_cpu.py holds oracle/loop.py to the reference without
a checkout of it.

    python oracle/make_golden_loop.py      (needs the reference tree, see oracle/refimport.py)

For each case (dpvo_b200.synthetic.make_loop_state, fast config) it stores the poses, the patch centres and the
intrinsics, and what the reference's own functions compute from them: the per-patch flow magnitudes and validity of
dpvo/projective_ops.py:flow_mag (beta = 0.5), for the candidate pairs of oracle.loop.loop_range, reduced here to one mean
per pair (more than 0.75 M valid patches, else +inf); and the (i, j) pairs the reference's numba reduce_edges
(dpvo/loop_closure/optim_utils.py) accepts among the pairs below the threshold.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402
from dpvo_b200 import synthetic  # noqa: E402
from oracle import loop as OL  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "loop_ref.pt")
LOOP = dict(removal=16, max_age=1000, freq=15, kf_index=4, thresh=64.0)
CASES = {
    "lap20_n60": dict(n_frames=60, period=20, radius=2.0, seed=11),
    "lap24_n90": dict(n_frames=90, period=24, radius=1.5, seed=12),
}


def reference_scores_and_pairs(poses, centres, intr, n, M):
    """(scores in candidate order [J * ni], accepted pairs [P, 2]) from the reference's flow_mag and reduce_edges"""
    from dpvo import projective_ops as pops
    from dpvo.lietorch import SE3
    from dpvo.loop_closure.optim_utils import reduce_edges
    i0, ni, j0, J = OL.loop_range(n, LOOP["removal"], LOOP["max_age"], LOOP["freq"], LOOP["kf_index"])
    pair_j = torch.arange(j0, j0 + J).repeat_interleave(ni)          # j-major, i-minor: the candidate order
    pair_i = torch.arange(i0, i0 + ni).repeat(J)
    kk = (pair_i[:, None] * M + torch.arange(M)[None, :]).reshape(-1)
    ii, jj = pair_i.repeat_interleave(M), pair_j.repeat_interleave(M)
    flow, valid = pops.flow_mag(SE3(poses[None]), centres.view(1, -1, 3, 1, 1), intr[None], ii, jj, kk, beta=0.5)
    flow, valid = flow.view(-1, M).float(), valid.view(-1, M)
    count = valid.sum(1)
    total = (flow * valid).sum(1)
    scores = torch.where(count > 0.75 * M, total / count.clamp(min=1), torch.full_like(total, float("inf")))
    below = scores < LOOP["thresh"]
    pairs = reduce_edges(scores[below].numpy(), pair_i[below].numpy(), pair_j[below].numpy(), max_num_edges=1000, nms=1)
    return scores, torch.as_tensor(pairs).view(-1, 2)


def main():
    out = dict(loop=LOOP, cases={})
    with refimport.reference_modules():
        for name, c in CASES.items():
            st = synthetic.make_loop_state("fast", device="cpu", features=False, **c)
            M, n = st.cfg["M"], st.n
            centres = st.patches[:n * M, :, 1, 1].clone()
            scores, pairs = reference_scores_and_pairs(st.poses[:n].clone(), centres, st.intrinsics[:n].clone(), n, M)
            out["cases"][name] = dict(params=c, M=M, n=n, poses=st.poses[:n].clone(), centres=centres,
                                      intrinsics=st.intrinsics[:n].clone(), scores=scores, pairs=pairs)
            print(name, "candidates", scores.numel(), "below thresh", int((scores < LOOP["thresh"]).sum()), "pairs", len(pairs))
    torch.save(out, OUT)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
