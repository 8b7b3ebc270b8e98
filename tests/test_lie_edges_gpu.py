"""The edge sweep of oracle/lie_edges.py through the lietorch_backends kernels (lie.cu) for all four groups in float and
double, against the cancellation-free fp64 reference oracle/lie_series.py: rotation angles and scales at 0, on both
sides of the 1e-6 switch, through the small-angle band and near pi; translations of 1e-3 to 1e3; elements with
denormalised and negated quaternions.  Each operator runs once on a single element and once as one launch of 300,000
elements, more than one grid-stride pass of either kernel (8 x 132 x 256 and 8 x 132 x 128 threads)."""
import pytest
import torch

from oracle import lie_edges as LE
from oracle import lie_series as LS

pytestmark = pytest.mark.gpu
DEV = "cuda"
BIG = 300_000


def _run(L, gid, op, ins):
    out = getattr(L, op)(gid, *[t.to(DEV) for t in ins])
    out = list(out) if isinstance(out, (list, tuple)) else [out]
    return [o.reshape(o.shape[0], -1) for o in out]


@pytest.mark.parametrize("gid", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("op", LS.OPS)
def test_edge_sweep_on_device(ext, gid, dtype, op):
    L = ext[2]
    ins = LE.inputs(gid, op, dtype)
    ref = LE.reference(gid, op, ins)
    n = ins[0].shape[0]
    # the whole sweep, tiled to one launch of BIG elements: every copy must match its reference row
    idx = torch.arange(BIG) % n
    big = [t[idx] for t in ins]
    got = _run(L, gid, op, big)
    assert all(o.shape[0] == BIG for o in got)
    LE.check(gid, op, dtype, big, [o.cpu() for o in got], [r[idx] for r in ref])
    # a single element
    i = n // 3
    one = [t[i:i + 1] for t in ins]
    LE.check(gid, op, dtype, one, [o.cpu() for o in _run(L, gid, op, one)], [r[i:i + 1] for r in ref])
