"""The edge sweep of oracle/lie_edges.py through the SO3 / RxSO3 / SE3 / Sim3 operators executed on the HOST
(lie_ops.cuh and lie_scaled.cuh are __host__ __device__), against the cancellation-free fp64 reference
oracle/lie_series.py.  Needs nvcc, no GPU: the small-angle numerics can be developed and checked on any machine."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import lie_edges as LE
from oracle import lie_series as LS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("lie") / "lie_host_check")
    subprocess.run([NVCC, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "dpvo_b200", "csrc"),
                    "-o", out, os.path.join(ROOT, "tools", "lie_host_check.cu")], check=True, capture_output=True)
    return out


def run_on_host(exe, tmp_path, gid, op, ins, widths, dtype):
    """outputs of operator `op` on the host, as [n, w] tensors of `dtype`"""
    n = ins[0].shape[0]
    np_t = np.float64 if dtype == torch.float64 else np.float32
    ins3 = ins + [torch.zeros(n, 1, dtype=dtype)] * (3 - len(ins))
    wo = widths + [1] * (2 - len(widths))
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        for t in ins3:
            f.write(t.numpy().astype(np_t).tobytes())
    subprocess.run([exe, str(gid), str(LS.OPS.index(op)), str(n)] + [str(t.shape[1]) for t in ins3] + [str(w) for w in wo]
                   + ["f64" if dtype == torch.float64 else "f32", fin, fout], check=True)
    raw = np.fromfile(fout, dtype=np_t)
    outs, off = [], 0
    for w in widths:
        outs.append(torch.from_numpy(raw[off:off + n * w].copy()).reshape(n, w))
        off += n * w
    return outs


@pytest.mark.parametrize("gid", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("op", LS.OPS)
def test_edge_sweep_on_host(exe, tmp_path, gid, dtype, op):
    ins = LE.inputs(gid, op, dtype)
    ref = LE.reference(gid, op, ins)
    got = run_on_host(exe, tmp_path, gid, op, ins, [r.shape[1] for r in ref], dtype)
    LE.check(gid, op, dtype, ins, got, ref)
