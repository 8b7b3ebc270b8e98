"""RxSO3 / Sim3 operators of dpvo_b200/csrc/lie_scaled.cuh executed on the HOST (the functions are __host__ __device__)
against the oracle, which the reference's own lietorch tests pin (oracle/pin_lie.py).  Needs nvcc, no GPU."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import importlib.util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the oracle backend with the pybind-like API, loaded under a private name: it must not shadow the product's
# `lietorch_backends` extension module for the other tests of the session
_spec = importlib.util.spec_from_file_location("oracle_lietorch_backends", os.path.join(ROOT, "oracle", "shims", "lietorch_backends.py"))
LB = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(LB)

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
OPS = ["expm", "expm_backward", "logm", "logm_backward", "inv", "inv_backward", "mul", "mul_backward", "adj", "adj_backward",
       "adjT", "adjT_backward", "act", "act_backward", "act4", "act4_backward", "as_matrix", "projector", "Jinv"]


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("lie") / "lie_host_check")
    subprocess.run([NVCC, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "dpvo_b200", "csrc"),
                    "-o", out, os.path.join(ROOT, "tools", "lie_host_check.cu")], check=True, capture_output=True)
    return out


def _case(gid, op, n, g):
    """inputs in the order of the pybind signature (without the group id) and the oracle's outputs"""
    G = LB._G(gid)
    N, K = G.N, G.K
    X = G.exp(0.6 * torch.randn(n, K, generator=g, dtype=torch.float64))
    Y = G.exp(0.6 * torch.randn(n, K, generator=g, dtype=torch.float64))
    a = 0.5 * torch.randn(n, K, generator=g, dtype=torch.float64)
    p3 = torch.randn(n, 3, generator=g, dtype=torch.float64)
    p4 = torch.randn(n, 4, generator=g, dtype=torch.float64)
    gN, gK = torch.randn(n, N, generator=g, dtype=torch.float64), torch.randn(n, K, generator=g, dtype=torch.float64)
    g3, g4 = torch.randn(n, 3, generator=g, dtype=torch.float64), torch.randn(n, 4, generator=g, dtype=torch.float64)
    ins = {"expm": [a], "expm_backward": [gN, a], "logm": [X], "logm_backward": [gK, X], "inv": [X], "inv_backward": [gN, X],
           "mul": [X, Y], "mul_backward": [gN, X, Y], "adj": [X, a], "adj_backward": [gK, X, a], "adjT": [X, a],
           "adjT_backward": [gK, X, a], "act": [X, p3], "act_backward": [g3, X, p3], "act4": [X, p4], "act4_backward": [g4, X, p4],
           "as_matrix": [X], "projector": [X], "Jinv": [X, a]}[op]
    ref = getattr(LB, op)(gid, *ins)
    ref = list(ref) if isinstance(ref, (list, tuple)) else [ref]
    return ins, [r.reshape(n, -1) for r in ref]


@pytest.mark.parametrize("gid", [2, 4])
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_scaled_groups_on_host_match_the_oracle(exe, tmp_path, gid, dtype):
    g = torch.Generator().manual_seed(100 + gid)
    n = 64
    np_t = np.float64 if dtype == "f64" else np.float32
    for code, op in enumerate(OPS):
        ins, ref = _case(gid, op, n, g)
        ins3 = ins + [torch.zeros(n, 1, dtype=torch.float64)] * (3 - len(ins))
        wo = [r.shape[1] for r in ref] + [1] * (2 - len(ref))
        fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
        with open(fin, "wb") as f:
            for t in ins3:
                f.write(t.numpy().astype(np_t).tobytes())
        subprocess.run([exe, str(gid), str(code), str(n)] + [str(t.shape[1]) for t in ins3] + [str(w) for w in wo] + [dtype, fin, fout], check=True)
        raw = np.fromfile(fout, dtype=np_t)
        off = 0
        for r, w in zip(ref, wo):
            got = torch.from_numpy(raw[off:off + n * w].astype(np.float64)).reshape(n, w)
            off += n * w
            scale = max(1.0, r.abs().max().item())
            tol = 1e-12 if dtype == "f64" else 2e-5
            err = (got - r).abs().max().item()
            assert err <= tol * scale, (op, dtype, err)
