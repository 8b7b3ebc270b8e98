import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def ext():
    """(cuda_corr, cuda_ba, lietorch_backends, dpvo_b200_ext) -- the real sm_90a build."""
    import dpvo_b200
    return dpvo_b200.extensions()


@pytest.fixture(scope="session")
def ref_ext():
    """The reference's own kernels compiled into oracle/_ref (None if not built)."""
    d = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(d):
        return None
    import torch  # noqa: F401
    if d not in sys.path:
        sys.path.insert(0, d)
    try:
        import ref_cuda_corr
        import ref_cuda_ba
    except ImportError:
        return None
    return ref_cuda_corr, ref_cuda_ba
