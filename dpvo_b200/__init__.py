"""dpvo_b200 -- H100-native (sm_90a) implementation of DPVO's per-frame update hot path.

Importing the package locates the in-tree build products and makes the three reference-named
torch extensions importable by their top-level names, exactly as the reference's Python files
expect (``import cuda_corr`` in dpvo/altcorr/correlation.py:2, ``import cuda_ba`` in
dpvo/fastba/ba.py:2, ``import lietorch_backends`` in dpvo/lietorch/group_ops.py:1).

There is no CPU or PyTorch fallback: if the CUDA library has not been built the import of any
operator module raises.  Build with ``python -m dpvo_b200.build`` (or ``__graft_entry__.build()``).
"""
import ctypes
import os
import sys

__version__ = "0.1.0"

_ROOT = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_ROOT, "lib", "libdpvo_b200.so")
EXT_DIR = os.path.join(_ROOT, "_ext")
INCLUDE_DIR = os.path.join(os.path.dirname(_ROOT), "include")

_lib = None


def library():
    """ctypes handle of libdpvo_b200.so (the C-ABI of include/dpvo_b200.h)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "dpvo_b200: %s is missing -- run `python -m dpvo_b200.build`; there is no CPU fallback" % LIB_PATH)
        _lib = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
        _lib.dpvo_version.restype = ctypes.c_char_p
        _lib.dpvo_last_error.restype = ctypes.c_char_p
        _lib.dpvo_launch_count.restype = ctypes.c_int64
    return _lib


def extensions():
    """Import and return (cuda_corr, cuda_ba, lietorch_backends, dpvo_b200_ext)."""
    import torch  # noqa: F401  (libtorch must be loaded before the shims)
    library()
    if EXT_DIR not in sys.path:
        sys.path.insert(0, EXT_DIR)
    try:
        import cuda_corr
        import cuda_ba
        import lietorch_backends
        import dpvo_b200_ext
    except ImportError as e:  # pragma: no cover
        raise ImportError("dpvo_b200: torch-extension shims are missing or stale (%s) -- run "
                          "`python -m dpvo_b200.build`; there is no CPU fallback" % e)
    for m in (cuda_corr, cuda_ba, lietorch_backends, dpvo_b200_ext):
        if not os.path.abspath(m.__file__).startswith(EXT_DIR):
            raise ImportError("dpvo_b200: module %s resolved to %s, not the in-tree build" % (m.__name__, m.__file__))
    return cuda_corr, cuda_ba, lietorch_backends, dpvo_b200_ext


def camera_extension():
    """Import and return dpvo_b200_camera, the torch shim of the camera-image preparation (csrc/undistort.cu).  It is a
    fifth module of the same shim object, under the same tensor contract; the four modules of extensions() keep the
    entry points that the per-argument contract table of tests/test_shim_args_gpu.py lists."""
    extensions()
    try:
        import dpvo_b200_camera
    except ImportError as e:  # pragma: no cover
        raise ImportError("dpvo_b200: the camera shim is missing or stale (%s) -- run `python -m dpvo_b200.build`" % e)
    if not os.path.abspath(dpvo_b200_camera.__file__).startswith(EXT_DIR):
        raise ImportError("dpvo_b200: module dpvo_b200_camera resolved to %s, not the in-tree build" % dpvo_b200_camera.__file__)
    return dpvo_b200_camera
