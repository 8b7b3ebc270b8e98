"""The C-ABI library loads without a GPU and exports every symbol include/dpvo_b200.h declares."""
import ctypes
import os
import re

import dpvo_b200

HDR = os.path.join(dpvo_b200.INCLUDE_DIR, "dpvo_b200.h")


def _declared():
    src = open(HDR).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dpvo_[a-zA-Z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported():
    lib = dpvo_b200.library()
    names = _declared()
    assert len(names) >= 30
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, "declared in dpvo_b200.h but not exported: %s" % missing


def test_version_and_error_text():
    lib = dpvo_b200.library()
    assert b"sm_90a" in lib.dpvo_version()
    assert isinstance(lib.dpvo_last_error(), bytes)
    assert lib.dpvo_launch_count() >= 0


def test_argument_validation_needs_no_gpu():
    """bad arguments are rejected on the host before any CUDA call"""
    lib = dpvo_b200.library()
    rc = lib.dpvo_corr_forward(None, None, None, None, None, None, None, None, ctypes.c_int64(1),
                               1, 1, 4, 128, 3, 1, 1, 8, 8, 3, None)
    assert rc == 1 and b"null" in lib.dpvo_last_error()
    lib.dpvo_ba_workspace_bytes.restype = ctypes.c_int64
    lib.dpvo_ba_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int]
    assert lib.dpvo_ba_workspace_bytes(47712, 10) > 47712 * 60 * 4


def test_argument_validation_of_the_fused_entry_points():
    """the entry points added for the fused update path reject inconsistent arguments on the host"""
    lib = dpvo_b200.library()
    buf = (ctypes.c_char * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    i64, i32 = ctypes.c_int64, ctypes.c_int
    # gated heads: gate without res
    rc = lib.dpvo_update_heads(p, p, i64(384), None, i64(384), p, p, None, i32(3), p, p, i64(1), i32(384), None)
    assert rc == 1 and b"gate and res come together" in lib.dpvo_last_error()
    # heads: dim must be a multiple of 128
    rc = lib.dpvo_update_heads(p, None, i64(0), None, i64(0), p, p, None, i32(3), p, p, i64(1), i32(100), None)
    assert rc == 1 and b"multiple of 128" in lib.dpvo_last_error()
    # LayerNorm: a scale for operand c without operand c
    dts = (ctypes.c_int * 3)(1, 0, 0)
    rc = lib.dpvo_add_layernorm(p, None, None, dts, None, p, i64(384), p, p, ctypes.c_float(1e-3), p, None, i32(0), i64(1), i32(384), None)
    assert rc == 1 and b"c_scale" in lib.dpvo_last_error()
    # paired grouping: the two problems need separate workspaces
    rc = lib.dpvo_group_edges_pair(p, None, None, p, p, p, p, None, p, p, p, None, None, p, p, p, p, None, p, p, i64(4), i64(4096), None)
    assert rc == 1 and b"separate workspaces" in lib.dpvo_last_error()
    # dense layer: the fp16 copy accompanies an fp32 result only; the split epilogue is a known value
    rc = lib.dpvo_linear_f16(p, i64(64), None, p, i64(64), None, None, i32(1), i64(0), None, i64(0), p, i32(0), i64(64), p, i64(64),
                             i64(8), i32(64), i32(64), i32(0), None)
    assert rc == 1 and b"fp16 copy" in lib.dpvo_last_error()
    rc = lib.dpvo_linear_f16(p, i64(64), None, p, i64(64), None, None, i32(1), i64(0), None, i64(0), p, i32(0), i64(64), None, i64(0),
                             i64(8), i32(64), i32(64), i32(9), None)
    assert rc == 1 and b"unknown epilogue" in lib.dpvo_last_error()
    lib.dpvo_corr_pyramid2_workspace_bytes.restype = ctypes.c_int64
    assert lib.dpvo_corr_pyramid2_workspace_bytes(i64(47712)) >= (47712 + 1) * 4


def test_shims_import_and_refuse_cpu_tensors():
    import pytest
    import torch
    cc, cb, lb, ex = dpvo_b200.extensions()
    assert {"forward", "backward", "patchify_forward", "patchify_backward"} <= set(dir(cc))
    assert {"forward", "neighbors", "reproject", "solve_system"} <= set(dir(cb))
    assert {"expm", "expm_backward", "logm", "logm_backward", "inv", "inv_backward", "mul", "mul_backward", "adj",
            "adj_backward", "adjT", "adjT_backward", "act", "act_backward", "act4", "act4_backward", "as_matrix",
            "projector", "Jinv"} <= set(dir(lb))
    with pytest.raises(RuntimeError, match="no CPU path"):
        lb.expm(3, torch.zeros(2, 6))
    with pytest.raises(RuntimeError, match="no CPU path"):
        cb.neighbors(torch.zeros(3, dtype=torch.long), torch.zeros(3, dtype=torch.long))
