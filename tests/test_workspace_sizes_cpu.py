"""Every *_workspace_bytes of the C ABI that needs no device returns the size its formula gives.

Callers allocate workspaces from these functions, so a size must never shrink under the kernels that write the
workspace.  The formulas below restate each workspace region by region; the batched bundle adjustment's size depends
on the SM count and is checked in test_workspace_sizes_gpu.py."""
import ctypes

import pytest

import dpvo_b200

EDGES = [0, 1, 63, 64, 255, 256, 47712, 1 << 20]
FREE_POSES = [0, 1, 10, 12, 13, 32]

BA_REC = 90               # floats per pair record of the bundle adjustment
BA_MAX_N = 32             # free poses held on chip
G_TILE, G_BINS = 1024, 1024
GROUP_HEADER = 56         # bytes of the grouping's header: barrier, pad and six 64-bit range maxima
CB_ITEM = 48              # edges per level-1 work item of the binned correlation


def a256(v):
    return (v + 255) // 256 * 256


def lib():
    L = dpvo_b200.library()
    i64, i32 = ctypes.c_int64, ctypes.c_int
    for name, args in [("dpvo_ba_workspace_bytes", [i64, i32]), ("dpvo_ba_grouped_workspace_bytes", [i64, i32]),
                       ("dpvo_ba_batched_workspace_bytes", [i64, i32, i32]), ("dpvo_group_workspace_bytes", [i64]),
                       ("dpvo_neighbors_workspace_bytes", [i64]), ("dpvo_corr_pyramid2_workspace_bytes", [i64])]:
        getattr(L, name).restype = i64
        getattr(L, name).argtypes = args
    return L


def group_bytes(E):
    ntiles = (E + G_TILE - 1) // G_TILE
    return a256(GROUP_HEADER) + 2 * a256(4 * E) + a256(4 * ntiles * G_BINS) + a256(4 * (ntiles + 1))


def ba_scratch_bytes(E, N, streams):
    """Ed rows of 6 max(N, 1) floats, Q_k, u_k, the pair records, one dX per stream"""
    return a256(4 * E * 6 * max(N, 1)) + 2 * a256(4 * E) + a256(4 * E * BA_REC) + a256(4 * streams * 6 * BA_MAX_N)


def ba_bytes(E, N):
    """the patch grouping and the pair grouping, the scratch, one grouping workspace each, and 256 B of alignment"""
    k = 2 * a256(4 * E) + a256(4 * (E + 1)) + a256(8 * E) + a256(4)
    p = 2 * a256(4 * E) + a256(4 * (E + 1)) + 2 * a256(8 * E) + a256(4)
    return k + p + ba_scratch_bytes(E, N, 1) + 2 * group_bytes(E) + 256


def ba_grouped_bytes(E, N):
    return ba_scratch_bytes(E, N, 1) + 512


def neighbors_bytes(E):
    return 2 * a256(4 * E) + a256(4 * (E + 1)) + a256(8 * E) + 256 + group_bytes(E)


def corr_pyramid2_bytes(M):
    """int32 words: header, list, order, key, rank, two counters per bin; then the int4 work items"""
    K = 2 * M + 4096
    items = K + (M + CB_ITEM - 1) // CB_ITEM
    return 4 * (4 + 4 * M + 2 * K) + 16 * items + 16


@pytest.mark.parametrize("N", FREE_POSES)
@pytest.mark.parametrize("E", EDGES)
def test_bundle_adjustment_workspaces(E, N):
    L = lib()
    assert L.dpvo_ba_workspace_bytes(E, N) == ba_bytes(E, N)
    assert L.dpvo_ba_grouped_workspace_bytes(E, N) == ba_grouped_bytes(E, N)


@pytest.mark.parametrize("E", EDGES)
def test_grouping_and_correlation_workspaces(E):
    L = lib()
    assert L.dpvo_group_workspace_bytes(E) == group_bytes(E)
    assert L.dpvo_neighbors_workspace_bytes(E) == neighbors_bytes(E)
    assert L.dpvo_corr_pyramid2_workspace_bytes(E) == corr_pyramid2_bytes(E)


def test_negative_sizes_count_as_zero_edges():
    L = lib()
    assert L.dpvo_ba_workspace_bytes(-5, 10) == ba_bytes(0, 10)
    assert L.dpvo_ba_grouped_workspace_bytes(-5, 10) == ba_grouped_bytes(0, 10)
    assert L.dpvo_group_workspace_bytes(-5) == group_bytes(0)
    assert L.dpvo_neighbors_workspace_bytes(-5) == neighbors_bytes(0)
