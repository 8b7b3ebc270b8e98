"""dpvo_ba_batched_workspace_bytes returns the size its formula gives on the current device (its partial-system
region scales with the SM count)."""
import pytest
import torch

from test_workspace_sizes_cpu import BA_MAX_N, EDGES, a256, ba_scratch_bytes, lib

pytestmark = pytest.mark.gpu

BA_FAST_MAX_N = 12        # widest window whose partial systems the reduce kernel forms


def ba_batched_bytes(E, B, N, sm_count):
    """stream bounds, the scratch with B dX slots, B x sm_count packed partial systems (fast path), 256 B of alignment"""
    N6 = 6 * N
    part = sm_count * (N6 * (N6 + 1) // 2 + N6) if 0 < N <= BA_FAST_MAX_N else 0
    return a256(4 * 2 * (B + 1)) + ba_scratch_bytes(E, N, B) + a256(4 * B * part) + 256


@pytest.mark.parametrize("N", [0, 1, 12, 13, BA_MAX_N])
@pytest.mark.parametrize("B", [1, 2, 8, 64])
@pytest.mark.parametrize("E", EDGES)
def test_batched_bundle_adjustment_workspace(E, B, N):
    torch.cuda.set_device(0)
    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    assert lib().dpvo_ba_batched_workspace_bytes(E, B, N) == ba_batched_bytes(E, B, N, sm_count)
