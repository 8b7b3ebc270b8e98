"""The workspace sizes that scale with the SM count answer for the current device: under torch.cuda.device(i), for every
visible device i, they follow device i's multiprocessor count, not that of the first device a process asked."""
import pytest
import torch

import dpvo_b200
from test_workspace_sizes_gpu import BA_FAST_MAX_N, ba_batched_bytes

pytestmark = pytest.mark.gpu

CH_SCRATCH_PER_CTA = 64 * 384 * (2 + 4)    # per chain CTA: a 64-row tile of the fp16 gate and of the fp32 input, 384 wide


@pytest.mark.parametrize("E,B", [(1, 1), (47712, 1), (47712, 8)])
def test_sm_count_sizes_follow_the_current_device(E, B):
    ext = dpvo_b200.extensions()[3]
    for i in range(torch.cuda.device_count()):
        sms = torch.cuda.get_device_properties(i).multi_processor_count
        with torch.cuda.device(i):
            assert ext.update_gru_workspace_bytes() == sms * CH_SCRATCH_PER_CTA, "device %d" % i
            for n in range(BA_FAST_MAX_N + 1):
                assert ext.ba_batched_workspace_bytes(E, B, n) == ba_batched_bytes(E, B, n, sms), "device %d, N=%d" % (i, n)
