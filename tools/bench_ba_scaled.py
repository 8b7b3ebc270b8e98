"""Bundle adjustment on a scaled synthetic graph (SURVEY 8(d): E >= 1e7 so that the per-edge traffic, not launch latency,
decides): a long synthetic video (8,100 frames x 96 patches x 13 observations = 10.1 M edges, 10 free poses at the
end, pairs of 96 edges as in the real graph).  Times ba_forward_grouped
(2 Gauss-Newton iterations: ba_reduce_kernel + ba_solve_kernel each) with CUDA events and reports the achieved
algorithmic bandwidth of the reduction -- SURVEY's 116 B/edge -- against the measured HBM peak.

    python tools/bench_ba_scaled.py [frames=8100]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import dpvo_b200
from dpvo_b200 import synthetic
from dpvo_b200.net import EdgeGroups

ex = dpvo_b200.extensions()[3]
dev = "cuda"
# a long video with the local structure of the real graph: NF frames, M patches per frame, every patch observed in the
# LIFE frames around its own (13 in default.yaml), so that an (i, j) pair holds M = 96 edges as in the real graph;
# only the last 10 poses are free, the rest of the trajectory is fixed (their edges still cost the same traffic)
M, LIFE = 96, 13
NF = int(sys.argv[1]) if len(sys.argv) > 1 else 8100
g = torch.Generator(device=dev).manual_seed(0)
n_patch = NF * M
k_all = torch.arange(n_patch, device=dev)
off = torch.arange(-(LIFE // 2), LIFE // 2 + 1, device=dev)
jj = (k_all // M)[:, None] + off[None, :]
keep = (jj >= 0) & (jj < NF)
kk = k_all[:, None].expand_as(jj)[keep]
jj = jj[keep]
ii = kk // M
E = kk.numel()
poses = torch.zeros(NF + 4, 7, device=dev); poses[:, 6] = 1
base = synthetic._trajectory(64, dev)
poses[:NF, :3] = base[torch.arange(NF, device=dev) % 64, :3] * 0.2
poses[:NF, 3:] = base[torch.arange(NF, device=dev) % 64, 3:]
h, w = 120, 160
patches = torch.zeros(n_patch, 3, 3, 3, device=dev)
offs = torch.tensor([-1.0, 0.0, 1.0], device=dev)
patches[:, 0] = (torch.rand(n_patch, generator=g, device=dev) * (w - 2) + 1)[:, None, None] + offs[None, None, :]
patches[:, 1] = (torch.rand(n_patch, generator=g, device=dev) * (h - 2) + 1)[:, None, None] + offs[None, :, None]
patches[:, 2] = (0.25 + 0.75 * torch.rand(n_patch, generator=g, device=dev))[:, None, None]
intr = torch.tensor([80.0, 80.0, 80.0, 60.0], device=dev).repeat(NF + 4, 1)
coords = ex.reproject_clamped(poses.view(1, -1, 7), patches.view(1, -1, 3, 3, 3), intr.view(1, -1, 4), ii, jj, kk)
target = coords[0, :, :, 1, 1].contiguous()[None] + 0.5 * torch.randn(1, E, 2, generator=g, device=dev)
weight = torch.rand(1, E, 2, generator=g, device=dev)
lmbda = torch.tensor([1e-4], device=dev)
gk, gp = EdgeGroups.pair((kk, None, jj), (ii, jj, None))
t0, t1, iters = NF - 10, NF, 2
p0, q0 = poses.clone(), patches.clone()


def run():
    poses.copy_(p0); patches.copy_(q0)
    ex.ba_forward_grouped(poses.view(1, -1, 7), patches.view(1, -1, 3, 3, 3), intr.view(1, -1, 4), target, weight, lmbda, ii, jj, kk, t0, t1, iters,
                          gk.order, gk.group_start, gk.key_a, gk.n, gp.order, gp.group_start, gp.key_a, gp.key_b, gp.n)


for _ in range(2):
    run()
torch.cuda.synchronize()
ts = []
for _ in range(5):
    poses.copy_(p0); patches.copy_(q0)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    ex.ba_forward_grouped(poses.view(1, -1, 7), patches.view(1, -1, 3, 3, 3), intr.view(1, -1, 4), target, weight, lmbda, ii, jj, kk, t0, t1, iters,
                          gk.order, gk.group_start, gk.key_a, gk.n, gp.order, gp.group_start, gp.key_a, gp.key_b, gp.n)
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))
ms = sorted(ts)[len(ts) // 2] / iters
peak = 3350.0                       # H100 SXM data-sheet HBM3 bandwidth (GB/s), not measured
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass
# per edge and Gauss-Newton iteration: each edge is linearised twice (once in its patch group, once in its pair group);
# 116 B (SURVEY 8(d)) is the once-per-edge figure: ii/jj/kk 24 B, target + weight 16 B, order entry 4 B, poses 2 x 28 B, patch 12 B + 4 B
alg = 116.0 * E
print(json.dumps({"what": "ba_forward_grouped on a scaled synthetic graph", "edges": E, "patches": n_patch, "free_poses": t1 - t0,
                  "ms_per_gauss_newton_iteration": ms, "algorithmic_bytes_per_iteration": alg, "algorithmic_GBps": alg / (ms * 1e-3) / 1e9,
                  "hbm_peak_GBps": peak, "frac_of_hbm_peak": alg / (ms * 1e-3) / 1e9 / peak,
                  "note": "every edge is linearised by two warps (patch item and pair item), so the kernel's own traffic is about twice the algorithmic figure"}))
