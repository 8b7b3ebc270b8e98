"""Times the three fused layer chains of the update operator (csrc/chain.cu) alone, CUDA events, E = 47,712, and prints
the weight bytes each launch streams: every 64-row tile reads every weight k-block (192 rows x 64 fp16 per column half),
and the CTAs of a cluster share each k-block, so L2 sends it once per group of CLUSTER tiles."""
import math, re, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import dpvo_b200

ex = dpvo_b200.extensions()[3]
E, DIM = int(os.environ.get("E", 47712)), 384
g = torch.Generator(device="cuda").manual_seed(0)
rw = lambda n, k: (torch.randn(n, k, generator=g, device="cuda") / k ** 0.5).half()
corr = torch.zeros(E, 896, device="cuda", dtype=torch.half); corr[:, :882] = torch.randn(E, 882, generator=g, device="cuda").half()
W0 = rw(DIM, 896); W25 = rw(2 * DIM, DIM); pA = torch.randn(7 * DIM, generator=g, device="cuda")
net = torch.randn(E, DIM, generator=g, device="cuda")
inp = torch.randn(3456, DIM, generator=g, device="cuda").half(); idx = torch.randint(0, 3456, (E,), generator=g, device="cuda")
n16 = torch.empty(1, E, DIM, device="cuda", dtype=torch.half); n16b = torch.empty_like(n16)
Wab = rw(2 * DIM, DIM); pC = torch.randn(2 * DIM, generator=g, device="cuda"); ix = torch.randint(-1, E, (E,), generator=g, device="cuda")
W6 = rw(6 * DIM, DIM); pG = torch.randn(14 * DIM + 4, generator=g, device="cuda")
hij = torch.randn(500, DIM, generator=g, device="cuda").half(); gof = torch.randint(0, 500, (E,), generator=g, device="cuda", dtype=torch.int32)
coords = torch.randn(E, 2, 3, 3, generator=g, device="cuda")
ws = torch.empty(ex.update_gru_workspace_bytes(), dtype=torch.uint8, device="cuda")
CLUSTER = int(re.search(r"constexpr int CH_CL = (\d+);", open(os.path.join(os.path.dirname(dpvo_b200.__file__), "csrc", "chain.cu")).read()).group(1))
KBLOCKS = {"corr_norm": 2 * (14 + 2 * 6), "neighbor_mlp": 2 * 2 * 6, "gru_heads": 2 * 6 * 6}     # per tile, both column halves
l2_bytes = {n: math.ceil(math.ceil(E / 64) / CLUSTER) * kb * 192 * 64 * 2 for n, kb in KBLOCKS.items()}
fl = {"corr_norm": 2.0 * E * (896 * 384 + 2 * 384 * 384), "neighbor_mlp": 2.0 * E * 2 * 384 * 384, "gru_heads": 2.0 * E * 6 * 384 * 384}
fn = {"corr_norm": lambda: ex.update_corr_norm(corr, W0, W25, pA, net, inp, idx, n16),
      "neighbor_mlp": lambda: ex.update_neighbor_mlp(n16, ix, Wab, pC, net, n16b),
      "gru_heads": lambda: ex.update_gru_heads(net, hij, gof, W6, pG, coords, ws)}
for name, f in fn.items():
    for _ in range(int(os.environ.get("WARM", 3))):
        f()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(int(os.environ.get("REPS", 20)))]
    for a, b in evs:
        a.record(); f(); b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in evs)
    med = t[len(t) // 2] * 1e-3
    print("%-13s median %.1f us  min %.1f us   %.0f TFLOP/s   weights %.3f GB into shared memory, %.3f GB from L2 (cluster %d), %.0f GB/s L2 -> SM (median)"
          % (name, med * 1e6, t[0] * 1e3, fl[name] / med / 1e12, l2_bytes[name] * CLUSTER / 1e9, l2_bytes[name] / 1e9, CLUSTER, l2_bytes[name] / med / 1e9))
