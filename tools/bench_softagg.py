"""Times the two SoftAgg aggregations of the update operator alone (net.py:_forward_chains), CUDA events, on the bench
state (synthetic.make_state("default", 36), E = 47,712) with both real groupings from EdgeGroups.pair and the group
bounds UpdateRunner uses.  Per aggregation it times, median of REPS launches each:
    fg       linear_f16 of the stacked f|g layer, E x 384 -> E x 768 fp16
    reduce   softagg_reduce over the [E,768] f|g rows
    h        linear_f16 of h on the group rows
    fused    softagg_fused (f|g layer + segment softmax on chip, with its combine launch), when the build has it
and prints the achieved TFLOP/s and the algorithmic HBM bytes of each (operands read once, results written once)."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import dpvo_b200
from dpvo_b200 import synthetic
from dpvo_b200.net import Update, EdgeGroups, DIM

ex = dpvo_b200.extensions()[3]
REPS, WARM = int(os.environ.get("REPS", 100)), int(os.environ.get("WARM", 5))
torch.manual_seed(0)
st = synthetic.make_state("default", 36, device="cuda", features=False)
E, M = st.E, st.cfg["M"]
max_kk = int((st.kk // M).unique().numel()) * M
max_ij = int(torch.unique(st.ii * 100000 + st.jj).numel())
gk, gp = EdgeGroups.pair((st.kk, None, st.jj), (st.ii, st.jj, None), max_kk, max_ij)
P = Update().cuda().eval().packed()
x = (torch.randn(1, E, DIM, device="cuda") / 2).half()
try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
except OSError:
    smi = torch.cuda.get_device_name()
print("device: %s   E = %d" % (smi, E))


def timeit(f):
    for _ in range(WARM):
        f()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(REPS)]
    for a, b in evs:
        a.record(); f(); b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in evs)
    return t[len(t) // 2] * 1e-3


for nm, grp, mg in (("kk", gk, max_kk), ("ij", gp, max_ij)):
    G = int(grp.n.item())
    fg = ex.linear_f16(x, P["fg_" + nm][0], P["fg_" + nm][1], 0)
    y = ex.softagg_reduce(fg, grp.order, grp.group_start, grp.n, mg)
    ops = {
        "fg": (lambda: ex.linear_f16(x, P["fg_" + nm][0], P["fg_" + nm][1], 0),
               2.0 * E * DIM * 2 * DIM, E * DIM * 2 + 2 * DIM * DIM * 2 + E * 2 * DIM * 2),
        "reduce": (lambda: ex.softagg_reduce(fg, grp.order, grp.group_start, grp.n, mg),
                   0.0, E * 2 * DIM * 2 + E * 4 + mg * DIM * 2),
        "h": (lambda: ex.linear_f16(y, P["h_" + nm][0], P["h_" + nm][1], 0),
              2.0 * mg * DIM * DIM, 2 * mg * DIM * 2 + DIM * DIM * 2),
    }
    if hasattr(ex, "softagg_fused"):
        ws = torch.empty(ex.softagg_fused_workspace_bytes(E), dtype=torch.uint8, device="cuda")
        ops["fused"] = (lambda: ex.softagg_fused(x, grp.order, grp.group_of, grp.group_start, grp.n, mg,
                                                 P["fgi_" + nm][0], P["fgi_" + nm][1], ws),
                        2.0 * E * DIM * 2 * DIM, E * DIM * 2 + E * 8 + 2 * DIM * DIM * 2 + mg * DIM * 2)
    times = {}
    print("agg_%s: %d groups (bound %d), %.1f rows per group" % (nm, G, mg, E / G))
    for k, (f, flop, nbytes) in ops.items():
        t = times[k] = timeit(f)
        print("  %-7s %7.1f us  %6.1f TFLOP/s  %6.1f MB HBM (algorithmic)  %6.0f GB/s"
              % (k, t * 1e6, flop / t / 1e12, nbytes / 1e6, nbytes / t / 1e9))
    two = times["fg"] + times["reduce"]
    print("  fg + reduce %.1f us" % (two * 1e6) + ("   fused / (fg + reduce) = %.2f" % (times["fused"] / two) if "fused" in times else ""))
