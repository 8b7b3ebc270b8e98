"""Loop-closure costs on one GPU (default configuration, M = 96, max_edge_age = 1000):
    proposal   LoopClosure.propose (scores + selection + emission, one proposal due) at n in {100, 500, 1200}, against
               the reference's PatchGraph.edges_loop on the same poses and patches (when oracle/_ref holds the staged
               reference package), median of REPS calls each
    update     one captured update over the normal slots and over the whole store (loop region full), against the
               same runner without loop closure
    global BA  LoopClosure.global_ba (normalize + 2 wide iterations, eager) against the inactive-store size, and the
               reference's own eff_impl kernels (oracle/_ref) on the same edges when they are built
CUDA events; the card's name, power limit and SM clocks are read before and after.

    python tools/bench_loop.py
"""
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

import dpvo_b200
from dpvo_b200 import synthetic
from dpvo_b200.loop import LoopClosure
from dpvo_b200.patchgraph import DevicePatchGraph
from dpvo_b200.runner import UpdateRunner

REPS, WARM = int(os.environ.get("REPS", 50)), int(os.environ.get("WARM", 5))


def smi():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def median_ms(f, reps=REPS, warm=WARM):
    for _ in range(warm):
        f()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        f()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def setup(st, loop_pairs=1000, inactive=1 << 20, capacity=None):
    g = DevicePatchGraph(capacity or st.E + 1024, st.cfg["M"], st.poses.shape[0] - 1, "cuda", loop_pairs=loop_pairs,
                         inactive_capacity=inactive)
    return g, LoopClosure(st.cfg, g)


def bench_proposal():
    from oracle import refimport
    for n in (100, 500, 1200):
        st = synthetic.make_loop_state("default", n, period=40, device="cuda", features=False)
        g, lc = setup(st)
        n_dev = torch.tensor([n], device="cuda")

        def ours():
            lc.last_global_ba.fill_(-1000)
            lc.propose(st.poses, st.patches, st.intrinsics, n_dev)
        t = median_ms(ours)
        k = int(lc.n_pairs.item())
        line = "proposal n=%5d: ours %.3f ms (%d pairs)" % (n, t, k)
        if refimport.staged():
            M = lc.M
            with refimport.reference_python():
                from dpvo.config import cfg as base
                from dpvo.patchgraph import PatchGraph
                cfg = base.clone()
                cfg.PATCHES_PER_FRAME, cfg.BUFFER_SIZE, cfg.REMOVAL_WINDOW = M, st.poses.shape[0], lc.removal
                pg = PatchGraph(cfg, 3, 384, lc.max_age, device="cuda", dtype=torch.half)
                pg.n = n
                pg.poses_[:] = st.poses
                pg.patches_[:] = st.patches.view(-1, M, 3, 3, 3)
                pg.intrinsics_[:] = st.intrinsics
                pg.index_[:] = torch.arange(pg.N, device="cuda")[:, None]
                tr = median_ms(pg.edges_loop, reps=max(5, REPS // 5), warm=2)
                kr = pg.edges_loop()[0].numel() // M
            line += "; reference edges_loop %.3f ms (%d pairs), %.1fx" % (tr, kr, tr / t)
        print(line, flush=True)


def bench_update():
    st = synthetic.make_loop_state("default", 36, period=12, radius=1.0, device="cuda")
    g, lc = setup(st, capacity=st.E + 2048)
    g.append(st.ii, st.jj, st.kk)
    st0 = synthetic.make_loop_state("default", 36, period=12, radius=1.0, device="cuda")
    g0 = DevicePatchGraph(st0.E + 2048, st0.cfg["M"], st0.poses.shape[0] - 1, "cuda")
    g0.append(st0.ii, st0.jj, st0.kk)
    r0 = UpdateRunner(st0, graph=g0)
    r0.capture()
    run = UpdateRunner(st, graph=g, loop=lc)
    run.capture()
    t_plain = median_ms(r0.graph.replay)
    t_norm = median_ms(run._loop_graphs[False][0].replay)
    lc.propose(st.poses, st.patches, st.intrinsics, torch.tensor([st.n], device="cuda"))
    npairs = int(lc.n_pairs.item())
    t_full = median_ms(run._loop_graphs[True][0].replay)
    print("update (graph): no loop closure %.3f ms; loop closure, normal slots %.3f ms; whole store (%d loop pairs, "
          "%d slots) %.3f ms" % (t_plain, t_norm, npairs, g.cap, t_full), flush=True)
    # eager steps (each reads the loop record; the first one runs the global bundle adjustment, in the warm-up)
    t_plain_e = median_ms(r0.step)
    t_loop_e = median_ms(run.step)
    used = run.loop.read_flags(st.n)[0]
    print("update (eager): no loop closure %.3f ms; loop closure with %d loop pairs active (normal slots + %d used "
          "loop-region slots) %.3f ms" % (t_plain_e, npairs, used, t_loop_e), flush=True)


def bench_global_ba(ref):
    n = 300
    st = synthetic.make_loop_state("default", n, period=40, device="cuda", features=False)
    M = st.cfg["M"]
    ex = dpvo_b200.extensions()[3]
    for count in (0, 100000, 400000, 1000000):
        g, lc = setup(st, loop_pairs=16, inactive=max(count, 1))
        g.append(st.ii, st.jj, st.kk)
        gen = torch.Generator(device="cuda").manual_seed(0)
        a = g.inactive_cap
        if count:
            i = torch.randint(0, n - 40, (count,), generator=gen, device="cuda")
            g.ii_all[a - count:a] = i
            g.jj_all[a - count:a] = (i + torch.randint(1, 12, (count,), generator=gen, device="cuda")).clamp(max=n - 1)
            g.kk_all[a - count:a] = i * M + torch.randint(0, M, (count,), generator=gen, device="cuda")
            lc.s_count.fill_(count)
        lo, hi = a - count, a + g.cap
        c = ex.reproject_clamped(st.poses.view(1, -1, 7), st.patches.view(1, -1, 3, 3, 3), st.intrinsics.view(1, -1, 4),
                                 g.ii_all[lo:hi], g.jj_all[lo:hi], g.kk_all[lo:hi])
        g.target_all[0, lo:hi] = c[0, :, :, 1, 1] + 0.5
        g.weight_all[0, lo:hi] = 1.0
        g.weight_all[0, a:] *= g.active.view(-1, 1)
        p0, q0 = st.poses.clone(), st.patches.clone()
        lm = torch.tensor([1e-4], device="cuda")

        def ours():
            st.poses.copy_(p0)
            st.patches.copy_(q0)
            lc.global_ba(st.poses, st.patches, st.intrinsics, n, 1, count, g.cap, lm)
        t = median_ms(ours, reps=max(5, REPS // 5), warm=2)
        line = "global BA n=%d, %7d inactive + %d active slots: ours %.2f ms" % (n, count, g.cap, t)
        if ref is not None:
            def theirs():
                st.poses.copy_(p0)
                st.patches.copy_(q0)
                ex.loop_normalize(st.poses, st.patches, n, M)
                ref[1].forward(st.poses.view(1, -1, 7), st.patches.view(1, -1, 3, 3, 3), st.intrinsics.view(1, -1, 4),
                               g.target_all[:, lo:hi], g.weight_all[:, lo:hi], lm, g.ii_all[lo:hi], g.jj_all[lo:hi],
                               g.kk_all[lo:hi], M, 1, n, 2, True)
            tr = median_ms(theirs, reps=max(5, REPS // 5), warm=2)
            line += "; reference eff_impl kernels %.2f ms" % tr
        print(line, flush=True)


def ref_kernels():
    d = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(d):
        return None
    sys.path.insert(0, d)
    try:
        import ref_cuda_ba
        import ref_cuda_corr
        return ref_cuda_corr, ref_cuda_ba
    except ImportError:
        return None


if __name__ == "__main__":
    print("GPU:", smi(), flush=True)
    bench_proposal()
    bench_update()
    bench_global_ba(ref_kernels())
    print("GPU:", smi(), flush=True)
