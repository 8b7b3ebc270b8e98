"""Keyframe-culling costs on one GPU:
    cull       Keyframes.cull alone (motion test, edge renumbering, KI - 1 shift steps) for a kept and a culled frame,
               default and fast configurations, B = 1, 4 and 8 streams: one batched call against B single-stream
               calls, and the B remove_frame launches of the batched call on their own.  The edge store and frame
               counters are restored between calls (outside the timed window), so every call sees the same state;
               median of REPS calls, each between CUDA events.
    keyframe   at B = 1, cull + the window removal against the reference's own DPVO.keyframe (which does both) on the
               same state, through the staged reference Python on this library's native modules (oracle/_ref; the
               row is skipped without it).
    tracking   a 200-frame loop on a stop-go stream (fast): new frame, add_frame, edge append, one update, cull, window
               removal and the read() record, against the same loop without culling; mean milliseconds per frame
               over the whole loop (host clock, ending in a synchronise).
The card's name, power limit and SM clocks are read in the same run.

    python tools/bench_keyframe.py
"""
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from dpvo_b200 import synthetic
from dpvo_b200.keyframe import Keyframes
from dpvo_b200.patchgraph import DevicePatchGraph
from dpvo_b200.runner import UpdateRunner
from dpvo_b200.streams import StreamBatch

REPS, WARM = int(os.environ.get("REPS", 200)), int(os.environ.get("WARM", 20))


def smi():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def median_ms(f, restore, reps=REPS, warm=WARM):
    for _ in range(warm):
        restore()
        f()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        restore()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        f()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def _state(config, n, seed, F, mem):
    # stop=60: frames up to 60 stand still (a culled frame); go=60 from the start of a period after it
    return synthetic.make_stop_go_state(config, n, total=F - 2, stop=60, go=60, buffer=F, mem=mem, device="cuda", seed=seed)


def bench_cull():
    F, mem = 128, 36
    for config in ("default", "fast"):
        for culled, n in ((True, 30), (False, 70)):
            for B in (1, 4, 8):
                states = [_state(config, n, 3 + b, F, mem) for b in range(B)]
                cfg, M = states[0].cfg, states[0].cfg["M"]
                singles = []
                for st in states:
                    g = DevicePatchGraph(2 * st.E + 4 * M * cfg["lifetime"], M, F - 1, "cuda")
                    g.append(st.ii, st.jj, st.kk)
                    singles.append(Keyframes(cfg, st, g))
                batch = StreamBatch(B, cfg, F, mem, device="cuda")
                for b, st in enumerate(states):
                    batch.load(b, st)
                store, graphs = DevicePatchGraph.stacked(B, 2 * states[0].E + 4 * M * cfg["lifetime"], M,
                                                         [b * F + F - 1 for b in range(B)], "cuda")
                for b, st in enumerate(states):
                    graphs[b].append(*batch.to_global(b, st.ii, st.jj, st.kk))
                kfb = Keyframes(cfg, batch, store)
                saved = [(t, t.clone()) for kf in singles + [kfb]
                         for t in (kf.pg.ii, kf.pg.jj, kf.pg.kk, kf.pg.active, kf.n_dev)]
                saved += [(g.n_active, g.n_active.clone()) for g in [kf.pg for kf in singles] + graphs]

                def restore():
                    for dst, src in saved:
                        dst.copy_(src)

                t_single = median_ms(lambda: [kf.cull() for kf in singles], restore)
                t_batch = median_ms(kfb.cull, restore)
                restore()
                kfb.cull()
                flags = kfb.flag.tolist()
                assert all(f == int(culled) for f in flags), (config, n, flags)

                def renumber():                  # the B remove_frame launches of a batched cull, on its flags and k
                    for b, gb in enumerate(graphs):
                        gb.remove_frame(kfb.k[b:b + 1], enable=kfb.flag[b:b + 1])
                t_ren = median_ms(renumber, restore)
                print("cull %-7s %-6s B=%d  batched %.1f us (of which %d remove_frame launches %.1f us)   "
                      "%d single-stream calls %.1f us" % (config, "culled" if culled else "kept", B, 1e3 * t_batch, B,
                                                          1e3 * t_ren, B, 1e3 * t_single), flush=True)
                if B == 1:
                    bench_reference(states[0], singles[0], restore, config, culled)


def bench_reference(st, kf, restore, config, culled):
    """cull + window removal against the reference's DPVO.keyframe (decision, shift and window removal) on the same
    state, through the staged reference Python on this library's native modules"""
    from oracle import keyframe as OK
    from oracle import refimport
    g = kf.pg
    removal = st.cfg["removal"]
    poses0, patches0, tstamp0 = st.poses.clone(), st.patches.clone(), kf.tstamp.clone()

    def restore_all():
        restore()
        st.poses.copy_(poses0)
        st.patches.copy_(patches0)
        kf.tstamp.copy_(tstamp0)

    def ours():
        kf.cull()
        g.remove_old(kf.n_dev, removal)
    t_ours = median_ms(ours, restore_all)
    line = "keyframe %-7s %-6s B=1  cull + remove_old %.1f us" % (config, "culled" if culled else "kept", 1e3 * t_ours)
    if refimport.staged():
        restore_all()
        a = g.active.bool()
        edges = torch.stack([g.ii[a], g.jj[a], g.kk[a]], 1).cpu()
        n = int(kf.n_dev[0])
        with refimport.reference_python():
            ref = OK.reference_dpvo(st, edges, n, kf.tstamp[0], kf.ki, kf.thresh)
            pg = ref.pg
            keep = dict(ii=pg.ii.clone(), jj=pg.jj.clone(), kk=pg.kk.clone(), net=pg.net.clone(), weight=pg.weight.clone(),
                        target=pg.target.clone(), tstamps_=pg.tstamps_.copy(), poses_=pg.poses_.clone(),
                        patches_=pg.patches_.clone(), inac=(pg.ii_inac, pg.jj_inac, pg.kk_inac, pg.weight_inac, pg.target_inac))

            def ref_restore():
                pg.ii, pg.jj, pg.kk = keep["ii"].clone(), keep["jj"].clone(), keep["kk"].clone()
                pg.net, pg.weight, pg.target = keep["net"].clone(), keep["weight"].clone(), keep["target"].clone()
                pg.ii_inac, pg.jj_inac, pg.kk_inac, pg.weight_inac, pg.target_inac = keep["inac"]
                pg.tstamps_[:] = keep["tstamps_"]
                pg.poses_.copy_(keep["poses_"])
                pg.patches_.copy_(keep["patches_"])
                pg.n, pg.m, pg.delta = n, n * ref.M, {}
            t_ref = median_ms(ref.keyframe, ref_restore)
            ref_restore()
            ref.keyframe()
            assert (pg.n == n - 1) == culled
        line += "   reference DPVO.keyframe %.1f us" % (1e3 * t_ref)
    else:
        line += "   (reference: oracle/_ref not staged)"
    print(line, flush=True)


def bench_tracking(frames=200, n0=16):
    for cull in (None, True, False):                   # None: a warm-up pass (module loads, first launches), not reported
        st = synthetic.make_stop_go_state("fast", n0, total=n0 + frames, stop=8, go=6, mem=36, device="cuda", seed=7)
        cfg, M = st.cfg, st.cfg["M"]
        g = DevicePatchGraph(2 * st.E + 4 * M * cfg["lifetime"], M, st.poses.shape[0] - 1, "cuda")
        g.append(st.ii, st.jj, st.kk)
        runner = UpdateRunner(st, graph=g)
        kf = Keyframes(cfg, st, g)
        traj, allp = st.extras["trajectory"], st.extras["patches"]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        culled = 0
        for f in range(frames):
            st.n += 1
            kf.n_dev += 1
            n = st.n
            st.poses[n - 1] = traj[n0 + f]
            st.patches[(n - 1) * M:n * M] = allp[(n0 + f) * M:(n0 + f + 1) * M]
            kf.add_frame()
            g.append_frame_edges(kf.n_dev, cfg["lifetime"])
            st.t0 = max(n - cfg["opt_window"], 1)
            runner.step()
            if cull is not False:
                kf.cull()
                culled += kf.read()[0][0]
            g.remove_old(kf.n_dev, cfg["removal"])
        torch.cuda.synchronize()
        assert int(g.overflow) == 0
        dt = (time.perf_counter() - t0) / frames
        if cull is None:
            continue
        print("tracking fast stop-go, %d frames, %s: %.3f ms / frame (%d culled, final n = %d)" % (
            frames, "with culling" if cull else "without culling", 1e3 * dt, culled, st.n), flush=True)


if __name__ == "__main__":
    print("gpu:", torch.cuda.get_device_name(0), "|", smi(), flush=True)
    bench_cull()
    bench_tracking()
    print("gpu:", smi(), flush=True)
