"""Aggregate throughput of B camera streams on one GPU, default and fast configurations, B in {1, 2, 4, 8}:
    (a) sequential  B single-stream UpdateRunner graphs replayed one after another on one CUDA stream
    (b) concurrent  the same B graphs, graph b replayed on CUDA stream b
    (c) batched     one UpdateRunner over a streams.StreamBatch of the B streams, one graph
Every stream is synthetic.make_state(config, 36) with its own seed (the bench's steady state).  As in bench.py, each
runner's poses and patches are reset before every replay (two small device copies per runner, inside the timed
window), so every replay sees the same geometry.  Aggregate frames/s = B x replays per second; CUDA events, median of
REPS replays after WARM warm-up replays.  Then the eager per-phase
breakdown of (c), mean of REPS eager steps: correlation, dense layers (every tensor-core launch of the update
operator), bundle adjustment, and the rest (reprojection, groupings, neighbours, reductions, launch gaps).
The card's name, power limit and SM clocks are read in the same run, before and after the timings.

    python tools/bench_streams.py [--configs default,fast] [--batches 1,2,4,8]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from dpvo_b200 import synthetic
from dpvo_b200.net import Update
from dpvo_b200.runner import UpdateRunner

REPS, WARM = int(os.environ.get("REPS", 200)), int(os.environ.get("WARM", 20))


def smi():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def median_time(f, reps=REPS, warm=WARM):
    for _ in range(warm):
        f()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in evs:
        a.record()
        f()
        b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in evs)
    return t[len(t) // 2] * 1e-3


def phases(run, reps=REPS):
    """eager per-phase means (ms) of run.step()"""
    ev = {k: [torch.cuda.Event(enable_timing=True) for _ in range(reps)] for k in ("t0", "corr0", "corr1", "ba0", "ba1", "t1")}
    for _ in range(3):                                  # lazy initialisation and first launches stay out of the means
        run.reset()
        run.step()
    gemm = []
    run.update.gemm_events = gemm
    for i in range(reps):
        run.reset()
        run.timers = {k: v[i] for k, v in ev.items()}
        ev["t0"][i].record()
        run.step()
        ev["t1"][i].record()
    torch.cuda.synchronize()
    run.timers = None
    run.update.gemm_events = None
    mean = lambda a, b: statistics.mean(x.elapsed_time(y) for x, y in zip(ev[a], ev[b]))
    total, corr, ba = mean("t0", "t1"), mean("corr0", "corr1"), mean("ba0", "ba1")
    dense = sum(a.elapsed_time(b) for a, b in gemm) / reps
    return dict(total=total, corr=corr, dense=dense, ba=ba, rest=total - corr - dense - ba)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="default,fast")
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--frames", type=int, default=36)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_streams: needs a CUDA device")
    print("device (name, power limit, SM clock, max SM clock): %s" % smi(), flush=True)
    torch.manual_seed(1234)
    update = Update(3).cuda().eval()
    rows = []
    for config in args.configs.split(","):
        for B in [int(x) for x in args.batches.split(",")]:
            seeds = [1234 + 17 * b for b in range(B)]
            batch = synthetic.make_batch(config, B, seeds, n_frames=args.frames, device="cuda")
            E = batch.E
            singles = [UpdateRunner(batch.copy_stream(b), update=update) for b in range(B)]
            for r in singles:
                r.capture()
            graphs = [r.graph for r in singles]

            def sequential():
                for r, g in zip(singles, graphs):
                    r.reset()
                    g.replay()

            side = [torch.cuda.Stream() for _ in range(B)]

            def concurrent():
                main = torch.cuda.current_stream()
                for s, r, g in zip(side, singles, graphs):
                    s.wait_stream(main)
                    with torch.cuda.stream(s):
                        r.reset()
                        g.replay()
                for s in side:
                    main.wait_stream(s)

            t_a = median_time(sequential)
            t_b = median_time(concurrent)
            del singles, graphs
            torch.cuda.empty_cache()
            run = UpdateRunner(batch, update=update)
            ph = phases(run)
            run.capture()

            def batched():
                run.reset()
                run.graph.replay()

            t_c = median_time(batched)
            row = dict(config=config, B=B, E=E, a=B / t_a, b=B / t_b, c=B / t_c, t_a=t_a, t_b=t_b, t_c=t_c, **ph)
            rows.append(row)
            print("[%s B=%d E=%d] frames/s: (a) sequential %.1f  (b) %d CUDA streams %.1f  (c) batched %.1f  "
                  "(c)/(a) %.3f  (c)/(b) %.3f | per replay: %.3f / %.3f / %.3f ms | eager (c) ms: total %.3f corr %.3f "
                  "dense %.3f BA %.3f rest %.3f"
                  % (config, B, E, row["a"], B, row["b"], row["c"], row["c"] / row["a"], row["c"] / row["b"],
                     t_a * 1e3, t_b * 1e3, t_c * 1e3, ph["total"], ph["corr"], ph["dense"], ph["ba"], ph["rest"]), flush=True)
            del run, batch
            torch.cuda.empty_cache()
    print("device after the timings: %s" % smi())
    print()
    print("| config | B | edges | (a) sequential | (b) B streams | (c) batched | (c)/(a) | (c)/(b) | eager (c): corr / dense / BA / rest ms |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %d | %d | %.1f | %.1f | %.1f | %.2f | %.2f | %.3f / %.3f / %.3f / %.3f |"
              % (r["config"], r["B"], r["E"], r["a"], r["b"], r["c"], r["c"] / r["a"], r["c"] / r["b"], r["corr"], r["dense"],
                 r["ba"], r["rest"]))


if __name__ == "__main__":
    main()
