"""What the map costs on one GPU:
    step     one captured update (UpdateRunner.capture / step_graph) with map=False and with map=True, the default and
             fast configurations and a batch of 8 fast streams.  The two graphs are replayed in alternation, ROUNDS
             rounds of REPS replays each, and the median of the per-round means is reported, with their difference: the
             point-cloud launch.
    ingest   ingest_image (one stream) and ingest_images (8 streams) with given centroids, on a state with and without
             colour buffers, alternated the same way: the added time of the colour threads in the centroid kernel.
Times are CUDA events around the replays / calls.  The card's name and power limit are read in the same run; one JSON
line per row.

    python tools/bench_map.py
"""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from dpvo_b200 import frontend, synthetic
from dpvo_b200.runner import UpdateRunner

REPS, ROUNDS = int(os.environ.get("REPS", 50)), int(os.environ.get("ROUNDS", 11))
DEV = "cuda"


def smi():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def alternate(fa, fb, reps=REPS, rounds=ROUNDS):
    """median over rounds of the mean ms per call of fa and of fb, each round timing fa then fb"""
    for f in (fa, fb):
        for _ in range(5):
            f()
    torch.cuda.synchronize()
    ta, tb = [], []
    for _ in range(rounds):
        for f, out in ((fa, ta), (fb, tb)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                f()
            b.record()
            b.synchronize()
            out.append(a.elapsed_time(b) / reps)
    return statistics.median(ta), statistics.median(tb)


def _runner(config, B, map, update):
    if B == 1:
        st = synthetic.make_state(config, 30, device=DEV, map=map)
    else:
        st = synthetic.make_batch(config, B, n_frames=[30 - 2 * b for b in range(B)], device=DEV, mem=30, map=map)
    run = UpdateRunner(st, update=update)
    run.capture()
    return run


def step_rows(update):
    rows = []
    for config, B in (("default", 1), ("fast", 1), ("fast", 8)):
        off, on = _runner(config, B, False, update), _runner(config, B, True, update)
        t_off, t_on = alternate(lambda: off.graph.replay(), lambda: on.graph.replay())
        rows.append(dict(row="step", config=config, B=B, map_off_ms=round(t_off, 4), map_on_ms=round(t_on, 4),
                         added_us=round(1000 * (t_on - t_off), 2)))
        del off, on
        torch.cuda.empty_cache()
    return rows


def ingest_rows(update):
    torch.manual_seed(4)
    enc = frontend.FrameEncoder(frontend.Patchifier().cuda().eval())
    rows = []
    for config, B in (("default", 1), ("fast", 1), ("fast", 8)):
        cfg = synthetic.CONFIGS[config]
        H, W = cfg["ht"], cfg["wd"]
        g = torch.Generator(device=DEV).manual_seed(1)
        imgs = torch.randint(0, 256, (B, 3, H, W), generator=g, device=DEV, dtype=torch.uint8)
        runs = []
        for map in (False, True):
            if B == 1:
                st = synthetic.make_state(config, 12, device=DEV, mem=12, map=map)
            else:
                st = synthetic.make_batch(config, B, n_frames=12, device=DEV, mem=12, map=map)
            runs.append(UpdateRunner(st, update=update, encoder=enc))
        M = cfg["M"]
        h, w = frontend.encoder_output_size(H, W)
        coords = torch.stack([torch.randint(1, w - 1, (B, M), generator=g, device=DEV),
                              torch.randint(1, h - 1, (B, M), generator=g, device=DEV)], -1).float()
        depth = torch.ones(B, M, device=DEV)
        if B == 1:
            calls = [lambda r=r: r.ingest_image(imgs[0], depth=depth.view(M, 1, 1), coords=coords[0]) for r in runs]
        else:
            calls = [lambda r=r: r.ingest_images(imgs, depth=depth, coords=coords) for r in runs]
        t_off, t_on = alternate(calls[0], calls[1])
        rows.append(dict(row="ingest", config=config, B=B, colors_off_ms=round(t_off, 4), colors_on_ms=round(t_on, 4),
                         added_us=round(1000 * (t_on - t_off), 2)))
        del runs
        torch.cuda.empty_cache()
    return rows


def main():
    assert torch.cuda.is_available(), "bench_map measures on a CUDA device"
    card = smi()
    torch.manual_seed(1234)
    from dpvo_b200.net import Update
    update = Update(3).to(DEV).eval()
    rows = step_rows(update) + ingest_rows(update)
    for r in rows:
        r["card"] = card
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
