"""Front end of B camera streams on one GPU, default (480 x 640, M = 96) and fast (480 x 752, M = 48), B in {1, 2, 4, 8}:
    (a) sequential  B UpdateRunner.ingest_image(stream=b) calls, eager
    (c) batched     one UpdateRunner.ingest_images call for the B images, eager
with the encoder TFLOP/s of each (both encoders at full resolution, bench_frontend.encoder_flops), then aggregate
image -> pose frames/s: one CUDA graph of the B ingest_image calls + the batched step(), against one graph of
ingest_images + the batched step() (coords and depths given, so nothing is drawn).  Every stream is
synthetic.make_state(config, 36) with its own seed, in one streams.StreamBatch; as in bench.py, poses and patches are
reset before every replay.  CUDA events, median of REPS calls after WARM warm-up calls.  The card's name, power limit
and SM clocks are read in the same run.

    python tools/bench_frontend_streams.py [--configs default,fast] [--batches 1,2,4,8]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bench_frontend import encoder_flops
from bench_streams import median_time, smi
from dpvo_b200 import frontend, synthetic
from dpvo_b200.runner import UpdateRunner


def graph_of(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="default,fast")
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--frames", type=int, default=36)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frontend_streams: needs a CUDA device")
    print("device (before): %s" % smi(), flush=True)
    rows = []
    for config in args.configs.split(","):
        cfg = synthetic.CONFIGS[config]
        H, W, M = cfg["ht"], cfg["wd"], cfg["M"]
        flop = encoder_flops(H, W, 128) + encoder_flops(H, W, 384)
        for B in (int(b) for b in args.batches.split(",")):
            batch = synthetic.make_batch(config, B, [1 + 17 * b for b in range(B)], n_frames=args.frames, device="cuda",
                                         frames_per_stream=64, mem=args.frames)
            torch.manual_seed(0)
            run = UpdateRunner(batch, encoder=frontend.FrameEncoder(frontend.Patchifier().cuda().eval()))
            g = torch.Generator(device="cuda").manual_seed(B)
            imgs = torch.randint(0, 256, (B, 3, H, W), generator=g, device="cuda", dtype=torch.uint8)

            def sequential():
                for b in range(B):
                    run.ingest_image(imgs[b], stream=b)

            def batched():
                run.ingest_images(imgs)

            t_a, t_c = median_time(sequential), median_time(batched)
            coords = torch.stack([run.encoder.centroids(imgs[b], M, "RANDOM") for b in range(B)])
            depth = torch.rand(B, M, device="cuda")

            def frame_a():
                for b in range(B):
                    run.ingest_image(imgs[b], depth=depth[b, :, None, None], coords=coords[b], stream=b)
                return run.step()

            def frame_c():
                run.ingest_images(imgs, depth=depth, coords=coords)
                return run.step()

            ga, gc = graph_of(frame_a), graph_of(frame_c)

            def replay(gr):
                def f():
                    run.reset()
                    gr.replay()
                return f

            f_a, f_c = median_time(replay(ga)), median_time(replay(gc))
            r = dict(config=config, B=B, a=t_a * 1e3, c=t_c * 1e3, tf_a=B * flop / t_a / 1e12, tf_c=B * flop / t_c / 1e12,
                     fps_a=B / f_a, fps_c=B / f_c)
            rows.append(r)
            print("[%s B=%d] (a) %d x ingest_image %.3f ms (%.1f TFLOP/s)  (c) ingest_images %.3f ms (%.1f TFLOP/s)  c/a %.3f   "
                  "image -> pose: graph (a) %.1f frames/s, graph (c) %.1f frames/s (%.3fx)"
                  % (config, B, B, r["a"], r["tf_a"], r["c"], r["tf_c"], r["c"] / r["a"], r["fps_a"], r["fps_c"], r["fps_c"] / r["fps_a"]),
                  flush=True)
            del run, batch, ga, gc
            torch.cuda.empty_cache()
    print("device (after): %s" % smi())
    print("| config | B | (a) B x ingest_image ms | (c) ingest_images ms | (c)/(a) | TFLOP/s (a) / (c) | graph (a) frames/s | graph (c) frames/s | (c)/(a) |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %d | %.3f | %.3f | %.3f | %.1f / %.1f | %.1f | %.1f | %.3f |" % (
            r["config"], r["B"], r["a"], r["c"], r["c"] / r["a"], r["tf_a"], r["tf_c"], r["fps_a"], r["fps_c"], r["fps_c"] / r["fps_a"]))


if __name__ == "__main__":
    main()
