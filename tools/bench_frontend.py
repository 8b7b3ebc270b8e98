"""Times the front end of one frame, CUDA events, median of REPS frames after WARM warm-up frames, for the default
(480 x 640, M = 96) and fast (480 x 752, M = 48) configurations:
    library    Patchifier under autocast(fp16) on cuDNN, plus the slot writes of dpvo.py:435-438 into the
               channels-last rings (what a user had to do before ingest_image existed)
    ingest     UpdateRunner.ingest_image: the sm_90a encoder kernels writing the slots directly
It prints the FLOP per frame computed from the shapes (both encoders at full resolution, as the library path computes
them) and the achieved TFLOP/s, then image -> pose frames/s: one CUDA graph of ingest_image(coords=...) + step() on
the bench's synthetic state (synthetic.make_state(config, 36)), next to the graph of step() alone."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from dpvo_b200 import frontend, synthetic
from dpvo_b200.runner import UpdateRunner

REPS, WARM = int(os.environ.get("REPS", 200)), int(os.environ.get("WARM", 20))


def encoder_flops(H, W, out_dim):
    h1, w1 = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    h2, w2 = frontend.encoder_output_size(H, W)
    macs = h1 * w1 * 32 * 3 * 49                       # stem
    macs += 4 * h1 * w1 * 32 * 32 * 9                  # layer1
    macs += h2 * w2 * 64 * (32 * 9 + 32 + 3 * 64 * 9)  # layer2: conv1 (3x3/2), projection, three 3x3
    macs += h2 * w2 * out_dim * 64                     # output convolution
    return 2.0 * macs


def timeit(f, reps=REPS, warm=WARM):
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


def image(H, W, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (3, H, W), generator=g, device="cuda", dtype=torch.uint8)


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("device: %s" % smi)
    for config in ("default", "fast"):
        cfg = synthetic.CONFIGS[config]
        H, W, M = cfg["ht"], cfg["wd"], cfg["M"]
        st = synthetic.make_state(config, 36, device="cuda", seed=1)
        torch.manual_seed(0)
        p = frontend.Patchifier().cuda().eval()
        run = UpdateRunner(st, encoder=frontend.FrameEncoder(p))
        img = image(H, W)
        slot, pslot = (st.n - 1) % run.mem, (st.n - 1) % run.pmem

        @torch.no_grad()
        def library():
            x = 2 * (img[None, None] / 255.0) - 0.5
            with torch.autocast("cuda", dtype=torch.float16):
                fmap, gmap, imap, patches, _ = p(x, patches_per_image=M)
            patches[:, :, 2] = torch.rand_like(patches[:, :, 2, 0, 0, None, None])
            st.patches[(st.n - 1) * M:st.n * M] = patches[0]
            st.imap[0, pslot * M:(pslot + 1) * M] = imap.view(M, -1)
            st.gmap[0, pslot * M:(pslot + 1) * M] = gmap.view(M, 128, 3, 3)
            st.fmap1[0, slot] = F.avg_pool2d(fmap[0, 0], 1, 1)
            st.fmap2[0, slot] = F.avg_pool2d(fmap[0, 0], 4, 4)

        def ingest():
            run.ingest_image(img)

        t_lib, t_ing = timeit(library), timeit(ingest)
        flop = encoder_flops(H, W, 128) + encoder_flops(H, W, 384)
        print("[%s %dx%d M=%d] library %.1f us  ingest_image %.1f us  (%.2fx)   %.2f GFLOP/frame: library %.1f TFLOP/s, ingest_image %.1f TFLOP/s"
              % (config, H, W, M, t_lib * 1e6, t_ing * 1e6, t_lib / t_ing, flop / 1e9, flop / t_lib / 1e12, flop / t_ing / 1e12))

        # image -> pose: one graph of ingest_image(coords) + step(), next to the graph of step() alone
        coords = run.encoder.centroids(img, M, "RANDOM")
        depth = torch.rand(M, 1, 1, device="cuda")

        def frame():
            run.ingest_image(img, depth=depth, coords=coords)
            return run.step()

        graphs = {}
        for nm, fn in (("step", run.step), ("image+step", frame)):
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
            graphs[nm] = g
        t_step = timeit(graphs["step"].replay)
        t_frame = timeit(graphs["image+step"].replay)
        print("[%s] graph of step(): %.1f us, %.1f updates/s   graph of ingest_image + step(): %.1f us, %.1f image -> pose frames/s"
              % (config, t_step * 1e6, 1 / t_step, t_frame * 1e6, 1 / t_frame))
        del run, st, graphs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
