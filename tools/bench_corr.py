"""Time the two-level correlation on the bench state (E = 47,712 edges, `synthetic.make_state("default", 36)` reprojected
as `runner.UpdateRunner.step` does) and set it against the bytes each design moves from L2 to the SMs.

  * whole call: CUDA events around `dpvo_corr_forward_pyramid2`, median of --iters launches after warm-up; with
    --parent-lib (a libdpvo_b200.so built from an earlier commit) the old build's call is timed in the same process,
    alternated launch by launch with the new one, on the same inputs, and its output is compared
  * per kernel: device time of every kernel inside the call (binning, level-1 pass, level-0 pass, list path) from
    torch.profiler, median over --prof-iters calls, in a run of its own
  * the old kernel on edges pre-sorted by (target frame, box origin): how much of its time is DRAM re-fetch
  * L2->SM bytes: per-edge boxes (level 0 + level 1 + patch) against the level-1 regions of the bins, from the shapes

Prints one JSON object; card name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import dpvo_b200  # noqa: E402
from dpvo_b200 import projective_ops as pops, synthetic  # noqa: E402
from dpvo_b200.runner import UpdateRunner  # noqa: E402

T1, APRON1, ITEM = 7, 9, 48      # level-1 tile side, apron and edges per work item of corr_bin.cu


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers are still reported, without the card
        return {"name": torch.cuda.get_device_name(), "error": str(e)[:200]}


class Corr:
    """dpvo_corr_forward_pyramid2 of one libdpvo_b200.so, called through its C ABI on the given inputs."""

    def __init__(self, lib, f1, l0, l1, coords, ii, jj, row):
        self.lib, self.keep = lib, (f1, l0, l1, coords, ii, jj)
        lib.dpvo_corr_pyramid2_workspace_bytes.restype = ctypes.c_int64
        M = coords.shape[1]
        self.wsb = lib.dpvo_corr_pyramid2_workspace_bytes(ctypes.c_int64(M))
        self.ws = torch.empty(self.wsb, dtype=torch.uint8, device=coords.device)
        self.out = torch.zeros(1, M, row, dtype=torch.half, device=coords.device)
        st = lambda t: (ctypes.c_int64 * 5)(*t.stride())
        self.s = (st(f1), st(l0), st(l1))
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        self.args = [p(f1), self.s[0], p(l0), self.s[1], l0.shape[3], l0.shape[4], p(l1), self.s[2], l1.shape[3], l1.shape[4],
                     ctypes.c_float(4.0), p(coords), p(ii), p(jj), p(self.out), ctypes.c_int64(row), 0, 1, M, 128, 3,
                     f1.shape[1], l0.shape[1], 3, p(self.ws), ctypes.c_int64(self.wsb)]

    def __call__(self):
        rc = self.lib.dpvo_corr_forward_pyramid2(*self.args, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, rc


def event_ms(fns, iters, warmup):
    """Median CUDA-event time of each callable, the callables alternated launch by launch."""
    for _ in range(warmup):
        for f in fns:
            f()
    ev = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)] for _ in fns]
    for i in range(iters):
        for f, e in zip(fns, ev):
            e[i][0].record(); f(); e[i][1].record()
    torch.cuda.synchronize()
    return [statistics.median(a.elapsed_time(b) for a, b in e) for e in ev]


def kernel_us(fn, iters):
    """Median device time per call of every kernel fn launches (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    per = {}
    for evt in prof.events():
        if evt.device_type == torch.autograd.DeviceType.CUDA:
            name = evt.name.split("(")[0].replace("void ", "").replace("dpvo::", "")
            per.setdefault(name, []).append(evt.device_time_total if hasattr(evt, "device_time_total") else evt.cuda_time_total)
    return {k: {"median_us": statistics.median(v), "launches": len(v)} for k, v in sorted(per.items())}


def box_stats(coords, div=4.0):
    """Per-edge box origins and sizes of both levels (the nine anchors' min / max, as corr_bin_count)."""
    c = coords[0].double()
    out = {}
    for lev, d in ((0, 1.0), (1, div)):
        a = torch.floor(c / d).long() - 3                       # [E, 2, 3, 3]
        mn, mx = a.flatten(2).min(-1).values, a.flatten(2).max(-1).values
        out[lev] = (mn, (mx - mn).clamp(max=64) + 8)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--prof-iters", type=int, default=50)
    ap.add_argument("--parent-lib", default=None, help="libdpvo_b200.so of the build to compare against")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_corr needs a CUDA device"
    dev = "cuda:0"
    torch.cuda.set_device(0)
    st = synthetic.make_state("default", 36, device=dev, seed=1234)
    run = UpdateRunner(st)
    coords = pops.transform_fused(st.poses.view(1, -1, 7), st.patches.view(1, -1, 3, 3, 3), st.intrinsics.view(1, -1, 4),
                                  st.ii, st.jj, st.kk).contiguous()
    f1, l0, l1 = st.gmap, st.fmap1, st.fmap2
    ii, jj = run.kk_ring.contiguous(), run.jj_ring.contiguous()
    E = coords.shape[1]
    res = {"card": card(), "E": E, "level0": list(l0.shape[3:]), "level1": list(l1.shape[3:]), "ring_slots": l0.shape[1]}

    # ---- bytes from the shapes
    bx = box_stats(coords.cpu())
    sz0 = bx[0][1][:, 0] * bx[0][1][:, 1]
    sz1 = bx[1][1][:, 0] * bx[1][1][:, 1]
    boxed = (bx[0][1][:, 0] <= 12) & (bx[0][1][:, 1] <= 12) & (sz0 <= 128) & (bx[1][1][:, 0] <= 10) & (bx[1][1][:, 1] <= 10)
    H1, W1 = l1.shape[3:]
    nty, ntx = (H1 + APRON1 + T1 - 1) // T1, (W1 + APRON1 + T1 - 1) // T1
    o1 = bx[1][0]
    ty = ((o1[:, 1] + APRON1).clamp(min=0) // T1).clamp(max=nty - 1)
    tx = ((o1[:, 0] + APRON1).clamp(min=0) // T1).clamp(max=ntx - 1)
    key = (jj.cpu() * nty + ty) * ntx + tx
    cnt = torch.bincount(key[boxed], minlength=l0.shape[1] * nty * ntx)
    items = int(((cnt + ITEM - 1) // ITEM).sum())
    patch = 9 * 256
    per_edge = float((sz0 + sz1).double().mean()) * 256 + patch
    res["bytes_L2_to_SM"] = {
        "per_edge_boxes_both_levels_GB": per_edge * E / 1e9,
        "level0_boxes_plus_patch_GB": (float(sz0.double().mean()) * 256 + patch) * E / 1e9,
        "level1_regions_GB": items * (T1 + APRON1) ** 2 * 256 / 1e9,
        "level1_patch_GB": patch * int(boxed.sum()) / 1e9,
        "mean_box_pixels": [float(sz0.double().mean()), float(sz1.double().mean())],
        "level1_bins_nonempty": int((cnt > 0).sum()), "level1_work_items": items,
        "edges_on_list_path": int((~boxed).sum()),
    }
    bb = res["bytes_L2_to_SM"]
    bb["binned_total_GB"] = bb["level0_boxes_plus_patch_GB"] + bb["level1_regions_GB"] + bb["level1_patch_GB"]

    # ---- timings
    row = 896
    new = Corr(dpvo_b200.library(), f1, l0, l1, coords, ii, jj, row)
    fns, names = [new], ["new"]
    if args.parent_lib:
        old_lib = ctypes.CDLL(os.path.abspath(args.parent_lib), mode=os.RTLD_LOCAL | os.RTLD_DEEPBIND)
        old = Corr(old_lib, f1, l0, l1, coords, ii, jj, row)
        # the old kernel on edges pre-sorted by (target frame, level-0 box origin in 16-pixel tiles)
        o0 = bx[0][0]
        skey = ((jj.cpu() * 64 + (o0[:, 1] + 11).clamp(0, 1023) // 16) * 64 + (o0[:, 0] + 11).clamp(0, 1023) // 16)
        perm = torch.argsort(skey).to(dev)
        old_sorted = Corr(old_lib, f1, l0, l1, coords[:, perm].contiguous(), ii[perm].contiguous(), jj[perm].contiguous(), row)
        fns += [old, old_sorted]
        names += ["parent", "parent_presorted_edges"]
    ms = event_ms(fns, args.iters, args.warmup)
    res["call_ms_median"] = dict(zip(names, ms))
    if args.parent_lib:
        new(); old(); torch.cuda.synchronize()
        d = (new.out.float() - old.out.float()).abs()
        lvl = d[..., :882].reshape(E, 441, 2)
        res["vs_parent"] = {"max_abs_diff_level0": float(lvl[..., 0].max()), "max_abs_diff_level1": float(lvl[..., 1].max()),
                            "max_abs_value": float(old.out.float().abs().max()),
                            "level0_bit_identical": bool(torch.equal(new.out.view(E, -1)[:, 0:882:2], old.out.view(E, -1)[:, 0:882:2]))}
        res["speedup_vs_parent"] = ms[1] / ms[0]
    res["kernels_new"] = kernel_us(new, args.prof_iters)
    if args.parent_lib:
        res["kernels_parent"] = kernel_us(old, args.prof_iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
