"""ORACLE harness (test infrastructure; GPU box): the reference's UNMODIFIED host code -- class DPVO of
dpvo/dpvo.py with dpvo/net.py:VONet -- driven on a synthetic image stream, on top of a selectable set
of native modules:

    native="ours"   cuda_corr / cuda_ba / lietorch_backends = dpvo_b200/_ext   (the drop-in, exercised)
    native="ref"    cuda_corr / cuda_ba = oracle/_ref (the reference's own kernels compiled for sm_90a);
                    lietorch_backends stays ours: the reference's is Eigen template code and Eigen is
                    not in the image (SURVEY 8(c)) -- it only serves pops.transform / the motion model here
    update="reference"  dpvo/net.py:Update in torch under autocast (dpvo.py:332), torch_scatter restated
    update="ours"       dpvo_b200.net.Update (wgmma kernels) loaded with the same state_dict

Used by tests/test_dropin_gpu.py (parity of one DPVO.update() from an identical state, ours vs the
reference kernels) and by bench.py's `reference_cuda` leg (the same-box denominator of north_star's
">= 5x the reference CUDA build" target).  Never imported by dpvo_b200/.

Weights are random (no checkpoint in the image, SURVEY 8(c)); the flow head's bias is shifted so that
dpvo.py:240-257 motion_probe lets the system initialise -- a property of the synthetic weights, not a
code change.  The stream is a fixed smooth random texture seen through a window sliding 3 px/frame.
"""
import contextlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402

SIZES = {"default": (480, 640, (320.0, 320.0, 320.0, 240.0)), "fast": (480, 752, (458.654, 457.296, 367.215, 248.375))}


def ref_native():
    d = os.path.join(ROOT, "oracle", "_ref")
    if d not in sys.path:
        sys.path.insert(0, d)
    import ref_cuda_corr
    import ref_cuda_ba
    return ref_cuda_corr, ref_cuda_ba


def make_stream(config, n_frames, seed=1234, device="cuda"):
    """[n,3,H,W] uint8 frames: a smooth random texture (N(128,40) blurred) seen through a window that slides
    3 px right and 1 px down per frame (SURVEY 8(d) config 2(ii), fronto-parallel plane)"""
    ht, wd, _ = SIZES[config]
    g = torch.Generator(device=device).manual_seed(seed)
    H, W = ht + n_frames + 8, wd + 3 * n_frames + 8
    tex = 128 + 40 * torch.randn(1, 3, H, W, generator=g, device=device)
    k = torch.tensor([1.0, 4.0, 6.0, 4.0, 1.0], device=device)
    k = (k[:, None] * k[None, :] / 256.0).expand(3, 1, 5, 5)
    for _ in range(2):
        tex = torch.nn.functional.conv2d(tex, k, padding=2, groups=3)
    tex = (128 + (tex - 128) * 3.0).clamp(0, 255).to(torch.uint8)[0]
    return torch.stack([tex[:, t:t + ht, 3 * t:3 * t + wd] for t in range(n_frames)]).contiguous()


class RefDPVO:
    """the reference DPVO object + the switches above.  Holds the reference package imported for its lifetime."""

    def __init__(self, config="default", native="ours", update="reference", seed=1234, buffer=256, channels_last=False):
        import dpvo_b200
        self._stack = contextlib.ExitStack()
        self.ours = dpvo_b200.extensions()
        self._stack.enter_context(refimport.reference_python(native=self.ours[:3]))
        import dpvo.dpvo as RD
        import dpvo.net as RN
        from dpvo.config import cfg as base
        self.mods = {k: v for k, v in sys.modules.items() if k.startswith("dpvo.")}
        self.RD, self.RN = RD, RN
        cfg = base.clone()
        cfg.update(refimport.read_config(config))
        cfg.BUFFER_SIZE = buffer
        self.config, self.cfg = config, cfg
        ht, wd, intr = SIZES[config]
        self.intrinsics = torch.tensor(intr, device="cuda")
        torch.manual_seed(seed)                      # evaluate_tartan.py:173
        net = RN.VONet()
        with torch.no_grad():
            net.update.d[1].bias.add_(2.0)           # |delta| median >= 2 px so that motion_probe passes (random weights)
        self.slam = RD.DPVO(cfg, net, ht=ht, wd=wd, viz=False)
        self.ref_update = self.slam.network.update
        self.our_update = None
        if channels_last:                            # INTEGRATION.md: the one-line allocation change of the fast path
            s = self.slam
            s.fmap1_ = torch.zeros_like(s.fmap1_.permute(0, 1, 3, 4, 2).contiguous()).permute(0, 1, 4, 2, 3)
            s.fmap2_ = torch.zeros_like(s.fmap2_.permute(0, 1, 3, 4, 2).contiguous()).permute(0, 1, 4, 2, 3)
            s.pyramid = (s.fmap1_, s.fmap2_)
            s.gmap_ = torch.zeros_like(s.gmap_.permute(0, 1, 3, 4, 2).contiguous()).permute(0, 1, 4, 2, 3)
        self.use(native, update)
        self.t = 0

    def close(self):
        self._stack.close()

    def use(self, native=None, update=None):
        if native is not None:
            cc, cb = (self.ours[0], self.ours[1]) if native == "ours" else ref_native()
            refimport.bind_native(self.mods, cc, cb)
            self.native = native
        if update is not None:
            if update == "ours":
                if self.our_update is None:
                    from dpvo_b200.net import Update
                    self.our_update = Update(3).cuda().eval()
                    self.our_update.load_state_dict(self.ref_update.state_dict())
                self.slam.network.update = self.our_update
            else:
                self.slam.network.update = self.ref_update
            self.update_kind = update

    def feed(self, images):
        with torch.no_grad():
            for im in images:
                self.slam(self.t, im, self.intrinsics)
                self.t += 1

    # ---- one DPVO.update() from a saved state
    def snapshot(self):
        pg = self.slam.pg
        return dict(poses=pg.poses_.clone(), patches=pg.patches_.clone(), net=pg.net.clone(), points=pg.points_.clone())

    def restore(self, snap):
        pg = self.slam.pg
        pg.poses_.copy_(snap["poses"]); pg.patches_.copy_(snap["patches"]); pg.points_.copy_(snap["points"])
        pg.net = snap["net"].clone()

    def update_once(self):
        with torch.no_grad():
            self.slam.update()
        pg = self.slam.pg
        return dict(poses=pg.poses_[:self.slam.n].clone(), depth=pg.patches_[:self.slam.n, :, 2, 1, 1].clone(),
                    net=pg.net.float().clone(), target=pg.target.clone(), weight=pg.weight.clone())

    def time_updates(self, iters=20, warmup=3):
        """ms per DPVO.update() (CUDA events), state restored before every call so each one does the same work"""
        snap = self.snapshot()
        for _ in range(warmup):
            self.restore(snap); self.update_once()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        tot = 0.0
        for _ in range(iters):
            self.restore(snap)
            torch.cuda.synchronize()
            a.record()
            with torch.no_grad():
                self.slam.update()
            b.record()
            torch.cuda.synchronize()
            tot += a.elapsed_time(b)
        self.restore(snap)
        return tot / iters

    def time_frames(self, images):
        """frames/s of DPVO.__call__ (front end + update + keyframe) over `images` (CUDA events around the loop)"""
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        self.feed(images)
        b.record()
        torch.cuda.synchronize()
        return len(images) / (a.elapsed_time(b) * 1e-3)


# ------------------------------------------------------------------ one update() on a dpvo_b200.synthetic state
class RefCudaStep:
    """The reference CUDA pipeline of ONE DPVO.update() (dpvo.py:328-360) on a dpvo_b200.synthetic state:
    pops.transform (oracle restatement on the device, pinned bit-exactly to projective_ops.py) ->
    ref_cuda_corr.forward x2 + stack (dpvo.py:200-207) -> Update in torch under autocast (dpvo.py:332; module =
    oracle/update.py, pinned to net.py by tests/golden/update_ref_*.pt) -> ref_cuda_ba.forward (2 iterations).
    Owns private NCHW copies of the feature rings (the reference's allocation, dpvo.py:62-72) and its own
    poses / patches / net, so it can run next to an UpdateRunner on the same state."""

    def __init__(self, st, update_module, ba_iterations=2):
        from oracle import ba as OB
        self.OB = OB
        self.cc, self.cb = ref_native()
        self.st = st
        self.mod = update_module
        self.M = st.cfg["M"]
        mem, pmem = st.fmap1.shape[1], st.imap.shape[1] // self.M
        self.fmap1 = st.fmap1.contiguous()
        self.fmap2 = st.fmap2.contiguous()
        self.gmap = st.gmap.contiguous()
        self.imap = st.imap
        self.kk_ring = st.kk % (self.M * pmem)
        self.jj_ring = st.jj % mem
        self.poses = st.poses.clone()
        self.patches = st.patches.clone()
        self.net = torch.zeros(1, st.E, 384, device=st.poses.device, dtype=torch.half)   # dpvo.py:220-221
        self.lmbda = torch.as_tensor([1e-4], device=st.poses.device)
        self.iters = ba_iterations

    def reset(self):
        self.poses.copy_(self.st.poses)
        self.patches.copy_(self.st.patches)

    @torch.no_grad()
    def step(self):
        st = self.st
        poses, patches, intr = self.poses[None], self.patches[None], st.intrinsics[None]
        coords = self.OB.transform(poses, patches, intr, st.ii, st.jj, st.kk).permute(0, 1, 4, 2, 3).contiguous()
        with torch.autocast("cuda", dtype=torch.half):
            c0, = self.cc.forward(self.gmap, self.fmap1, coords, self.kk_ring, self.jj_ring, 3)
            c1, = self.cc.forward(self.gmap, self.fmap2, coords / 4, self.kk_ring, self.jj_ring, 3)
            corr = torch.stack([c0, c1], -1).view(1, st.E, -1)
            ctx = self.imap[:, self.kk_ring]
            self.net, (delta, weight, _) = self.mod(self.net, ctx, corr, None, st.ii, st.jj, st.kk)
        weight = weight.float()
        target = coords[..., 1, 1] + delta.float()
        self.cb.forward(poses, patches, intr, target, weight, self.lmbda, st.ii, st.jj, st.kk, self.M, st.t0, st.n,
                        self.iters, False)
        return target, weight, corr
