"""One DPVO `update()` iteration on the sm_90a kernels -- the public call a user makes.

Mirrors DPVO.update (dpvo/dpvo.py:328-360):
    reproject -> correlation (2 levels) -> context gather -> update operator -> target/weight ->
    2 Gauss-Newton bundle-adjustment iterations
over state tensors laid out like dpvo/dpvo.py:58-73 / dpvo/patchgraph.py:26-35.  `ingest_frame`
is the per-frame host->device traffic of DPVO.__call__ (dpvo.py:426-438): the new frame's feature
maps, patch features and patches copied from pinned host memory into their ring-buffer slots.
"""
import torch

from . import extensions
from . import altcorr, fastba
from . import projective_ops as pops
from .net import Update, EdgeGroups, DIM


class UpdateRunner:
    def __init__(self, state, update=None, ba_iterations=2, seed=1234, graph=None):
        """graph: optional DevicePatchGraph (patchgraph.py).  With it the edge lists and the recurrent state are the
        store's fixed-capacity arrays: every kernel runs over all `cap` slots, parked slots are dummy edges in groups of
        their own whose confidence weights are zeroed before bundle adjustment, and a captured CUDA graph of step()
        stays valid while edges are appended and removed between replays."""
        self.s = state
        self.pg = graph
        dev = state.poses.device
        if update is None:
            torch.manual_seed(seed)                    # evaluate_tartan.py:173
            update = Update(3)
        self.update = update.to(dev).eval()
        self.update.inplace_state = True               # `self.net` is one buffer, updated in place
        self.update.packed()
        self.graph = None
        self.M = state.cfg["M"]
        self.mem = state.fmap1.shape[1]
        self.pmem = state.imap.shape[1] // self.M
        self.ba_iterations = ba_iterations
        self.lmbda = torch.as_tensor([1e-4], device=dev)
        self.poses0 = state.poses.clone()
        self.patches0 = state.patches.clone()
        self.timers = None
        if graph is None:
            self.E = state.E
            self.ii, self.jj, self.kk = state.ii, state.jj, state.kk
            self.net = torch.zeros(1, state.E, DIM, device=dev, dtype=torch.float32)
            # host-known bounds on the number of groups (no device->host sync in the step)
            n_live_frames = int((state.kk // self.M).unique().numel())
            self.max_patch_groups = n_live_frames * self.M
            self.max_pair_groups = int(torch.unique(state.ii * 100000 + state.jj).numel())
            self.kk_ring = state.kk % (self.M * self.pmem)
            self.jj_ring = state.jj % self.mem
        else:
            self.E = graph.cap
            self.ii, self.jj, self.kk = graph.ii, graph.jj, graph.kk
            self.net = graph.net                                      # [1, cap, 384] fp32, updated in place
            # bounds that hold for any topology the store can take: every live patch + the dummy patch; every ordered
            # frame pair inside the removal window + the dummy pair
            live = state.cfg["removal"] + 2
            self.max_patch_groups = min(graph.cap, live * self.M + 1)
            self.max_pair_groups = min(graph.cap, live * live + 1)
            self.kk_ring = self.jj_ring = None                       # the ring indices follow the edges: computed per step
        self.corr_buf = torch.zeros(1, self.E, 896, device=dev, dtype=torch.half)   # padding columns stay zero

    def reset(self):
        self.s.poses.copy_(self.poses0)
        self.s.patches.copy_(self.patches0)

    # -------------------------------------------------------------------------------- one update
    @torch.no_grad()
    def step(self):
        s = self.s
        ev = self.timers
        poses = s.poses.view(1, -1, 7)
        patches = s.patches.view(1, -1, 3, 3, 3)
        intr = s.intrinsics.view(1, -1, 4)
        ii, jj, kk = self.ii, self.jj, self.kk
        kk_ring = self.kk_ring if self.pg is None else kk % (self.M * self.pmem)
        jj_ring = self.jj_ring if self.pg is None else jj % self.mem
        coords = pops.transform_fused(poses, patches, intr, ii, jj, kk)               # [1,E,2,3,3]
        if ev is not None:
            ev["corr0"].record()
        corr = altcorr.corr_pyramid(s.gmap, (s.fmap1, s.fmap2), coords, kk_ring, jj_ring, 3, 4.0, 896, self.corr_buf)
        if ev is not None:
            ev["corr1"].record()
        groups_kk, groups_ij = EdgeGroups.pair((kk, None, jj), (ii, jj, None), self.max_patch_groups, self.max_pair_groups)
        # context gather (dpvo.py:334) and target = centre + delta (dpvo.py:341) are folded into the
        # first LayerNorm pass and the heads kernel
        self.net, (target, weight, _) = self.update(self.net, s.imap, corr, None, ii, jj, kk, groups_kk, groups_ij,
                                                    inp_index=kk_ring, coords=coords)
        if self.pg is not None:
            weight = weight * self.pg.active.view(1, -1, 1)          # parked edges carry no confidence into bundle adjustment
        if ev is not None:
            ev["ba0"].record()
        fastba.BA_grouped(poses, patches, intr, target, weight, self.lmbda, ii, jj, kk, s.t0, s.n,
                          self.ba_iterations, groups_kk, groups_ij)
        if ev is not None:
            ev["ba1"].record()
        return target, weight

    # ----------------------------------------------------------------------------- CUDA graph
    def capture(self):
        """Record one update() -- ~38 kernel launches, two memsets, no host decisions -- into a CUDA graph.
        Every buffer the step touches is persistent (state, ring buffers, corr rows) or comes from the graph's
        private pool, and the recurrent state is updated in place, so replaying the graph IS the next update."""
        if self.timers is not None:
            raise RuntimeError("capture(): event timers cannot be recorded inside a graph")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                      # warm-up off the capture: lazy inits, attribute calls
            for _ in range(2):
                self.step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._graph_out = self.step()
        return self.graph

    def step_graph(self):
        self.graph.replay()
        return self._graph_out

    # ----------------------------------------------------------------- end to end (host buffers)
    def make_host_frame(self, seed=0):
        """pinned host copies of everything DPVO.__call__ writes for one new frame"""
        s = self.s
        g = torch.Generator().manual_seed(seed)
        h, w = s.fmap1.shape[3], s.fmap1.shape[4]
        f = dict(
            fmap1=(torch.randn(h, w, 128, generator=g) / 4).half(),
            fmap2=(torch.randn(h // 4, w // 4, 128, generator=g) / 4).half(),
            gmap=(torch.randn(self.M, 3, 3, 128, generator=g) / 4).half(),
            imap=(torch.randn(self.M, DIM, generator=g) / 4).half(),
            patches=s.patches[(s.n - 1) * self.M:s.n * self.M].cpu().clone(),
            pose=s.poses[s.n - 1].cpu().clone(),
        )
        return {k: v.pin_memory() for k, v in f.items()}

    def ingest_frame(self, hf):
        """H2D of one frame into ring slot n-1 (channels-last buffers take the host layout as is)."""
        s = self.s
        slot = (s.n - 1) % self.mem
        pslot = (s.n - 1) % self.pmem
        s.fmap1[0, slot].permute(1, 2, 0).copy_(hf["fmap1"], non_blocking=True)
        s.fmap2[0, slot].permute(1, 2, 0).copy_(hf["fmap2"], non_blocking=True)
        s.gmap[0, pslot * self.M:(pslot + 1) * self.M].permute(0, 2, 3, 1).copy_(hf["gmap"], non_blocking=True)
        s.imap[0, pslot * self.M:(pslot + 1) * self.M].copy_(hf["imap"], non_blocking=True)
        s.patches[(s.n - 1) * self.M:s.n * self.M].copy_(hf["patches"], non_blocking=True)
        s.poses[s.n - 1].copy_(hf["pose"], non_blocking=True)
        return sum(v.numel() * v.element_size() for v in hf.values())

    # A streaming front end has frame t+1 in pinned memory while update t runs: its H2D copy goes to a staging
    # buffer on a copy stream (overlapping the update), and only the short device-to-device move into the ring
    # slots sits on the compute stream.
    def upload(self, hf):
        """start the H2D copy of a frame into the staging buffers (copy stream); returns the bytes copied"""
        if not hasattr(self, "_staging"):
            self._staging = {k: torch.empty_like(v, device=self.s.poses.device) for k, v in hf.items()}
            self._copy_stream = torch.cuda.Stream()
            self._ev_uploaded, self._ev_consumed = torch.cuda.Event(), torch.cuda.Event()
            self._ev_consumed.record()
        self._copy_stream.wait_event(self._ev_consumed)          # the previous frame has left the staging buffers
        with torch.cuda.stream(self._copy_stream):
            for k, v in hf.items():
                self._staging[k].copy_(v, non_blocking=True)
            self._ev_uploaded.record()
        return sum(v.numel() * v.element_size() for v in hf.values())

    def step_e2e_pipelined(self, hf_next, out_poses, out_depth):
        """consume the uploaded frame, start uploading the next one (if any), update, read the results back"""
        s = self.s
        main = torch.cuda.current_stream()
        main.wait_event(self._ev_uploaded)
        self.ingest_frame(self._staging)                           # device-to-device, a few microseconds
        self._ev_consumed.record()
        h2d = self.upload(hf_next) if hf_next is not None else 0
        if self.graph is not None:
            self.graph.replay()
        else:
            self.step()
        out_poses.copy_(s.poses[:s.n], non_blocking=True)
        out_depth.copy_(s.patches[:s.n * self.M, 2, 1, 1], non_blocking=True)
        # the results of this frame are on the host once this event has completed: the caller waits for it AFTER
        # issuing the next frame (two result buffers in rotation), so the device never idles on the host
        if not hasattr(self, "_ev_done"):
            self._ev_done, self._ev_i = [torch.cuda.Event(), torch.cuda.Event()], 0
        ev = self._ev_done[self._ev_i]
        self._ev_i ^= 1
        ev.record()
        return h2d, out_poses.numel() * 4 + out_depth.numel() * 4, ev

    def step_e2e(self, hf, out_poses, out_depth):
        """ingest a frame from pinned host memory, update, read poses + patch depths back to host"""
        s = self.s
        h2d = self.ingest_frame(hf)
        if self.graph is not None:
            self.graph.replay()
        else:
            self.step()
        out_poses.copy_(s.poses[:s.n], non_blocking=True)
        out_depth.copy_(s.patches[:s.n * self.M, 2, 1, 1], non_blocking=True)
        return h2d, out_poses.numel() * 4 + out_depth.numel() * 4
