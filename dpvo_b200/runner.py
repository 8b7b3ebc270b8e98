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
from .camera import undistort_frames
from .frontend import encoder_output_size
from .streams import StreamBatch
from .synthetic import check_map


class UpdateRunner:
    def __init__(self, state, update=None, ba_iterations=2, seed=1234, graph=None, encoder=None, loop=None):
        """state: one stream's state (synthetic.SyntheticState layout), or a streams.StreamBatch of B streams that every
        step updates together: one launch per kernel for all of them, bundle adjustment by fastba.BA_batched.
        encoder: optional frontend.FrameEncoder, which `ingest_image` runs.
        graph: optional DevicePatchGraph (patchgraph.py).  With it the edge lists and the recurrent state are the
        store's fixed-capacity arrays: every kernel runs over all `cap` slots, parked slots are dummy edges in groups of
        their own whose confidence weights are zeroed before bundle adjustment, and a captured CUDA graph of step()
        stays valid while edges are appended and removed between replays.  For a batch: DevicePatchGraph.stacked.
        loop: optional loop.LoopClosure on `graph` (one stream).  While no loop edge is active a step runs over the
        graph's normal slots only, exactly as without loop closure; while one is, over the normal slots and the used
        part of the loop region (a captured graph: over the whole store).  Each step then
        reads one small record from the device to decide this, and runs the global bundle adjustment in place of the
        local one when an active edge has ii < n - removal - 1 and none ran at this n (dpvo.py:348).  The rings must
        hold pmem = max_edge_age patch frames (dpvo.py:58-61).
        A state with map buffers (synthetic.make_state(map=True), StreamBatch(map=True)) also gets the map: every step
        ends with the points of frames [0, n) (dpvo.py:358-360), and ingest_image(s) write the new frame's colours
        (dpvo.py:404).  `map()` returns them."""
        check_map(state, "UpdateRunner")
        self.s = state
        self.batch = state if isinstance(state, StreamBatch) else None
        self.pg = graph
        self.loop = loop
        self.encoder = encoder
        dev = state.poses.device
        if update is None:
            torch.manual_seed(seed)                    # evaluate_tartan.py:173
            update = Update(3)
        self.update = update.to(dev).eval()
        self.update.inplace_state = True               # `self.net` is one buffer, updated in place
        self.update.packed()
        self.graph = None
        self.M = state.cfg["M"]
        if self.batch is None:
            self.mem = state.fmap1.shape[1]
            self.pmem = state.imap.shape[1] // self.M
        else:
            self.mem, self.pmem = state.mem, state.pmem                # ring sizes of one stream
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
            if self.batch is None:
                self.kk_ring = state.kk % (self.M * self.pmem)
                self.jj_ring = state.jj % self.mem
            else:
                self.kk_ring, self.jj_ring = state.ring_rows(state.kk, state.jj)
        else:
            self.E = graph.cap
            self.ii, self.jj, self.kk = graph.ii, graph.jj, graph.kk
            self.net = graph.net                                      # [1, cap, 384] fp32, updated in place
            # bounds that hold for any topology the store can take: every live patch + the dummy patch; every ordered
            # frame pair inside the removal window + the dummy pair, per stream
            live = state.cfg["removal"] + 2
            nb = 1 if self.batch is None else self.batch.B
            self.max_patch_groups = min(graph.normal_cap, nb * (live * self.M + 1))
            self.max_pair_groups = min(graph.normal_cap, nb * (live * live + 1))
            if loop is not None:
                if self.batch is not None or loop.pg is not graph:
                    raise ValueError("UpdateRunner: loop closure needs one stream and a LoopClosure on this runner's graph")
                if self.pmem != loop.max_age:
                    raise ValueError("UpdateRunner: the patch rings hold %d frames; loop closure needs pmem = max_edge_age = %d"
                                     % (self.pmem, loop.max_age))
                # with the loop region stepped: up to loop_pairs more pairs and loop_pairs * M more (old) patches
                self.loop_groups = (min(graph.cap, self.max_patch_groups + graph.loop_pairs * self.M),
                                    min(graph.cap, self.max_pair_groups + graph.loop_pairs))
            self.kk_ring = self.jj_ring = None                       # the ring indices follow the edges: computed per step
        self.corr_buf = torch.zeros(1, self.E, 896, device=dev, dtype=torch.half)   # padding columns stay zero

    def reset(self):
        self.s.poses.copy_(self.poses0)
        self.s.patches.copy_(self.patches0)

    # -------------------------------------------------------------------------------- one update
    @torch.no_grad()
    def step(self, loop_edges=None, loop_record=None):
        """One update.  With loop closure, loop_edges=None reads the device's loop record (one small D2H; or takes
        `loop_record`, a LoopClosure.read_flags result the caller read for this frame) and picks the slots and the
        bundle adjustment from it; True / False fixes the slots (the whole store / the normal ones) without reading
        anything and runs the local bundle adjustment, as a captured graph does."""
        s = self.s
        ev = self.timers
        poses = s.poses.view(1, -1, 7)
        patches = s.patches.view(1, -1, 3, 3, 3)
        intr = s.intrinsics.view(1, -1, 4)
        ii, jj, kk = self.ii, self.jj, self.kk
        net, corr_buf, gmax = self.net, self.corr_buf, (self.max_patch_groups, self.max_pair_groups)
        global_ba = None
        if self.loop is not None:
            if loop_edges is None:
                rec = self.loop.read_flags(s.n) if loop_record is None else loop_record
                loop_edges, long_range, t0, count = rec
                if long_range and s.n not in self.loop.ran_global_ba:
                    global_ba = (t0, count)
            if loop_edges is True:
                E = self.pg.cap                                       # the captured form: the whole store
            elif loop_edges:
                # eager, from the record: the normal slots and the used part of the loop region only (rounded up to
                # 128 slots); the parked remainder of the region would only add one large group of dummy edges
                E = min(self.pg.cap, self.pg.normal_cap + (int(loop_edges) + 127) // 128 * 128)
            else:
                E = self.pg.normal_cap
            ii, jj, kk, net, corr_buf = ii[:E], jj[:E], kk[:E], net[:, :E], corr_buf[:, :E]
            if loop_edges:
                gmax = (min(E, self.loop_groups[0]), min(E, self.loop_groups[1]))
        if self.pg is None:
            kk_ring, jj_ring = self.kk_ring, self.jj_ring
        elif self.batch is None:
            kk_ring, jj_ring = kk % (self.M * self.pmem), jj % self.mem
        else:
            kk_ring, jj_ring = self.batch.ring_rows(kk, jj)
        coords = pops.transform_fused(poses, patches, intr, ii, jj, kk)               # [1,E,2,3,3]
        if ev is not None:
            ev["corr0"].record()
        corr = altcorr.corr_pyramid(s.gmap, (s.fmap1, s.fmap2), coords, kk_ring, jj_ring, 3, 4.0, 896, corr_buf)
        if ev is not None:
            ev["corr1"].record()
        groups_kk, groups_ij = EdgeGroups.pair((kk, None, jj), (ii, jj, None), gmax[0], gmax[1])
        # context gather (dpvo.py:334) and target = centre + delta (dpvo.py:341) are folded into the
        # first LayerNorm pass and the heads kernel
        net, (target, weight, _) = self.update(net, s.imap, corr, None, ii, jj, kk, groups_kk, groups_ij,
                                               inp_index=kk_ring, coords=coords)
        if self.loop is None:
            self.net = net
        if self.pg is not None:
            weight = weight * self.pg.active[:ii.numel()].view(1, -1, 1)   # parked edges carry no confidence into bundle adjustment
        if self.loop is not None:
            # every slot's last target / weight: what LoopClosure.remove keeps and the global bundle adjustment reads
            self.pg.target[:, :ii.numel()].copy_(target)
            self.pg.weight[:, :ii.numel()].copy_(weight)
        if ev is not None:
            ev["ba0"].record()
        if global_ba is not None:
            self.loop.global_ba(s.poses, s.patches, s.intrinsics, s.n, global_ba[0], global_ba[1], ii.numel(), self.lmbda,
                                self.ba_iterations)
        elif self.batch is None:
            fastba.BA_grouped(poses, patches, intr, target, weight, self.lmbda, ii, jj, kk, s.t0, s.n,
                              self.ba_iterations, groups_kk, groups_ij)
        else:
            t0s, t1s = self.batch.windows()
            fastba.BA_batched(poses, patches, intr, target, weight, self.lmbda, ii, jj, kk, self.batch.F, t0s, t1s,
                              self.ba_iterations, groups_kk, groups_ij)
        if ev is not None:
            ev["ba1"].record()
        if getattr(s, "points", None) is not None:
            # dpvo.py:358-360, after whichever bundle adjustment ran; n is a launch parameter, as the BA window is
            if self.batch is None:
                F, ns = s.poses.shape[0], [s.n]
            else:
                F, ns = self.batch.F, [self.batch.stream(b).n for b in range(self.batch.B)]
            extensions()[3].point_cloud(s.poses, s.patches, s.intrinsics, F, ns, s.points)
        return target, weight

    def map(self, stream=None):
        """demo.py:53-54's arrays of one stream, read-only views: (points [n M, 3] fp32, colors [n M, 3] uint8), the
        points of the last step and the colours of the ingested frames.  In a batch, `stream` names the stream."""
        s = self._stream_state(stream, "map")
        if getattr(s, "points", None) is None or getattr(s, "colors", None) is None:
            raise RuntimeError("map: this state has no map buffers (make_state(map=True) / StreamBatch(map=True))")
        m = s.n * self.M
        return s.points[:m], s.colors.view(-1, 3)[:m]

    # ----------------------------------------------------------------------------- CUDA graph
    def capture(self):
        """Record one update() -- ~38 kernel launches, two memsets, no host decisions -- into a CUDA graph.
        Every buffer the step touches is persistent (state, ring buffers, corr rows) or comes from the graph's
        private pool, and the recurrent state is updated in place, so replaying the graph IS the next update."""
        if self.timers is not None:
            raise RuntimeError("capture(): event timers cannot be recorded inside a graph")
        if self.loop is not None:
            # one graph over the normal slots, one over the whole store; step_graph picks by the loop record
            self._loop_graphs = {}
            for mode in (False, True):
                self._loop_graphs[mode] = (self._capture(lambda: self.step(loop_edges=mode)), self._graph_out)
            self.graph = self._loop_graphs[False][0]
            return self.graph
        return self._capture(self.step)

    def _capture(self, fn):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                      # warm-up off the capture: lazy inits, attribute calls
            for _ in range(2):
                fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._graph_out = fn()
        return self.graph

    def step_graph(self):
        if self.loop is not None:
            # the global bundle adjustment is eager (dense solve); every other frame replays one of the two graphs
            rec = self.loop.read_flags(self.s.n)
            loop_edges, long_range, _, _ = rec
            if long_range and self.s.n not in self.loop.ran_global_ba:
                return self.step(loop_record=rec)            # the record already read: one D2H for the frame
            g, out = self._loop_graphs[bool(loop_edges)]
            g.replay()
            return out
        self.graph.replay()
        return self._graph_out

    # ----------------------------------------------------------------- end to end (host buffers)
    def _stream_state(self, stream, what):
        """the single-stream state a per-frame call writes: the state itself, or stream `stream` of a batch"""
        if self.batch is None:
            if stream is not None:
                raise RuntimeError("%s: stream=%s given, but this UpdateRunner holds one stream" % (what, stream))
            return self.s
        if stream is None:
            raise RuntimeError("%s: this UpdateRunner holds %d streams; say which with stream=b" % (what, self.batch.B))
        return self.batch.stream(stream)

    def make_host_frame(self, seed=0, stream=None):
        """pinned host copies of everything DPVO.__call__ writes for one new frame"""
        s = self._stream_state(stream, "make_host_frame")
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

    def ingest_frame(self, hf, stream=None):
        """H2D of one frame into ring slot n-1 (channels-last buffers take the host layout as is); in a batch, into
        stream `stream`'s slots (its own n)."""
        s = self._stream_state(stream, "ingest_frame")
        slot = (s.n - 1) % self.mem
        pslot = (s.n - 1) % self.pmem
        s.fmap1[0, slot].permute(1, 2, 0).copy_(hf["fmap1"], non_blocking=True)
        s.fmap2[0, slot].permute(1, 2, 0).copy_(hf["fmap2"], non_blocking=True)
        s.gmap[0, pslot * self.M:(pslot + 1) * self.M].permute(0, 2, 3, 1).copy_(hf["gmap"], non_blocking=True)
        s.imap[0, pslot * self.M:(pslot + 1) * self.M].copy_(hf["imap"], non_blocking=True)
        s.patches[(s.n - 1) * self.M:s.n * self.M].copy_(hf["patches"], non_blocking=True)
        s.poses[s.n - 1].copy_(hf["pose"], non_blocking=True)
        return sum(v.numel() * v.element_size() for v in hf.values())

    def _prepare(self, images, cameras):
        """the raw images [B', 3, H, W] prepared by their cameras (camera.undistort_frames) into a buffer the runner
        keeps, as [B', 3, h, w] views of HWC storage.  The buffer grows and is kept, like the encoder workspace, so a call
        with coords and depth given can be captured (a graph captured before a call that grows it must be captured
        again)."""
        h, w = cameras[0].size
        nb = len(cameras) * h * w * 3
        buf = getattr(self, "_prepared", None)
        if buf is None or buf.numel() < nb or buf.device != images.device:
            self._prepared = buf = torch.empty(nb, dtype=torch.uint8, device=images.device)
        out = buf[:nb].view(len(cameras), h, w, 3)
        return undistort_frames(images, cameras, out).permute(0, 3, 1, 2)

    @torch.no_grad()
    def ingest_image(self, image, depth=None, coords=None, stream=None, camera=None):
        """Encode a uint8 camera image [3, H, W] (CHW or HWC strides) straight into the slots `ingest_frame` writes:
        fmap1 / fmap2 slot (n-1) % mem, gmap / imap slot (n-1) % pmem, patches[(n-1) M : n M] (dpvo.py:389-438), and
        colors[n-1] (dpvo.py:404) when the state has map buffers.
        Centroids are drawn as Patchifier.forward draws them, unless `coords` [M, 2] is given (CUDA-graph capture);
        the patch depths are then one torch.rand draw (dpvo.py:427), or `depth` (the median the caller computes once
        initialised, dpvo.py:429-431).  Poses, intrinsics and the motion model stay with the caller.  In a batch,
        `stream` names the stream whose slots (at its own n) receive the frame.  Returns the centroids.
        With a `camera` (camera.Camera), `image` is the raw camera image: it is first prepared on the device
        (undistorted, halved if the camera says so, cropped) and the prepared image is encoded, centroids and colours
        included; intrinsics[n-1] is then set to camera.intrinsics / 4 (dpvo.py:401)."""
        if self.encoder is None:
            raise RuntimeError("ingest_image: this UpdateRunner was built without an encoder")
        s, M = self._stream_state(stream, "ingest_image"), self.M
        if camera is not None:
            if not isinstance(image, torch.Tensor) or image.dim() != 3:
                raise RuntimeError("ingest_image: the raw image must be a uint8 tensor [3, H, W]")
            image = self._prepare(image[None], [camera])[0]
        h, w = s.fmap1.shape[3], s.fmap1.shape[4]
        if image.dim() != 3 or encoder_output_size(image.shape[1], image.shape[2]) != (h, w):
            raise RuntimeError("ingest_image: a %s image encodes to %s features, the rings hold %dx%d"
                               % (tuple(image.shape), encoder_output_size(*image.shape[-2:]) if image.dim() >= 2 else None, h, w))
        slot = (s.n - 1) % self.mem
        pslot = (s.n - 1) % self.pmem
        patches = s.patches[(s.n - 1) * M:s.n * M]
        coords = self.encoder.encode_into(image, M, self.encoder.strategy, s.fmap1[0, slot].permute(1, 2, 0),
                                          s.fmap2[0, slot].permute(1, 2, 0),
                                          s.gmap[0, pslot * M:(pslot + 1) * M].permute(0, 2, 3, 1),
                                          s.imap[0, pslot * M:(pslot + 1) * M], patches, coords=coords,
                                          colors_slot=None if getattr(s, "colors", None) is None else s.colors[s.n - 1])
        if depth is None:
            depth = torch.rand(M, 1, 1, device=patches.device, dtype=patches.dtype)
        patches[:, 2] = depth
        if camera is not None:
            s.intrinsics.view(-1, 4)[s.n - 1].copy_(camera.ring_intrinsics(patches.device))
        return coords

    @torch.no_grad()
    def ingest_images(self, images, depth=None, coords=None, streams=None, cameras=None):
        """Encode the images of several streams of a batch in one pass of the encoders: uint8 [B', 3, H, W] (or the
        permuted [B', H, W, 3] view), image i into stream streams[i]'s slots at that stream's own n -- the slots
        `ingest_image(images[i], stream=streams[i])` writes, with the same bytes.  `streams` lists B' distinct streams
        (default: all B, in order), so a rig where a camera dropped a frame passes the others.
        Without `coords` [B', M, 2] and `depth` (fp32, broadcastable to [B', M]) the CUDA generator is drawn as those
        ingest_image calls draw it, image by image: centroid x, centroid y, then the depths.  With both given nothing
        is drawn and the call can be captured in a CUDA graph.  Returns the centroids [B', M, 2].
        With `cameras` (B' camera.Camera sharing raw size, half and crop), the images are raw camera images: one launch
        prepares all of them, the prepared images are encoded, and each stream's intrinsics[n-1] is set to its camera's
        intrinsics / 4 -- what `ingest_image(images[i], stream=streams[i], camera=cameras[i])` does."""
        if self.batch is None:
            raise RuntimeError("ingest_images: this UpdateRunner holds one stream; use ingest_image")
        if self.encoder is None:
            raise RuntimeError("ingest_images: this UpdateRunner was built without an encoder")
        batch, M = self.batch, self.M
        if not (isinstance(images, torch.Tensor) and images.is_cuda):
            raise RuntimeError("ingest_images: the images must be a CUDA tensor (there is no CPU path)")
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[1] != 3:
            raise RuntimeError("ingest_images: the images must be uint8 [B', 3, H, W], got %s %s" % (images.dtype, tuple(images.shape)))
        n = images.shape[0]
        streams = list(range(batch.B)) if streams is None else [int(b) for b in streams]
        if len(streams) != n:
            raise RuntimeError("ingest_images: %d images for %d streams %s" % (n, len(streams), streams))
        if len(set(streams)) != n:
            raise RuntimeError("ingest_images: streams %s name a stream twice" % streams)
        bad = [b for b in streams if not 0 <= b < batch.B]
        if bad:
            raise RuntimeError("ingest_images: streams %s outside the batch of %d" % (bad, batch.B))
        if cameras is not None:
            cameras = list(cameras)
            if len(cameras) != n:
                raise RuntimeError("ingest_images: %d cameras for %d images" % (len(cameras), n))
            images = self._prepare(images, cameras)
        h, w = batch.fmap1.shape[3], batch.fmap1.shape[4]
        if encoder_output_size(images.shape[2], images.shape[3]) != (h, w):
            raise RuntimeError("ingest_images: a %s image encodes to %s features, the rings hold %dx%d"
                               % (tuple(images.shape[1:]), encoder_output_size(*images.shape[-2:]), h, w))
        empty = [b for b in streams if batch.stream(b).n < 1]
        if empty:
            raise RuntimeError("ingest_images: streams %s have no frame slot yet (n = 0)" % empty)
        dev = batch.patches.device
        if coords is None or depth is None:
            drawn_c, drawn_d = [], []
            for i in range(n):                                      # ingest_image's order, image by image
                if coords is None:
                    drawn_c.append(self.encoder.centroids(images[i], M, self.encoder.strategy))
                if depth is None:
                    drawn_d.append(torch.rand(M, 1, 1, device=dev, dtype=batch.patches.dtype))
            coords = torch.stack(drawn_c) if coords is None else coords
            depth = torch.stack(drawn_d).view(n, M) if depth is None else depth
        depth = torch.broadcast_to(torch.as_tensor(depth, device=dev, dtype=torch.float32), (n, M)).contiguous()
        rows = [batch.frame_rows(b) for b in streams]
        coords = self.encoder.encode_frames_into(images, M, self.encoder.strategy, batch.fmap1[0].permute(0, 2, 3, 1),
                                                 batch.fmap2[0].permute(0, 2, 3, 1), batch.gmap[0].permute(0, 2, 3, 1),
                                                 batch.imap[0], batch.patches, [r[0] for r in rows], [r[1] for r in rows],
                                                 [r[2] for r in rows], coords=coords, depth=depth,
                                                 colors_ring=getattr(batch, "colors", None))
        if cameras is not None:
            for b, cam in zip(streams, cameras):
                s = batch.stream(b)
                s.intrinsics[s.n - 1].copy_(cam.ring_intrinsics(dev))
        return coords

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
