"""Several camera streams stepped together on one GPU: the stacked state that UpdateRunner(StreamBatch) updates with one
launch per kernel for all streams.

B streams share one configuration (M, image size, ring sizes `mem` / `pmem`, dtype) and keep their own poses,
intrinsics, patches, feature rings and edges.  Stream b owns

    frames   [b F, (b+1) F)                 of poses [B F, 7] and intrinsics [B F, 4]   (F = frames_per_stream)
    patches  [b F M, (b+1) F M)             of patches [B F M, 3, 3, 3]
    ring rows [b mem, (b+1) mem)            of fmap1 [1, B mem, 128, h, w] and fmap2 [1, B mem, 128, h/4, w/4]
    ring rows [b pmem M, (b+1) pmem M)      of gmap [1, B pmem M, 128, 3, 3] and imap [1, B pmem M, 384]
    with map=True also
    patches  [b F M, (b+1) F M)             of points [B F M, 3]   (fp32 world points, pg.points_'s layout)
    frames   [b F, (b+1) F)                 of colors [B F, M, 3]  (uint8 viewer colours, pg.colors_'s layout)

Every tensor has the single-stream layout (feature maps channels-last).  Edges carry global frame / patch numbers, so
every per-edge and per-group kernel of the update sees one graph; no edge may join two streams.  `stream(b)` is a
SyntheticState whose tensors are views of stream b's rows, holding that stream's LOCAL edge lists and its frame counter
`n` and window start `t0`: the per-frame bookkeeping of one stream works on it exactly as on a single state.
"""
import torch

from .synthetic import SyntheticState

MAX_FREE_POSES = 32            # the on-chip bundle adjustment solve holds up to 32 free poses per window
MAX_STREAMS = 64


class StreamBatch:
    def __init__(self, B, cfg, frames_per_stream, mem, pmem=None, device="cuda", dtype=torch.half, map=False):
        B, F, mem = int(B), int(frames_per_stream), int(mem)
        pmem = mem if pmem is None else int(pmem)
        if not 1 <= B <= MAX_STREAMS:
            raise ValueError("StreamBatch: %d streams, 1 to %d supported" % (B, MAX_STREAMS))
        if F < 2 or mem < 1 or pmem < 1:
            raise ValueError("StreamBatch: frames_per_stream >= 2 and ring sizes >= 1 needed")
        self.B, self.F, self.mem, self.pmem = B, F, mem, pmem
        self.cfg = dict(cfg)
        self.M = M = int(cfg["M"])
        self.ht, self.wd = int(cfg["ht"]), int(cfg["wd"])
        h, w = self.ht // 4, self.wd // 4
        dev = torch.device(device)
        self.poses = torch.zeros(B * F, 7, device=dev)
        self.poses[:, 6] = 1.0
        self.patches = torch.zeros(B * F * M, 3, 3, 3, device=dev)
        self.intrinsics = torch.zeros(B * F, 4, device=dev)
        # channels-last storage, logical NCHW (synthetic.make_state's layout)
        self.fmap1 = torch.zeros(1, B * mem, h, w, 128, device=dev, dtype=dtype).permute(0, 1, 4, 2, 3)
        self.fmap2 = torch.zeros(1, B * mem, h // 4, w // 4, 128, device=dev, dtype=dtype).permute(0, 1, 4, 2, 3)
        self.gmap = torch.zeros(1, B * pmem * M, 3, 3, 128, device=dev, dtype=dtype).permute(0, 1, 4, 2, 3)
        self.imap = torch.zeros(1, B * pmem * M, 384, device=dev, dtype=dtype)
        self.points = torch.zeros(B * F * M, 3, device=dev) if map else None
        self.colors = torch.zeros(B * F, M, 3, dtype=torch.uint8, device=dev) if map else None
        z = torch.zeros(0, dtype=torch.long, device=dev)
        self._streams = []
        for b in range(B):
            fs, ps = slice(b * F, (b + 1) * F), slice(b * F * M, (b + 1) * F * M)
            rs, gs = slice(b * mem, (b + 1) * mem), slice(b * pmem * M, (b + 1) * pmem * M)
            self._streams.append(SyntheticState(cfg=self.cfg, n=0, t0=0, ii=z, jj=z, kk=z, poses=self.poses[fs],
                                                patches=self.patches[ps], intrinsics=self.intrinsics[fs],
                                                fmap1=self.fmap1[:, rs], fmap2=self.fmap2[:, rs], gmap=self.gmap[:, gs],
                                                imap=self.imap[:, gs],
                                                points=self.points[ps] if map else None,
                                                colors=self.colors[fs] if map else None))
        self.ii, self.jj, self.kk = z, z, z

    # ------------------------------------------------------------------------------------------------ streams
    def stream(self, b):
        """stream b as a single-stream state: views of its rows, its local edges, its `n` and `t0`"""
        if not 0 <= int(b) < self.B:
            raise IndexError("stream %d of a batch of %d" % (b, self.B))
        return self._streams[int(b)]

    def load(self, b, state):
        """copy a single-stream state (its poses, patches, intrinsics, feature rings, edges, n and t0) into stream b; in a
        batch with map buffers also its points and colours (zeros where the state has none)"""
        s = self.stream(b)
        if self.points is not None:
            from .synthetic import check_map
            check_map(state, "StreamBatch.load")
        if int(state.cfg["M"]) != self.M or (int(state.cfg["ht"]), int(state.cfg["wd"])) != (self.ht, self.wd):
            raise ValueError("StreamBatch.load: stream %d has M=%s and a %sx%s image, the batch M=%d and %dx%d: one "
                             "configuration and one image size per batch" % (b, state.cfg["M"], state.cfg["ht"],
                                                                              state.cfg["wd"], self.M, self.ht, self.wd))
        mine = {k: v for k, v in self.cfg.items() if k != "intrinsics"}          # cameras may differ per stream
        theirs = {k: v for k, v in state.cfg.items() if k != "intrinsics"}
        if mine != theirs:
            raise ValueError("StreamBatch.load: stream %d's configuration %s differs from the batch's %s" % (b, theirs, mine))
        for name in ("fmap1", "fmap2", "gmap", "imap"):
            src, dst = getattr(state, name), getattr(s, name)
            if src is None or tuple(src.shape) != tuple(dst.shape) or src.dtype != dst.dtype:
                raise ValueError("StreamBatch.load: %s of stream %d is %s %s, the batch holds %s %s per stream" % (
                    name, b, None if src is None else tuple(src.shape), None if src is None else src.dtype,
                    tuple(dst.shape), dst.dtype))
            dst.copy_(src)
        if state.poses.shape[0] > self.F:
            raise ValueError("StreamBatch.load: %d pose slots > %d frames per stream" % (state.poses.shape[0], self.F))
        nf = state.poses.shape[0]
        s.poses[:nf].copy_(state.poses)
        s.patches[:nf * self.M].copy_(state.patches)
        s.intrinsics[:nf].copy_(state.intrinsics)
        if self.points is not None:
            for name, rows in (("points", nf * self.M), ("colors", nf)):
                src, dst = getattr(state, name), getattr(s, name)
                dst.zero_()
                if src is not None:
                    dst[:rows].copy_(src)
        s.ii, s.jj, s.kk = (t.to(self.poses.device) for t in (state.ii, state.jj, state.kk))
        s.n, s.t0 = int(state.n), int(state.t0)

    def copy_stream(self, b):
        """a standalone single-stream state equal to stream b (cloned tensors, same layouts)"""
        s = self.stream(b)
        return SyntheticState(cfg=dict(self.cfg), n=s.n, t0=s.t0, ii=s.ii.clone(), jj=s.jj.clone(), kk=s.kk.clone(),
                              poses=s.poses.clone(), patches=s.patches.clone(), intrinsics=s.intrinsics.clone(),
                              fmap1=s.fmap1.clone(), fmap2=s.fmap2.clone(), gmap=s.gmap.clone(), imap=s.imap.clone(),
                              points=None if s.points is None else s.points.clone(),
                              colors=None if s.colors is None else s.colors.clone())

    # ------------------------------------------------------------------------------------------------ index maps
    def to_global(self, b, ii=None, jj=None, kk=None):
        """stream b's local frame / patch numbers -> the batch's: ii + b F, jj + b F, kk + b F M"""
        f0, k0 = int(b) * self.F, int(b) * self.F * self.M
        return (None if ii is None else ii + f0, None if jj is None else jj + f0, None if kk is None else kk + k0)

    def to_local(self, ii=None, jj=None, kk=None):
        """global numbers -> (stream, local number) for each list given"""
        out = []
        for x, per in ((ii, self.F), (jj, self.F), (kk, self.F * self.M)):
            out.append(None if x is None else (torch.div(x, per, rounding_mode="floor"), torch.remainder(x, per)))
        return tuple(out)

    def ring_rows(self, kk, jj):
        """ring rows of global patches kk (gmap / imap) and global frames jj (fmap1 / fmap2): stream b's rings start at
        b pmem M and b mem, and within them a patch / frame takes the slot a single stream gives it:
            kk_ring = b pmem M + (kk_local mod pmem M),   jj_ring = b mem + (jj_local mod mem)
        Elementwise device ops, no synchronisation (capturable)."""
        FM, PM = self.F * self.M, self.pmem * self.M
        bk = torch.div(kk, FM, rounding_mode="floor")
        bj = torch.div(jj, self.F, rounding_mode="floor")
        return bk * PM + torch.remainder(kk - bk * FM, PM), bj * self.mem + torch.remainder(jj - bj * self.F, self.mem)

    def frame_rows(self, b):
        """rows that stream b's newest frame (local n - 1) occupies in the stacked buffers: (fmap1 / fmap2 ring row,
        first gmap / imap ring row, first patch row).  Its M patch features and patches are the rows that follow."""
        s = self.stream(b)
        f = int(s.n) - 1
        return (int(b) * self.mem + f % self.mem, (int(b) * self.pmem + f % self.pmem) * self.M, (int(b) * self.F + f) * self.M)

    # ------------------------------------------------------------------------------------------------ edges, windows
    def check_edges(self, ii, jj, kk):
        """reject global edge lists with an edge outside the batch or joining two streams (one host synchronisation)"""
        if not (ii.shape == jj.shape == kk.shape and ii.dim() == 1):
            raise ValueError("StreamBatch: ii, jj, kk must be 1-D lists of one length")
        if ii.numel() == 0:
            return
        (si, _), (sj, _), (sk, _) = self.to_local(ii, jj, kk)
        bad_range = (si < 0) | (si >= self.B) | (sj < 0) | (sj >= self.B) | (sk < 0) | (sk >= self.B)
        bad_join = (si != sj) | (si != sk)
        if bool(bad_range.any()):
            e = int(torch.nonzero(bad_range)[0])
            raise ValueError("StreamBatch: edge %d (ii=%d, jj=%d, kk=%d) lies outside the %d streams' frames / patches" % (
                e, int(ii[e]), int(jj[e]), int(kk[e]), self.B))
        if bool(bad_join.any()):
            e = int(torch.nonzero(bad_join)[0])
            raise ValueError("StreamBatch: edge %d (ii=%d, jj=%d, kk=%d) joins streams %d, %d and %d: edges must stay "
                             "inside one stream" % (e, int(ii[e]), int(jj[e]), int(kk[e]), int(si[e]), int(sj[e]), int(sk[e])))

    def set_edges(self, ii=None, jj=None, kk=None):
        """the batch's edge lists.  Without arguments: every stream's local lists, offset to global numbers and
        concatenated in stream order.  With global lists: checked, then split into the streams' local lists (order kept)."""
        if ii is None:
            parts = [self.to_global(b, s.ii, s.jj, s.kk) for b, s in enumerate(self._streams)]
            ii, jj, kk = (torch.cat([p[i] for p in parts]) for i in range(3))
            self.check_edges(ii, jj, kk)
        else:
            ii, jj, kk = (t.to(device=self.poses.device, dtype=torch.long) for t in (ii, jj, kk))
            self.check_edges(ii, jj, kk)
            sk = torch.div(kk, self.F * self.M, rounding_mode="floor")
            for b, s in enumerate(self._streams):
                m = sk == b
                s.ii, s.jj, s.kk = ii[m] - b * self.F, jj[m] - b * self.F, kk[m] - b * self.F * self.M
        self.ii, self.jj, self.kk = ii, jj, kk

    @property
    def E(self):
        return self.ii.numel()

    def windows(self):
        """host lists (t0s, t1s) of the streams' bundle adjustment windows in global frame numbers: stream b optimises
        its frames [t0, n).  An empty window (t0 == n) leaves the stream untouched."""
        t0s, t1s = [], []
        for b, s in enumerate(self._streams):
            t0, n = int(s.t0), int(s.n)
            if not 0 <= t0 <= n <= self.F:
                raise ValueError("StreamBatch: stream %d's window [t0=%d, n=%d) is not inside its %d frames" % (b, t0, n, self.F))
            if n - t0 > MAX_FREE_POSES:
                raise ValueError("StreamBatch: stream %d has %d free poses, bundle adjustment holds up to %d" % (
                    b, n - t0, MAX_FREE_POSES))
            t0s.append(b * self.F + t0)
            t1s.append(b * self.F + n)
        return t0s, t1s
