"""Keyframe culling on the device (csrc/keyframe.cu): DPVO.keyframe's motion test, the frame shift, the record of every
culled frame's relative pose, and terminate()'s trajectory (dpvo/dpvo.py:166-198, 257-300, 400-444).

Every frame, after the update, `cull` decides on the device whether frame k = n - KEYFRAME_INDEX stays: when the mean
flow between its neighbours i = k - 1 and j = k + 1 is below KEYFRAME_THRESH, the edges touching k are parked and the
frames above it renumbered (DevicePatchGraph.remove_frame under the decision flag), the per-frame buffers and feature
rings of frames k + 1 .. n - 1 move down one slot, k's pose relative to k - 1 is recorded under its timestamp, and the
device frame counter drops by one.  Nothing waits for the host: `add_frame` + `cull` can be captured in a CUDA graph,
and `read` is the frame's one device-to-host copy.  For a streams.StreamBatch every call is one launch for all streams
(the edge renumbering: one remove_frame per stream), each stream deciding for itself.
"""
import torch

from . import extensions
from .synthetic import check_map

# the reference's defaults (dpvo/config.py: KEYFRAME_INDEX, KEYFRAME_THRESH)
KEYFRAME_DEFAULTS = dict(keyframe_index=4, keyframe_thresh=15.0)


class Keyframes:
    def __init__(self, cfg, state, graph, keyframe_index=None, keyframe_thresh=None, max_timestamps=4096, loop=None):
        """cfg: the stream configuration (synthetic.CONFIGS layout); keyframe_index / keyframe_thresh default to cfg's
        entries of those names, then to the reference's (4 and 15.0).  state: one stream's state (synthetic.SyntheticState
        layout) or a streams.StreamBatch; graph: its patchgraph.DevicePatchGraph (for a batch, the stacked store).
        max_timestamps: the delta table's size, the most input frames (kept, culled or skipped) a stream may see.
        loop: the loop.LoopClosure on the same graph, if any; it must use the same keyframe index, and its normalize
        then scales the recorded relative poses with the map.

        The frames the state holds already count as kept frames with timestamps 0 .. n - 1."""
        def param(name, given):
            return given if given is not None else cfg.get(name, KEYFRAME_DEFAULTS[name])

        check_map(state, "Keyframes")
        self.ki = int(param("keyframe_index", keyframe_index))
        self.thresh = float(param("keyframe_thresh", keyframe_thresh))
        if self.ki < 1:
            raise ValueError("Keyframes: keyframe_index=%d must be at least 1" % self.ki)
        if loop is None and graph.loop_pairs > 0:
            # its global bundle adjustment would leave the recorded relative poses unscaled
            raise ValueError("Keyframes: the graph has a loop region; pass its LoopClosure as loop=")
        if loop is not None and loop.pg is not graph:
            raise ValueError("Keyframes: the LoopClosure runs on another graph")
        if loop is not None and int(loop.kf_index) != self.ki:
            raise ValueError("Keyframes: keyframe_index=%d but the LoopClosure on this graph uses %d" % (self.ki, loop.kf_index))
        self.state, self.pg, self.loop = state, graph, loop
        self.batch = hasattr(state, "stream")
        if self.batch:
            self.B, self.F, self.M = state.B, state.F, state.M
            if getattr(graph, "streams", None) is None or len(graph.streams) != self.B:
                raise ValueError("Keyframes: a StreamBatch culls through its stacked store (DevicePatchGraph.stacked)")
            if graph.loop_pairs > 0:
                raise ValueError("Keyframes: loop closure runs on one stream, not on a batch")
            streams = [state.stream(b) for b in range(self.B)]
        else:
            self.B, self.F, self.M = 1, state.poses.shape[0], int(cfg["M"])
            if getattr(graph, "streams", None) is not None:
                raise ValueError("Keyframes: a stacked store belongs to a StreamBatch")
            streams = [state]
        if graph.M != self.M:
            raise ValueError("Keyframes: cfg M=%d but the graph holds M=%d" % (self.M, graph.M))
        self.T = int(max_timestamps)
        if self.T < self.F:
            raise ValueError("Keyframes: max_timestamps=%d is smaller than the %d frame slots" % (self.T, self.F))
        self.bufs, self.rows = [], []
        # colors: the viewer colours of a state with map buffers (dpvo.py:289); points are recomputed by the next update
        for name in ("poses", "patches", "intrinsics", "fmap1", "fmap2", "gmap", "imap", "colors"):
            t = getattr(state, name, None)
            if t is None:                                       # features=False, or no map
                continue
            rows = self.F
            if name in ("fmap1", "fmap2"):
                rows = t.shape[1] // self.B
            elif name in ("gmap", "imap"):
                rows = t.shape[1] // (self.B * self.M)
            if rows < self.ki:
                raise ValueError("Keyframes: the %s ring holds %d frames, fewer than keyframe_index=%d" % (name, rows, self.ki))
            self.bufs.append(t)
            self.rows.append(rows)
        dev = state.poses.device
        B, T = self.B, self.T
        n0 = [int(s.n) for s in streams]
        self.n_dev = torch.tensor(n0, dtype=torch.long, device=dev)
        self.tstamp = torch.zeros(B, self.F, dtype=torch.long, device=dev)
        for b, n in enumerate(n0):
            self.tstamp[b, :n] = torch.arange(n, device=dev)
        self.bufs.append(self.tstamp)
        self.rows.append(self.F)
        self.counter = torch.tensor(n0, dtype=torch.long, device=dev)
        self.delta = torch.zeros(B, T, 7, device=dev)
        self.delta[..., 6] = 1.0
        self.delta_src = torch.full((B, T), -1, dtype=torch.long, device=dev)
        # the per-frame record, one buffer so that read() is one copy: flag int32 [B], overflow int32 [B], k int64 [B],
        # m fp64 [B]
        self._rec = torch.zeros(24 * B, dtype=torch.uint8, device=dev)
        self.flag = self._rec[:4 * B].view(torch.int32)
        self.overflow = self._rec[4 * B:8 * B].view(torch.int32)
        self.k = self._rec[8 * B:16 * B].view(torch.long)
        self.m = self._rec[16 * B:24 * B].view(torch.float64)
        self._streams = streams
        if loop is not None:
            loop.keyframes = self                               # its global bundle adjustment scales self.delta

    # ------------------------------------------------------------------------ dpvo.py:400, 440-444
    def add_frame(self):
        """tstamp[n - 1] = counter, counter += 1 for every stream, n read from n_dev (the caller has counted the new
        frame in n_dev); capturable"""
        extensions()[3].keyframe_count(0, self.n_dev, self.tstamp, self.F, self.counter, self.delta, self.delta_src, self.overflow)

    def skip_frame(self):
        """a frame dropped before initialisation (dpvo.py:441-444): delta[c] = (c - 1, identity), counter += 1"""
        extensions()[3].keyframe_count(1, self.n_dev, self.tstamp, self.F, self.counter, self.delta, self.delta_src, self.overflow)

    # ------------------------------------------------------------------------ dpvo.py:257-300
    def cull(self):
        """the keyframe decision of every stream, and under it the edge removal and renumbering, the shift of every
        buffer, the delta record and n_dev -= 1; capturable.  Call it after the frame's update and before the window
        removal (remove_old / LoopClosure.remove with n_dev), as dpvo.py:266-310 orders them."""
        ex = extensions()[3]
        g = self.pg
        st = self.state
        ex.keyframe_motion(st.poses, st.patches, st.intrinsics, self.F, g.ii, g.jj, g.kk, g.active, self.n_dev, self.tstamp,
                           self.delta, self.delta_src, self.ki, self.thresh, self.flag, self.k, self.m, self.overflow)
        if self.batch:
            for b, gb in enumerate(g.streams):
                gb.remove_frame(self.k[b:b + 1], enable=self.flag[b:b + 1])
        else:
            g.remove_frame(self.k, enable=self.flag)
        ex.keyframe_shift(self.bufs, self.rows, self.F, self.ki, self.flag, self.k)

    def read(self):
        """the frame's one device-to-host copy: [(removed, m)] per stream.  The host frame count `n` of every stream that
        lost a frame drops by one, as n_dev did on the device, before an overflow of the delta table is raised."""
        rec = self._rec.cpu()
        B = self.B
        flag = rec[:4 * B].view(torch.int32).tolist()
        over = rec[4 * B:8 * B].view(torch.int32).tolist()
        m = rec[16 * B:24 * B].view(torch.float64).tolist()
        for b in range(B):
            if flag[b]:
                self._streams[b].n -= 1
        if any(over):
            raise RuntimeError("Keyframes: a timestamp of stream(s) %s reached max_timestamps=%d"
                               % ([b for b in range(B) if over[b]], self.T))
        return [(bool(f), v) for f, v in zip(flag, m)]

    # ------------------------------------------------------------------------ dpvo.py:166-198
    def trajectory(self, stream=None):
        """terminate()'s poses: [counter, 7] fp32 on the device, pose(t)^-1 for every timestamp t (a live keyframe's pose,
        else dP_t pose(src_t) along the delta chain).  stream: which one of a batch (required for B > 1)."""
        if stream is None:
            if self.B > 1:
                raise ValueError("Keyframes.trajectory: say which stream of the batch")
            stream = 0
        err = torch.zeros(self.B, dtype=torch.int32, device=self.n_dev.device)
        out = extensions()[3].keyframe_trajectory(self.state.poses, self.tstamp, self.n_dev, self.F, self.delta, self.delta_src,
                                                  self.counter, err)
        if int(self.overflow[stream].item()):
            raise RuntimeError("Keyframes.trajectory: stream %d saw more than max_timestamps=%d frames" % (stream, self.T))
        if int(err[stream].item()):
            raise RuntimeError("Keyframes.trajectory: a timestamp of stream %d has neither a live keyframe nor a recorded "
                               "delta" % stream)
        c = int(self.counter[stream].item())
        return out[stream, :c]
