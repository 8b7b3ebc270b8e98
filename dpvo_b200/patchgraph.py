"""Device-resident patch graph: fixed-capacity edge arrays + per-edge recurrent state (csrc/pgraph.cu).

The reference's patch graph (dpvo/patchgraph.py:26-35 ii / jj / kk / net, dpvo/dpvo.py:215-238 append_factors /
remove_factors, :266-310 keyframe) grows and shrinks every frame with torch.cat and boolean-mask indexing, which costs
host synchronisations and changes tensor shapes -- a captured CUDA graph of update() cannot follow it.  Here the arrays
have a fixed capacity; a slot holds an active edge or a parked dummy edge that points at a reserved frame / patch and so
lives in groups of its own in every grouping of the update operator.  Removal parks slots in place, append fills parked
slots in index order and zeroes the state rows of the new edges; all decisions read device scalars.
"""
import torch

from . import extensions
from .net import DIM


class DevicePatchGraph:
    def __init__(self, capacity, M, dummy_frame, device="cuda", loop_pairs=0, inactive_capacity=0):
        """capacity: edge slots (rounded up to a multiple of 128); dummy_frame: a frame slot no real edge ever uses (its
        pose / intrinsics / patches must be valid data, e.g. the last slot of the pose buffer).
        loop_pairs > 0 adds a loop region of loop_pairs * M slots (rounded up to a multiple of 128) after the normal
        ones, where loop.LoopClosure writes the edges of accepted loop pairs, and inactive_capacity slots of an inactive
        edge store directly BEFORE the store (ii / jj / kk and the fp32 `target` / `weight` [1, cap, 2] rows the
        runner keeps per slot), so that the used inactive edges and the active store form one edge list."""
        self.normal_cap = (int(capacity) + 127) // 128 * 128
        self.loop_pairs = int(loop_pairs)
        self.M = int(M)
        self.loop_region = (self.loop_pairs * self.M + 127) // 128 * 128
        self.cap = self.normal_cap + self.loop_region
        self.inactive_cap = int(inactive_capacity)
        self.dummy_frame = int(dummy_frame)
        self.dummy_patch = self.dummy_frame * self.M
        dev = torch.device(device)
        full = self.inactive_cap + self.cap
        self.ii_all = torch.full((full,), self.dummy_frame, dtype=torch.long, device=dev)
        self.jj_all = torch.full((full,), self.dummy_frame, dtype=torch.long, device=dev)
        self.kk_all = torch.full((full,), self.dummy_patch, dtype=torch.long, device=dev)
        a = self.inactive_cap
        self.ii, self.jj, self.kk = self.ii_all[a:], self.jj_all[a:], self.kk_all[a:]
        if self.loop_pairs > 0 or self.inactive_cap > 0:
            self.target_all = torch.zeros(1, full, 2, device=dev)
            self.weight_all = torch.zeros(1, full, 2, device=dev)
            self.target, self.weight = self.target_all[:, a:], self.weight_all[:, a:]
        self.active = torch.zeros(self.cap, dtype=torch.uint8, device=dev)
        self.n_active = torch.zeros(1, dtype=torch.int32, device=dev)
        self.overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        self.net = torch.zeros(1, self.cap, DIM, device=dev)                  # the recurrent state `net` (dpvo.py:53), fp32

    @classmethod
    def stacked(cls, B, capacity, M, dummy_frames, device="cuda"):
        """One store for the B streams of a streams.StreamBatch: B slices of `capacity` slots (rounded up to a multiple of
        128) in stream order, and B per-stream graphs whose arrays and recurrent state are views of their slice.
        dummy_frames[b] is stream b's reserved frame in global numbering (e.g. its last pose slot, b F + F - 1): its
        parked slots point there, so they stay inside stream b's frames and rings.  Appends and removals go through the
        per-stream graphs, with global frame numbers, and touch only that slice -- removing a keyframe renumbers only
        that stream's edges; UpdateRunner steps the whole store.  Returns (store, [graph of stream b])."""
        dummy_frames = [int(f) for f in dummy_frames]
        if len(dummy_frames) != int(B):
            raise ValueError("DevicePatchGraph.stacked: one dummy frame per stream")
        cap = (int(capacity) + 127) // 128 * 128
        store = cls(B * cap, M, dummy_frames[0], device)
        store.dummy_frame = store.dummy_patch = None            # per stream: see store.streams
        store.n_active = store.overflow = None
        store.streams = []
        for b, f in enumerate(dummy_frames):
            sl = slice(b * cap, (b + 1) * cap)
            store.ii[sl] = f
            store.jj[sl] = f
            store.kk[sl] = f * store.M
            g = cls.__new__(cls)
            g.normal_cap, g.loop_pairs, g.loop_region, g.inactive_cap = cap, 0, 0, 0
            g.cap, g.M, g.dummy_frame, g.dummy_patch = cap, store.M, f, f * store.M
            g.ii, g.jj, g.kk, g.active = store.ii[sl], store.jj[sl], store.kk[sl], store.active[sl]
            g.net = store.net[:, sl]
            g.n_active = torch.zeros(1, dtype=torch.int32, device=store.ii.device)
            g.overflow = torch.zeros(1, dtype=torch.int32, device=store.ii.device)
            store.streams.append(g)
        return store, store.streams

    def _per_stream(self, what):
        if self.dummy_frame is None:
            raise RuntimeError("DevicePatchGraph.%s: a stacked store changes through its per-stream graphs (store.streams)" % what)

    def _normal_rule(self, what):
        # the loop region is written by LoopClosure.propose and emptied by LoopClosure.remove; keyframe renumbering
        # (remove_frame) runs over the whole store, loop region included
        if what == "remove_old" and self.loop_pairs > 0:
            raise RuntimeError("DevicePatchGraph.remove_old: a graph with a loop region removes through LoopClosure.remove")

    # -------------------------------------------------------------------------------- dpvo.py:215-222
    def append(self, ii, jj, kk, enable=None):
        """add edges (ii = source frame, jj = target frame, kk = patch); their state rows start at zero.
        Returns the slot of every new edge (int32, -1 = store full, `overflow` is then set).  With a loop region, the
        edges go to the normal slots only."""
        self._per_stream("append")
        n = self.normal_cap
        return extensions()[3].pgraph_append(self.ii[:n], self.jj[:n], self.kk[:n], self.active[:n], ii, jj, kk, enable,
                                             self.net[0, :n], self.n_active, self.overflow)

    def append_frame_edges(self, n_dev, lifetime, enable=None):
        """the forward + backward edges of the newest frame n - 1 (dpvo.py:457-459 with :362-375), n on the device"""
        ii, jj, kk = extensions()[3].pgraph_new_edges(n_dev, self.M, lifetime)
        return self.append(ii, jj, kk, enable)

    # -------------------------------------------------------------------------------- dpvo.py:224-238, 300-306
    def remove_old(self, n_dev, window, enable=None):
        """park the edges whose patch left the removal window: ix[kk] < n - window"""
        self._per_stream("remove_old")
        self._normal_rule("remove_old")
        extensions()[3].pgraph_remove(self.ii, self.jj, self.kk, self.active, 0, n_dev, int(window), enable,
                                      self.dummy_frame, self.dummy_patch, self.M, self.n_active)

    # -------------------------------------------------------------------------------- dpvo.py:279-286
    def remove_frame(self, k_dev, enable=None):
        """keyframe removal: park the edges that touch frame k and renumber frames / patches above it"""
        self._per_stream("remove_frame")
        self._normal_rule("remove_frame")
        extensions()[3].pgraph_remove(self.ii, self.jj, self.kk, self.active, 1, k_dev, 0, enable,
                                      self.dummy_frame, self.dummy_patch, self.M, self.n_active)

    # -------------------------------------------------------------------------------- host-side views (synchronise)
    def edges(self):
        m = self.active.bool()
        return self.ii[m], self.jj[m], self.kk[m]

    def net_rows(self):
        """[cap, 384] view of the recurrent state"""
        return self.net[0]
