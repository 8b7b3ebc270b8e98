"""Proximity loop closure on the device-resident patch graph (csrc/loop.cu): the DPV-SLAM back end of the reference
(LOOP_CLOSURE=True, dpvo/config.py:28-31).

Every frame whose n - last_global_ba >= GLOBAL_OPT_FREQ, `propose` scores every (old frame i, recent frame j) pair by
the mean flow of frame i's patch centres (PatchGraph.edges_loop, dpvo/patchgraph.py:56-82), greedily accepts the pairs
below BACKEND_THRESH (reduce_edges) and writes their M edges each into the graph's loop region.  `remove` is keyframe()'s
window removal with the loop exception, and it keeps the removed edges in an inactive store (remove_factors(store=True),
dpvo/dpvo.py:223-238, 300-310).  `global_ba` normalizes the map and runs the wide bundle adjustment over the inactive and
the active edges (__run_global_BA, dpvo.py:312-326), which runner.UpdateRunner calls in place of the local one when the
condition of dpvo.py:348 holds.  Every call but global_ba reads the frame counter from a device scalar and can be
captured in a CUDA graph.
"""
import torch

from . import extensions
from . import fastba

# the reference's defaults (dpvo/config.py:16, 29-31)
LOOP_DEFAULTS = dict(backend_thresh=64.0, max_edge_age=1000, global_opt_freq=15, keyframe_index=4)


class LoopClosure:
    def __init__(self, cfg, graph, backend_thresh=None, max_edge_age=None, global_opt_freq=None, keyframe_index=None):
        """cfg: the stream's configuration (synthetic.CONFIGS layout: M, removal, opt_window); the loop parameters
        default to cfg's entries of the same names, then to the reference's defaults.  graph: a patchgraph.DevicePatchGraph
        built with loop_pairs > 0 (the most pairs one proposal accepts, 1,000 in the reference) and an inactive store
        (inactive_capacity > 0)."""
        if graph.loop_pairs <= 0 or graph.inactive_cap <= 0:
            raise ValueError("LoopClosure: the graph needs a loop region (loop_pairs > 0) and an inactive store (inactive_capacity > 0)")
        if getattr(graph, "streams", None) is not None:
            raise ValueError("LoopClosure: loop closure runs on one stream's graph, not a stacked store")

        def param(name, given):
            return given if given is not None else cfg.get(name, LOOP_DEFAULTS[name])

        self.pg = graph
        self.M = int(cfg["M"])
        if self.M != graph.M:
            raise ValueError("LoopClosure: cfg M=%d but the graph holds M=%d" % (self.M, graph.M))
        self.removal = int(cfg["removal"])
        self.opt_window = int(cfg["opt_window"])
        self.thresh = float(param("backend_thresh", backend_thresh))
        self.max_age = int(param("max_edge_age", max_edge_age))
        self.freq = int(param("global_opt_freq", global_opt_freq))
        self.kf_index = int(param("keyframe_index", keyframe_index))
        if self.opt_window > self.freq + self.kf_index:
            # a loop edge of frame n0 has j <= n0 - kf_index - 1; the next proposal comes at n >= n0 + freq, after the
            # removal at n - 1 has parked every loop edge with j <= n - 1 - opt_window.  With a wider optimisation window
            # a proposal could find loop edges still active in the region it writes
            raise ValueError("LoopClosure: opt_window=%d exceeds global_opt_freq + keyframe_index = %d: loop edges would "
                             "still be active at the next proposal" % (self.opt_window, self.freq + self.kf_index))
        self.pairs_cap = graph.loop_pairs
        dev = graph.ii.device
        a = graph.inactive_cap
        # the inactive store: the first `inactive_cap` entries of the graph's buffers, filled from the end
        self.s_ii, self.s_jj, self.s_kk = graph.ii_all[:a], graph.jj_all[:a], graph.kk_all[:a]
        self.s_target, self.s_weight = graph.target_all[:, :a], graph.weight_all[:, :a]
        self.s_count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.s_overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        self.last_global_ba = torch.full((1,), -1000, dtype=torch.long, device=dev)     # dpvo.py:60
        self.pairs = torch.zeros(self.pairs_cap, 2, dtype=torch.long, device=dev)
        self.n_pairs = torch.zeros(1, dtype=torch.int32, device=dev)
        self.region_overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        self.flags = torch.zeros(4, dtype=torch.long, device=dev)
        self.ran_global_ba = set()                                                     # dpvo.py:42, host side
        self.scores = None
        self.keyframes = None                                                          # keyframe.Keyframes, if one culls

    # ------------------------------------------------------------------------ dpvo.py:449-455 + patchgraph.py:56-82
    def candidates(self):
        """(J, max_age): the layout of `scores`, slot (j - (n - freq)) * max_age + (i - max(n - removal - max_age, 0))"""
        return self.freq - self.kf_index, self.max_age

    def score(self, poses, patches, intrinsics, n_dev):
        """fp32 [J * max_age] candidate scores (+inf outside the range, or everywhere when no proposal is due)"""
        return extensions()[3].loop_scores(poses, patches, intrinsics, n_dev, self.last_global_ba, self.M, self.removal,
                                           self.max_age, self.freq, self.kf_index)

    def propose(self, poses, patches, intrinsics, n_dev):
        """score, select and emit the loop edges of frame n (device n_dev); call it before the frame's forward and
        backward edges are appended, as dpvo.py:448-459 does.  poses [N, 7], patches [N M, 3, 3, 3], intrinsics [N, 4]."""
        g = self.pg
        self.scores = self.score(poses, patches, intrinsics, n_dev)
        r0, r1 = g.normal_cap, g.cap
        extensions()[3].loop_select(self.scores, n_dev, self.last_global_ba, self.M, self.removal, self.max_age, self.freq,
                                    self.kf_index, self.thresh, self.pairs, self.n_pairs, g.ii[r0:r1], g.jj[r0:r1],
                                    g.kk[r0:r1], g.active[r0:r1], g.net[0, r0:r1], g.n_active, self.region_overflow)
        return self.scores

    # ------------------------------------------------------------------------ dpvo.py:223-238, 300-310
    def remove(self, n_dev, enable=None):
        """park the edges that left the removal window, except the loop edges still in use, and keep them in the
        inactive store with their last target and weight (the runner writes those per slot in g.target / g.weight)"""
        g = self.pg
        extensions()[3].pgraph_remove_store(g.ii, g.jj, g.kk, g.active, g.target[0], g.weight[0], n_dev, self.removal,
                                            self.opt_window, enable, g.dummy_frame, g.dummy_patch, self.M, g.n_active,
                                            self.s_ii, self.s_jj, self.s_kk, self.s_target[0], self.s_weight[0],
                                            self.s_count, self.s_overflow)

    # ------------------------------------------------------------------------ the host's per-frame decision
    def read_flags(self, n):
        """(loop-region slots in use: 1 + the last active one, 0 when no loop edge is active; an edge with
        ii < n - removal - 1; minimum active ii; inactive count): one D2H copy"""
        g = self.pg
        extensions()[3].loop_flags(g.ii, g.active, g.normal_cap, int(n), self.removal, self.s_count, self.flags)
        f = self.flags.tolist()
        return int(f[0]), bool(f[1]), int(f[2]), int(f[3])

    def inactive(self):
        """host-synchronising view of the used inactive store: (ii, jj, kk, target [1, c, 2], weight [1, c, 2])"""
        c = int(self.s_count.item())
        a = self.pg.inactive_cap
        return (self.s_ii[a - c:], self.s_jj[a - c:], self.s_kk[a - c:], self.s_target[:, a - c:], self.s_weight[:, a - c:])

    # ------------------------------------------------------------------------ dpvo.py:312-326, patchgraph.py:84-91
    def normalize(self, poses, patches, n, delta=None):
        """delta: a keyframe delta table (fp32 [T, 7]) whose translations are scaled with the poses', or None"""
        extensions()[3].loop_normalize(poses, patches, int(n), self.M, delta)

    def global_ba(self, poses, patches, intrinsics, n, t0, count, E, lmbda, iterations=2):
        """normalize, then the wide (eff_impl) bundle adjustment of poses [t0, n) over the `count` inactive edges and the
        first E active slots (their weights already multiplied by `active`).  Eager, host-synchronised by its dense
        solve; raises if the inactive store overflowed or a frame has more observers than the wide path holds.
        When a keyframe.Keyframes culls this stream (it registers itself as `keyframes`), normalize scales its
        recorded relative poses with the map (patchgraph.py:89-90)."""
        if int(self.s_overflow.item()):
            raise RuntimeError("LoopClosure.global_ba: the inactive store (%d edges) overflowed; removed edges were lost"
                               % self.pg.inactive_cap)
        if int(self.region_overflow.item()):
            raise RuntimeError("LoopClosure.global_ba: a proposal overwrote loop edges that were still active")
        g = self.pg
        self.normalize(poses, patches, n, None if self.keyframes is None else self.keyframes.delta[0])
        lo, hi = g.inactive_cap - int(count), g.inactive_cap + int(E)
        fastba.BA(poses.view(1, -1, 7), patches.view(1, -1, 3, 3, 3), intrinsics.view(1, -1, 4), g.target_all[:, lo:hi],
                  g.weight_all[:, lo:hi], lmbda, g.ii_all[lo:hi], g.jj_all[lo:hi], g.kk_all[lo:hi], int(t0), int(n),
                  self.M, iterations, eff_impl=True)
        self.ran_global_ba.add(int(n))
