"""Keyframe culling on the device (csrc/keyframe.cu, dpvo_b200/keyframe.py) against oracle/keyframe.py."""
import math

import pytest
import torch

from dpvo_b200 import synthetic
from dpvo_b200.keyframe import Keyframes
from dpvo_b200.loop import LoopClosure
from dpvo_b200.patchgraph import DevicePatchGraph
from dpvo_b200.runner import UpdateRunner
from dpvo_b200.streams import StreamBatch
from oracle import keyframe as OK
from oracle import loop as OL

pytestmark = pytest.mark.gpu
DEV = "cuda"
KI, THRESH = 4, 15.0
RINGS = ("fmap1", "fmap2", "gmap", "imap")


def _graph(st, **kw):
    M = st.cfg["M"]
    g = DevicePatchGraph(2 * st.E + 4 * M * st.cfg["lifetime"], M, st.poses.shape[0] - 1, DEV, **kw)
    g.append(st.ii, st.jj, st.kk)
    return g


def _edges(g, lo=0, hi=None):
    hi = g.cap if hi is None else hi
    a = g.active[lo:hi].bool().cpu()
    return sorted(zip(g.ii[lo:hi].cpu()[a].tolist(), g.jj[lo:hi].cpu()[a].tolist(), g.kk[lo:hi].cpu()[a].tolist()))


def _host(st, kf, g, b=0):
    """HostKeyframes from the device state of one stream (CPU copies, same dtypes) and its active edges"""
    hg = OL.HostGraph(st.cfg["M"], st.cfg["removal"], st.cfg["opt_window"])
    hg.act = [list(e) for e in _edges(g)]
    rings = {r: (None if getattr(st, r) is None else getattr(st, r).cpu()) for r in RINGS}
    return OK.HostKeyframes(st.cfg["M"], st.poses.cpu(), st.patches.cpu(), st.intrinsics.cpu(), int(kf.n_dev[b]),
                            tstamp=kf.tstamp[b].cpu(), counter=int(kf.counter[b]), graph=hg, **rings)


def _same_buffers(st, host):
    assert torch.equal(st.poses.cpu(), host.poses) and torch.equal(st.patches.cpu(), host.patches)
    assert torch.equal(st.intrinsics.cpu(), host.intrinsics)
    for r in RINGS:
        if getattr(st, r) is not None:
            assert torch.equal(getattr(st, r).cpu(), getattr(host, r)), r


def _close(m, m_ref):
    """the kernel's fp64 mean of fp32 flows against the fp64 oracle: each flow is a difference of fp32 pixel coordinates,
    so the bar is 1e-5 of m, but not less than 1e-5 px"""
    return abs(m - m_ref) <= 1e-5 * max(abs(m_ref), 1.0)


def _same(a, b):
    """(removed, m) records, NaN equal to NaN"""
    return a[0] == b[0] and (a[1] == b[1] or (math.isnan(a[1]) and math.isnan(b[1])))


def _margin_ok(m, removed):
    """the kernel's decision against the fp64 oracle's, wherever m / 2 is farther from the threshold than 1e-5 of it"""
    return removed == (m / 2 < THRESH) or abs(m / 2 - THRESH) <= 1e-5 * THRESH


# -------------------------------------------------------------------------------- 1. the motion test
def test_motion_matches_oracle_is_deterministic_and_keeps_frames_without_edges():
    seen = set()
    cases = [synthetic.make_stop_go_state("fast", n, total=40, device=DEV, features=False, seed=n) for n in range(8, 34, 3)]
    for seed in (3, 4):
        st = synthetic.make_state("default" if seed == 4 else "fast", 24, device=DEV, features=False, seed=seed, buffer=26)
        g = torch.Generator(device="cpu").manual_seed(seed)
        st.poses[:24, :3] += (0.2 * torch.randn(24, 3, generator=g)).to(DEV)
        q = torch.randn(24, 4, generator=g) * 0.05
        q[:, 3] += 1.0
        st.poses[:24, 3:] = (q / q.norm(dim=1, keepdim=True)).to(DEV)
        cases.append(st)
    for st in cases:
        g = _graph(st)
        host = _host(st, Keyframes(st.cfg, st, g), g)
        m_ref, _ = host.motion(KI, THRESH)
        probe = Keyframes(st.cfg, st, g, keyframe_thresh=-1.0)            # decides nothing: m only
        probe.cull()
        a = probe.m.clone()
        probe.cull()
        assert torch.equal(a, probe.m) and not probe.flag.any()
        kf = Keyframes(st.cfg, st, g)
        kf.cull()
        (removed, m), = kf.read()
        assert m == float(a[0])
        assert _close(m, m_ref), (m, m_ref)
        assert removed == (m / 2 < THRESH) and _margin_ok(m_ref, removed)
        seen.add(removed)
    assert seen == {True, False}
    st = synthetic.make_stop_go_state("fast", KI, total=20, device=DEV, features=False)      # n < KI + 2: no (i, j) edge
    g = _graph(st)
    kf = Keyframes(st.cfg, st, g)
    kf.cull()
    (removed, m), = kf.read()
    assert math.isnan(m) and not removed and int(kf.n_dev[0]) == KI


# -------------------------------------------------------------------------------- 2. one cull, bit for bit
def test_one_cull_matches_oracle_bit_for_bit_with_a_wrapping_ring():
    # n = 22: frames 17 .. 21 stand still, k = 18 is culled, and slots 18 .. 21 wrap around mem = 10
    st = synthetic.make_stop_go_state("fast", 22, total=40, mem=10, device=DEV, seed=5)
    g = _graph(st)
    kf = Keyframes(st.cfg, st, g)
    host = _host(st, kf, g)
    host_poses0 = host.poses.clone()
    net0 = g.net.clone()
    n_act0 = int(g.n_active)
    kf.cull()
    (removed, m), = kf.read()
    m_ref, dec = host.motion(KI, THRESH)
    assert removed and dec and _close(m, m_ref)
    host.keyframe(KI, THRESH, removed=True)
    _same_buffers(st, host)
    assert torch.equal(kf.tstamp[0].cpu(), host.tstamp)
    assert _edges(g) == sorted(map(tuple, host.graph.act))
    assert int(g.n_active) == len(host.graph.act) < n_act0
    assert torch.equal(g.net, net0)                           # removal parks in place: every state row stays with its edge
    assert int(kf.n_dev[0]) == 21 and st.n == 21
    k = 22 - KI
    t0, dP = host.delta[k]
    assert int(kf.delta_src[0, k]) == t0 == k - 1 and (kf.delta_src[0] >= 0).sum() == 1
    assert torch.allclose(kf.delta[0, k].cpu().double(), dP, rtol=0, atol=2e-6)
    # bit for bit: the same product through the library's SE3 operators (lie.cu), P_k P_{k-1}^-1 from the pre-cull poses
    from dpvo_b200.lietorch import SE3
    P = host_poses0.to(DEV)
    want = (SE3(P[k:k + 1]) * SE3(P[k - 1:k]).inv()).data[0]
    assert torch.equal(kf.delta[0, k], want)


def test_a_kept_frame_changes_nothing():
    st = synthetic.make_stop_go_state("fast", 14, total=40, mem=10, device=DEV, seed=6)      # k = 10 moves
    g = _graph(st)
    kf = Keyframes(st.cfg, st, g)
    before = {r: getattr(st, r).clone() for r in ("poses", "patches", "intrinsics") + RINGS}
    gb = [t.clone() for t in (g.ii, g.jj, g.kk, g.active, g.n_active, g.net)]
    ts, dl, ds = kf.tstamp.clone(), kf.delta.clone(), kf.delta_src.clone()
    kf.cull()
    (removed, _), = kf.read()
    assert not removed and st.n == 14 and int(kf.n_dev[0]) == 14
    for r, t in before.items():
        assert torch.equal(getattr(st, r), t), r
    assert all(torch.equal(a, b) for a, b in zip(gb, (g.ii, g.jj, g.kk, g.active, g.n_active, g.net)))
    assert torch.equal(kf.tstamp, ts) and torch.equal(kf.delta, dl) and torch.equal(kf.delta_src, ds)


# -------------------------------------------------------------------------------- 3. the reference's own keyframe()
@pytest.mark.parametrize("n,seed,mem", [(22, 5, 10), (14, 6, 10), (27, 8, 36), (31, 9, 7)])
def test_cull_equals_the_reference_dpvo_keyframe(n, seed, mem):
    """DPVO.keyframe (motion test, delta record, remove_factors, renumbering, shift, then the window removal) of the
    reference's unmodified Python on our native modules, on a DPVO object built on a copy of the same state, against
    cull + remove_old: the same decision and bit-identical buffers, edges, timestamps and delta record"""
    from oracle import refimport
    if not refimport.staged():
        pytest.skip("the reference's Python package is not staged in oracle/_ref")
    st = synthetic.make_stop_go_state("fast", n, total=40, mem=mem, device=DEV, seed=seed)
    cfg = st.cfg
    g = _graph(st)
    kf = Keyframes(cfg, st, g)
    edges = torch.tensor(_edges(g), dtype=torch.long)
    with refimport.reference_python():
        ref = OK.reference_dpvo(st, edges, n, kf.tstamp[0], KI, THRESH)
        ref.keyframe()
        torch.cuda.synchronize()
        delta = {t: (int(t0), dP.data.reshape(7).clone()) for t, (t0, dP) in ref.pg.delta.items()}
        pg = ref.pg
        r_edges = sorted(zip(pg.ii.tolist(), pg.jj.tolist(), pg.kk.tolist()))
        r_n, r_tstamp = pg.n, torch.as_tensor(pg.tstamps_)
        r = dict(poses=pg.poses_, patches=pg.patches_.view(-1, 3, 3, 3), intrinsics=pg.intrinsics_, fmap1=ref.fmap1_,
                 fmap2=ref.fmap2_, gmap=ref.gmap_.flatten(0, 1)[None], imap=ref.imap_.reshape(1, -1, 384))
    kf.cull()
    g.remove_old(kf.n_dev, cfg["removal"])
    (removed, _), = kf.read()
    assert removed == (r_n == n - 1) and st.n == r_n == int(kf.n_dev[0])
    for name, t in r.items():
        assert torch.equal(getattr(st, name), t), name
    assert torch.equal(kf.tstamp[0].cpu(), r_tstamp)
    assert _edges(g) == r_edges
    rec = (kf.delta_src[0] >= 0).nonzero().view(-1).tolist()
    assert rec == sorted(delta)
    for t in rec:
        assert int(kf.delta_src[0, t]) == delta[t][0] and torch.equal(kf.delta[0, t], delta[t][1]), t


# -------------------------------------------------------------------------------- 4. a tracking loop
def _ring_ids(st):
    """rings of row ids with the device rings' slot layout, for the oracle to permute"""
    M = st.cfg["M"]
    mem, pmem = st.fmap1.shape[1], st.gmap.shape[1] // M
    return dict(fmap1=torch.arange(mem)[None], fmap2=torch.arange(mem)[None], gmap=torch.arange(pmem * M)[None],
                imap=torch.arange(pmem * M)[None])


def _new_frame(st, kf, c):
    """the frame of timestamp c into slot n - 1 (the caller's part of dpvo.py:386-440)"""
    M, n = st.cfg["M"], st.n
    st.poses[n - 1] = st.extras["trajectory"][c]
    st.patches[(n - 1) * M:n * M] = st.extras["patches"][c * M:(c + 1) * M]


def test_tracking_loop_with_device_decisions_matches_oracle():
    frames, n0 = 120, 16
    st = synthetic.make_stop_go_state("fast", n0, total=n0 + frames, stop=8, go=6, mem=36, device=DEV, seed=7)
    cfg, M = st.cfg, st.cfg["M"]
    g = _graph(st)
    runner = UpdateRunner(st, graph=g)
    kf = Keyframes(cfg, st, g)
    hg = OL.HostGraph(M, cfg["removal"], cfg["opt_window"])
    hg.act = [list(e) for e in _edges(g)]
    culled = kept = 0
    for f in range(frames):
        c = int(kf.counter[0])
        st.n += 1
        kf.n_dev += 1
        _new_frame(st, kf, c)
        kf.add_frame()
        n = st.n
        g.append_frame_edges(kf.n_dev, cfg["lifetime"])
        r = cfg["lifetime"]
        fk = list(range(M * (n - r), M * (n - 1)))
        bk = list(range(M * (n - 1), M * n))
        hg.append([k // M for k in fk], [n - 1] * len(fk), fk)
        hg.append([b // M for b in bk for _ in range(r)], [jx for b in bk for jx in range(n - r, n)], [b for b in bk for _ in range(r)])
        st.t0 = max(n - cfg["opt_window"], 1)
        runner.step()
        host = OK.HostKeyframes(M, st.poses.cpu(), st.patches.cpu(), st.intrinsics.cpu(), n, tstamp=kf.tstamp[0].cpu(),
                                counter=int(kf.counter[0]), graph=hg, **_ring_ids(st))
        pre = {r_: getattr(st, r_).clone() for r_ in RINGS}
        kf.cull()
        (removed, m), = kf.read()
        m_ref, _ = host.motion(KI, THRESH)
        # after bundle adjustment on random features some patches sit near the projection's depth clamp, where the fp32
        # flows lose more digits than on the synthetic poses: 1e-4 here
        assert abs(m - m_ref) <= 1e-4 * max(abs(m_ref), 1.0) and _margin_ok(m_ref, removed), "frame %d" % f
        host.keyframe(KI, THRESH, removed=removed)
        culled, kept = culled + removed, kept + (not removed)
        assert st.n == host.n and int(kf.n_dev[0]) == host.n
        assert torch.equal(st.poses.cpu(), host.poses) and torch.equal(st.patches.cpu(), host.patches)
        assert torch.equal(kf.tstamp[0].cpu(), host.tstamp)
        for r_ in RINGS:
            assert torch.equal(getattr(st, r_), pre[r_][:, host.__dict__[r_][0].to(DEV)]), "frame %d %s" % (f, r_)
        # the window removal (dpvo.py:300-306) with the frame count cull left
        g.remove_old(kf.n_dev, cfg["removal"])
        hg.act = [e for e in hg.act if e[2] // M >= st.n - cfg["removal"]]
        assert _edges(g) == sorted(map(tuple, hg.act)), "frame %d" % f
        assert int(g.n_active) == len(hg.act) and int(g.overflow) == 0
    assert culled >= 20 and kept >= 20, (culled, kept)


# -------------------------------------------------------------------------------- 5. with loop closure
def test_culling_on_a_loop_closure_graph_leaves_the_inactive_store_and_scales_deltas():
    n0, frames = 30, 40
    st = synthetic.make_loop_state("fast", n0 + frames, period=24, radius=1.5, device=DEV, features=False)
    st.n, st.t0 = n0, n0 - st.cfg["opt_window"]
    cfg, M = st.cfg, st.cfg["M"]
    ii, jj, kk = synthetic.replay_edges(n0, M, cfg["lifetime"], cfg["removal"])
    g = DevicePatchGraph(2 * ii.numel(), M, st.poses.shape[0] - 1, DEV, loop_pairs=1000, inactive_capacity=200000)
    g.append(ii.to(DEV), jj.to(DEV), kk.to(DEV))
    lc = LoopClosure(cfg, g)
    kf = Keyframes(cfg, st, g, loop=lc)
    gen = torch.Generator(device=DEV).manual_seed(3)
    deltas, culled = {}, 0
    for f in range(frames):
        st.n += 1
        kf.n_dev += 1
        kf.add_frame()
        lc.propose(st.poses, st.patches, st.intrinsics, kf.n_dev)
        g.append_frame_edges(kf.n_dev, cfg["lifetime"])
        g.target.copy_(torch.rand(g.target.shape, generator=gen, device=DEV))
        g.weight.copy_(torch.rand(g.weight.shape, generator=gen, device=DEV))
        store = [t.clone() for t in (lc.s_ii, lc.s_jj, lc.s_kk, lc.s_target, lc.s_weight, lc.s_count)]
        host = _host(st, kf, g)
        host.delta = deltas
        kf.cull()
        assert all(torch.equal(a, b) for a, b in zip(store, (lc.s_ii, lc.s_jj, lc.s_kk, lc.s_target, lc.s_weight, lc.s_count)))
        (removed, m), = kf.read()
        host.keyframe(KI, THRESH, removed=removed)
        culled += removed
        assert _edges(g) == sorted(map(tuple, host.graph.act)), "frame %d" % f
        lc.remove(kf.n_dev)
    assert culled >= 3
    # the global bundle adjustment's normalize scales every recorded delta with the map
    n = st.n
    s = float(st.patches[:n * M, 2].double().mean())
    d0 = kf.delta.clone()
    count = int(lc.s_count)
    g.weight.mul_(g.active[None, :, None].float())
    lc.global_ba(st.poses, st.patches, st.intrinsics, n, 1, count, g.cap, torch.as_tensor([1e-4], device=DEV))
    rec = kf.delta_src[0] >= 0
    assert torch.allclose(kf.delta[0, rec, :3], d0[0, rec, :3] * s, rtol=2e-6, atol=1e-7)
    assert torch.equal(kf.delta[0, :, 3:], d0[0, :, 3:])
    want = OK.terminate(st.poses.cpu(), kf.tstamp[0].cpu(), n, OK.scale_deltas(deltas, s), int(kf.counter[0]))
    got = kf.trajectory().cpu()
    dt, da = OK.pose_distance(got, want)
    assert (dt <= 1e-4).all() and (da <= 1e-5).all(), (dt.max(), da.max())


# -------------------------------------------------------------------------------- 6. several streams
def test_batch_matches_single_streams_bit_for_bit():
    B, n0, F, mem, frames = 3, 14, 48, 10, 12
    states = [synthetic.make_stop_go_state("fast", n0, total=n0 + frames, stop=s, go=g_, buffer=F, mem=mem, device=DEV, seed=11 + b)
              for b, (s, g_) in enumerate(((6, 4), (3, 9), (12, 2)))]
    cfg, M = states[0].cfg, states[0].cfg["M"]
    batch = StreamBatch(B, cfg, F, mem, device=DEV)
    for b, st in enumerate(states):
        batch.load(b, st)
    store, graphs = DevicePatchGraph.stacked(B, 2 * states[0].E + 4 * M * cfg["lifetime"], M, [b * F + F - 1 for b in range(B)], DEV)
    for b, st in enumerate(states):
        graphs[b].append(*batch.to_global(b, st.ii, st.jj, st.kk))
    kfb = Keyframes(cfg, batch, store)
    singles = []
    for st in states:
        g = _graph(st)
        singles.append((st, g, Keyframes(cfg, st, g)))
    outcomes = set()
    for f in range(frames):
        for b, (st, g, kf) in enumerate(singles):
            c = int(kf.counter[0])
            st.n += 1
            kf.n_dev += 1
            _new_frame(st, kf, c)
            s = batch.stream(b)
            s.n += 1
            s.poses[s.n - 1] = st.poses[st.n - 1]
            s.patches[(s.n - 1) * M:s.n * M] = st.patches[(st.n - 1) * M:st.n * M]
            kf.add_frame()
            g.append_frame_edges(kf.n_dev, cfg["lifetime"])
            graphs[b].append_frame_edges(torch.tensor([b * F + s.n], device=DEV), cfg["lifetime"])
        kfb.n_dev += 1
        kfb.add_frame()
        kfb.cull()
        rb = kfb.read()
        for b, (st, g, kf) in enumerate(singles):
            kf.cull()
            (removed, m), = kf.read()
            outcomes.add(removed)
            assert _same(rb[b], (removed, m)), "frame %d stream %d" % (f, b)
            s = batch.stream(b)
            assert s.n == st.n
            g.remove_old(kf.n_dev, cfg["removal"])
            graphs[b].remove_old(torch.tensor([b * F + s.n], device=DEV), cfg["removal"])
            assert int(g.overflow) == 0 and int(graphs[b].overflow) == 0
            for r in ("poses", "patches", "intrinsics") + RINGS:
                assert torch.equal(getattr(s, r), getattr(st, r)), "frame %d stream %d %s" % (f, b, r)
            assert torch.equal(kfb.tstamp[b], kf.tstamp[0]) and torch.equal(kfb.delta[b], kf.delta[0])
            assert torch.equal(kfb.delta_src[b], kf.delta_src[0]) and torch.equal(kfb.counter[b], kf.counter[0])
            off = torch.tensor([b * F, b * F, b * F * M])
            assert _edges(graphs[b]) == sorted(tuple((torch.tensor(e) + off).tolist()) for e in _edges(g))
    assert outcomes == {True, False}


# -------------------------------------------------------------------------------- 7. CUDA graph capture
def test_captured_add_frame_and_cull_equals_eager():
    frames, n0 = 24, 14
    runs = []
    for _ in range(2):
        st = synthetic.make_stop_go_state("fast", n0, total=n0 + frames, stop=5, go=4, mem=10, device=DEV, seed=13)
        g = _graph(st)
        runs.append((st, g, Keyframes(st.cfg, st, g)))
    st_g, g_g, kf_g = runs[1]

    def frame(st, g, kf):
        kf.n_dev.add_(1)
        kf.add_frame()
        g.append_frame_edges(kf.n_dev, st.cfg["lifetime"])
        kf.cull()
        g.remove_old(kf.n_dev, st.cfg["removal"])

    def body():
        frame(st_g, g_g, kf_g)

    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):              # capture only: nothing runs until replay
        body()
    outcomes = set()
    for f in range(frames):
        for st, g, kf in runs:
            st.n += 1                          # the new frame's slot; read() takes a culled frame off again
            _new_frame(st, kf, int(kf.counter[0]))
        kf0 = runs[0][2]
        frame(*runs[0])
        graph.replay()
        (r0, m0), = kf0.read()
        (r1, m1), = kf_g.read()
        assert _same((r0, m0), (r1, m1)) and not math.isnan(m0), "frame %d" % f
        outcomes.add(r0)
        a, b = runs
        for r in ("poses", "patches", "intrinsics") + RINGS:
            assert torch.equal(getattr(a[0], r), getattr(b[0], r)), r
        for x, y in zip((a[1].ii, a[1].jj, a[1].kk, a[1].active, a[1].n_active), (b[1].ii, b[1].jj, b[1].kk, b[1].active, b[1].n_active)):
            assert torch.equal(x, y)
        for x, y in zip((a[2].tstamp, a[2].delta, a[2].delta_src, a[2].counter, a[2].n_dev),
                        (b[2].tstamp, b[2].delta, b[2].delta_src, b[2].counter, b[2].n_dev)):
            assert torch.equal(x, y)
    assert outcomes == {True, False}


# -------------------------------------------------------------------------------- 8. the trajectory
def test_trajectory_matches_oracle_over_long_chains_and_reports_overflow():
    n0, frames, skips = 8, 90, 60
    st = synthetic.make_stop_go_state("fast", n0, total=n0 + skips + frames, stop=60, go=6, device=DEV, features=False, seed=17)
    cfg, M = st.cfg, st.cfg["M"]
    g = _graph(st)
    kf = Keyframes(cfg, st, g)
    host = _host(st, kf, g)
    for _ in range(skips):                   # frames dropped before initialisation
        kf.skip_frame()
        host.skip_frame()
    run = best = 0
    for f in range(frames):
        c = int(kf.counter[0])
        st.n += 1
        kf.n_dev += 1
        host.n += 1
        _new_frame(st, kf, c - skips)
        host.poses, host.patches = st.poses.cpu(), st.patches.cpu()
        kf.add_frame()
        host.add_frame()
        g.append_frame_edges(kf.n_dev, cfg["lifetime"])
        host.graph.act = [list(e) for e in _edges(g)]
        kf.cull()
        (removed, _), = kf.read()
        host.keyframe(KI, THRESH, removed=removed)
        run = run + 1 if removed else 0
        best = max(best, run)
        g.remove_old(kf.n_dev, cfg["removal"])
    assert best >= 50, best
    assert torch.equal(kf.tstamp[0].cpu()[:host.n], host.tstamp[:host.n])
    got = kf.trajectory().cpu()
    want = OK.terminate(host.poses, host.tstamp, host.n, host.delta, host.counter)
    assert got.shape == want.shape == (n0 + skips + frames, 7)
    # chain length of every timestamp: the number of relative poses between it and its live keyframe
    live = {int(t) for t in host.tstamp[:host.n]}
    for t in range(host.counter):
        L, u = 0, t
        while u not in live:
            u, L = host.delta[u][0], L + 1
        dt, da = OK.pose_distance(got[t:t + 1], want[t:t + 1])
        bar = OK.chain_bar(L, scale=float(want[t, :3].abs().max()))
        assert dt.item() <= bar and da.item() <= bar, (t, L, dt.item(), da.item(), bar)
    # a delta table too small for the stream: reported, not silently wrapped
    st2 = synthetic.make_stop_go_state("fast", n0, total=40, device=DEV, features=False, seed=18)
    g2 = _graph(st2)
    kf2 = Keyframes(cfg, st2, g2, max_timestamps=st2.poses.shape[0])
    for _ in range(st2.poses.shape[0]):
        kf2.skip_frame()
    with pytest.raises(RuntimeError, match="max_timestamps"):
        kf2.read()
    with pytest.raises(RuntimeError, match="max_timestamps"):
        kf2.trajectory()
    # a culled frame whose timestamp overflows: read() raises after the host n has followed n_dev
    st3 = synthetic.make_stop_go_state("fast", 22, total=40, mem=10, device=DEV, features=False, seed=5)      # k culled
    g3 = _graph(st3)
    kf3 = Keyframes(cfg, st3, g3, max_timestamps=st3.poses.shape[0])
    kf3.tstamp[0, 22 - KI] = kf3.T                                  # frame k's timestamp lies outside the table
    kf3.cull()
    with pytest.raises(RuntimeError, match="max_timestamps"):
        kf3.read()
    assert st3.n == int(kf3.n_dev[0]) == 21
    # a broken chain in one stream of a batch leaves the other stream's trajectory readable
    F = 24
    batch = StreamBatch(2, cfg, F, KI, device=DEV)
    for b in range(2):
        s = batch.stream(b)
        s.n = 8
        s.poses[:8] = st.extras["trajectory"][:8]
    store, _ = DevicePatchGraph.stacked(2, 256, M, [F - 1, 2 * F - 1], DEV)
    kfb = Keyframes(cfg, batch, store)
    kfb.tstamp[1, 3] = kfb.T + 5                                    # timestamp 3 of stream 1: neither live nor recorded
    want = OK.terminate(batch.stream(0).poses.cpu(), kfb.tstamp[0].cpu(), 8, {}, 8)
    assert torch.allclose(kfb.trajectory(stream=0).cpu().double(), want, rtol=0, atol=1e-6)
    with pytest.raises(RuntimeError, match="stream 1"):
        kfb.trajectory(stream=1)
