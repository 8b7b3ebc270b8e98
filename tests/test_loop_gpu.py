"""Proximity loop closure on the device (csrc/loop.cu, dpvo_b200/loop.py) against oracle/loop.py and the reference."""
import pytest
import torch

from dpvo_b200 import synthetic
from dpvo_b200.loop import LoopClosure
from dpvo_b200.patchgraph import DevicePatchGraph
from dpvo_b200.runner import UpdateRunner
from oracle import loop as OL
from oracle import ba as OB

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _setup(st, loop_pairs=1000, inactive=200000, capacity=None, **kw):
    M = st.cfg["M"]
    dummy = st.poses.shape[0] - 1
    g = DevicePatchGraph(capacity or st.E + 4 * M * st.cfg["lifetime"], M, dummy, DEV, loop_pairs=loop_pairs,
                         inactive_capacity=inactive)
    lc = LoopClosure(st.cfg, g, **kw)
    return g, lc


def _n(v):
    return torch.tensor([v], dtype=torch.long, device=DEV)


def _oracle_scores(st, lc, n, last_ba=-1000):
    return OL.scores(st.poses.cpu(), st.patches.cpu(), st.intrinsics.cpu(), n, lc.M, lc.removal, lc.max_age, lc.freq,
                     lc.kf_index, last_ba)


def _propose(st, lc, n):
    sc = lc.propose(st.poses, st.patches, st.intrinsics, _n(n))
    torch.cuda.synchronize()
    k = int(lc.n_pairs.item())
    return sc, [tuple(p) for p in lc.pairs[:k].tolist()]


def test_scores_match_oracle_and_are_deterministic():
    st = synthetic.make_loop_state("fast", 90, period=24, radius=1.5, device=DEV, features=False)
    g, lc = _setup(st)
    a = lc.score(st.poses, st.patches, st.intrinsics, _n(st.n))
    b = lc.score(st.poses, st.patches, st.intrinsics, _n(st.n))
    assert torch.equal(a, b)
    ref = _oracle_scores(st, lc, st.n)
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isfinite(a.cpu()), fin) and fin.sum() > 500
    err = (a.cpu().double()[fin] - ref[fin]).abs()
    assert (err <= 1e-5 * ref[fin].abs() + 2e-5).all(), err.max().item()


def test_selection_equals_oracle_and_emits_edges():
    st = synthetic.make_loop_state("fast", 90, period=24, radius=1.5, device=DEV, features=False)
    g, lc = _setup(st)
    sc, pairs = _propose(st, lc, st.n)
    want = OL.select(sc.cpu(), st.n, lc.removal, lc.max_age, lc.freq, lc.kf_index, lc.thresh, lc.pairs_cap)
    assert pairs == want and len(pairs) > 100
    assert int(lc.last_global_ba.item()) == st.n
    M, r0 = lc.M, g.normal_cap
    k = len(pairs) * M
    ii, jj, kk = g.ii[r0:r0 + k].cpu(), g.jj[r0:r0 + k].cpu(), g.kk[r0:r0 + k].cpu()
    pi = torch.tensor([p[0] for p in pairs]).repeat_interleave(M)
    pj = torch.tensor([p[1] for p in pairs]).repeat_interleave(M)
    assert torch.equal(ii, pi) and torch.equal(jj, pj) and torch.equal(kk, pi * M + torch.arange(M).repeat(len(pairs)))
    assert g.active[r0:r0 + k].all() and not g.active[r0 + k:].any() and int(g.n_active.item()) == k
    assert not g.net[0, r0:r0 + k].any()
    # no proposal is due at the same n any more: nothing changes
    sc2, pairs2 = _propose(st, lc, st.n)
    assert torch.isinf(sc2).all() and pairs2 == [] and int(g.n_active.item()) == k


def test_selection_equals_reference_edges_loop():
    from oracle import refimport
    if not refimport.staged():
        pytest.skip("the reference's Python package is not staged in oracle/_ref")
    st = synthetic.make_loop_state("fast", 90, period=24, radius=1.5, device=DEV, features=False)
    g, lc = _setup(st)
    _, pairs = _propose(st, lc, st.n)
    M, n = lc.M, st.n
    with refimport.reference_python():
        from dpvo.config import cfg as base
        from dpvo.patchgraph import PatchGraph
        cfg = base.clone()
        cfg.PATCHES_PER_FRAME, cfg.BUFFER_SIZE, cfg.REMOVAL_WINDOW = M, st.poses.shape[0], lc.removal
        cfg.MAX_EDGE_AGE, cfg.GLOBAL_OPT_FREQ, cfg.KEYFRAME_INDEX, cfg.BACKEND_THRESH = lc.max_age, lc.freq, lc.kf_index, lc.thresh
        pg = PatchGraph(cfg, 3, 384, lc.max_age, device=DEV, dtype=torch.half)
        pg.n = n
        pg.poses_[:] = st.poses
        pg.patches_[:] = st.patches.view(-1, M, 3, 3, 3)
        pg.intrinsics_[:] = st.intrinsics
        pg.index_[:] = torch.arange(pg.N, device=DEV)[:, None]
        kk, jj = pg.edges_loop()
    ref = [(int(k) // M, int(j)) for k, j in zip(kk[::M].tolist(), jj[::M].tolist())]
    assert pairs == ref


def _flat_state(n, M_cfg="fast"):
    """poses all identical: every candidate scores 0, the selection visits pairs in candidate order"""
    st = synthetic.make_loop_state(M_cfg, n, device=DEV, features=False, noise=0.0)
    st.poses[:] = st.poses[0]
    return st


def test_no_candidates_at_or_below_the_removal_window():
    st = _flat_state(40)
    g, lc = _setup(st)
    for n in (lc.removal - 3, lc.removal):
        sc, pairs = _propose(st, lc, n)
        assert torch.isinf(sc).all() and pairs == [] and int(lc.last_global_ba.item()) == -1000


def test_gap_29_30_31_and_neighbour_suppression():
    st = _flat_state(80)
    g, lc = _setup(st)
    sc, pairs = _propose(st, lc, 80)
    assert (sc.cpu()[torch.isfinite(sc.cpu())] == 0).all()
    assert pairs == OL.select(sc.cpu(), 80, lc.removal, lc.max_age, lc.freq, lc.kf_index, lc.thresh)
    gaps = {j - i for i, j in pairs}
    assert 29 not in gaps and min(gaps) == 30 and 31 in gaps
    s = set(pairs)
    assert not any((i + 1, j) in s or (i - 1, j) in s for i, j in pairs)


def test_fewer_than_three_quarters_valid_is_inf():
    st = _flat_state(60)
    M = st.cfg["M"]
    j = 60 - 8                                         # a target frame of the proposal at n = 60
    st.poses[j, 2] -= 1.0                              # relative translation tz = -1: Z = 1 - d
    st.patches[:, 2] = 0.5
    nbad = {3: M - int(0.75 * M), 4: M - int(0.75 * M) - 1}     # frame 3: exactly 0.75 M valid; frame 4: one more
    for i, b in nbad.items():
        st.patches[i * M:i * M + b, 2] = 0.9
    g, lc = _setup(st)
    sc = lc.score(st.poses, st.patches, st.intrinsics, _n(60)).cpu()
    i0, ni, j0, J = OL.loop_range(60, lc.removal, lc.max_age, lc.freq, lc.kf_index)
    row = sc.view(J, lc.max_age)[j - j0]
    assert torch.isinf(row[3 - i0]) and torch.isfinite(row[4 - i0]) and torch.isfinite(row[5 - i0])
    ref = _oracle_scores(st, lc, 60)
    assert torch.equal(torch.isfinite(sc), torch.isfinite(ref))


def test_more_than_1000_acceptable_pairs():
    st = _flat_state(260)
    g, lc = _setup(st, inactive=1024)
    sc, pairs = _propose(st, lc, 260)
    assert len(pairs) == 1000
    assert pairs == OL.select(sc.cpu(), 260, lc.removal, lc.max_age, lc.freq, lc.kf_index, lc.thresh, 1000)


def _edges(g, lo, hi):
    a = g.active[lo:hi].bool().cpu()
    return sorted(zip(g.ii[lo:hi].cpu()[a].tolist(), g.jj[lo:hi].cpu()[a].tolist(), g.kk[lo:hi].cpu()[a].tolist()))


def _slot_values(g):
    """{(ii, jj, kk): target + weight} of every active edge"""
    a = g.active.bool()
    e = torch.stack([g.ii[a], g.jj[a], g.kk[a]], 1).tolist()
    return {tuple(x): tuple(t) + tuple(w) for x, t, w in zip(e, g.target[0][a].tolist(), g.weight[0][a].tolist())}


def _drive(frames, n0=30, keyframe_every=7, seed=3, run=False):
    """the per-frame bookkeeping of dpvo.py:449-459 (propose, append), :328-360 (the update, with the global bundle
    adjustment of :348 when due) and :266-310 (keyframe removal, then the window removal that keeps edges) on the device
    and on oracle.loop.HostGraph.  run=True steps an UpdateRunner every frame, whose targets / weights the removal
    keeps; otherwise every slot gets random ones."""
    st = synthetic.make_loop_state("fast", n0 + frames, period=24, radius=1.5, device=DEV, features=run)
    cfg, M = st.cfg, st.cfg["M"]
    g, lc = _setup(st, capacity=2 * st.E)
    hg = OL.HostGraph(M, cfg["removal"], cfg["opt_window"])
    ii, jj, kk = synthetic.replay_edges(n0, M, cfg["lifetime"], cfg["removal"])
    g.append(ii.to(DEV), jj.to(DEV), kk.to(DEV))
    hg.append(ii.tolist(), jj.tolist(), kk.tolist())
    runner = UpdateRunner(st, graph=g, loop=lc) if run else None
    gen = torch.Generator(device=DEV).manual_seed(seed)
    n, last_ba, ran, stored = n0, -1000, set(), 0
    for f in range(frames):
        n += 1
        n_dev = _n(n)
        sc, pairs = _propose(st, lc, n)
        if n - last_ba >= lc.freq:
            want = OL.select(sc.cpu(), n, lc.removal, lc.max_age, lc.freq, lc.kf_index, lc.thresh, lc.pairs_cap)
            assert pairs == want
            if want:
                last_ba = n
                hg.append_pairs(want)
        else:
            assert pairs == []
        assert int(lc.last_global_ba.item()) == last_ba
        g.append_frame_edges(n_dev, cfg["lifetime"])
        r = cfg["lifetime"]
        fk = list(range(M * (n - r), M * (n - 1)))
        bk = list(range(M * (n - 1), M * n))
        hg.append([k // M for k in fk], [n - 1] * len(fk), fk)
        hg.append([k // M for b in bk for k in [b] * r], [jx for b in bk for jx in range(n - r, n)], [b for b in bk for _ in range(r)])
        if run:
            # dpvo.py:348: the global bundle adjustment runs when an edge has ii < n - removal - 1, once per n
            if any(e[0] < n - cfg["removal"] - 1 for e in hg.act) and n not in ran:
                ran.add(n)
            st.n, st.t0 = n, max(n - cfg["opt_window"], 1)
            runner.step()
            torch.cuda.synchronize()
            assert lc.ran_global_ba == ran, "frame %d" % f
        else:
            g.target.copy_(torch.rand(g.target.shape, generator=gen, device=DEV))
            g.weight.copy_(torch.rand(g.weight.shape, generator=gen, device=DEV))
        if f % keyframe_every == keyframe_every - 1:
            k = n - lc.kf_index
            g.remove_frame(_n(k))
            hg.remove_keyframe(k)
            n -= 1
            n_dev = _n(n)
        tw = _slot_values(g)
        lc.remove(n_dev)
        hg.remove_window(n, lambda e: tw[tuple(e)])
        assert _edges(g, 0, g.cap) == sorted(map(tuple, hg.act)), "frame %d" % f
        assert int(g.n_active.item()) == len(hg.act)
        # this frame's removals: the block just below the previous ones in the store
        s_ii, s_jj, s_kk, s_t, s_w = lc.inactive()
        new = len(hg.inac) - stored
        assert s_ii.numel() == len(hg.inac), "frame %d" % f
        dev_new = sorted(zip(s_ii[:new].tolist(), s_jj[:new].tolist(), s_kk[:new].tolist(), *s_t[0, :new].t().tolist(),
                             *s_w[0, :new].t().tolist()))
        assert dev_new == sorted(map(tuple, hg.inac[stored:])), "frame %d" % f
        stored = len(hg.inac)
    s_ii, s_jj, s_kk, s_t, s_w = lc.inactive()
    dev_inac = sorted(zip(s_ii.tolist(), s_jj.tolist(), s_kk.tolist(), *s_t[0].t().tolist(), *s_w[0].t().tolist()))
    assert dev_inac == sorted(map(tuple, hg.inac))
    return st, g, lc, hg, n, ran


def test_driver_matches_host_restatement():
    st, g, lc, hg, n, ran = _drive(120, run=True)
    assert len(hg.inac) > 10000 and any(j - i > 30 for i, j, k, *_ in hg.inac)
    assert ran, "the loop closures must have run global bundle adjustments"
    assert int(lc.s_overflow.item()) == 0 and int(lc.region_overflow.item()) == 0


def _runner_state(n=40, age=64):
    st = synthetic.make_loop_state("fast", n, period=12, radius=1.0, max_edge_age=age, device=DEV)
    return st


def test_loop_off_is_bit_identical_and_loop_on_runs_global_ba():
    stA, stB = _runner_state(), _runner_state()
    M, cap = stA.cfg["M"], stA.E + 1024
    gA = DevicePatchGraph(cap, M, stA.poses.shape[0] - 1, DEV)
    gB, lc = _setup(stB, loop_pairs=64, inactive=100000, capacity=cap, max_edge_age=64)
    for g, st in ((gA, stA), (gB, stB)):
        g.append(st.ii, st.jj, st.kk)
    rA = UpdateRunner(stA, graph=gA)
    rB = UpdateRunner(stB, graph=gB, loop=lc)
    for _ in range(2):
        rA.step()
        rB.step()
    torch.cuda.synchronize()
    assert torch.equal(stA.poses, stB.poses) and torch.equal(stA.patches, stB.patches)
    assert torch.equal(gA.net, gB.net[:, :gB.normal_cap])
    # a loop proposal at n, then one update: the whole store is stepped and the global bundle adjustment runs
    sc, pairs = _propose(stB, lc, stB.n)
    assert pairs, "the closed loop must give loop pairs"
    fl = lc.read_flags(stB.n)
    assert fl[0] and fl[1]
    p0 = stB.poses.clone()
    rB.step()
    torch.cuda.synchronize()
    assert stB.n in lc.ran_global_ba and torch.isfinite(stB.poses).all() and not torch.equal(p0, stB.poses)


def test_global_ba_matches_fp64_oracle_and_reference_kernels(ref_ext):
    st, g, lc, hg, n, _ = _drive(50)
    M = lc.M
    poses0, patches0 = st.poses.clone(), st.patches.clone()
    fl = lc.read_flags(n)
    count, E = fl[3], g.cap
    assert count > 0, "the drive must have moved edges to the inactive store"
    lo, hi = g.inactive_cap - count, g.inactive_cap + E
    loop_edges = (g.jj_all[lo:hi] - g.ii_all[lo:hi] > 30) & torch.cat([torch.ones(count, dtype=torch.bool, device=DEV),
                                                                       g.active.bool()])
    assert loop_edges.any(), "the problem must contain loop edges (jj - ii > 30)"
    g.weight.mul_(g.active.view(1, -1, 1))
    # targets: the reprojections plus half a pixel of noise (the driver's are random numbers)
    coords = synthetic_ext().reproject_clamped(st.poses.view(1, -1, 7), st.patches.view(1, -1, 3, 3, 3),
                                               st.intrinsics.view(1, -1, 4), g.ii_all[lo:hi], g.jj_all[lo:hi], g.kk_all[lo:hi])
    gen = torch.Generator(device=DEV).manual_seed(5)
    g.target_all[0, lo:hi] = coords[0, :, :, 1, 1] + 0.5 * torch.randn(hi - lo, 2, generator=gen, device=DEV)
    t0 = fl[2]
    lmbda = torch.tensor([1e-4], device=DEV)
    lc.global_ba(st.poses, st.patches, st.intrinsics, n, t0, count, E, lmbda)
    torch.cuda.synchronize()
    # the real edges only: the used inactive ones and the active ones (parked slots carry zero weight)
    real = torch.cat([torch.ones(count, dtype=torch.bool), g.active.bool().cpu()])
    edges = [x[lo:hi].cpu()[real] for x in (g.ii_all, g.jj_all, g.kk_all)]
    target, weight = g.target_all[0, lo:hi].cpu()[real], g.weight_all[0, lo:hi].cpu()[real]
    used = torch.unique(edges[2])
    used = used[used < n * M]

    rp, rq = OL.normalize(poses0.cpu(), patches0.cpu(), n, M)
    rp, rq = OB.fastba_forward(rp, rq, st.intrinsics.cpu().double(), target.double(), weight.double(),
                               torch.tensor([1e-4], dtype=torch.float64), *edges, t0, n, 2)
    ep = ((st.poses[:n].cpu().double() - rp[:n]).abs().max() / rp[:n].abs().max()).item()
    ed = ((st.patches[used, 2].cpu().double() - rq[used, 2]).abs().max() / rq[used, 2].abs().max()).item()
    assert ep < 1e-4 and ed < 1e-4, (ep, ed)
    if ref_ext is None:
        return
    # the reference's __run_global_BA path on the same edges: normalize, then its own eff_impl kernels
    p, q = poses0.clone(), patches0.clone()
    lc.normalize(p, q, n)
    d_edges = [x.to(DEV) for x in edges]
    ref_ext[1].forward(p.view(1, -1, 7), q.view(1, -1, 3, 3, 3), st.intrinsics.view(1, -1, 4), target.to(DEV)[None],
                       weight.to(DEV)[None], lmbda, *d_edges, M, t0, n, 2, True)
    torch.cuda.synchronize()
    ep = ((st.poses[:n] - p[:n]).abs().max() / p[:n].abs().max()).item()
    ed = ((st.patches[used, 2].cpu() - q[used, 2].cpu()).abs().max() / q[used, 2].cpu().abs().max()).item()
    assert ep < 1e-4 and ed < 1e-4, (ep, ed)


def synthetic_ext():
    import dpvo_b200
    return dpvo_b200.extensions()[3]


def _graph_setup(n0, frames):
    """a stream at n0 whose device frame counter will advance `frames` frames over a closed loop; the host n (the local
    bundle adjustment's window) stays at n0, as a captured step keeps it"""
    st = synthetic.make_loop_state("fast", n0 + frames, period=12, radius=1.0, max_edge_age=64, device=DEV)
    cfg, M = st.cfg, st.cfg["M"]
    ii, jj, kk = synthetic.replay_edges(n0, M, cfg["lifetime"], cfg["removal"])
    st.ii, st.jj, st.kk = ii.to(DEV), jj.to(DEV), kk.to(DEV)
    st.n, st.t0 = n0, n0 - cfg["opt_window"]
    g, lc = _setup(st, loop_pairs=64, inactive=200000, capacity=2 * st.E, max_edge_age=64)
    g.append(st.ii, st.jj, st.kk)
    run = UpdateRunner(st, graph=g, loop=lc)
    return st, g, lc, run


def test_captured_frame_replays_bit_equal_to_eager():
    n0, frames = 50, 20
    sA, gA, lA, rA = _graph_setup(n0, frames)
    sB, gB, lB, rB = _graph_setup(n0, frames)
    r = sA.cfg["lifetime"]
    nA, nB = _n(n0), _n(n0)

    def frame(st, g, lc, run, n_dev):
        lc.propose(st.poses, st.patches, st.intrinsics, n_dev)
        g.append_frame_edges(n_dev, r)
        run.step(loop_edges=True)
        lc.remove(n_dev)

    accepted_A, accepted_B = [], []
    for f in range(frames):
        nA.fill_(n0 + 1 + f)
        frame(sA, gA, lA, rA, nA)
        accepted_A.append(int(lA.n_pairs.item()))
    # B: the first frame eagerly (lazy initialisation stays out of the capture), the others as replays of one graph
    # that reads the frame counter from nB
    nB.fill_(n0 + 1)
    frame(sB, gB, lB, rB, nB)
    accepted_B.append(int(lB.n_pairs.item()))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        frame(sB, gB, lB, rB, nB)
    for f in range(1, frames):
        nB.fill_(n0 + 1 + f)
        graph.replay()
        accepted_B.append(int(lB.n_pairs.item()))
    torch.cuda.synchronize()
    assert accepted_A == accepted_B
    assert accepted_B[0] > 0 and any(k > 0 for k in accepted_B[1:]), accepted_B    # a replay accepted pairs
    assert torch.equal(lA.pairs, lB.pairs) and torch.equal(lA.last_global_ba, lB.last_global_ba)
    assert torch.equal(sA.poses, sB.poses) and torch.equal(sA.patches, sB.patches)
    for x, y in ((gA.ii_all, gB.ii_all), (gA.jj_all, gB.jj_all), (gA.kk_all, gB.kk_all), (gA.active, gB.active),
                 (gA.net, gB.net), (gA.target_all, gB.target_all), (gA.weight_all, gB.weight_all),
                 (lA.s_count, lB.s_count), (gA.n_active, gB.n_active)):
        assert torch.equal(x, y)
    assert int(lB.s_count.item()) > 0
