"""B camera streams stepped together (streams.StreamBatch, UpdateRunner on a batch, fastba.BA_batched) against the
same streams stepped one at a time.  Three streams with different seeds and frame counts, hence different windows
t0 / N_b, one of them with N_b < 10, on the default and the fast configuration."""
import pytest
import torch

from oracle import ba as OB
from dpvo_b200 import synthetic, fastba
from dpvo_b200.net import EdgeGroups
from dpvo_b200.runner import UpdateRunner
from dpvo_b200.patchgraph import DevicePatchGraph

pytestmark = pytest.mark.gpu
DEV = "cuda"
FRAMES = {"fast": [30, 5, 20], "default": [36, 8, 25]}      # N_b = 7, 4, 7 (fast) and 10, 7, 10 (default)
SEEDS = [11, 12, 13]


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp(min=1e-12)).item()


def _batch(config, frames=None, mem=36):
    return synthetic.make_batch(config, 3, SEEDS, n_frames=frames or FRAMES[config], device=DEV, frames_per_stream=64, mem=mem)


def _edge_ranges(batch):
    out, e0 = [], 0
    for b in range(batch.B):
        out.append((e0, e0 + batch.stream(b).E))
        e0 += batch.stream(b).E
    return out


# ------------------------------------------------------------------------------------------------ 1. BA alone
def _ba_targets(batch, seed):
    """per stream: reprojections under its own camera plus noise, confidence weights; concatenated in edge order"""
    g = torch.Generator().manual_seed(seed)
    tg, wg = [], []
    for b in range(batch.B):
        s = batch.stream(b)
        c = OB.fastba_reproject(s.poses.cpu().double(), s.patches.cpu().double(), s.intrinsics.cpu().double(),
                                s.ii.cpu(), s.jj.cpu(), s.kk.cpu())
        tg.append((c[:, :, 1, 1] + torch.randn(s.E, 2, generator=g).double()).float())
        wg.append(torch.rand(s.E, 2, generator=g))
    return torch.cat(tg).to(DEV), torch.cat(wg).to(DEV)


def _run_batched(batch, target, weight, iters=2):
    poses, patches = batch.poses.clone(), batch.patches.clone()
    gk, gp = EdgeGroups.pair((batch.kk, None, batch.jj), (batch.ii, batch.jj, None))
    t0s, t1s = batch.windows()
    fastba.BA_batched(poses.view(1, -1, 7), patches.view(1, -1, 3, 3, 3), batch.intrinsics.view(1, -1, 4), target[None],
                      weight[None], torch.tensor([1e-4], device=DEV), batch.ii, batch.jj, batch.kk, batch.F, t0s, t1s, iters,
                      gk, gp)
    torch.cuda.synchronize()
    return poses, patches


def _run_single(batch, b, target, weight, iters=2):
    s = batch.stream(b)
    poses, patches = s.poses.clone(), s.patches.clone()
    if s.E == 0:
        return poses, patches
    gk, gp = EdgeGroups.pair((s.kk, None, s.jj), (s.ii, s.jj, None))
    fastba.BA_grouped(poses.view(1, -1, 7), patches.view(1, -1, 3, 3, 3), s.intrinsics.view(1, -1, 4), target[None],
                      weight[None], torch.tensor([1e-4], device=DEV), s.ii, s.jj, s.kk, s.t0, s.n, iters, gk, gp)
    torch.cuda.synchronize()
    return poses, patches


def _single_takes_fast_path(N, E):
    """ba.cu's choice for one window: the fast path when 0 < N <= 12 and the per-SM partial systems fit the workspace"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n6 = 6 * N
    return 0 < N <= 12 and sms * (n6 * (n6 + 1) // 2 + n6) <= E * 90


@pytest.mark.parametrize("config", ["fast", "default"])
@pytest.mark.parametrize("path", ["fast", "general"])
def test_batched_ba_matches_each_stream_alone_and_the_oracle(ext, config, path):
    batch = _batch(config)
    if path == "general":                              # stream 0 opens a 28-free-pose window: the whole batch takes the general path
        batch.stream(0).t0 = batch.stream(0).n - 28
    # the streams have their own cameras: stream 1's focal lengths differ
    batch.stream(1).intrinsics[:, :2] *= 1.15
    target, weight = _ba_targets(batch, 5)
    F, M = batch.F, batch.M
    poses, patches = _run_batched(batch, target, weight)
    poses2, patches2 = _run_batched(batch, target, weight)
    assert torch.equal(poses, poses2) and torch.equal(patches, patches2), "two launches differ"
    lm = torch.tensor([1e-4], dtype=torch.float64)
    for b, (e0, e1) in enumerate(_edge_ranges(batch)):
        s = batch.stream(b)
        p1, q1 = _run_single(batch, b, target[e0:e1], weight[e0:e1])
        pb, qb = poses[b * F:(b + 1) * F], patches[b * F * M:(b + 1) * F * M]
        live = s.kk.unique()
        po, qo = OB.fastba_forward(s.poses.cpu().double(), s.patches.cpu().double(), s.intrinsics.cpu().double(),
                                   target[e0:e1].cpu().double(), weight[e0:e1].cpu().double(), lm, s.ii.cpu(), s.jj.cpu(),
                                   s.kk.cpu(), s.t0, s.n, 2)
        d_single = (_rel(pb[:s.n], p1[:s.n]), _rel(qb[live, 2], q1[live, 2]))
        d_oracle = (_rel(pb[:s.n].cpu(), po[:s.n]), _rel(qb[live, 2].cpu(), qo[live.cpu(), 2]))
        print("\n[%s %s] stream %d N_b=%d E=%d: vs BA_grouped alone pose %.3g depth %.3g (bit-equal %s), vs fp64 oracle "
              "pose %.3g depth %.3g" % (config, path, b, s.n - s.t0, s.E, *d_single,
                                        torch.equal(pb, p1) and torch.equal(qb, q1), *d_oracle))
        assert (pb - s.poses).abs().max() > 1e-4, "degenerate problem: BA did not move stream %d's poses" % b
        assert max(d_single) < 1e-4 and max(d_oracle) < 1e-4
        # where the stream alone takes the path the batch takes, the batched launch computes the same bits
        if (path == "fast") == _single_takes_fast_path(s.n - s.t0, s.E):
            assert torch.equal(pb, p1) and torch.equal(qb, q1), "stream %d differs from BA_grouped on the same path" % b
        # poses outside the window and every x / y stay untouched
        assert torch.equal(pb[:s.t0], s.poses[:s.t0]) and torch.equal(pb[s.n:], s.poses[s.n:])
        assert torch.equal(qb[:, :2], s.patches[:, :2])


def test_streams_without_edges_or_window_are_untouched_and_do_not_disturb_the_others(ext):
    batch = _batch("fast")
    F, M = batch.F, batch.M
    # stream 1 loses its edges; stream 2 keeps its edges but has an empty window
    keep = (batch.kk // (F * M)) != 1
    batch.set_edges(batch.ii[keep], batch.jj[keep], batch.kk[keep])
    batch.stream(2).t0 = batch.stream(2).n
    target, weight = _ba_targets(batch, 9)
    poses, patches = _run_batched(batch, target, weight)
    for b in (1, 2):
        assert torch.equal(poses[b * F:(b + 1) * F], batch.stream(b).poses), "stream %d's poses moved" % b
        assert torch.equal(patches[b * F * M:(b + 1) * F * M], batch.stream(b).patches), "stream %d's patches moved" % b
    e0, e1 = _edge_ranges(batch)[0]
    p1, q1 = _run_single(batch, 0, target[e0:e1], weight[e0:e1])
    s = batch.stream(0)
    assert _rel(poses[:s.n], p1[:s.n]) < 1e-5 and _rel(patches[s.kk.unique(), 2], q1[s.kk.unique(), 2]) < 1e-5
    # a batch in which no stream has a window is a no-op
    for b in range(3):
        batch.stream(b).t0 = batch.stream(b).n
    poses, patches = _run_batched(batch, target, weight)
    assert torch.equal(poses, batch.poses) and torch.equal(patches, batch.patches)


def test_batched_ba_rejects_wide_windows_and_bad_arguments(ext):
    batch = _batch("fast")
    target, weight = _ba_targets(batch, 1)
    gk, gp = EdgeGroups.pair((batch.kk, None, batch.jj), (batch.ii, batch.jj, None))
    args = lambda t0s, t1s, F=batch.F: (batch.poses.clone().view(1, -1, 7), batch.patches.clone().view(1, -1, 3, 3, 3),
                                        batch.intrinsics.view(1, -1, 4), target[None], weight[None],
                                        torch.tensor([1e-4], device=DEV), batch.ii, batch.jj, batch.kk, F, t0s, t1s, 2, gk, gp)
    t0s, t1s = batch.windows()
    with pytest.raises(RuntimeError, match="free poses"):
        fastba.BA_batched(*args([0] + t0s[1:], [33] + t1s[1:]))             # 33 free poses in stream 0
    with pytest.raises(RuntimeError, match="window"):
        fastba.BA_batched(*args(t0s, [t1s[0] + 64] + t1s[1:]))              # window reaches into stream 1
    with pytest.raises(RuntimeError, match="frames"):
        fastba.BA_batched(*args(t0s, t1s, F=48))
    with pytest.raises(RuntimeError, match="one entry per stream"):
        fastba.BA_batched(*args(t0s, t1s[:2]))


# ------------------------------------------------------------------------------------------------ 2./3. full step
@pytest.mark.parametrize("config", ["fast", "default"])
def test_batched_step_matches_each_stream_stepped_alone(ext, config):
    batch = _batch(config)
    singles = [batch.copy_stream(b) for b in range(batch.B)]
    run = UpdateRunner(batch, seed=5)
    tgt, wgt = run.step()
    torch.cuda.synchronize()
    F, M = batch.F, batch.M
    gkb, gpb = EdgeGroups.pair((batch.kk, None, batch.jj), (batch.ii, batch.jj, None))
    for b, (e0, e1) in enumerate(_edge_ranges(batch)):
        st = singles[b]
        r1 = UpdateRunner(st, update=run.update)
        t1, w1 = r1.step()
        torch.cuda.synchronize()
        assert torch.equal(run.corr_buf[0, e0:e1], r1.corr_buf[0]), "stream %d: correlation rows differ" % b
        # groupings: stream b's patch groups and pair groups, offsets removed, equal its own groupings
        gks, gps = EdgeGroups.pair((st.kk, None, st.jj), (st.ii, st.jj, None))
        for gb, gs, per in ((gkb, gks, F * M), (gpb, gps, F)):
            nb, ns = int(gb.n), int(gs.n)
            keys = gb.key_a[:nb]
            sel = torch.nonzero(torch.div(keys, per, rounding_mode="floor") == b).flatten()
            assert sel.numel() == ns and bool((sel[1:] - sel[:-1] == 1).all()), "stream %d's groups are not one range" % b
            g0, g1 = int(sel[0]), int(sel[-1]) + 1
            assert torch.equal(gb.key_a[g0:g1] - b * per, gs.key_a[:ns])
            if per == F:                               # the pair grouping's second key
                assert torch.equal(gb.key_b[g0:g1] - b * F, gs.key_b[:ns])
            starts = gb.group_start[g0:g1 + 1]
            assert torch.equal(starts - starts[0], gs.group_start[:ns + 1])
            assert torch.equal(gb.order[int(starts[0]):int(starts[-1])] - e0, gs.order[:st.E])
        s = batch.stream(b)
        live = st.kk.unique()
        d = dict(pose=_rel(s.poses[:s.n], st.poses[:st.n]), depth=_rel(s.patches[live, 2, 1, 1], st.patches[live, 2, 1, 1]),
                 target=(tgt[0, e0:e1] - t1[0]).abs().max().item(), weight=(wgt[0, e0:e1] - w1[0]).abs().max().item(),
                 net=(run.net[0, e0:e1] - r1.net[0]).abs().max().item())
        print("\n[%s] stream %d (E=%d, N_b=%d) batched vs alone: %s" % (config, b, st.E, st.n - st.t0,
                                                                      {k: "%.3g" % v for k, v in d.items()}))
        assert d["pose"] < 1e-4 and d["depth"] < 1e-4
        assert d["target"] < 1e-2 and d["weight"] < 5e-3 and d["net"] < 2e-2


def test_three_batched_updates_track_each_stream_alone(ext):
    batch = _batch("fast")
    singles = [batch.copy_stream(b) for b in range(batch.B)]
    run = UpdateRunner(batch, seed=5)
    runs = [UpdateRunner(st, update=run.update) for st in singles]
    ranges = _edge_ranges(batch)
    for it in range(3):
        run.step()
        for r in runs:
            r.step()
        torch.cuda.synchronize()
        for b, (e0, e1) in enumerate(ranges):
            s, st = batch.stream(b), singles[b]
            live = st.kk.unique()
            e_net = (run.net[0, e0:e1] - runs[b].net[0]).abs().max().item()
            e_pose = _rel(s.poses[:s.n], st.poses[:st.n])
            e_depth = _rel(s.patches[live, 2, 1, 1], st.patches[live, 2, 1, 1])
            print("update %d stream %d: net abs %.3g, pose rel %.3g, depth rel %.3g" % (it, b, e_net, e_pose, e_depth))
            assert e_net < 5e-2 and e_pose < 2e-3 and e_depth < 2e-2


# ------------------------------------------------------------------------------------------------ 4. graphs
def test_captured_batched_step_replays_bit_equal_to_eager(ext):
    batch = _batch("fast")
    run = UpdateRunner(batch, seed=5)
    poses0, patches0 = batch.poses.clone(), batch.patches.clone()
    run.capture()
    run.reset(); run.net.zero_()
    tgt, wgt = run.step()
    torch.cuda.synchronize()
    eager = [t.clone() for t in (batch.poses, batch.patches, tgt, wgt, run.net, run.corr_buf)]
    run.reset(); run.net.zero_()
    assert torch.equal(batch.poses, poses0) and torch.equal(batch.patches, patches0)
    tgt, wgt = run.step_graph()
    torch.cuda.synchronize()
    for a, b in zip(eager, (batch.poses, batch.patches, tgt, wgt, run.net, run.corr_buf)):
        assert torch.equal(a, b), "graph replay differs from eager launches"


def test_stacked_store_graph_survives_per_stream_topology_changes(ext):
    batch = _batch("fast")
    B, F, M = batch.B, batch.F, batch.M
    dummies = [b * F + F - 1 for b in range(B)]
    store, graphs = DevicePatchGraph.stacked(B, max(batch.stream(b).E for b in range(B)) + 700, M, dummies)
    for b, g in enumerate(graphs):
        s = batch.stream(b)
        g.append(*batch.to_global(b, s.ii, s.jj, s.kk))
    run = UpdateRunner(batch, graph=store, seed=5)
    poses0, patches0 = batch.poses.clone(), batch.patches.clone()
    run.capture()
    dev = lambda v: torch.tensor([v], dtype=torch.long, device=DEV)
    for round_ in range(4):
        before = [t.clone() for t in (store.ii, store.jj, store.kk, store.active)]
        if round_ == 1:                                # stream 0: drop the edges of its oldest live frame's patches
            g = graphs[0]
            oldest = int((g.kk[g.active.bool()] // M).min())
            g.remove_old(dev(oldest + 1 + 16), 16)
        if round_ == 2:                                # stream 2: keyframe removal of frame n - 3 (global numbering)
            s = batch.stream(2)
            graphs[2].remove_frame(dev(2 * F + s.n - 3))
        if round_ == 3:                                # stream 1: new edges into its parked slots
            s = batch.stream(1)
            k_new = torch.arange(M * (s.n - 1), M * s.n, device=DEV).repeat_interleave(3)
            j_new = torch.arange(s.n - 3, s.n, device=DEV).repeat(M)
            graphs[1].append(*batch.to_global(1, k_new // M, j_new, k_new))
        changed = {1: 0, 2: 2, 3: 1}.get(round_)
        cap = graphs[0].cap
        for b in range(B):
            if b != changed:                           # the other streams' slices are bit-unchanged
                sl = slice(b * cap, (b + 1) * cap)
                assert all(torch.equal(x[sl], y[sl]) for x, y in zip(before, (store.ii, store.jj, store.kk, store.active)))
        if changed is not None:
            sl = slice(changed * cap, (changed + 1) * cap)
            assert not all(torch.equal(x[sl], y[sl]) for x, y in zip(before, (store.ii, store.jj, store.kk, store.active)))
        state_rows = store.net.clone()
        batch.poses.copy_(poses0); batch.patches.copy_(patches0)
        tgt_e, wgt_e = run.step()
        torch.cuda.synchronize()
        eager = [t.clone() for t in (batch.poses, batch.patches, tgt_e, wgt_e, store.net)]
        store.net.copy_(state_rows)
        batch.poses.copy_(poses0); batch.patches.copy_(patches0)
        tgt_g, wgt_g = run.step_graph()
        torch.cuda.synchronize()
        for a, b_ in zip(eager, (batch.poses, batch.patches, tgt_g, wgt_g, store.net)):
            assert torch.equal(a, b_), "graph replay differs from eager launches in round %d" % round_
        parked = ~store.active.bool()
        assert (wgt_g[0][parked] == 0).all(), "parked edges must carry zero confidence"
        # parked slots point at their own stream's reserved frame
        for b in range(B):
            sl = slice(b * cap, (b + 1) * cap)
            assert bool((store.ii[sl][parked[sl]] == dummies[b]).all())
        for g in graphs:
            assert int(g.overflow) == 0


# ------------------------------------------------------------------------------------------------ 5. encoding
def test_ingest_image_writes_only_its_streams_slots(ext):
    from dpvo_b200 import frontend
    batch = _batch("fast", frames=[12, 9, 14], mem=16)
    torch.manual_seed(4)
    fe = frontend.FrameEncoder(frontend.Patchifier().cuda().eval())
    run = UpdateRunner(batch, encoder=fe)
    for t in (batch.fmap1, batch.fmap2, batch.gmap, batch.imap):
        t.fill_(7.0)
    batch.patches.fill_(-3.0)
    names = ("fmap1", "fmap2", "gmap", "imap", "patches", "poses", "intrinsics")
    before = {k: getattr(batch, k).clone() for k in names}
    img = torch.randint(0, 256, (3, 480, 752), dtype=torch.uint8, device=DEV)
    b = 1
    s = batch.stream(b)
    torch.manual_seed(21)
    run.ingest_image(img, depth=torch.tensor(0.5, device=DEV), stream=b)
    torch.cuda.synchronize()
    M, mem, pmem, F = batch.M, batch.mem, batch.pmem, batch.F
    slot, pslot = b * mem + (s.n - 1) % mem, b * pmem * M + ((s.n - 1) % pmem) * M
    written = {"fmap1": (1, slot, slot + 1), "fmap2": (1, slot, slot + 1), "gmap": (1, pslot, pslot + M),
               "imap": (1, pslot, pslot + M), "patches": (0, b * F * M + (s.n - 1) * M, b * F * M + s.n * M)}
    for k in names:
        a, o = getattr(batch, k), before[k]
        if k not in written:
            assert torch.equal(a, o), k
            continue
        dim, lo, hi = written[k]
        assert not torch.equal(a.narrow(dim, lo, hi - lo), o.narrow(dim, lo, hi - lo)), k
        assert torch.equal(a.narrow(dim, 0, lo), o.narrow(dim, 0, lo)), k
        assert torch.equal(a.narrow(dim, hi, a.shape[dim] - hi), o.narrow(dim, hi, a.shape[dim] - hi)), k
    assert bool((batch.patches[b * F * M + (s.n - 1) * M:b * F * M + s.n * M, 2] == 0.5).all())
    # the same image encoded by a single-stream runner writes the same bytes
    st = batch.copy_stream(b)
    r1 = UpdateRunner(st, encoder=fe, update=run.update)
    torch.manual_seed(21)
    r1.ingest_image(img, depth=torch.tensor(0.5, device=DEV))
    torch.cuda.synchronize()
    ls = (s.n - 1) % mem
    assert torch.equal(st.fmap1[0, ls], batch.fmap1[0, slot]) and torch.equal(st.imap[0, ((s.n - 1) % pmem) * M:((s.n - 1) % pmem + 1) * M],
                                                                             batch.imap[0, pslot:pslot + M])
    with pytest.raises(RuntimeError, match="stream=b"):
        run.ingest_image(img)
    with pytest.raises(RuntimeError, match="one stream"):
        r1.ingest_image(img, stream=0)
