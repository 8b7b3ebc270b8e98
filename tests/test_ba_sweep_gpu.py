"""Bundle adjustment at every window width the on-chip solver holds, on both of its solve paths and in batches of 1 to
64 streams, against the fp64 oracle (oracle.ba.fastba_forward).

ba.cu branches on N = t1 - t0, the number of free poses:
  fast path     0 < N <= 12 and sm_count * 6N(6N+3)/2 <= 90 E (single window; the batched entry takes it whenever
                every window is at most 12 wide): the reduce kernel builds packed per-SM partial reduced systems
  general path  otherwise, up to N = 32: the 8-CTA solve cluster forms the reduced system itself -- Schur products in
                32-patch chunks, pair records staged 64 at a time, Cholesky in 6-column panels
  wide path     N > 32 or eff_impl=True (ba_wide.cu)
Every problem states the path it means to reach and asserts that takes_fast_path agrees, so a device with another SM
count fails here instead of quietly testing the other path.  Where two entries take different paths their sums run in
different orders and their bits differ; where they take the same path their bits are equal.

The bar everywhere: the window's poses and the inverse depths of every patch an edge refers to within 1e-4 relative of
the oracle; poses outside the window, patch x / y and patches without edges bit-identical; every problem moves its
poses (no test passes on a no-op)."""
import pytest
import torch

from oracle import ba as OB
from dpvo_b200 import synthetic, fastba
from dpvo_b200.net import EdgeGroups

pytestmark = pytest.mark.gpu
DEV = "cuda"
ITERS = 2
LMBDA = 1e-4
BAR = 1e-4                    # device vs fp64 oracle
# one problem through two entries that sum in different orders.  On two large sliding windows the entries agree to
# 1e-5 (test_ba_grouped_entry_matches_plain_entry); the streams here are small, with few edges per patch, and a depth
# update Q_k (u_k - E_k dX) of such a patch amplifies the last bits of the pose step: the 64-stream batch with only its
# edges shuffled -- the same path, the group members in another order -- moves poses by 1.5e-5 and depths by 2.4e-5
PATH_BAR = 5e-5
BA_FAST_MAX_N, BA_MAX_N, BA_MAX_STREAMS = 12, 32, 64
BA_CLUSTER, BA_ECH, BA_REC_CHUNK, BA_REC = 8, 32, 64, 90


# ------------------------------------------------------------------------------------------------ paths
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _packed_entries(N):
    n6 = 6 * N
    return n6 * (n6 + 1) // 2 + n6


def takes_fast_path(N, E):
    """ba_run's choice for one window (cuda_ba.forward, BA_grouped) on this device: the fast path when 0 < N <= 12 and
    the sm_count packed partial systems fit where the E pair records of the general path would go"""
    return 0 < N <= BA_FAST_MAX_N and _sms() * _packed_entries(N) <= E * BA_REC


def batched_takes_fast_path(Ns):
    """dpvo_ba_forward_batched's choice: the fast path for the whole batch when every window is at most 12 wide"""
    return 0 < max(Ns) <= BA_FAST_MAX_N


def fast_edge_bound(N):
    """the fewest edges with which a window of N free poses takes the fast path"""
    return -(-_sms() * _packed_entries(N) // BA_REC)


# ------------------------------------------------------------------------------------------------ problems
def make_problem(n_frames, N, M, seed, edge_fraction=1.0, lifetime=6, focal=1.0, buffer=None, sigma=1.0):
    """A sliding-window problem on synthetic.make_state(features=False): frames [0, n_frames), the window is the last N
    of them (N = 0: an empty window at t0 = t1 = n_frames), M patches per frame.  Every edge of the replayed graph is
    kept (the removal window is longer than the video) unless edge_fraction < 1, which keeps that share of the edges at
    random and then one more edge between two different frames on every free pose that lost all of its own.  Targets
    are the fp64 reprojections under the problem's camera (focal lengths scaled by `focal`) plus `sigma` px of noise;
    weights lie in (0, 1).  Returns (state, target, weight, t0, t1)."""
    assert 0 <= N < n_frames
    cfg = dict(M=M, lifetime=lifetime, removal=n_frames + 1, opt_window=N, ht=480, wd=640,
               intrinsics=(320.0 * focal, 321.0 * focal, 320.0, 240.0))
    buffer = n_frames + 1 if buffer is None else buffer
    st = synthetic.make_state(cfg, n_frames, device="cpu", features=False, seed=seed, buffer=buffer, mem=n_frames)
    t0, t1 = n_frames - N, n_frames
    st.t0 = t0
    g = torch.Generator().manual_seed(seed + 1)
    if edge_fraction < 1.0:
        perm = torch.randperm(st.E, generator=g)
        keep = torch.zeros(st.E, dtype=torch.bool)
        keep[perm[:max(1, int(edge_fraction * st.E))]] = True
        for p in range(t0, t1):
            touch = (st.ii == p) | (st.jj == p)
            if not bool((keep & touch & (st.ii != st.jj)).any()):
                cand = perm[(touch & (st.ii != st.jj))[perm]]
                keep[cand[0]] = True
        st.ii, st.jj, st.kk = st.ii[keep], st.jj[keep], st.kk[keep]
    target, weight = _targets(st, g, sigma)
    return st, target, weight, t0, t1


def _targets(st, g, sigma=1.0):
    coords = OB.fastba_reproject(st.poses.double(), st.patches.double(), st.intrinsics.double(), st.ii, st.jj, st.kk)
    target = (coords[:, :, 1, 1] + sigma * torch.randn(st.E, 2, generator=g).double()).float()
    weight = torch.rand(st.E, 2, generator=g).clamp(min=1e-3)
    return target, weight


def _keep_edges(st, keep):
    st.ii, st.jj, st.kk = st.ii[keep], st.jj[keep], st.kk[keep]


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-12)).item()


# ------------------------------------------------------------------------------------------------ entries
def oracle(st, target, weight, t0, t1):
    threads = torch.get_num_threads()
    torch.set_num_threads(1)          # systems of at most 192 unknowns: starting the thread pool costs more than the work
    try:
        return OB.fastba_forward(st.poses.double(), st.patches.double(), st.intrinsics.double(), target.double(),
                                 weight.double(), torch.tensor([LMBDA], dtype=torch.float64), st.ii, st.jj, st.kk, t0, t1,
                                 ITERS)
    finally:
        torch.set_num_threads(threads)


def run_forward(mod, st, target, weight, t0, t1, eff_impl=False):
    """cuda_ba.forward (ours or the reference's): builds its own groupings"""
    poses, patches = st.poses.clone().to(DEV)[None], st.patches.clone().to(DEV)[None]
    mod.forward(poses, patches, st.intrinsics.to(DEV)[None], target.to(DEV)[None], weight.to(DEV)[None],
                torch.tensor([LMBDA], device=DEV), st.ii.to(DEV), st.jj.to(DEV), st.kk.to(DEV), st.cfg["M"], t0, t1, ITERS,
                eff_impl)
    torch.cuda.synchronize()
    return poses[0].cpu(), patches[0].cpu()


def _groups(ii, jj, kk):
    return EdgeGroups.pair((kk, None, jj), (ii, jj, None))


def run_grouped(st, target, weight, t0, t1):
    ii, jj, kk = st.ii.to(DEV), st.jj.to(DEV), st.kk.to(DEV)
    poses, patches = st.poses.clone().to(DEV)[None], st.patches.clone().to(DEV)[None]
    if ii.numel():
        gk, gp = _groups(ii, jj, kk)
        fastba.BA_grouped(poses, patches, st.intrinsics.to(DEV)[None], target.to(DEV)[None], weight.to(DEV)[None],
                          torch.tensor([LMBDA], device=DEV), ii, jj, kk, t0, t1, ITERS, gk, gp)
        torch.cuda.synchronize()
    return poses[0].cpu(), patches[0].cpu()


def run_batched(poses, patches, intrinsics, target, weight, ii, jj, kk, F, t0s, t1s):
    """BA_batched over streams of F frames each; all tensors global (stream b owns frames [b F, (b+1) F))"""
    ii, jj, kk = ii.to(DEV), jj.to(DEV), kk.to(DEV)
    poses, patches = poses.clone().to(DEV), patches.clone().to(DEV)
    gk, gp = _groups(ii, jj, kk)
    fastba.BA_batched(poses[None], patches[None], intrinsics.to(DEV)[None], target.to(DEV)[None], weight.to(DEV)[None],
                      torch.tensor([LMBDA], device=DEV), ii, jj, kk, F, t0s, t1s, ITERS, gk, gp)
    torch.cuda.synchronize()
    return poses.cpu(), patches.cpu()


def run_batched_one(st, target, weight, t0, t1):
    """BA_batched with B = 1: the problem as the only stream"""
    return run_batched(st.poses, st.patches, st.intrinsics, target, weight, st.ii, st.jj, st.kk, st.poses.shape[0],
                       [t0], [t1])


# ------------------------------------------------------------------------------------------------ checks
def check_oracle(tag, st, t0, t1, out, ref):
    """the north-star bar for one result; returns (pose, depth) relative errors"""
    poses, patches = out
    rp, rq = ref
    live = st.kk.unique()
    dead = torch.ones(patches.shape[0], dtype=torch.bool)
    dead[live] = False
    e = (_rel(poses[t0:t1], rp[t0:t1]) if t1 > t0 else 0.0, _rel(patches[live, 2], rq[live, 2]))
    print("  %-34s vs oracle: pose %.3g depth %.3g" % (tag, *e))
    assert torch.isfinite(poses).all() and torch.isfinite(patches).all(), tag
    assert e[0] < BAR and e[1] < BAR, "%s: pose %.3g depth %.3g vs the fp64 oracle" % (tag, *e)
    assert torch.equal(poses[:t0], st.poses[:t0]) and torch.equal(poses[t1:], st.poses[t1:]), \
        "%s: a pose outside the window moved" % tag
    assert torch.equal(patches[:, :2], st.patches[:, :2]), "%s: patch x / y moved" % tag
    assert torch.equal(patches[dead], st.patches[dead]), "%s: a patch without edges moved" % tag
    if t1 > t0:
        assert (poses[t0:t1] - st.poses[t0:t1]).abs().max() > 1e-4, "%s: degenerate problem, the poses did not move" % tag
    return e


def check_same_problem(tag, a, b, same_path, st):
    """two entries on one problem: equal bits on the same path; otherwise within PATH_BAR and NOT the same bits (equal
    bits from two paths would mean that one entry did not take the path it was meant to)"""
    live = st.kk.unique()
    bit_equal = torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    d = (_rel(a[0], b[0]), _rel(a[1][live, 2], b[1][live, 2]))
    print("  %-34s pose %.3g depth %.3g, bit-equal %s (same path: %s)" % (tag, *d, bit_equal, same_path))
    if same_path:
        assert bit_equal, "%s: the same path gave different bits" % tag
    else:
        assert max(d) < PATH_BAR, "%s: the two paths differ by pose %.3g depth %.3g" % (tag, *d)
        assert not bit_equal, "%s: two paths gave identical bits -- one entry took the other path" % tag


def solve_everywhere(st, target, weight, t0, t1, ref_ext=None, ext=None):
    """cuda_ba.forward, BA_grouped and BA_batched (B = 1) on one problem, each against the oracle; the reference's own
    cuda_ba.forward too when it is built.  Returns the results."""
    N, E = t1 - t0, st.E
    ref = oracle(st, target, weight, t0, t1)
    assert (ref[0] - st.poses.double()).abs().max() > 1e-4, "degenerate problem: the oracle did not move the poses"
    single_fast = takes_fast_path(N, E)
    batch_fast = batched_takes_fast_path([N])
    print("\nN=%d E=%d patches=%d: single window %s path, batched %s path" % (
        N, E, st.kk.unique().numel(), "fast" if single_fast else "general", "fast" if batch_fast else "general"))
    out = {}
    if ext is not None:
        out["forward"] = run_forward(ext[1], st, target, weight, t0, t1)
    out["grouped"] = run_grouped(st, target, weight, t0, t1)
    out["batched"] = run_batched_one(st, target, weight, t0, t1)
    if ref_ext is not None:
        out["reference"] = run_forward(ref_ext[1], st, target, weight, t0, t1)
    for k, v in out.items():
        check_oracle(k, st, t0, t1, v, ref)
    check_same_problem("batched (B=1) vs grouped", out["batched"], out["grouped"], single_fast == batch_fast, st)
    if "forward" in out:          # same path, kk group members in another order
        live = st.kk.unique()
        d = (_rel(out["forward"][0], out["grouped"][0]), _rel(out["forward"][1][live, 2], out["grouped"][1][live, 2]))
        assert max(d) < PATH_BAR, "forward vs grouped: pose %.3g depth %.3g" % d
    return out, ref


# ------------------------------------------------------------------------------------------------ 0. the fast-path width
def test_library_fast_path_width(ext):
    """the batched workspace holds one set of sm_count packed partial systems per stream exactly when the batch takes
    the fast path: read the library's fast-path width from it"""
    E = 5000
    for N in range(1, BA_MAX_N + 1):
        per_stream = ext[3].ba_batched_workspace_bytes(E, 2, N) - ext[3].ba_batched_workspace_bytes(E, 1, N)
        parts = _sms() * _packed_entries(N) * 4
        if batched_takes_fast_path([N]):
            assert per_stream >= parts, "N=%d: the library does not take the fast path (%d B per stream)" % (N, per_stream)
        else:
            assert per_stream < 1024, "N=%d: the library takes the fast path (%d B per stream)" % (N, per_stream)


# ------------------------------------------------------------------------------------------------ 1./2./3. width sweep
def _general_problem(N, seed):
    """a problem that takes the general path: for N <= 12, 4 patches per frame and 80 % of the edges (at most 90 % of
    the fast-path bound), so that every patch keeps a few edges; wider windows keep every edge of 8 patches per frame"""
    n_frames = N + 2
    if N > BA_FAST_MAX_N:
        return make_problem(n_frames, N, 8, seed)
    st, *_ = make_problem(n_frames, N, 4, seed)
    return make_problem(n_frames, N, 4, seed, edge_fraction=min(0.8, 0.9 * fast_edge_bound(N) / st.E))


def _fast_problem(N, seed):
    """a problem that takes the fast path: E well above the fast-path bound"""
    return make_problem(N + 2, N, 48, seed)


@pytest.mark.parametrize("N", range(1, BA_MAX_N + 1))
def test_width_sweep_general_path(ext, ref_ext, N):
    st, target, weight, t0, t1 = _general_problem(N, 100 + N)
    assert not takes_fast_path(N, st.E), "N=%d E=%d was meant for the general path" % (N, st.E)
    assert batched_takes_fast_path([N]) == (N <= BA_FAST_MAX_N)
    solve_everywhere(st, target, weight, t0, t1, ref_ext, ext)


@pytest.mark.parametrize("N", range(1, BA_FAST_MAX_N + 1))
def test_width_sweep_fast_path(ext, ref_ext, N):
    st, target, weight, t0, t1 = _fast_problem(N, 200 + N)
    assert takes_fast_path(N, st.E), "N=%d E=%d was meant for the fast path" % (N, st.E)
    solve_everywhere(st, target, weight, t0, t1, ref_ext, ext)


# ------------------------------------------------------------------------------------------------ 4. structure
STRUCT_N = 8


def _struct_problem(seed, n_frames=STRUCT_N + 2, M=8):
    """N = 8 with E below the fast-path bound: BA_grouped takes the general path, BA_batched the fast path"""
    return make_problem(n_frames, STRUCT_N, M, seed, lifetime=5)


def _both_paths(st, target, weight, t0, t1, ext):
    assert not takes_fast_path(t1 - t0, st.E) and batched_takes_fast_path([t1 - t0]), "meant for both paths"
    return solve_everywhere(st, target, weight, t0, t1, None, ext)


def test_free_pose_without_edges(ext):
    st, _, _, t0, t1 = _struct_problem(301)
    p = t0 + 3
    _keep_edges(st, (st.ii != p) & (st.jj != p))
    target, weight = _targets(st, torch.Generator().manual_seed(1))
    out, ref = _both_paths(st, target, weight, t0, t1, ext)
    # its block is the damping identity and its gradient zero: a zero step
    assert torch.allclose(ref[0][p], st.poses[p].double(), rtol=0, atol=1e-12)
    for k, (poses, _) in out.items():
        assert (poses[p] - st.poses[p]).abs().max() <= 1e-6, "%s: the pose without edges moved" % k


@pytest.mark.parametrize("side", ["source_only", "target_only"])
def test_free_pose_seen_from_one_side(ext, side):
    st, _, _, t0, t1 = _struct_problem(302)
    p = t0 + 2
    if side == "source_only":                  # pose p appears only as ii
        keep = st.jj != p
        _keep_edges(st, keep)
        assert bool((st.ii == p).any()) and not bool((st.jj == p).any())
    else:
        _keep_edges(st, st.ii != p)
        assert bool((st.jj == p).any()) and not bool((st.ii == p).any())
    target, weight = _targets(st, torch.Generator().manual_seed(2))
    _both_paths(st, target, weight, t0, t1, ext)


def test_self_edges_inside_the_window(ext):
    st, target, weight, t0, t1 = _struct_problem(303)
    self_e = (st.ii == st.jj) & (st.ii >= t0)
    assert int(self_e.sum()) >= STRUCT_N * st.cfg["M"], "the replayed graph (__edges_back) carries self edges"
    _both_paths(st, target, weight, t0, t1, ext)


def test_frame_pair_with_zero_weights(ext):
    st, target, weight, t0, t1 = _struct_problem(304)
    pair = (st.ii == t0 + 1) & (st.jj == t0 + 4)
    assert int(pair.sum()) > 0
    weight[pair] = 0.0
    _both_paths(st, target, weight, t0, t1, ext)


def _patch_subset(st, n_groups, seed):
    """keep the edges of n_groups patches chosen at random: exactly n_groups patch groups"""
    live = st.kk.unique()
    sel = live[torch.randperm(live.numel(), generator=torch.Generator().manual_seed(seed))[:n_groups]]
    keep = torch.isin(st.kk, sel)
    _keep_edges(st, keep)
    assert st.kk.unique().numel() == n_groups


def test_fewer_patch_groups_than_cluster_ctas(ext):
    """5 patch groups over the 8 CTAs of the solve cluster: three CTAs own no patch"""
    st, _, _, t0, t1 = make_problem(4, 2, 8, 305)
    # one patch of every frame plus one more of frame 0: every free pose is a target of several of them
    sel = torch.tensor([0, 8, 16, 24, 3])
    _keep_edges(st, torch.isin(st.kk, sel))
    assert st.kk.unique().numel() == 5 < BA_CLUSTER
    target, weight = _targets(st, torch.Generator().manual_seed(3))
    assert not takes_fast_path(t1 - t0, st.E)
    solve_everywhere(st, target, weight, t0, t1, None, ext)


@pytest.mark.parametrize("n_groups", [BA_CLUSTER * BA_ECH - 1, BA_CLUSTER * BA_ECH, BA_CLUSTER * BA_ECH + 1])
def test_patch_groups_at_schur_chunk_edges(ext, n_groups):
    """8 x 32 - 1, 8 x 32 and 8 x 32 + 1 patch groups: each cluster CTA's slice ends one short of, at, or one past a
    32-patch Schur chunk (N = 10: BA_grouped on the general path, BA_batched on the fast path)"""
    st, _, _, t0, t1 = make_problem(12, 10, 32, 306 + n_groups, lifetime=5)
    _patch_subset(st, n_groups, n_groups)
    target, weight = _targets(st, torch.Generator().manual_seed(n_groups))
    assert not takes_fast_path(t1 - t0, st.E) and batched_takes_fast_path([t1 - t0])
    solve_everywhere(st, target, weight, t0, t1, None, ext)


@pytest.mark.parametrize("n_pairs", [BA_CLUSTER * BA_REC_CHUNK - 1, BA_CLUSTER * BA_REC_CHUNK, BA_CLUSTER * BA_REC_CHUNK + 1])
def test_pair_groups_at_record_chunk_edges(ext, n_pairs):
    """8 x 64 - 1, 8 x 64 and 8 x 64 + 1 frame-pair groups: each cluster CTA stages its pair records in one round of 64
    or spills one record into a second round (N = 22, general path on every entry)"""
    n_frames = 24
    st, _, _, t0, t1 = make_problem(n_frames, 22, 3, 309, lifetime=n_frames + 1)     # every patch sees every frame
    assert st.E == n_frames * 3 * n_frames
    g = torch.Generator().manual_seed(n_pairs)
    pair_id = st.ii * n_frames + st.jj
    cross = torch.tensor([i * n_frames + j for i in range(n_frames) for j in range(n_frames) if i != j])
    drop = cross[torch.randperm(cross.numel(), generator=g)[:n_frames * n_frames - n_pairs]]
    _keep_edges(st, ~torch.isin(pair_id, drop))
    assert torch.unique(st.ii * n_frames + st.jj).numel() == n_pairs
    target, weight = _targets(st, g)
    assert not batched_takes_fast_path([t1 - t0])
    solve_everywhere(st, target, weight, t0, t1, None, ext)


# ------------------------------------------------------------------------------------------------ 5. batched entry
def _stack(problems, F, M):
    """concatenate single-stream problems of F pose slots each into one batch (global frame and patch numbers)"""
    cat = lambda xs: torch.cat(xs)
    poses = cat([p[0].poses for p in problems])
    patches = cat([p[0].patches for p in problems])
    intr = cat([p[0].intrinsics for p in problems])
    ii = cat([p[0].ii + b * F for b, p in enumerate(problems)])
    jj = cat([p[0].jj + b * F for b, p in enumerate(problems)])
    kk = cat([p[0].kk + b * F * M for b, p in enumerate(problems)])
    target, weight = cat([p[1] for p in problems]), cat([p[2] for p in problems])
    t0s = [b * F + p[3] for b, p in enumerate(problems)]
    t1s = [b * F + p[4] for b, p in enumerate(problems)]
    return poses, patches, intr, target, weight, ii, jj, kk, t0s, t1s


@pytest.mark.parametrize("N", [1, BA_FAST_MAX_N, BA_FAST_MAX_N + 1, BA_MAX_N])
def test_batched_single_stream_at_its_limits(ext, N):
    """B = 1 against BA_grouped on the same stream and against the oracle; the stream's problem is small, so BA_grouped
    takes the general path and the batch the fast path up to N = 12"""
    st, target, weight, t0, t1 = _general_problem(N, 400 + N)
    assert not takes_fast_path(N, st.E)
    assert batched_takes_fast_path([N]) == (N <= BA_FAST_MAX_N)
    solve_everywhere(st, target, weight, t0, t1, None, None)


B64_M, B64_LIFETIME = 8, 4


@pytest.mark.parametrize("mode", ["fast", "general"])
def test_batched_64_streams(ext, mode):
    """BA_MAX_STREAMS streams, each with its own camera, windows cycling through 0..12 (the whole batch on the fast path)
    or 0..32 (general path).  Every stream equals BA_grouped on the stream alone -- bit-identical where both take the
    same path, within PATH_BAR otherwise -- and the oracle; streams with an empty window are bit-unchanged.  The same
    edges interleaved across the streams give the same result within PATH_BAR."""
    B, M = BA_MAX_STREAMS, B64_M
    cycle = BA_FAST_MAX_N + 1 if mode == "fast" else BA_MAX_N + 1
    Ns = [b % cycle for b in range(B)]
    F = max(Ns) + 3
    problems = [make_problem(N + 2, N, M, 500 + b, lifetime=B64_LIFETIME, focal=0.8 + 0.01 * b, buffer=F)
                for b, N in enumerate(Ns)]
    assert batched_takes_fast_path(Ns) == (mode == "fast")
    poses, patches, intr, target, weight, ii, jj, kk, t0s, t1s = _stack(problems, F, M)
    assert len(set(intr[::F, 0].tolist())) == B, "every stream has its own focal length"
    out = run_batched(poses, patches, intr, target, weight, ii, jj, kk, F, t0s, t1s)
    batch_fast = batched_takes_fast_path(Ns)
    n_same = 0
    for b, (st, tg, wt, t0, t1) in enumerate(problems):
        pb, qb = out[0][b * F:(b + 1) * F], out[1][b * F * M:(b + 1) * F * M]
        if t1 == t0:
            assert torch.equal(pb, st.poses) and torch.equal(qb, st.patches), "stream %d (empty window) changed" % b
            continue
        print("stream %d: N=%d E=%d" % (b, t1 - t0, st.E))
        ref = oracle(st, tg, wt, t0, t1)
        check_oracle("stream %d batched" % b, st, t0, t1, (pb, qb), ref)
        same = takes_fast_path(t1 - t0, st.E) == batch_fast
        n_same += same
        check_same_problem("stream %d vs grouped alone" % b, (pb, qb), run_grouped(st, tg, wt, t0, t1), same, st)
    print("%d of %d streams on the batch's path when alone" % (n_same, B))
    # the streams' edges interleaved: the device finds each stream's groups from the sorted keys alone
    perm = torch.randperm(ii.numel(), generator=torch.Generator().manual_seed(7))
    assert not torch.equal(perm, torch.arange(ii.numel()))
    shuf = run_batched(poses, patches, intr, target[perm], weight[perm], ii[perm], jj[perm], kk[perm], F, t0s, t1s)
    live = kk.unique()
    d = (_rel(shuf[0], out[0]), _rel(shuf[1][live, 2], out[1][live, 2]))
    print("interleaved edges vs stream order: pose %.3g depth %.3g" % d)
    assert max(d) < PATH_BAR
    assert torch.equal(shuf[0][:t0s[0]], poses[:t0s[0]]) and torch.equal(shuf[1][:, :2], patches[:, :2])
    for b, (st, tg, wt, t0, t1) in enumerate(problems):
        if t1 > t0 and b % 8 == 1:            # a sample of streams against the oracle (all are within PATH_BAR of the above)
            check_oracle("stream %d interleaved" % b, st, t0, t1,
                         (shuf[0][b * F:(b + 1) * F], shuf[1][b * F * M:(b + 1) * F * M]), oracle(st, tg, wt, t0, t1))


def test_batched_rejects_65_streams(ext):
    B, M, F = BA_MAX_STREAMS + 1, 2, 4
    problems = [make_problem(3, 1, M, 600 + b, buffer=F) for b in range(B)]
    poses, patches, intr, target, weight, ii, jj, kk, t0s, t1s = _stack(problems, F, M)
    with pytest.raises(RuntimeError, match="65 streams > 64"):
        run_batched(poses, patches, intr, target, weight, ii, jj, kk, F, t0s, t1s)


def test_empty_window_batched_untouched_single_structure_only(ext):
    """t1 == t0: the batched entry leaves the stream untouched; BA_grouped (and cuda_ba.forward) run the structure-only
    step that updates the depths alone"""
    M, F = 8, 10
    problems = [make_problem(8, 5, M, 700, buffer=F), make_problem(8, 0, M, 701, buffer=F)]
    poses, patches, intr, target, weight, ii, jj, kk, t0s, t1s = _stack(problems, F, M)
    out = run_batched(poses, patches, intr, target, weight, ii, jj, kk, F, t0s, t1s)
    st, tg, wt, t0, t1 = problems[1]
    assert t0 == t1
    assert torch.equal(out[0][F:], st.poses) and torch.equal(out[1][F * M:], st.patches)
    st0 = problems[0]
    check_oracle("stream 0 beside an empty window", st0[0], st0[3], st0[4], (out[0][:F], out[1][:F * M]), oracle(*st0))
    ref = oracle(st, tg, wt, t0, t1)
    live = st.kk.unique()
    assert (ref[1][live, 2] - st.patches[live, 2].double()).abs().max() > 1e-4, "the structure-only step moves depths"
    for name, res in (("grouped", run_grouped(st, tg, wt, t0, t1)), ("forward", run_forward(ext[1], st, tg, wt, t0, t1))):
        assert torch.equal(res[0], st.poses), name
        check_oracle("%s structure-only" % name, st, t0, t1, res, ref)


# ------------------------------------------------------------------------------------------------ 6. wide path
@pytest.mark.parametrize("N,eff_impl", [(BA_MAX_N + 1, False), (1, True), (BA_FAST_MAX_N, True)])
def test_wide_path_at_its_edges(ext, ref_ext, N, eff_impl):
    """N = 33, the first width past the on-chip solver, and eff_impl=True at N = 1 and 12 (ba_wide.cu)"""
    st, target, weight, t0, t1 = make_problem(N + 2, N, 8, 800 + N)
    assert N > BA_MAX_N or eff_impl
    ref = oracle(st, target, weight, t0, t1)
    print("\nwide N=%d E=%d eff_impl=%s" % (N, st.E, eff_impl))
    check_oracle("forward (wide)", st, t0, t1, run_forward(ext[1], st, target, weight, t0, t1, eff_impl), ref)
    if ref_ext is not None:
        check_oracle("reference", st, t0, t1, run_forward(ref_ext[1], st, target, weight, t0, t1, eff_impl), ref)
