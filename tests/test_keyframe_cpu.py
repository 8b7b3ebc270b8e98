"""oracle/keyframe.py against the reference's own flow_mag (tests/golden/keyframe_ref.pt) and against a line-by-line
transcription of DPVO.keyframe / terminate; the keyframe entry points' host-side argument checks."""
import ctypes
import math
import os

import pytest
import torch

import dpvo_b200
from dpvo_b200 import synthetic
from dpvo_b200.keyframe import Keyframes
from dpvo_b200.loop import LoopClosure
from dpvo_b200.patchgraph import DevicePatchGraph
from oracle import keyframe as OK
from oracle import loop as OL

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "keyframe_ref.pt")


def _golden():
    return torch.load(GOLDEN, weights_only=False)


def test_oracle_flows_and_decisions_match_the_reference():
    """the reference computes in fp32: a flow is a difference of pixel coordinates of up to the image width W, each
    rounded at 2^-24 W, so a flow (and a mean of flows) is held to 1e-6 of max(|flow|, W)"""
    g = _golden()
    assert len(g["cases"]) >= 7
    seen = set()
    for name, c in g["cases"].items():
        W = 2.0 * float(c["intrinsics"][0, 2])
        means = []
        for s in c["sets"]:
            if s["ii"].numel() == 0:
                means.append(float("nan"))
                continue
            f = OK.flow9(c["poses"], c["patches"], c["intrinsics"], s["ii"], s["jj"], s["kk"])
            ref = s["flow"].double()
            assert ((f - ref).abs() <= 1e-6 * ref.abs().clamp(min=W)).all(), name
            mean = OK.motionmag(c["poses"], c["patches"], c["intrinsics"], list(zip(s["ii"].tolist(), s["jj"].tolist(), s["kk"].tolist())),
                                int(s["ii"][0]), int(s["jj"][0]))
            assert abs(mean - s["mean"]) <= 1e-6 * max(abs(s["mean"]), W), name
            means.append(mean)
        m = means[0] + means[1]
        edges = [e for s in c["sets"] for e in zip(s["ii"].tolist(), s["jj"].tolist(), s["kk"].tolist())]
        om, removed = OK.motion(c["poses"], c["patches"], c["intrinsics"], edges, c["n"], g["ki"], g["thresh"])
        if math.isnan(c["m"]):
            assert math.isnan(om) and not removed and not c["removed"], name
        else:
            assert abs(om - c["m"]) <= 2e-6 * max(abs(c["m"]), W) and removed == c["removed"], name
        seen.add(c["removed"])
    assert seen == {True, False}


# -------------------------------------------------------------------------------- a transcription of the reference
class _PG:
    """the reference's buffers in its own layouts (patches_ [N, M, 3, 3, 3], imap_ [pmem, M, D], fmap1_ [1, mem, ...])"""


def _ref_keyframe(self, pg, ki, M, mem, pmem):
    """dpvo.py:273-300 with the decision taken (remove_factors without store, lists as tensors)"""
    k = self.n - ki
    t0 = pg.tstamps_[k - 1]
    t1 = pg.tstamps_[k]
    dP = OL._mul(OL._norm(pg.poses_[k].double()[None]), OL._inv(OL._norm(pg.poses_[k - 1].double()[None])))[0]
    pg.delta[int(t1)] = (int(t0), dP)
    to_remove = (pg.ii == k) | (pg.jj == k)
    pg.ii, pg.jj, pg.kk = pg.ii[~to_remove], pg.jj[~to_remove], pg.kk[~to_remove]
    pg.kk[pg.ii > k] -= M
    pg.ii[pg.ii > k] -= 1
    pg.jj[pg.jj > k] -= 1
    for i in range(k, self.n - 1):
        pg.tstamps_[i] = pg.tstamps_[i + 1]
        pg.poses_[i] = pg.poses_[i + 1]
        pg.patches_[i] = pg.patches_[i + 1]
        pg.intrinsics_[i] = pg.intrinsics_[i + 1]
        self.imap_[i % pmem] = self.imap_[(i + 1) % pmem]
        self.gmap_[i % pmem] = self.gmap_[(i + 1) % pmem]
        self.fmap1_[0, i % mem] = self.fmap1_[0, (i + 1) % mem]
        self.fmap2_[0, i % mem] = self.fmap2_[0, (i + 1) % mem]
    self.n -= 1


def _ref_terminate(pg, n, counter):
    """dpvo.py:166-198's interpolation, poses.inv()"""
    traj = {int(pg.tstamps_[i]): OL._norm(pg.poses_[i].double()[None])[0] for i in range(n)}

    def get_pose(t):
        if t in traj:
            return traj[t]
        t0, dP = pg.delta[t]
        return OL._mul(dP[None], get_pose(t0)[None])[0]

    return torch.stack([OL._inv(get_pose(t)[None])[0] for t in range(counter)])


@pytest.mark.parametrize("ki,mem,pmem", [(4, 4, 6), (2, 3, 3), (5, 7, 5)])
def test_oracle_shift_and_interpolation_match_a_transcription(ki, mem, pmem):
    torch.manual_seed(ki * 100 + mem)
    M, F, n0, D = 3, 40, 14, 5
    self, pg = _PG(), _PG()
    pg.poses_ = torch.randn(F, 7)
    pg.poses_[:, 3:] /= pg.poses_[:, 3:].norm(dim=1, keepdim=True)
    pg.patches_ = torch.randn(F, M, 3, 3, 3)
    pg.intrinsics_ = torch.rand(F, 4) + 1
    pg.tstamps_ = torch.zeros(F, dtype=torch.long)
    pg.tstamps_[:n0] = torch.arange(n0)
    pg.delta = {}
    self.imap_, self.gmap_ = torch.randn(pmem, M, D), torch.randn(pmem, M, 2, 3, 3)
    self.fmap1_, self.fmap2_ = torch.randn(1, mem, 2, 4, 4), torch.randn(1, mem, 2, 2, 2)
    ii, jj, kk = synthetic.replay_edges(n0, M, 5, 9)
    pg.ii, pg.jj, pg.kk = ii.clone(), jj.clone(), kk.clone()
    self.n = n0
    hg = OL.HostGraph(M, 9, 4)
    hg.append(ii.tolist(), jj.tolist(), kk.tolist())
    host = OK.HostKeyframes(M, pg.poses_.clone(), pg.patches_.reshape(F * M, 3, 3, 3).clone(), pg.intrinsics_.clone(), n0,
                            fmap1=self.fmap1_.clone(), fmap2=self.fmap2_.clone(), gmap=self.gmap_.reshape(1, pmem * M, 2, 3, 3).clone(),
                            imap=self.imap_.reshape(1, pmem * M, D).clone(), graph=hg)
    counter = n0
    for step in range(6):
        # a new frame (dpvo.py:400, 440), a skipped one on odd steps, then the culling of the frame KI back
        if step % 2:
            host.skip_frame()
            pg.delta[counter] = (counter - 1, torch.tensor([0, 0, 0, 0, 0, 0, 1.0], dtype=torch.float64))
            counter += 1
        self.n += 1
        host.n += 1
        pg.tstamps_[self.n - 1] = counter
        counter += 1
        host.add_frame()
        _ref_keyframe(self, pg, ki, M, mem, pmem)
        host.keyframe(ki, 15.0, removed=True)
        assert host.n == self.n and host.counter == counter
        assert torch.equal(host.tstamp, pg.tstamps_) and torch.equal(host.poses, pg.poses_)
        assert torch.equal(host.patches, pg.patches_.reshape(F * M, 3, 3, 3)) and torch.equal(host.intrinsics, pg.intrinsics_)
        assert torch.equal(host.fmap1, self.fmap1_) and torch.equal(host.fmap2, self.fmap2_)
        assert torch.equal(host.gmap, self.gmap_.reshape(1, pmem * M, 2, 3, 3)) and torch.equal(host.imap, self.imap_.reshape(1, pmem * M, D))
        assert sorted(map(tuple, hg.act)) == sorted(zip(pg.ii.tolist(), pg.jj.tolist(), pg.kk.tolist()))
        assert host.delta.keys() == pg.delta.keys()
        for t in pg.delta:
            assert host.delta[t][0] == pg.delta[t][0] and torch.allclose(host.delta[t][1], pg.delta[t][1], rtol=0, atol=1e-12)
    want = _ref_terminate(pg, self.n, counter)
    got = OK.terminate(host.poses, host.tstamp, host.n, host.delta, host.counter)
    assert got.shape == (counter, 7) and torch.allclose(got, want, rtol=0, atol=1e-12)
    # normalize's dP.scale(s) scales translations only
    sc = OK.scale_deltas(host.delta, 2.5)
    for t, (t0, dP) in sc.items():
        assert t0 == host.delta[t][0] and torch.equal(dP[:3], 2.5 * host.delta[t][1][:3]) and torch.equal(dP[3:], host.delta[t][1][3:])


def test_stop_go_state_has_both_outcomes_far_from_the_threshold():
    st = synthetic.make_stop_go_state("fast", 30, total=30, device="cpu", features=False)
    cfg = st.cfg
    out = []
    for n in range(6, 31):
        edges = torch.stack(synthetic.replay_edges(n, cfg["M"], cfg["lifetime"], cfg["removal"]), 1).tolist()
        out.append(OK.motion(st.poses, st.patches, st.intrinsics, edges, n, 4, 15.0))
    assert sum(r for _, r in out) >= 6 and sum(not r for _, r in out) >= 6
    assert all(abs(m / 2 - 15.0) > 10.0 for m, _ in out)


# -------------------------------------------------------------------------------- host-side argument checks
def test_keyframe_entry_points_reject_bad_arguments_without_a_gpu():
    lib = dpvo_b200.library()
    buf = (ctypes.c_char * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    i64, i32, f64 = ctypes.c_int64, ctypes.c_int, ctypes.c_double

    def motion(F=8, B=1, slots=16, T=64, ki=4, ptr=p, ws=4096):
        return lib.dpvo_keyframe_motion(p, p, p, i64(F), i32(B), p, p, p, p, i64(slots), ptr, p, p, p, i64(T), i32(ki), f64(15.0),
                                        p, p, p, p, p, i64(ws), None)
    assert motion(ki=0) == 1 and b"keyframe_index" in lib.dpvo_last_error()
    assert motion(T=4) == 1 and b"delta table" in lib.dpvo_last_error()
    assert motion(ptr=None) == 1 and b"null" in lib.dpvo_last_error()
    assert motion(B=0) == 1 and b"bad sizes" in lib.dpvo_last_error()
    assert motion(B=2, ws=100) == 1 and b"workspace" in lib.dpvo_last_error()

    bases = (ctypes.c_void_p * 2)(p.value, p.value)
    rb = (ctypes.c_int64 * 2)(28, 64)

    def shift(rows, ki=4, rbytes=rb, b=bases):
        rw = (ctypes.c_int64 * 2)(*rows)
        return lib.dpvo_keyframe_shift(b, rbytes, rw, i32(2), i64(8), i32(1), i32(ki), p, p, None)
    assert shift((8, 3)) == 1 and b"fewer than keyframe_index" in lib.dpvo_last_error()      # a ring of mem < KI
    assert shift((8, 8), ki=0) == 1 and b"keyframe_index" in lib.dpvo_last_error()
    assert shift((8, 8), rbytes=(ctypes.c_int64 * 2)(28, 6)) == 1 and b"multiple of 4" in lib.dpvo_last_error()
    assert shift((8, 8), b=(ctypes.c_void_p * 2)(p.value, None)) == 1 and b"null" in lib.dpvo_last_error()
    assert lib.dpvo_keyframe_count(i32(2), p, p, i64(8), i32(1), p, p, p, i64(64), p, None) == 1
    assert b"mode" in lib.dpvo_last_error()
    assert lib.dpvo_keyframe_count(i32(0), None, p, i64(8), i32(1), p, p, p, i64(64), p, None) == 1
    assert lib.dpvo_keyframe_trajectory(p, p, p, i64(8), i32(1), p, p, i64(4), p, p, p, p, None) == 1
    assert b"bad sizes" in lib.dpvo_last_error()
    assert lib.dpvo_loop_normalize_deltas(p, p, i64(4), i32(8), i32(3), None, i64(5), None) == 1
    assert b"null" in lib.dpvo_last_error()


def test_keyframes_rejects_bad_configurations():
    st = synthetic.make_stop_go_state("fast", 12, total=20, device="cpu", features=False)
    M, dummy = st.cfg["M"], st.poses.shape[0] - 1
    g = DevicePatchGraph(4096, M, dummy, "cpu")
    with pytest.raises(ValueError, match="at least 1"):
        Keyframes(st.cfg, st, g, keyframe_index=0)
    with pytest.raises(ValueError, match="max_timestamps"):
        Keyframes(st.cfg, st, g, max_timestamps=8)
    st.gmap = torch.zeros(1, 3 * M, 128, 3, 3)
    with pytest.raises(ValueError, match="fewer than keyframe_index"):
        Keyframes(st.cfg, st, g)
    st.gmap = None
    gl = DevicePatchGraph(4096, M, dummy, "cpu", loop_pairs=10, inactive_capacity=100)
    lc = LoopClosure(st.cfg, gl, keyframe_index=3)
    with pytest.raises(ValueError, match="loop region"):
        Keyframes(st.cfg, st, gl, keyframe_index=3)                  # its deltas would miss normalize's scaling
    with pytest.raises(ValueError, match="another graph"):
        Keyframes(st.cfg, st, g, keyframe_index=3, loop=lc)
    with pytest.raises(ValueError, match="LoopClosure"):
        Keyframes(st.cfg, st, gl, loop=lc)
    kf = Keyframes(st.cfg, st, gl, keyframe_index=3, loop=lc)
    assert lc.keyframes is kf and kf.thresh == 15.0 and kf.tstamp[0, :st.n].tolist() == list(range(st.n))
