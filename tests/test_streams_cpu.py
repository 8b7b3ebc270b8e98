"""The stream batch layout (dpvo_b200/streams.py) without a GPU: the local <-> global numbering and the ring rows against
a per-stream restatement, the stacked edge store's slices, and the host-side rejection of batches that cannot be
stepped together."""
import pytest
import torch

from dpvo_b200 import synthetic
from dpvo_b200.streams import StreamBatch
from dpvo_b200.patchgraph import DevicePatchGraph

# a small configuration so that the synthetic streams build quickly on the CPU
CFG = dict(M=4, lifetime=3, removal=5, opt_window=3, ht=64, wd=96, intrinsics=(40.0, 40.0, 48.0, 32.0))


def _batch(B=3, frames=(9, 4, 7), F=16, mem=10):
    return synthetic.make_batch(CFG, B, seeds=[3 + b for b in range(B)], n_frames=list(frames), device="cpu",
                                frames_per_stream=F, mem=mem)


def test_global_numbering_and_ring_rows_match_a_per_stream_restatement():
    batch = _batch()
    F, M, mem, pmem = batch.F, batch.M, batch.mem, batch.pmem
    kk_ring, jj_ring = batch.ring_rows(batch.kk, batch.jj)
    e0 = 0
    for b in range(batch.B):
        s = batch.stream(b)
        e1 = e0 + s.E
        # the batch's lists are the streams' local lists, offset and concatenated in stream order
        assert torch.equal(batch.ii[e0:e1], s.ii + b * F) and torch.equal(batch.jj[e0:e1], s.jj + b * F)
        assert torch.equal(batch.kk[e0:e1], s.kk + b * F * M)
        # a single stream's ring rows (runner.py: kk % (M pmem), jj % mem), moved to stream b's block of the rings
        assert torch.equal(kk_ring[e0:e1], b * pmem * M + s.kk % (M * pmem))
        assert torch.equal(jj_ring[e0:e1], b * mem + s.jj % mem)
        (si, li), (sj, lj), (sk, lk) = batch.to_local(batch.ii[e0:e1], batch.jj[e0:e1], batch.kk[e0:e1])
        assert bool((si == b).all() and (sj == b).all() and (sk == b).all())
        assert torch.equal(li, s.ii) and torch.equal(lj, s.jj) and torch.equal(lk, s.kk)
        e0 = e1
    assert e0 == batch.E
    # every local frame / patch number, not only the ones the edges use
    f = torch.arange(F)
    k = torch.arange(F * M)
    for b in range(batch.B):
        gi, gj, gk = batch.to_global(b, f, f, k)
        kr, jr = batch.ring_rows(gk, gj)
        assert torch.equal(kr, b * pmem * M + k % (pmem * M)) and torch.equal(jr, b * mem + f % mem)
        assert torch.equal(gi, f + b * F)


def test_stream_views_alias_the_stacked_buffers_and_copies_do_not():
    batch = _batch()
    b = 1
    s = batch.stream(b)
    F, M, mem = batch.F, batch.M, batch.mem
    s.poses[2, 0] = 42.0
    s.patches[5, 2] = 0.125
    s.intrinsics[0, 0] = 77.0
    s.fmap1[0, 3, 7, 1, 2] = 5.0
    s.imap[0, 11, 9] = -2.0
    assert batch.poses[b * F + 2, 0] == 42.0 and bool((batch.patches[b * F * M + 5, 2] == 0.125).all())
    assert batch.intrinsics[b * F, 0] == 77.0 and batch.fmap1[0, b * mem + 3, 7, 1, 2] == 5.0
    assert batch.imap[0, b * batch.pmem * M + 11, 9] == -2.0
    assert batch.fmap1.stride() == s.fmap1.stride() and s.fmap1.permute(0, 1, 3, 4, 2).is_contiguous()
    c = batch.copy_stream(b)
    c.poses[2, 0] = 0.0
    assert batch.poses[b * F + 2, 0] == 42.0 and c.fmap1.stride() == s.fmap1.stride()
    # windows in global numbering
    t0s, t1s = batch.windows()
    for i in range(batch.B):
        assert (t0s[i], t1s[i]) == (i * F + batch.stream(i).t0, i * F + batch.stream(i).n)


def test_mismatched_configurations_and_image_sizes_are_rejected():
    batch = StreamBatch(2, CFG, 16, 6, device="cpu")
    ok = synthetic.make_state(CFG, 5, device="cpu", seed=1, buffer=16, mem=6)
    batch.load(0, ok)
    other_cam = dict(CFG, intrinsics=(50.0, 50.0, 48.0, 32.0))          # cameras may differ per stream
    batch.load(1, synthetic.make_state(other_cam, 5, device="cpu", seed=2, buffer=16, mem=6))
    for cfg, msg in ((dict(CFG, M=8), "M=8"), (dict(CFG, wd=128), "image"), (dict(CFG, removal=7), "configuration")):
        bad = synthetic.make_state(cfg, 5, device="cpu", seed=1, buffer=16, mem=6)
        with pytest.raises(ValueError, match=msg):
            batch.load(1, bad)
    with pytest.raises(ValueError, match="fmap1"):
        batch.load(1, synthetic.make_state(CFG, 5, device="cpu", seed=1, buffer=16, mem=8))
    with pytest.raises(ValueError, match="pose slots"):
        batch.load(1, synthetic.make_state(CFG, 5, device="cpu", seed=1, buffer=20, mem=6))
    with pytest.raises(ValueError, match="one seed"):
        synthetic.make_batch(CFG, 2, seeds=[1], n_frames=5, device="cpu", frames_per_stream=16, mem=6)
    with pytest.raises(ValueError, match="streams"):
        StreamBatch(0, CFG, 16, 6, device="cpu")


def test_an_edge_joining_two_streams_is_rejected():
    batch = _batch()
    F, M = batch.F, batch.M
    ii, jj, kk = batch.ii.clone(), batch.jj.clone(), batch.kk.clone()
    batch.set_edges(ii, jj, kk)                       # the batch's own lists pass and split back into the same streams
    for b in range(batch.B):
        assert torch.equal(batch.to_global(b, kk=batch.stream(b).kk)[2], kk[batch.to_local(kk=kk)[2][0] == b])
    for field, shift in (("jj", F), ("ii", F), ("kk", F * M)):
        bad = {"ii": ii.clone(), "jj": jj.clone(), "kk": kk.clone()}
        bad[field][0] += shift                          # stream 0's first edge reaches into stream 1
        with pytest.raises(ValueError, match="joins streams"):
            batch.set_edges(bad["ii"], bad["jj"], bad["kk"])
    bad_kk = kk.clone()
    bad_kk[-1] = batch.B * F * M                       # past the last stream
    with pytest.raises(ValueError, match="outside"):
        batch.set_edges(ii, jj, bad_kk)
    with pytest.raises(ValueError, match="outside"):
        batch.check_edges(ii - 10 ** 6, jj, kk)


def test_windows_outside_a_stream_or_wider_than_the_solver_are_rejected():
    batch = _batch(F=48)
    s = batch.stream(2)
    s.t0, s.n = 5, 4                                   # t0 > n
    with pytest.raises(ValueError, match="not inside"):
        batch.windows()
    s.t0, s.n = 3, 49                                  # n past the stream's frames
    with pytest.raises(ValueError, match="not inside"):
        batch.windows()
    s.t0, s.n = -1, 4
    with pytest.raises(ValueError, match="not inside"):
        batch.windows()
    s.t0, s.n = 2, 35                                  # 33 free poses
    with pytest.raises(ValueError, match="33 free poses"):
        batch.windows()
    s.t0, s.n = 3, 35                                  # 32: the widest window the solver holds
    assert batch.windows()[1][2] == 2 * 48 + 35
    s.t0 = s.n = 7                                     # an empty window is allowed: the stream is left untouched
    batch.windows()


def test_stacked_store_slices_and_dummy_frames():
    B, cap, M, F = 3, 200, 4, 16
    dummies = [b * F + F - 1 for b in range(B)]
    store, graphs = DevicePatchGraph.stacked(B, cap, M, dummies, device="cpu")
    assert store.cap == B * 256 and len(graphs) == B
    for b, g in enumerate(graphs):
        assert g.cap == 256 and g.dummy_frame == dummies[b] and g.dummy_patch == dummies[b] * M
        sl = slice(b * 256, (b + 1) * 256)
        assert bool((store.ii[sl] == dummies[b]).all() and (store.jj[sl] == dummies[b]).all())
        assert bool((store.kk[sl] == dummies[b] * M).all())
        # views: a write through the stream's graph lands in its slice of the store
        g.ii[3] = 1000 + b
        g.net[0, 5, 7] = float(b + 1)
        assert store.ii[b * 256 + 3] == 1000 + b and store.net[0, b * 256 + 5, 7] == b + 1
        assert g.net.is_contiguous() and g.n_active.data_ptr() != store.ii.data_ptr()
    with pytest.raises(RuntimeError, match="per-stream"):
        store.append(store.ii[:1], store.jj[:1], store.kk[:1])
    with pytest.raises(RuntimeError, match="per-stream"):
        store.remove_old(torch.tensor([3]), 2)
    with pytest.raises(ValueError, match="dummy frame"):
        DevicePatchGraph.stacked(2, cap, M, [15], device="cpu")
