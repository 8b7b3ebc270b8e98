"""fastba host interface over cuda_ba: same surface as dpvo/fastba/ba.py:4-8."""
from . import extensions


def neighbors(ii, jj):
    return extensions()[1].neighbors(ii, jj)


def reproject(poses, patches, intrinsics, ii, jj, kk):
    return extensions()[1].reproject(poses, patches, intrinsics, ii, jj, kk)


def BA(poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, t0, t1, M, iterations, eff_impl=False):
    """In-place Gauss-Newton bundle adjustment (poses[t0:t1] and the depths of the patches in kk)."""
    return extensions()[1].forward(poses.data, patches, intrinsics, target, weight, lmbda, ii, jj, kk, M, t0, t1,
                                   iterations, eff_impl)


def BA_grouped(poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, t0, t1, iterations, groups_kk, groups_ij):
    """BA on the edge groupings the update operator already built for this graph (net.EdgeGroups):
    saves the two radix-sort launches cuda_ba.forward would repeat."""
    gk, gp = groups_kk, groups_ij
    return extensions()[3].ba_forward_grouped(poses.data, patches, intrinsics, target, weight, lmbda, ii, jj, kk, t0, t1,
                                              iterations, gk.order, gk.group_start, gk.key_a, gk.n,
                                              gp.order, gp.group_start, gp.key_a, gp.key_b, gp.n)


def BA_batched(poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, frames_per_stream, t0s, t1s, iterations,
               groups_kk, groups_ij):
    """BA_grouped for B streams in one reduce and one solve launch per iteration.  Stream b owns frames
    [b F, (b+1) F) and patches [b F M, (b+1) F M) (F = frames_per_stream); its window is [t0s[b], t1s[b]) in global
    frame numbers and intrinsics row b F is its camera.  The edge lists and groupings span all streams, and no edge may
    join two streams (streams.StreamBatch builds and checks such lists).  Each stream's result is that of BA_grouped on
    the stream alone, with one exception: a stream with an empty window (t0s[b] == t1s[b]) is left untouched, where
    BA_grouped runs its structure-only step and updates the depths.  A stream without edges is left untouched too."""
    gk, gp = groups_kk, groups_ij
    return extensions()[3].ba_forward_batched(poses.data, patches, intrinsics, target, weight, lmbda, ii, jj, kk,
                                              int(frames_per_stream), [int(t) for t in t0s], [int(t) for t in t1s],
                                              iterations, gk.order, gk.group_start, gk.key_a, gk.n,
                                              gp.order, gp.group_start, gp.key_a, gp.key_b, gp.n)
