"""The tensor contract of the torch shims (csrc/shim.cpp): every tensor argument of every entry point is a CUDA tensor on
the op's device, and where the op requires them of one dtype and contiguous.  A violation raises RuntimeError naming the
op before anything is launched, so no host or peer-device pointer ever reaches a kernel.

ROWS holds one small valid call per entry point of the four modules; test_shim_args_cpu.py checks that it covers every
exported name.  Each tensor argument is wrapped by what the op requires of it beyond the device: `need` (dtype and
contiguity), `typed` (dtype, any layout) or `dense` (contiguity, any dtype); a bare tensor is converted by the op."""
import re
from types import SimpleNamespace

import pytest
import torch

from dpvo_b200 import frontend, synthetic
from dpvo_b200.keyframe import Keyframes
from dpvo_b200.loop import LoopClosure
from dpvo_b200.patchgraph import DevicePatchGraph

DEV = "cuda:0"
MODULES = ("cuda_corr", "cuda_ba", "lietorch_backends", "dpvo_b200_ext")
SE3 = 3


class Req:
    def __init__(self, t, dtype, contiguous):
        self.t, self.dtype, self.contiguous = t, dtype, contiguous


def need(t):
    return Req(t, True, True)


def typed(t):
    return Req(t, True, False)


def dense(t):
    return Req(t, False, True)


def f32(*s, scale=0.1):
    return torch.randn(*s, device=DEV) * scale


def f16(*s):
    return f32(*s).half()


def ar(n, dtype=torch.long):
    return torch.arange(n, device=DEV, dtype=dtype)


def zeros(*s, dtype=torch.float32):
    return torch.zeros(*s, device=DEV, dtype=dtype)


def scalar(v, dtype):
    return torch.tensor([v], device=DEV, dtype=dtype)


def _se3(n):
    return _ext()[2].expm(SE3, f32(n, 6, scale=0.3))


def _ext():
    import dpvo_b200
    return dpvo_b200.extensions()


def _groups(key):
    return _ext()[3].group_edges(key)


# ------------------------------------------------------------------------------------------------ cuda_corr, cuda_ba
def _corr(c, backward):
    f1, f2 = f32(1, 8, 128, 3, 3), f32(1, 2, 128, 10, 12)
    coords, ii, jj = torch.rand(1, 8, 2, 3, 3, device=DEV) * 9, ar(8), zeros(8, dtype=torch.long)
    return [f1, f2 if backward else typed(f2), coords, ii, jj] + ([f32(1, 8, 3, 3, 3, 3)] if backward else []) + [1]


def _ba_edges(c):
    st = c.st
    return [st.poses.clone().view(1, -1, 7), st.patches.clone().view(1, -1, 3, 3, 3), st.intrinsics.view(1, -1, 4).clone()]


def _ba_obs(c):
    E = c.st.E
    return [zeros(1, E, 2) + 10.0, zeros(1, E, 2) + 0.5, scalar(1e-4, torch.float32), c.st.ii.clone(), c.st.jj.clone(),
            c.st.kk.clone()]


def _ba(c):
    p, q, i = _ba_edges(c)
    return [need(p), need(q), i] + _ba_obs(c)


def _groupings(c):
    ex, st = _ext()[3], c.st
    f = ex.group_edges_pair(st.kk, None, st.jj, st.ii, st.jj, None)
    return [need(f[0]), need(f[2]), need(f[3]), need(f[5]), need(f[6]), need(f[8]), need(f[9]), need(f[10]), need(f[11])]


def _solve_system():
    ii, jj = torch.tensor([0, 1, 2, 0, 1, 2], device=DEV), torch.tensor([1, 2, 3, 2, 3, 3], device=DEV)
    return [f32(6, 7, 7), f32(6, 7, 7), ii, jj, f32(6, 7), 1e-3, 1e-4, 2]


# ------------------------------------------------------------------------------------------------ lietorch_backends
def _lie(name):
    X, Y, a, p, p4 = _se3(4), _se3(4), f32(4, 6), f32(4, 3), f32(4, 4)
    second = {"mul": (Y, 7), "adj": (a, 6), "adjT": (a, 6), "act": (p, 3), "act4": (p4, 4), "Jinv": (a, 6)}
    if name == "expm":
        return [SE3, dense(a)]
    if name == "expm_backward":
        return [SE3, dense(f32(4, 7)), dense(a)]
    if name in ("logm", "inv", "as_matrix", "projector"):
        return [SE3, dense(X)]
    if name == "logm_backward":
        return [SE3, dense(f32(4, 6)), dense(X)]
    if name == "inv_backward":
        return [SE3, dense(f32(4, 7)), dense(X)]
    if name.endswith("_backward"):
        y, _ = second[name[:-len("_backward")]]
        out_dim = {"mul": 7, "adj": 6, "adjT": 6, "act": 3, "act4": 4}[name[:-len("_backward")]]
        return [SE3, dense(f32(4, out_dim)), dense(X), dense(y)]
    return [SE3, dense(X), need(second[name][0])]


LIE = ["expm", "expm_backward", "logm", "logm_backward", "inv", "inv_backward", "mul", "mul_backward", "adj", "adj_backward",
       "adjT", "adjT_backward", "act", "act_backward", "act4", "act4_backward", "as_matrix", "projector", "Jinv"]


# ------------------------------------------------------------------------------------------------ dpvo_b200_ext
def _chains():
    E = 64
    return SimpleNamespace(E=E, net32=f32(E, 384), corr=f16(E, 896), W0=f16(384 * 896), W25=f16(768 * 384), pA=f32(7 * 384),
                           inp=f16(E, 384), n16=f16(E, 384), Wab=f16(768 * 384), pC=f32(2 * 384), W6=f16(6 * 384 * 384),
                           pG=f32(14 * 384 + 4))


def _loop(c):
    g = c.lg
    r0, r1 = g.normal_cap, g.cap
    return [need(g.ii[r0:r1].clone()), need(g.jj[r0:r1].clone()), need(g.kk[r0:r1].clone()), need(g.active[r0:r1].clone()),
            need(g.net[0, r0:r1].clone())]


def _encoder_slots(c, R, Rg, B=1):
    h, w = frontend.encoder_output_size(64, 64)
    lead = (R,) if B > 1 else ()
    w16, b32 = c.fe.packed()
    return [need(w16), need(b32), need(torch.rand(*((B,) if B > 1 else ()), 8, 2, device=DEV) * 12 + 1),
            typed(torch.empty(*lead, h, w, 128, device=DEV, dtype=torch.half)),
            typed(torch.empty(*lead, h // 4, w // 4, 128, device=DEV, dtype=torch.half)),
            typed(torch.empty(Rg, 3, 3, 128, device=DEV, dtype=torch.half)), typed(torch.empty(Rg, 384, device=DEV, dtype=torch.half)),
            need(torch.empty(Rg, 3, 3, 3, device=DEV))]


def _image(*lead):
    return torch.randint(0, 256, (*lead, 3, 64, 64), device=DEV, dtype=torch.uint8)


def _rows():
    rows = {
        "cuda_corr.forward": lambda c: _corr(c, False),
        "cuda_corr.backward": lambda c: _corr(c, True),
        "cuda_corr.patchify_forward": lambda c: [f32(1, 16, 10, 12), torch.rand(1, 5, 2, device=DEV) * 8 + 1, 1],
        "cuda_corr.patchify_backward": lambda c: [f32(1, 16, 10, 12), torch.rand(1, 5, 2, device=DEV) * 8 + 1, f32(1, 5, 16, 4, 4), 1],
        "cuda_ba.forward": lambda c: _ba(c) + [c.st.cfg["M"], c.st.t0, c.st.n, 1, False],
        "cuda_ba.neighbors": lambda c: [c.st.ii.clone(), c.st.jj.clone()],
        "cuda_ba.reproject": lambda c: _ba_edges(c) + [c.st.ii.clone(), c.st.jj.clone(), c.st.kk.clone()],
        "cuda_ba.solve_system": lambda c: _solve_system(),
        "dpvo_b200_ext.corr_pyramid2": lambda c: [f16(1, 8, 128, 3, 3), f16(1, 2, 128, 16, 20), f16(1, 2, 128, 4, 5),
                                                  torch.rand(1, 8, 2, 3, 3, device=DEV) * 12, ar(8), zeros(8, dtype=torch.long), 3, 4.0,
                                                  896, need(zeros(1, 8, 896, dtype=torch.half))],
        "dpvo_b200_ext.group_edges_pair": lambda c: [c.st.kk.clone(), None, c.st.jj.clone(), c.st.ii.clone(), c.st.jj.clone(), None],
        "dpvo_b200_ext.group_edges": lambda c: [c.st.ii.clone(), c.st.jj.clone(), c.st.kk.clone()],
        "dpvo_b200_ext.ba_forward_grouped": lambda c: _ba(c) + [c.st.t0, c.st.n, 1] + _groupings(c),
        "dpvo_b200_ext.ba_forward_batched": lambda c: _ba(c) + [c.st.poses.shape[0], [c.st.t0], [c.st.n], 1] + _groupings(c),
        "dpvo_b200_ext.ba_batched_workspace_bytes": lambda c: [64, 1, 8],
        "dpvo_b200_ext.reproject_clamped": lambda c: _ba_edges(c) + [c.st.ii.clone(), c.st.jj.clone(), c.st.kk.clone()],
        "dpvo_b200_ext.add_layernorm": lambda c: [f32(64, 384), f16(16, 384), f32(64, 384), f32(384), f32(384), 1e-3, True, True, True,
                                                  ar(64) % 16, False, typed(f16(64, 384))],
        "dpvo_b200_ext.gather_rows_masked": lambda c: [f32(64, 384), ar(32) * 2, True],
        "dpvo_b200_ext.residual_add_": lambda c: [need(f32(64, 384)), f16(16, 384), ar(64, torch.int32) % 16, True],
        "dpvo_b200_ext.residual_sum16": lambda c: [need(f32(64, 384)), f16(16, 384), ar(64, torch.int32) % 16],
        "dpvo_b200_ext.gated_residual": lambda c: [typed(f32(64, 384)), typed(f16(64, 384)), typed(f16(64, 384)), True],
        "dpvo_b200_ext.softagg_reduce": lambda c: _softagg(False),
        "dpvo_b200_ext.softagg_fused": lambda c: _softagg(True),
        "dpvo_b200_ext.softagg_fused_workspace_bytes": lambda c: [64],
        "dpvo_b200_ext.update_heads": lambda c: [need(f32(64, 384)), f32(4, 384), f32(4), f32(64, 2, 3, 3), typed(f16(64, 384)),
                                                 typed(f16(64, 384))],
        "dpvo_b200_ext.linear_f16": lambda c: [typed(f16(64, 64)), typed(f16(64, 64)), f32(64), 4, f32(32, 64), typed(f16(32, 64)),
                                               ar(32) * 2, True, need(zeros(1, 32, 64)), need(zeros(1, 32, 64, dtype=torch.half))],
        "dpvo_b200_ext.update_corr_norm": lambda c: _corr_norm(_chains()),
        "dpvo_b200_ext.update_neighbor_mlp": lambda c: _neighbor_mlp(_chains()),
        "dpvo_b200_ext.update_gru_heads": lambda c: _gru_heads(_chains()),
        "dpvo_b200_ext.update_gru_workspace_bytes": lambda c: [],
        "dpvo_b200_ext.pgraph_remove": lambda c: _store(c.kg) + [0, need(scalar(c.st.n, torch.long)), 8, need(scalar(1, torch.int32)),
                                                                 c.kg.dummy_frame, c.kg.dummy_patch, c.kg.M,
                                                                 need(c.kg.n_active.clone())],
        "dpvo_b200_ext.pgraph_append": lambda c: _store(c.kg, c.kg.normal_cap) + [c.st.ii[:8].clone(), c.st.jj[:8].clone(),
                                                                                  c.st.kk[:8].clone(), need(scalar(1, torch.int32)),
                                                                                  need(c.kg.net[0, :c.kg.normal_cap].clone()),
                                                                                  need(c.kg.n_active.clone()), need(c.kg.overflow.clone())],
        "dpvo_b200_ext.pgraph_new_edges": lambda c: [need(scalar(c.st.n, torch.long)), c.st.cfg["M"], c.st.cfg["lifetime"]],
        "dpvo_b200_ext.loop_scores": lambda c: [need(c.st.poses.clone()), need(c.st.patches.clone()), need(c.st.intrinsics.clone()),
                                                need(scalar(c.st.n, torch.long)), need(c.lc.last_global_ba.clone()), c.lc.M, c.lc.removal,
                                                c.lc.max_age, c.lc.freq, c.lc.kf_index],
        "dpvo_b200_ext.loop_select": lambda c: _loop_select(c),
        "dpvo_b200_ext.pgraph_remove_store": lambda c: _remove_store(c),
        "dpvo_b200_ext.loop_flags": lambda c: [need(c.lg.ii.clone()), need(c.lg.active.clone()), c.lg.normal_cap, c.st.n, c.lc.removal,
                                               need(c.lc.s_count.clone()), need(c.lc.flags.clone())],
        "dpvo_b200_ext.loop_normalize": lambda c: [need(c.st.poses.clone()), need(c.st.patches.clone()), c.st.n, c.st.cfg["M"],
                                                   need(torch.tensor([[0.0] * 6 + [1.0]] * 4, device=DEV))],
        "dpvo_b200_ext.keyframe_motion": lambda c: _keyframe_motion(c),
        "dpvo_b200_ext.keyframe_shift": lambda c: [[b.clone() for b in c.kf.bufs], list(c.kf.rows), c.kf.F, c.kf.ki,
                                                   need(zeros(1, dtype=torch.int32)), need(c.kf.k.clone())],
        "dpvo_b200_ext.keyframe_count": lambda c: [0, need(c.kf.n_dev.clone()), need(c.kf.tstamp.clone()), c.kf.F,
                                                   need(c.kf.counter.clone()), need(c.kf.delta.clone()), need(c.kf.delta_src.clone()),
                                                   need(zeros(1, dtype=torch.int32))],
        "dpvo_b200_ext.keyframe_trajectory": lambda c: [need(c.st.poses.clone()), need(c.kf.tstamp.clone()), need(c.kf.n_dev.clone()),
                                                        c.kf.F, need(c.kf.delta.clone()), need(c.kf.delta_src.clone()),
                                                        need(c.kf.counter.clone()), need(zeros(1, dtype=torch.int32))],
        "dpvo_b200_ext.neighbors_from_groups": lambda c: (lambda f: [need(f[0]), need(f[1])])(_groups(c.st.kk)),
        "dpvo_b200_ext.encoder_conv": lambda c: [1, need(f16(16, 16, 32)), need(f16(9 * 4 * 32 * 8)), need(f32(32)),
                                                 need(f32(2, 32) + 1.0), True, need(f16(16, 16, 32)), need(f32(2, 32) + 1.0), False,
                                                 True, True, False, 1.0],
        "dpvo_b200_ext.encode_frame": lambda c: [typed(_image())] + _encoder_slots(c, 1, 8) +
                                                [dense(zeros(_ext()[3].encode_frame_workspace_bytes(64, 64), dtype=torch.uint8)),
                                                 need(zeros(8, 3, dtype=torch.uint8))],
        "dpvo_b200_ext.encode_frame_workspace_bytes": lambda c: [64, 64],
        "dpvo_b200_ext.encode_frames": lambda c: [typed(_image(2))] + _encoder_slots(c, 3, 16, B=2) +
                                                 [[0, 1], [0, 8], [0, 8], need(zeros(2, 8) + 1.0),
                                                  dense(zeros(_ext()[3].encode_frames_workspace_bytes(2, 64, 64), dtype=torch.uint8)),
                                                  need(zeros(16, 3, dtype=torch.uint8))],
        "dpvo_b200_ext.encode_frames_workspace_bytes": lambda c: [2, 64, 64],
        "dpvo_b200_ext.point_cloud": lambda c: [need(c.st.poses.clone()), need(c.st.patches.clone()), need(c.st.intrinsics.clone()),
                                                c.st.poses.shape[0], [c.st.n],
                                                need(zeros(c.st.patches.shape[0], 3))],
        "dpvo_b200_ext.launch_count": lambda c: [],
        "dpvo_b200_ext.version": lambda c: [],
    }
    for name in LIE:
        rows["lietorch_backends." + name] = lambda c, name=name: _lie(name)
    return rows


def _softagg(fused):
    E, G = 64, 16
    f = _groups(ar(E) // (E // G))
    grouping = [need(f[0])] + ([need(f[1])] if fused else []) + [need(f[2]), need(f[5]), G]
    if not fused:
        return [need(f16(E, 768))] + grouping
    ws = zeros(_ext()[3].softagg_fused_workspace_bytes(E), dtype=torch.uint8)
    return [typed(f16(E, 384))] + grouping + [need(f16(768, 384)), need(f32(768)), dense(ws)]


def _corr_norm(k):
    return [typed(k.corr), need(k.W0), need(k.W25), need(k.pA), need(k.net32), need(k.inp), ar(k.E), need(k.n16)]


def _neighbor_mlp(k):
    return [need(k.inp), ar(k.E), need(k.Wab), need(k.pC), need(k.net32), need(k.n16)]


def _gru_heads(k):
    ws = zeros(_ext()[3].update_gru_workspace_bytes(), dtype=torch.uint8)
    return [need(k.net32), need(k.inp), ar(k.E, torch.int32), need(k.W6), need(k.pG), f32(k.E, 2, 3, 3), dense(ws), need(k.n16),
            ar(k.E, torch.int32), need(zeros(k.E, 2)), need(zeros(k.E, 2))]


def _store(g, n=None):
    n = g.cap if n is None else n
    return [need(g.ii[:n].clone()), need(g.jj[:n].clone()), need(g.kk[:n].clone()), need(g.active[:n].clone())]


def _loop_select(c):
    lc, st = c.lc, c.st
    scores = lc.score(st.poses, st.patches, st.intrinsics, scalar(st.n, torch.long)).clone()
    ii, jj, kk, active, state = _loop(c)
    return [need(scores), need(scalar(st.n, torch.long)), need(lc.last_global_ba.clone()), lc.M, lc.removal, lc.max_age, lc.freq,
            lc.kf_index, lc.thresh, need(lc.pairs.clone()), need(lc.n_pairs.clone()), ii, jj, kk, active, state,
            need(c.lg.n_active.clone()), need(lc.region_overflow.clone())]


def _remove_store(c):
    g, lc = c.lg, c.lc
    return _store(g) + [need(g.target[0].clone()), need(g.weight[0].clone()), need(scalar(c.st.n, torch.long)), lc.removal,
                        lc.opt_window, need(scalar(1, torch.int32)), g.dummy_frame, g.dummy_patch, lc.M, need(g.n_active.clone()),
                        need(lc.s_ii.clone()), need(lc.s_jj.clone()), need(lc.s_kk.clone()), need(lc.s_target[0].clone()),
                        need(lc.s_weight[0].clone()), need(lc.s_count.clone()), need(lc.s_overflow.clone())]


def _keyframe_motion(c):
    kf, st = c.kf, c.st
    return [need(st.poses.clone()), need(st.patches.clone()), need(st.intrinsics.clone()), kf.F] + _store(c.kg) + \
        [need(kf.n_dev.clone()), need(kf.tstamp.clone()), need(kf.delta.clone()), need(kf.delta_src.clone()), kf.ki, kf.thresh,
         need(kf.flag.clone()), need(kf.k.clone()), need(kf.m.clone()), need(kf.overflow.clone())]


ROWS = _rows()


# ------------------------------------------------------------------------------------------------ the tests
@pytest.fixture(scope="module")
def c():
    torch.manual_seed(0)
    st = synthetic.make_state("fast", 12, device=DEV, seed=7)
    M = st.cfg["M"]
    dummy = st.poses.shape[0] - 1
    kg = DevicePatchGraph(2 * st.E + 4 * M * st.cfg["lifetime"], M, dummy, DEV)
    kg.append(st.ii, st.jj, st.kk)
    lg = DevicePatchGraph(st.E + 4 * M * st.cfg["lifetime"], M, dummy, DEV, loop_pairs=4, inactive_capacity=256)
    lg.append(st.ii, st.jj, st.kk)
    lc = LoopClosure(st.cfg, lg)
    kf = Keyframes(st.cfg, st, kg)
    fe = frontend.FrameEncoder(frontend.Patchifier().to(DEV).eval())
    torch.cuda.synchronize()
    return SimpleNamespace(st=st, kg=kg, lg=lg, lc=lc, kf=kf, fe=fe)


def _slots(args):
    """(index, item index or None, Req or tensor) of every tensor argument"""
    out = []
    for i, a in enumerate(args):
        if isinstance(a, (torch.Tensor, Req)):
            out.append((i, None, a))
        elif isinstance(a, list):
            out += [(i, j, x) for j, x in enumerate(a) if isinstance(x, (torch.Tensor, Req))]
    return out


def _plain(a):
    if isinstance(a, Req):
        return a.t
    if isinstance(a, list):
        return [_plain(x) for x in a]
    return a


def _with(args, i, j, value):
    out = [_plain(a) for a in args]
    if j is None:
        out[i] = value
    else:
        out[i] = list(out[i])
        out[i][j] = value
    return out


def _fn(ext, name):
    mod, fn = name.split(".")
    return getattr(ext[MODULES.index(mod)], fn)


def _rejected(ext, name, args, i, j, value, why):
    ex = ext[3]
    n0 = ex.launch_count()
    with pytest.raises(RuntimeError, match=re.escape(name)):
        _fn(ext, name)(*_with(args, i, j, value))
    assert ex.launch_count() == n0, "%s: argument %d%s (%s) launched a kernel" % (name, i, "" if j is None else "[%d]" % j, why)


def _wrong_dtype(t):
    return t.to(torch.float32 if t.dtype == torch.float64 else torch.float64)


def _strided(t):
    s = torch.empty(*t.shape, 2, dtype=t.dtype, device=t.device)[..., 0]
    s.copy_(t)
    assert not s.is_contiguous()
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ROWS))
def test_every_tensor_argument_is_checked_before_launch(ext, c, name):
    _fn(ext, name)(*_plain(ROWS[name](c)))             # the valid call
    torch.cuda.synchronize()
    args = ROWS[name](c)
    for i, j, a in _slots(args):
        t = _plain(a)
        _rejected(ext, name, args, i, j, t.cpu(), "a host tensor")
        if isinstance(a, Req) and a.dtype:
            _rejected(ext, name, args, i, j, _wrong_dtype(t), "dtype %s" % _wrong_dtype(t).dtype)
        if isinstance(a, Req) and a.contiguous and t.numel() > 1:
            _rejected(ext, name, args, i, j, _strided(t), "a strided view")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ROWS))
def test_every_tensor_argument_on_another_gpu_is_rejected(ext, c, name):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    args = ROWS[name](c)
    slots = _slots(args)
    if len(slots) < 2:
        pytest.skip("one tensor argument: it sets the op's device")
    for i, j, a in slots:
        _rejected(ext, name, args, i, j, _plain(a).to("cuda:1"), "a tensor on cuda:1")
