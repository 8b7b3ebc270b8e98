"""dpvo_softagg_fused (the SoftAgg f|g layer fused with its segment softmax) vs the two-kernel form it replaces:
linear_f16 of the stacked f|g layer followed by softagg_reduce, on the same inputs and groupings."""
import ctypes

import pytest
import torch

import dpvo_b200
from dpvo_b200 import synthetic
from dpvo_b200.net import Update, EdgeGroups, DIM

DEV = "cuda"
gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def packed():
    torch.manual_seed(5)
    return Update().to(DEV).eval().packed()


def _fp16_ulps(y, ref):
    """|y - ref| in units of the fp16 spacing at ref"""
    a = ref.float().abs().clamp(min=2.0 ** -14)
    return ((y.float() - ref.float()).abs() / torch.exp2(torch.floor(torch.log2(a)) - 10)).max().item()


def _check(ex, P, x, grp, max_groups, nm="kk"):
    fg = ex.linear_f16(x, P["fg_" + nm][0], P["fg_" + nm][1], 0)
    ref = ex.softagg_reduce(fg, grp.order, grp.group_start, grp.n, max_groups)
    y = ex.softagg_fused(x, grp.order, grp.group_of, grp.group_start, grp.n, max_groups, *P["fgi_" + nm])
    y2 = ex.softagg_fused(x, grp.order, grp.group_of, grp.group_start, grp.n, max_groups, *P["fgi_" + nm])
    assert y.shape == ref.shape == (1, max_groups, DIM)
    assert torch.isfinite(y).all()
    assert torch.equal(y, y2), "two launches differ"
    G = int(grp.n.item())
    assert _fp16_ulps(y[0, :G], ref[0, :G]) <= 2
    assert (y[0, G:] == 0).all() and not torch.signbit(y[0, G:]).any(), "padding rows must be exactly zero"
    return G


def _grouping(sizes, seed):
    """a grouping with the given group sizes, rows dealt to groups in a random order"""
    g = torch.Generator().manual_seed(seed)
    key = torch.repeat_interleave(torch.arange(len(sizes)), torch.as_tensor(sizes))
    key = key[torch.randperm(key.numel(), generator=g)]
    return EdgeGroups(key.to(DEV))


@gpu
def test_bench_groupings(ext, packed):
    """both groupings of the bench graph (E = 47,712): patches (kk, ~22 rows) and frame pairs (ij, ~96 rows)"""
    st = synthetic.make_state("default", 36, device=DEV, features=False)
    assert st.E == 47712
    x = (torch.randn(1, st.E, DIM, device=DEV) / 2).half()
    gk, gp = EdgeGroups.pair((st.kk, None, st.jj), (st.ii, st.jj, None))
    _check(ext[3], packed, x, gk, gk.max_groups, "kk")
    _check(ext[3], packed, x, gp, gp.max_groups, "ij")


@gpu
@pytest.mark.parametrize("case", ["ragged", "large_groups", "single_rows", "padded"])
def test_group_shapes(ext, packed, case):
    g = torch.Generator().manual_seed(11)
    E = 132 * 64 + 5
    if case == "single_rows":
        sizes = [1] * E
    else:                               # large_groups: every group spans more than two 64-row tiles
        lo, hi = (130, 400) if case == "large_groups" else (1, 150)
        sizes = []
        while sum(sizes) < E:
            sizes.append(int(torch.randint(lo, hi, (1,), generator=g)))
        sizes[-1] -= sum(sizes) - E     # the last group takes the remainder (>= 1 row)
    x =(torch.randn(1, E, DIM, device=DEV) * 2).half()
    grp = _grouping(sizes, 12)
    G = len(sizes)
    max_groups = min(E, G + 77) if case == "padded" else G
    assert _check(ext[3], packed, x, grp, max_groups, "ij") == G


@gpu
def test_bad_arguments(ext, packed):
    ex = ext[3]
    E = 256
    x = torch.randn(1, E, DIM, device=DEV).half()
    grp = _grouping([64] * 4, 3)
    w, b = packed["fgi_kk"]
    args = (grp.order, grp.group_of, grp.group_start, grp.n, 4)
    with pytest.raises(RuntimeError, match="float16"):
        ex.softagg_fused(x.float(), *args, w, b)
    with pytest.raises(RuntimeError, match=r"\[2\*dim, dim\]"):
        ex.softagg_fused(x, *args, w[:DIM], b)
    with pytest.raises(RuntimeError, match="float32"):
        ex.softagg_fused(x, *args, w, b.half())
    with pytest.raises(RuntimeError, match="one entry per row"):
        ex.softagg_fused(x[:, :100], *args, w, b)
    with pytest.raises(RuntimeError, match="max_groups"):
        ex.softagg_fused(x, grp.order, grp.group_of, grp.group_start, grp.n, E + 1, w, b)
    with pytest.raises(RuntimeError, match="workspace"):
        ex.softagg_fused(x, *args, w, b, torch.empty(16, dtype=torch.uint8, device=DEV))
    with pytest.raises(RuntimeError, match="dim"):            # the kernel is built for 384 channels
        ex.softagg_fused(x[..., :192].contiguous(), *args, w[:384, :192].contiguous(), b[:384])


def test_c_abi_validation_needs_no_gpu():
    """bad arguments are rejected on the host before any CUDA call"""
    lib = dpvo_b200.library()
    lib.dpvo_softagg_fused_workspace_bytes.restype = ctypes.c_int64
    lib.dpvo_softagg_fused_workspace_bytes.argtypes = [ctypes.c_int64]
    assert lib.dpvo_softagg_fused_workspace_bytes(47712) == 746 * 2 * 3 * 384 * 4
    i64 = ctypes.c_int64
    buf = ctypes.create_string_buffer(64)
    rc = lib.dpvo_softagg_fused(buf, i64(384), None, None, buf, buf, buf, buf, i64(100), i64(10), buf, buf, i64(1 << 20), 384, None)
    assert rc == 1 and b"null" in lib.dpvo_last_error()
    rc = lib.dpvo_softagg_fused(buf, i64(384), buf, buf, buf, buf, buf, buf, i64(100), i64(10), buf, buf, i64(1 << 20), 256, None)
    assert rc == 1 and b"dim" in lib.dpvo_last_error()
    rc = lib.dpvo_softagg_fused(buf, i64(384), buf, buf, buf, buf, buf, buf, i64(100), i64(10), buf, buf, i64(16), 384, None)
    assert rc == 1 and b"workspace" in lib.dpvo_last_error()
