"""The map buffers without a GPU: the colour formula the encoders compute (a host transcription of csrc/encoder.cu's
centroid_color against the reference's torch expression), the layouts and views of map=True states and batches, what
StreamBatch.load / copy_stream carry, and the rejection of map buffers of the wrong shape or dtype."""
import ctypes

import numpy as np
import pytest
import torch

import dpvo_b200
from dpvo_b200 import synthetic
from dpvo_b200.keyframe import Keyframes
from dpvo_b200.patchgraph import DevicePatchGraph
from dpvo_b200.runner import UpdateRunner
from dpvo_b200.streams import StreamBatch

F32 = np.float32


# ------------------------------------------------------------------------------------------------ the colour formula
def host_color(img, fx, fy, c):
    """centroid_color of csrc/encoder.cu, one fp32 operation per step: img uint8 [3, H, W], centroid (fx, fy) in
    feature pixels, output channel c (image channel 2 - c)"""
    H, W = img.shape[1], img.shape[2]
    inv255 = F32(1.0) / F32(255.0)
    px, py = F32(4.0) * (F32(fx) + F32(0.5)), F32(4.0) * (F32(fy) + F32(0.5))
    flx, fly = np.floor(px), np.floor(py)
    dx, dy = px - flx, py - fly
    x0, y0 = int(flx), int(fly)
    v = np.zeros((2, 2), dtype=F32)
    for i in range(2):
        for j in range(2):
            y, x = y0 + i, x0 + j
            if 0 <= y < H and 0 <= x < W:
                v[i, j] = F32(2.0) * (F32(img[2 - c, y, x]) * inv255) - F32(0.5)
    omx, omy = F32(1.0) - dx, F32(1.0) - dy
    s = (((omy * omx) * v[0, 0] + (omy * dx) * v[0, 1]) + (dy * omx) * v[1, 0]) + (dy * dx) * v[1, 1]
    return np.uint8(np.int64(np.trunc((s + F32(0.5)) * F32(127.5))) & 255)


def torch_colors(img, coords, divide=False):
    """Patchifier.forward(return_color=True)'s colour (net.py:142-143 as frontend.Patchifier writes it) and dpvo.py:404,
    in torch on the CPU.  The normalisation 2 (img / 255.0) - 0.5 of dpvo.py:389 runs on the GPU in the reference,
    where PyTorch multiplies by the fp32 reciprocal of a scalar divisor; divide=True takes the CPU kernel's division."""
    x = img.float()
    x = x / 255.0 if divide else x * (torch.tensor(1.0) / torch.tensor(255.0))
    images = 2 * x - 0.5                                                  # [3, H, W]
    H, W = images.shape[1:]
    pc = 4 * (coords + 0.5)                                               # [M, 2]
    fl = pc.floor()
    frac = pc - fl
    dx, dy = frac[:, 0, None], frac[:, 1, None]
    x0, y0 = fl[:, 0].long(), fl[:, 1].long()

    def px(y, x):                                                          # altcorr.patchify's zero-filled window
        ok = (y >= 0) & (y < H) & (x >= 0) & (x < W)
        v = images[:, y.clamp(0, H - 1), x.clamp(0, W - 1)].T           # [M, 3]
        return torch.where(ok[:, None], v, torch.zeros_like(v))

    clr = ((1 - dy) * (1 - dx) * px(y0, x0) + (1 - dy) * dx * px(y0, x0 + 1) +
           dy * (1 - dx) * px(y0 + 1, x0) + dy * dx * px(y0 + 1, x0 + 1))
    return ((clr[:, [2, 1, 0]] + 0.5) * (255.0 / 2)).to(torch.uint8)


def _every_byte_image(H=12, W=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (3, H, W), generator=g, dtype=torch.uint8)
    img.view(-1)[:256] = torch.arange(256, dtype=torch.uint8)             # every byte value in every channel's reach
    return img


def _check(img, coords):
    ref = torch_colors(img, coords)
    for m in range(coords.shape[0]):
        for c in range(3):
            got = host_color(img.numpy(), float(coords[m, 0]), float(coords[m, 1]), c)
            assert got == int(ref[m, c]), "centroid %s channel %d: %d != %d" % (coords[m].tolist(), c, got, int(ref[m, c]))


def test_host_transcription_matches_torch_on_every_byte():
    """integer centroids sample one pixel (weights 1, 0, 0, 0): every byte value 0..255 through the round trip"""
    for v in range(256):
        img = torch.full((3, 8, 8), v, dtype=torch.uint8)
        img[1] = 255 - v
        _check(img, torch.tensor([[0.0, 0.0], [1.0, 1.0]]))
    img = _every_byte_image()
    ys, xs = torch.meshgrid(torch.arange(3), torch.arange(6), indexing="ij")
    _check(img, torch.stack([xs.reshape(-1), ys.reshape(-1)], -1).float())


def test_host_transcription_matches_torch_on_fractional_offsets_and_borders():
    img = _every_byte_image(seed=3)
    g = torch.Generator().manual_seed(5)
    frac = torch.rand(64, 2, generator=g) * torch.tensor([6.0, 3.0]) - 0.6          # x in [-0.6, 5.4), y in [-0.6, 2.4)
    edge = torch.tensor([[-0.6, -0.6], [5.9, 2.9], [5.5, 0.3], [0.25, 2.75], [-0.125, 1.0], [5.75, -0.3]])
    _check(img, torch.cat([frac, edge]))


def test_round_trip_loses_the_low_bytes_and_the_division_matters():
    """fp32 2 (v / 255) - 0.5 back to bytes is not the identity: with the GPU's reciprocal product the bytes 1..23 come
    back one lower, with the CPU's division 1..31 (so the two normalisations differ at 24..31)"""
    v = torch.arange(256, dtype=torch.uint8).view(1, 1, 256).expand(3, 1, 256).contiguous()
    coords = torch.stack([torch.arange(256.0) / 4 - 0.5, torch.full((256,), -0.5)], -1)       # 4 (c + 0.5) = pixel (v, 0)
    gpu, cpu = torch_colors(v, coords)[:, 0].long(), torch_colors(v, coords, divide=True)[:, 0].long()
    assert (gpu != torch.arange(256)).nonzero().view(-1).tolist() == list(range(1, 24))
    assert (cpu != torch.arange(256)).nonzero().view(-1).tolist() == list(range(1, 32))
    assert ((gpu == torch.arange(256)) | (gpu == torch.arange(256) - 1)).all()


# ------------------------------------------------------------------------------------------------ layouts
def test_map_buffers_of_a_state():
    st = synthetic.make_state("fast", 12, device="cpu", features=False, buffer=20, map=True)
    M = st.cfg["M"]
    assert st.points.shape == (20 * M, 3) and st.points.dtype == torch.float32 and st.points.is_contiguous()
    assert st.colors.shape == (20, M, 3) and st.colors.dtype == torch.uint8 and st.colors.is_contiguous()
    plain = synthetic.make_state("fast", 12, device="cpu", features=False, buffer=20)
    assert plain.points is None and plain.colors is None


def test_map_buffers_of_a_batch_are_stacked_and_streams_view_their_rows():
    cfg = synthetic.CONFIGS["fast"]
    B, F, M = 3, 10, cfg["M"]
    batch = StreamBatch(B, cfg, F, 2, device="cpu", map=True)
    assert batch.points.shape == (B * F * M, 3) and batch.colors.shape == (B * F, M, 3)
    for b in range(B):
        s = batch.stream(b)
        assert s.points.shape == (F * M, 3) and s.colors.shape == (F, M, 3)
        assert s.points.data_ptr() == batch.points[b * F * M].data_ptr()
        assert s.colors.data_ptr() == batch.colors[b * F].data_ptr()
        s.points.fill_(b + 1.0)
        s.colors.fill_(b + 1)
    for b in range(B):
        assert (batch.points[b * F * M:(b + 1) * F * M] == b + 1.0).all()
        assert (batch.colors[b * F:(b + 1) * F] == b + 1).all()
    plain = StreamBatch(B, cfg, F, 2, device="cpu")
    assert plain.points is None and plain.colors is None and plain.stream(1).points is None


def test_load_and_copy_stream_carry_the_map():
    cfg = synthetic.CONFIGS["fast"]
    batch = StreamBatch(2, cfg, 8, 4, device="cpu", map=True)
    st = synthetic.make_state("fast", 4, device="cpu", buffer=6, mem=4, map=True)
    g = torch.Generator().manual_seed(1)
    st.points.copy_(torch.randn(st.points.shape, generator=g))
    st.colors.copy_(torch.randint(0, 256, st.colors.shape, generator=g, dtype=torch.uint8))
    batch.points.fill_(9.0)
    batch.colors.fill_(9)
    batch.load(1, st)
    s = batch.stream(1)
    assert torch.equal(s.points[:6 * st.cfg["M"]], st.points) and (s.points[6 * st.cfg["M"]:] == 0).all()
    assert torch.equal(s.colors[:6], st.colors) and (s.colors[6:] == 0).all()
    assert (batch.stream(0).points == 9.0).all() and (batch.stream(0).colors == 9).all()
    c = batch.copy_stream(1)
    assert torch.equal(c.points, s.points) and torch.equal(c.colors, s.colors)
    assert c.points.data_ptr() != s.points.data_ptr() and c.colors.data_ptr() != s.colors.data_ptr()
    # a state without a map loads as an empty map
    batch.load(0, synthetic.make_state("fast", 4, device="cpu", buffer=6, mem=4))
    assert (batch.stream(0).points == 0).all() and (batch.stream(0).colors == 0).all()


# ------------------------------------------------------------------------------------------------ rejection
BAD = [("points", lambda M, N: torch.zeros(N * M, 4)), ("points", lambda M, N: torch.zeros(N * M, 3, dtype=torch.float64)),
       ("points", lambda M, N: torch.zeros(N * M - 1, 3)), ("points", lambda M, N: torch.zeros(3, N * M).T),
       ("colors", lambda M, N: torch.zeros(N, M, 3)), ("colors", lambda M, N: torch.zeros(N, M, 4, dtype=torch.uint8)),
       ("colors", lambda M, N: torch.zeros(N * M, 3, dtype=torch.uint8)), ("colors", lambda M, N: torch.zeros(N + 1, M, 3, dtype=torch.uint8))]


@pytest.mark.parametrize("k", range(len(BAD)))
def test_wrong_map_buffers_are_rejected(k):
    name, make = BAD[k]
    st = synthetic.make_stop_go_state("fast", 12, total=20, device="cpu", features=False)
    synthetic.add_map(st)
    M, N = st.cfg["M"], st.poses.shape[0]
    setattr(st, name, make(M, N))
    with pytest.raises(ValueError, match=name):
        UpdateRunner(st)
    g = DevicePatchGraph(4096, M, N - 1, "cpu")
    with pytest.raises(ValueError, match=name):
        Keyframes(st.cfg, st, g)
    batch = StreamBatch(1, st.cfg, N, 2, device="cpu", map=True)
    with pytest.raises(ValueError, match=name):
        batch.load(0, st)


def test_map_needs_map_buffers():
    st = synthetic.make_state("fast", 12, device="cpu", features=False, buffer=20)
    run = UpdateRunner.__new__(UpdateRunner)
    run.s, run.batch, run.M = st, None, st.cfg["M"]
    with pytest.raises(RuntimeError, match="no map buffers"):
        run.map()


def test_entry_points_reject_bad_arguments_without_a_gpu():
    lib = dpvo_b200.library()
    buf = (ctypes.c_char * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    i64, i32 = ctypes.c_int64, ctypes.c_int
    n = (ctypes.c_int64 * 2)(4, 9)
    assert lib.dpvo_point_cloud(p, p, p, i64(8), i32(48), i32(0), n, p, None) == 1 and b"B=0" in lib.dpvo_last_error()
    assert lib.dpvo_point_cloud(p, p, p, i64(8), i32(48), i32(65), n, p, None) == 1
    assert lib.dpvo_point_cloud(p, p, p, i64(8), i32(48), i32(2), n, p, None) == 1 and b"n=9" in lib.dpvo_last_error()
    assert lib.dpvo_point_cloud(p, None, p, i64(8), i32(48), i32(1), n, p, None) == 1 and b"null" in lib.dpvo_last_error()
    # the byte-granular shift: the slot checks of dpvo_keyframe_shift, without the multiple of 4
    bases = (ctypes.c_void_p * 2)(p.value, p.value)
    rw = (ctypes.c_int64 * 2)(8, 8)
    assert lib.dpvo_keyframe_shift_bytes(bases, (ctypes.c_int64 * 2)(126, 0), rw, i32(2), i64(8), i32(1), i32(4), p, p, None) == 1
    assert b"positive" in lib.dpvo_last_error()
    assert lib.dpvo_keyframe_shift_bytes(bases, (ctypes.c_int64 * 2)(126, 6), (ctypes.c_int64 * 2)(8, 3), i32(2), i64(8), i32(1),
                                         i32(4), p, p, None) == 1
    assert b"fewer than keyframe_index" in lib.dpvo_last_error()
    assert lib.dpvo_keyframe_shift_bytes(bases, (ctypes.c_int64 * 10)(*[4] * 10), (ctypes.c_int64 * 10)(*[8] * 10), i32(10), i64(8),
                                         i32(1), i32(4), p, p, None) == 1
    assert b"buffers=10" in lib.dpvo_last_error()
    # the colour encode: no colour destination
    rows = (ctypes.c_int64 * 1)(0)
    args = [p, i64(0), i64(1), i64(640), i64(1), i32(1), i32(480), i32(640), p, p, p, i32(8), p, i64(0), i64(20480), i64(128),
            p, i64(0), i64(5120), i64(128), i64(1), p, i64(1152), i64(384), i64(128), p, i64(384), i64(8), p, i64(8), rows, rows,
            rows, None, None, p, i64(1 << 30), None]
    assert lib.dpvo_encode_frames_colors(*args) == 1 and b"null colour" in lib.dpvo_last_error()
