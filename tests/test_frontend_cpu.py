"""Frame-encoder pieces that need no GPU: frontend.Encoder4 pinned to the reference's BasicEncoder4, the packed weight
layout, and the host-side validation of the encoder entry points of the C-ABI."""
import ctypes
import os

import torch

import dpvo_b200
from dpvo_b200 import frontend
from oracle.make_golden_encoder import OUT, rule_weights


def test_encoder4_matches_reference_basic_encoder4():
    """fnet / inet of frontend.Encoder4 equal dpvo/extractor.py:BasicEncoder4 on the stored fixture (fp32, CPU)"""
    gold = torch.load(OUT)
    for nm, dim, norm, salt in (("fnet", 128, "instance", 0), ("inet", 384, "none", 100)):
        enc = rule_weights(frontend.Encoder4(dim, norm), salt).eval()
        with torch.no_grad():
            y = enc(gold["image"])
        assert y.shape == gold[nm].shape
        err = ((y - gold[nm]).abs().max() / gold[nm].abs().max()).item()
        assert err <= 1e-5, "%s: rel err %g" % (nm, err)


def test_pack_round_trip():
    torch.manual_seed(3)
    p = frontend.Patchifier()
    fe = frontend.FrameEncoder(p)
    w16, b32 = fe.packed()
    assert w16.dtype == torch.half and b32.shape == (2, 11, 384)
    got = fe.unpack()
    for e, enc in enumerate((p.fnet, p.inet)):
        for l, conv in enumerate(frontend.encoder_layers(enc)):
            w, b = got[(e, l)]
            assert torch.equal(w, conv.weight.detach().half()), (e, l)
            assert torch.equal(b, conv.bias.detach().float()), (e, l)
    assert w16.numel() == sum(frontend.pack_conv(c.weight).numel() for enc in (p.fnet, p.inet) for c in frontend.encoder_layers(enc))
    # repacked when a parameter changes in place
    with torch.no_grad():
        p.inet.conv2.bias.add_(1.0)
    assert torch.equal(fe.packed()[1][1, 10, :384], p.inet.conv2.bias.detach().float())


def test_encoder_output_size():
    assert frontend.encoder_output_size(480, 640) == (120, 160)
    assert frontend.encoder_output_size(480, 752) == (120, 188)
    assert frontend.encoder_output_size(250, 330) == (63, 83)


def test_encoder_entry_points_validate_on_the_host():
    lib = dpvo_b200.library()
    i64 = ctypes.c_int64
    lib.dpvo_encode_frame_workspace_bytes.restype = ctypes.c_int64
    lib.dpvo_encoder_conv_workspace_bytes.restype = ctypes.c_int64
    assert lib.dpvo_encode_frame_workspace_bytes(480, 640) > 2 * 4 * 240 * 320 * 32 * 2
    assert lib.dpvo_encoder_conv_workspace_bytes(0, 480, 640) > 0
    assert lib.dpvo_encoder_conv_workspace_bytes(9, 480, 640) == 0
    buf = (ctypes.c_char * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    rc = lib.dpvo_encoder_conv(9, 64, 64, 1, p, None, i64(0), None)
    assert rc == 1 and b"unknown shape" in lib.dpvo_last_error()
    rc = lib.dpvo_encoder_conv(1, 64, 64, 3, p, None, i64(0), None)
    assert rc == 1 and b"nenc" in lib.dpvo_last_error()
    rc = lib.dpvo_encoder_conv(1, 64, 64, 1, None, None, i64(0), None)
    assert rc == 1 and b"null io" in lib.dpvo_last_error()
    rc = lib.dpvo_encoder_conv(1, 64, 64, 1, p, None, i64(0), None)           # zeroed io: no x / w / y
    assert rc == 1 and b"null pointer" in lib.dpvo_last_error()
    args = [p, i64(3), i64(640), i64(1), 480, 640, p, p, p, 96, p, i64(160 * 128), i64(128), p, i64(40 * 128), i64(128),
            p, i64(9 * 128), i64(3 * 128), i64(128), p, i64(384), p, p, i64(1 << 40), None]
    bad = list(args)
    bad[0] = None
    assert lib.dpvo_encode_frame(*bad) == 1 and b"null pointer" in lib.dpvo_last_error()
    bad = list(args)
    bad[9] = 0
    assert lib.dpvo_encode_frame(*bad) == 1 and b"M=0" in lib.dpvo_last_error()
    bad = list(args)
    bad[12] = i64(64)
    assert lib.dpvo_encode_frame(*bad) == 1 and b"channels-last" in lib.dpvo_last_error()
    bad = list(args)
    bad[24] = i64(16)
    assert lib.dpvo_encode_frame(*bad) == 1 and b"workspace" in lib.dpvo_last_error()


def test_shims_refuse_cpu_tensors():
    import pytest
    ex = dpvo_b200.extensions()[3]
    img = torch.zeros(3, 64, 64, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ex.encoder_conv(0, img, torch.zeros(5120, dtype=torch.half), torch.zeros(32))
    z = torch.zeros(1)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ex.encode_frame(img, z, z, z, z, z, z, z, z, z)
    fe = frontend.FrameEncoder(frontend.Patchifier())
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        fe.encode_into(img, 8, "RANDOM", None, None, None, None, None)
