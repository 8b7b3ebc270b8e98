"""dpvo_encode_frames (several images in one pass of the frame encoders) rejects bad arguments on the host, before any
CUDA call, so no GPU is needed here."""
import ctypes

import dpvo_b200

i64 = ctypes.c_int64
M, H, W = 8, 64, 96


def _lib():
    lib = dpvo_b200.library()
    lib.dpvo_encode_frames_workspace_bytes.restype = ctypes.c_int64
    lib.dpvo_encode_frame_workspace_bytes.restype = ctypes.c_int64
    return lib


def _rows(*v):
    return (ctypes.c_int64 * max(len(v), 1))(*v)


def _args(B, frame_row, feat_row, patch_row, p, frame_rows=4, feat_rows=4 * M, patch_rows=4 * M, ws_bytes=1 << 40):
    h, w = 16, 24
    return [p, i64(3 * H * W), i64(H * W), i64(W), i64(1), B, H, W, p, p, p, M,
            p, i64(h * w * 128), i64(w * 128), i64(128),
            p, i64(4 * 6 * 128), i64(6 * 128), i64(128), i64(frame_rows),
            p, i64(9 * 128), i64(3 * 128), i64(128), p, i64(384), i64(feat_rows),
            p, i64(patch_rows), frame_row, feat_row, patch_row, None, p, i64(ws_bytes), None]


def _buf():
    buf = (ctypes.c_char * 4096)()
    addr = (ctypes.addressof(buf) + 15) // 16 * 16
    return buf, ctypes.c_void_p(addr)


def _rejects(lib, args, text):
    rc = lib.dpvo_encode_frames(*args)
    err = lib.dpvo_last_error()
    assert rc == 1 and text in err, (rc, err)


def test_workspace_is_one_block_per_image():
    lib = _lib()
    one = lib.dpvo_encode_frame_workspace_bytes(480, 640)
    assert one > 0
    for B in (1, 2, 8, 64):
        assert lib.dpvo_encode_frames_workspace_bytes(B, 480, 640) == B * one
    assert lib.dpvo_encode_frames_workspace_bytes(0, 480, 640) == 0
    assert lib.dpvo_encode_frames_workspace_bytes(65, 480, 640) == 0


def test_image_count_outside_1_to_64_is_rejected():
    lib = _lib()
    buf, p = _buf()
    r = _rows(*range(65))
    _rejects(lib, _args(0, r, r, r, p), b"B=0 images, 1 to 64")
    _rejects(lib, _args(65, r, r, r, p), b"B=65 images, 1 to 64")


def test_null_pointers_are_rejected():
    lib = _lib()
    buf, p = _buf()
    r = _rows(0, 1)
    for i in (0, 8, 12, 16, 21, 25, 28):                        # images, w16, fmap1, fmap2, gmap, imap, patches
        a = _args(2, r, _rows(0, M), _rows(0, M), p)
        a[i] = None
        _rejects(lib, a, b"null pointer")
    a = _args(2, None, _rows(0, M), _rows(0, M), p)             # a row list
    _rejects(lib, a, b"null pointer")


def test_misaligned_pointers_and_rows_are_rejected():
    lib = _lib()
    buf, p = _buf()
    q = ctypes.c_void_p(p.value + 8)
    a = _args(2, _rows(0, 1), _rows(0, M), _rows(0, M), p)
    a[12] = q                                                   # fmap1
    _rejects(lib, a, b"misaligned")
    a = _args(2, _rows(0, 1), _rows(0, M), _rows(0, M), p)
    a[13] = i64(16 * 24 * 128 + 4)                              # fmap1 ring-row stride
    _rejects(lib, a, b"misaligned")


def test_rows_outside_their_ring_are_rejected():
    lib = _lib()
    buf, p = _buf()
    _rejects(lib, _args(2, _rows(0, 4), _rows(0, M), _rows(0, M), p), b"frame row 4 outside the 4-row")
    _rejects(lib, _args(2, _rows(0, -1), _rows(0, M), _rows(0, M), p), b"frame row -1 outside")
    _rejects(lib, _args(2, _rows(0, 1), _rows(0, 3 * M + 1), _rows(0, M), p), b"gmap / imap ring")
    _rejects(lib, _args(2, _rows(0, 1), _rows(0, M), _rows(0, 4 * M), p), b"patch rows")


def test_two_images_writing_one_row_are_rejected():
    lib = _lib()
    buf, p = _buf()
    _rejects(lib, _args(3, _rows(0, 2, 2), _rows(0, M, 2 * M), _rows(0, M, 2 * M), p), b"images 1 and 2 write the same destination fmap1")
    _rejects(lib, _args(2, _rows(0, 1), _rows(0, M - 1), _rows(0, M), p), b"images 0 and 1 write the same destination gmap / imap")
    _rejects(lib, _args(2, _rows(0, 1), _rows(0, M), _rows(M, 3), p), b"images 0 and 1 write the same destination patch")


def test_a_short_workspace_is_rejected():
    lib = _lib()
    buf, p = _buf()
    need = lib.dpvo_encode_frames_workspace_bytes(2, H, W)
    _rejects(lib, _args(2, _rows(0, 1), _rows(0, M), _rows(0, M), p, ws_bytes=need - 1), b"workspace")
