"""Loop closure without a GPU: oracle/loop.py against the reference's own edges_loop (tests/golden/loop_ref.pt, written
by oracle/make_golden_loop.py), and the host-side rejections of the loop-closure C-ABI (csrc/loop.cu), which happen
before any CUDA call."""
import ctypes
import os

import torch

import dpvo_b200
from oracle import loop as OL

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loop_ref.pt")
i64, f32 = ctypes.c_int64, ctypes.c_float


def _golden():
    return torch.load(GOLDEN)


def _case_scores(c, L):
    M, n = c["M"], c["n"]
    patches = torch.zeros(n * M, 3, 3, 3, dtype=torch.float64)
    patches[:, :, 1, 1] = c["centres"].double()
    sc = OL.scores(c["poses"], patches, c["intrinsics"], n, M, L["removal"], L["max_age"], L["freq"], L["kf_index"])
    return sc


def test_oracle_scores_match_the_reference_flow_mag():
    g = _golden()
    L = g["loop"]
    for name, c in g["cases"].items():
        sc = _case_scores(c, L)
        i0, ni, j0, J = OL.loop_range(c["n"], L["removal"], L["max_age"], L["freq"], L["kf_index"])
        compact = sc.view(J, L["max_age"])[:, :ni].reshape(-1)
        ref = c["scores"].double()
        assert torch.isfinite(ref).all()
        # the reference computes in fp32: its rounding leaves ~1e-5 px on scores of up to tens of px
        err = (compact - ref).abs()
        assert (err <= 2e-5 + 1e-6 * ref.abs()).all(), (name, err.max().item())
        assert torch.isinf(sc.view(J, L["max_age"])[:, ni:]).all()


def test_oracle_selection_matches_the_reference_reduce_edges():
    g = _golden()
    L = g["loop"]
    for name, c in g["cases"].items():
        sc = _case_scores(c, L)
        pairs = OL.select(sc, c["n"], L["removal"], L["max_age"], L["freq"], L["kf_index"], L["thresh"])
        assert len(pairs) > 100, name
        assert pairs == [tuple(p) for p in c["pairs"].tolist()], name


def test_oracle_selection_rules():
    # all scores equal: visited in candidate order; j - i >= 30 only; no two accepted pairs are neighbours in i
    n, removal, age, freq, kfi = 80, 16, 1000, 15, 4
    i0, ni, j0, J = OL.loop_range(n, removal, age, freq, kfi)
    sc = torch.full((J * age,), float("inf"), dtype=torch.float64)
    sc.view(J, age)[:, :ni] = 1.0
    pairs = OL.select(sc, n, removal, age, freq, kfi)
    assert all(j - i >= 30 for i, j in pairs) and any(j - i == 30 for i, j in pairs)
    s = set(pairs)
    assert not any((i + 1, j) in s for i, j in pairs)
    assert len(OL.select(sc, n, removal, age, freq, kfi, max_pairs=7)) == 7
    assert OL.select(sc, n, removal, age, freq, kfi, thresh=1.0) == []


def test_host_graph_keeps_removed_edges_and_loop_edges():
    hg = OL.HostGraph(M=2, removal=4, opt_window=3)
    hg.append([0, 0, 6], [1, 40, 7], [0, 1, 12])
    hg.remove_window(10, lambda e: (1.0, 2.0, 3.0, 4.0))
    # (0, 40) is a loop edge with jj > n - opt_window: kept; (0, 1) goes to the store; (6, 7) is inside the window
    assert sorted(map(tuple, hg.act)) == [(0, 40, 1), (6, 7, 12)]
    assert hg.inac == [[0, 1, 0, 1.0, 2.0, 3.0, 4.0]]
    hg.remove_keyframe(5)
    assert sorted(map(tuple, hg.act)) == [(0, 39, 1), (5, 6, 10)]
    assert hg.inac == [[0, 1, 0, 1.0, 2.0, 3.0, 4.0]]


# ------------------------------------------------------------------------------------ C-ABI host rejections
def _lib():
    lib = dpvo_b200.library()
    lib.dpvo_loop_candidates.restype = ctypes.c_int64
    return lib


def _buf():
    buf = (ctypes.c_char * 4096)()
    return buf, ctypes.c_void_p((ctypes.addressof(buf) + 15) // 16 * 16)


def _rejects(rc, lib, code, text):
    err = lib.dpvo_last_error()
    assert rc == code and text in err, (rc, err)


def test_candidate_count():
    lib = _lib()
    assert lib.dpvo_loop_candidates(1000, 15, 4) == 11000
    assert lib.dpvo_loop_candidates(1000, 4, 4) == 0
    assert lib.dpvo_loop_candidates(0, 15, 4) == 0


def test_scores_rejections():
    lib = _lib()
    buf, p = _buf()
    _rejects(lib.dpvo_loop_scores(p, p, p, p, p, 48, 16, 1000, 4, 4, p, None), lib, 1, b"loop: bad range")
    _rejects(lib.dpvo_loop_scores(p, p, p, p, p, 0, 16, 1000, 15, 4, p, None), lib, 1, b"loop: bad range")
    _rejects(lib.dpvo_loop_scores(p, p, p, p, p, 48, 16, 2000, 15, 4, p, None), lib, 2, b"22000 candidate pairs")
    _rejects(lib.dpvo_loop_scores(p, None, p, p, p, 48, 16, 1000, 15, 4, p, None), lib, 1, b"loop_scores: null pointer")


def test_select_rejections():
    lib = _lib()
    buf, p = _buf()

    def call(max_pairs=10, region=480, scores=p, thresh=64.0, age=1000):
        return lib.dpvo_loop_select(scores, p, p, 48, 16, age, 15, 4, f32(thresh), max_pairs, p, p, p, p, p, p,
                                    i64(region), None, p, None, None)
    _rejects(call(max_pairs=0), lib, 1, b"max_pairs=0")
    _rejects(call(region=479), lib, 1, b"loop region of 479 slots cannot hold 10 pairs of 48 edges")
    _rejects(call(scores=None), lib, 1, b"loop_select: null pointer")
    _rejects(call(age=20000), lib, 2, b"candidate pairs per proposal")


def test_remove_store_rejections():
    lib = _lib()
    buf, p = _buf()

    def call(cap=128, s_cap=256, M=48, removal=16, opt=7, target=p, s_ii=p):
        return lib.dpvo_pgraph_remove_store(p, p, p, p, target, p, i64(cap), p, removal, opt, None, i64(100), i64(4800), M,
                                            p, s_ii, p, p, p, p, i64(s_cap), p, p, None)
    _rejects(call(cap=-1), lib, 1, b"pgraph_remove_store: bad arguments")
    _rejects(call(M=0), lib, 1, b"pgraph_remove_store: bad arguments")
    _rejects(call(opt=0), lib, 1, b"pgraph_remove_store: bad arguments")
    _rejects(call(s_cap=1 << 31), lib, 1, b"exceeds the int32 count")
    _rejects(call(target=None), lib, 1, b"pgraph_remove_store: null pointer")
    _rejects(call(s_ii=None), lib, 1, b"null store pointer")
    assert call(cap=0) == 0


def test_flags_and_normalize_rejections():
    lib = _lib()
    buf, p = _buf()
    _rejects(lib.dpvo_loop_flags(p, p, i64(100), i64(101), i64(50), 16, None, p, None), lib, 1, b"loop_flags: bad sizes")
    _rejects(lib.dpvo_loop_flags(p, p, i64(100), i64(100), i64(50), 16, None, None, None), lib, 1, b"loop_flags: null pointer")
    _rejects(lib.dpvo_loop_normalize(p, p, i64(-1), 48, 3, None), lib, 1, b"loop_normalize: bad sizes")
    _rejects(lib.dpvo_loop_normalize(None, p, i64(5), 48, 3, None), lib, 1, b"loop_normalize: null pointer")
    assert lib.dpvo_loop_normalize(None, None, i64(0), 48, 3, None) == 0
