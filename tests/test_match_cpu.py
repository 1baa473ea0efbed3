"""CPU tests of frame correspondences: the brute-force restatement (tests/match_reference.py) against scipy's cKDTree in
fp64, the argument checks of match_frames (raised before anything reaches the device), the workspace sizes, and the C entry
points' argument checks on host pointers (no kernel is launched)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import match_reference as R


def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_agrees_with_kdtree(seed):
    spatial = pytest.importorskip("scipy.spatial")
    rs = np.random.RandomState(seed)
    target = rs.randn(1, 17, 23, 3).astype(np.float32) * np.float32(0.3)
    query = rs.randn(1, 11, 13, 3).astype(np.float32) * np.float32(0.3)
    index, distance, _, _ = R.match(query, target)
    t64 = target.reshape(-1, 3).astype(np.float64)
    q64 = query.reshape(-1, 3).astype(np.float64)
    d64, i64 = spatial.cKDTree(t64).query(q64)
    ours = index.reshape(-1)
    diff = ours != i64
    # where the fp32 choice differs, the two candidates' fp64 distances differ by less than fp32 rounding
    d_ours = np.linalg.norm(t64[ours] - q64, axis=1)
    assert np.all(np.abs(d_ours[diff] - d64[diff]) <= 4e-7 * np.maximum(d64[diff], 1e-30) ** 1 + 1e-12)
    assert diff.mean() < 0.02
    assert np.allclose(distance.reshape(-1), d64, rtol=1e-6, atol=1e-7)


def test_restatement_rules():
    q = np.zeros((1, 1, 2, 3), np.float32)
    q[0, 0, 1] = [5, 0, 0]
    t = np.zeros((1, 2, 2, 3), np.float32)
    t[0, 0, 0] = [1, 0, 0]
    t[0, 0, 1] = [-1, 0, 0]              # a tie with index 0: the smaller index wins
    t[0, 1, 0] = [np.nan, 0, 0]          # never valid
    t[0, 1, 1] = [4, 0, 0]
    idx, dist, flow, cons = R.match(q, t, round_trip=True, round_trip_pixels=0.5)
    assert idx.tolist() == [[[0, 3]]] and dist.tolist() == [[[1.0, 1.0]]]
    assert flow[0, 0, 0].tolist() == [0.0, 0.0] and flow[0, 0, 1].tolist() == [0.0, 1.0]
    assert cons.tolist() == [[[True, True]]]
    idx, dist, flow, _ = R.match(q, t, max_distance=np.nextafter(np.float32(1), np.float32(0)))
    assert idx.tolist() == [[[-1, -1]]] and np.isinf(dist).all() and np.isnan(flow).all()
    idx, _, _, _ = R.match(q, t, target_mask=np.array([[[0, 1], [1, 0]]]))
    assert idx.tolist() == [[[1, 1]]]


def test_match_frames_refuses_before_launch():
    from nonrigid_nerf_b200 import correspondence as M
    q = torch.zeros(2, 3, 4, 3)
    bad = [
        (lambda: M.match_frames(q, torch.zeros(3, 3, 4, 3)), "do not pair"),
        (lambda: M.match_frames(q, torch.zeros(2, 3, 4)), "must be [F, H, W, 3]"),
        (lambda: M.match_frames(q.reshape(2, 12, 3), q), "needs its frame size"),
        (lambda: M.match_frames(q.reshape(2, 12, 3), q, size=(5, 2)), "points per frame"),
        (lambda: M.match_frames(q, q, size=(4, 3)), "not frames of"),
        (lambda: M.match_frames(q, q, max_distance=-1.0), "max_distance"),
        (lambda: M.match_frames(q, q, max_distance=float("nan")), "max_distance"),
        (lambda: M.match_frames(q, q, round_trip=True, round_trip_pixels=float("nan")), "round_trip_pixels"),
        (lambda: M.match_frames(q, q, query_mask=torch.ones(2, 4, 3, dtype=torch.bool)), "query_mask"),
        (lambda: M.match_frames(q, q, target_mask=torch.ones(1, 3, 4, dtype=torch.bool)), "target_mask"),
        (lambda: M.match_frames(torch.zeros(1, 0, 4, 3), q), "height and width"),
        (lambda: M.match_frames(q, q), "CUDA tensors"),
        (lambda: M.match_frames(q.numpy(), q), "CUDA tensor"),
    ]
    for call, text in bad:
        with pytest.raises(RuntimeError, match=None) as e:
            call()
        assert text in str(e.value), (text, str(e.value))


def _cloud(F, N):
    n = max(1, int(round((max(1, N // 2)) ** (1 / 3))))
    while n ** 3 > max(1, N // 2):
        n -= 1
    while (n + 1) ** 3 <= max(1, N // 2):
        n += 1
    a = lambda b: (b + 255) // 256 * 256
    C_ = n ** 3
    return a(32 * F) + a(4 * F * C_) + a(4 * F * (C_ + 1)) + a(16 * F * N)


def test_workspace_sizes():
    _, lib = _lib()
    ws = lib.nrn_match_workspace_bytes
    for fq, hq, wq, ft, ht, wt in [(1, 1, 1, 1, 1, 1), (86, 378, 504, 86, 378, 504), (1, 378, 504, 86, 378, 504),
                                   (5, 7, 9, 1, 11, 13), (1, 756, 1008, 1, 756, 1008)]:
        assert ws(fq, hq, wq, ft, ht, wt, 0) == _cloud(ft, ht * wt)
        assert ws(fq, hq, wq, ft, ht, wt, 1) == _cloud(ft, ht * wt) + _cloud(fq, hq * wq)
    # pinned: 86 frames at 504 x 378 (45^3 cells each) and one 1008 x 756 frame (72^3 cells)
    assert ws(86, 378, 504, 86, 378, 504, 0) == 324_841_984
    assert ws(1, 756, 1008, 1, 756, 1008, 1) == 30_358_528
    assert ws(1, 1, 1, 1, 1, 1, 0) == 1024
    for args in [(2, 4, 4, 3, 4, 4, 0), (-1, 4, 4, -1, 4, 4, 0), (1, 0, 4, 1, 4, 4, 0), (1, 4, 4, 1, 1 << 25, 1, 0),
                 (1, 65536, 65536, 1, 4, 4, 0), (65536, 4, 4, 65536, 4, 4, 0)]:
        assert ws(*args) == 0, args


def test_c_entry_point_checks():
    L, lib = _lib()
    assert lib.nrn_match(None) == -1 and b"null args" in lib.nrn_last_error()

    def args(**kw):
        a = L.NrnMatchArgs()
        a.n_query_frames, a.query_height, a.query_width = 2, 3, 4
        a.n_target_frames, a.target_height, a.target_width = 2, 3, 4
        a.max_distance, a.round_trip, a.round_trip_pixels = math.inf, 0, 1.0
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    buf = (C.c_uint8 * 4096)()
    base = (C.addressof(buf) + 255) // 256 * 256
    full = dict(query=base, target=base, index=base, distance=base, flow=base, workspace=base, workspace_bytes=1 << 20)
    cases = [
        (dict(n_query_frames=2, n_target_frames=3), b"do not pair"),
        (dict(n_query_frames=-1), b"do not pair"),
        (dict(query_height=0), b"height and width"),
        (dict(target_width=-4), b"height and width"),
        (dict(max_distance=-1.0), b"max_distance"),
        (dict(max_distance=math.nan), b"max_distance"),
        (dict(round_trip=1, round_trip_pixels=-0.5), b"round_trip_pixels"),
        (dict(), b"null argument"),
        (dict(full, round_trip=1), b"null argument"),
        (dict(full, query=base + 2), b"4-byte aligned"),
        (dict(full, flow=base + 1), b"4-byte aligned"),
        (dict(full, workspace=base + 16), b"256-byte aligned"),
        (dict(full, workspace_bytes=100), b"needed"),
    ]
    for kw, text in cases:
        a = args(**kw)
        assert lib.nrn_match(C.byref(a)) == -1, kw
        assert text in lib.nrn_last_error(), (kw, lib.nrn_last_error())
    # no frame pairs: nothing to do, nothing launched
    assert lib.nrn_match(C.byref(args(n_query_frames=0, n_target_frames=0))) == 0
    assert lib.nrn_match(C.byref(args(n_query_frames=1, n_target_frames=0))) == 0
