"""CPU tests of occupancy grids: the numpy restatement (tests/occupancy_reference.py) against brute force, the refusals of
occupancy_grid and render(..., occupancy=) (raised before anything reaches the device), the workspace sizes, and the C
entry points' argument checks on host pointers (no kernel is launched)."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from tests import occupancy_reference as R


def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


def test_restatement_build_matches_brute_force():
    rs = np.random.RandomState(0)
    sigma = rs.randn(6, 5, 8).astype(np.float32)
    sigma[2, 3, 4] = np.nan
    for d in (0, 1, 3):
        occ = R.build(sigma, 1.2, d)
        nz, ny, nx = occ.shape
        base = np.zeros_like(occ)
        for k, j, i in itertools.product(range(nz), range(ny), range(nx)):
            c = sigma[k:k + 2, j:j + 2, i:i + 2]
            base[k, j, i] = bool(np.any(~(c <= np.float32(1.2))))
        want = np.zeros_like(occ)
        for k, j, i in itertools.product(range(nz), range(ny), range(nx)):
            want[k, j, i] = base[max(k - d, 0):k + d + 1, max(j - d, 0):j + d + 1, max(i - d, 0):i + d + 1].any()
        assert np.array_equal(occ, want)


def test_restatement_pack_and_lookup():
    rs = np.random.RandomState(1)
    occ = rs.rand(3, 4, 11) < 0.4
    bits = R.pack(occ)
    assert bits.dtype == np.int32 and bits.size == (occ.size + 31) // 32
    assert np.array_equal(R.unpack(bits, occ.shape), occ)
    lo, hi = np.float32([-1, 0, 2]), np.float32([1, 2, 5])
    pts = np.array([[-1, 0, 2], [1, 2, 5], [np.nan, 1, 3], [0, np.inf, 3], [2, 1, 3], [0.999, 1.999, 4.999]], np.float32)
    k = R.keep(pts, occ, lo, hi)
    assert k[2] and k[3] and k[4]                         # non-finite and outside: kept
    assert k[0] == occ[0, 0, 0] and k[1] == occ[2, 3, 10]  # box faces: the first and (clamped) last cell
    xyz, idx = R.compact(pts, occ, lo, hi)
    assert np.all(np.diff(idx) > 0) and np.array_equal(xyz, pts[idx], equal_nan=True)


def test_workspace_sizes():
    L, lib = _lib()
    assert lib.nrn_occupancy_words(1, 1, 1) == 1
    assert lib.nrn_occupancy_words(96, 112, 80) == 96 * 112 * 80 // 32
    assert lib.nrn_occupancy_words(0, 1, 1) == 0 and lib.nrn_occupancy_words(4097, 1, 1) == 0
    assert lib.nrn_occupancy_build_workspace_bytes(3, 4, 5) == 120
    assert lib.nrn_occupancy_compact_workspace_bytes(0) == 256
    assert lib.nrn_occupancy_compact_workspace_bytes(1024 * 300) == 1280   # 301 ints, in 256-byte units
    assert lib.nrn_occupancy_compact_workspace_bytes(-1) == 0
    P = 1000 * 64
    assert lib.nrn_occupancy_workspace_bytes(1000, 64, 5, 1) == 16 * P + 12 * P + 4 * P + 20 * P + 256 + 256
    assert lib.nrn_occupancy_workspace_bytes(1000, 64, 4, 0) == 12 * P + 4 * P + 16 * P + 256 + 256
    assert lib.nrn_occupancy_workspace_bytes(1000, 64, 6, 0) == 0


def _grid(L, **kw):
    g = L.NrnOccupancyGrid()
    g.bits, g.nx, g.ny, g.nz = kw.get("bits", 4096), kw.get("nx", 4), kw.get("ny", 4), kw.get("nz", 4)
    g.min_point[:] = kw.get("lo", [-1.0, -1.0, -1.0])
    g.max_point[:] = kw.get("hi", [1.0, 1.0, 1.0])
    return g


def test_c_argument_checks():
    L, lib = _lib()
    err = lambda: lib.nrn_last_error().decode()
    buf = (C.c_float * 64)()
    ws = C.c_void_p(4096)
    # build
    assert lib.nrn_occupancy_build(buf, 0, 2, 2, 0.5, 1, ws, buf, None) == -1 and "out of range" in err()
    assert lib.nrn_occupancy_build(buf, 2, 2, 2, 0.5, -1, ws, buf, None) == -1 and "dilation" in err()
    assert lib.nrn_occupancy_build(buf, 2, 2, 2, float("nan"), 1, ws, buf, None) == -1 and "NaN" in err()
    assert lib.nrn_occupancy_build(None, 2, 2, 2, 0.5, 1, ws, buf, None) == -1 and "null" in err()
    assert lib.nrn_occupancy_build(buf, 2, 2, 2, 0.5, 1, ws, C.c_void_p(4098), None) == -1 and "aligned" in err()
    # compact
    cnt = C.c_void_p(4096)
    bad_grids = [({"nx": 0}, "out of range"), ({"bits": None}, "bits"), ({"bits": 4098}, "bits"),
                 ({"lo": [1.0, 0.0, 0.0], "hi": [1.0, 1.0, 1.0]}, "max > min"), ({"hi": [float("inf"), 1.0, 1.0]}, "finite"),
                 ({"lo": [0.0, 0.0, 0.0], "hi": [1e-44, 1.0, 1.0]}, "fp32 range")]
    for kw, msg in bad_grids:
        g = _grid(L, **kw)
        assert lib.nrn_occupancy_compact(C.byref(g), buf, 4, 3, buf, buf, cnt, ws, None) == -1 and msg in err(), (kw, err())
    g = _grid(L)
    assert lib.nrn_occupancy_compact(None, buf, 4, 3, buf, buf, cnt, ws, None) == -1 and "null grid" in err()
    assert lib.nrn_occupancy_compact(C.byref(g), buf, -1, 3, buf, buf, cnt, ws, None) == -1 and "n_points" in err()
    assert lib.nrn_occupancy_compact(C.byref(g), buf, 2 ** 31, 3, buf, buf, cnt, ws, None) == -1 and "n_points" in err()
    assert lib.nrn_occupancy_compact(C.byref(g), buf, 4, 2, buf, buf, cnt, ws, None) == -1 and "points_stride" in err()
    assert lib.nrn_occupancy_compact(C.byref(g), None, 4, 3, buf, buf, cnt, ws, None) == -1 and "null" in err()
    assert lib.nrn_occupancy_compact(C.byref(g), buf, 4, 3, buf, buf, cnt, C.c_void_p(4096 + 16), None) == -1 and "256-byte" in err()
    # the render pass
    a = L.NrnFieldArgs()
    a.rays, a.z_vals, a.n_rays, a.n_samples, a.out_ch, a.nerf_packed, a.raw = 4096, 4096, 10, 64, 5, 4096, 4096
    need = lib.nrn_occupancy_workspace_bytes(10, 64, 5, 0)
    assert lib.nrn_field_forward_occupancy(C.byref(a), None, ws, need) == -1 and "null grid" in err()
    assert lib.nrn_field_forward_occupancy(C.byref(a), C.byref(g), ws, need - 1) == -1 and "workspace" in err()
    assert lib.nrn_field_forward_occupancy(C.byref(a), C.byref(g), C.c_void_p(4096 + 16), need) == -1 and "workspace" in err()
    a.stash, a.relu_mask = 4096, 4096
    assert lib.nrn_field_forward_occupancy(C.byref(a), C.byref(g), ws, need) == -1 and "inference only" in err()
    a.stash = a.relu_mask = None
    a.points, a.points_stride = 4096, 3
    assert lib.nrn_field_forward_occupancy(C.byref(a), C.byref(g), ws, need) == -1 and "ray mode" in err()
    a.points = None
    a.raw = None
    assert lib.nrn_field_forward_occupancy(C.byref(a), C.byref(g), ws, need) == -1 and "raw" in err()
    a.raw, a.out_ch = 4096, 6
    assert lib.nrn_field_forward_occupancy(C.byref(a), C.byref(g), ws, need) == -1 and "out_ch" in err()


def _nets(**kw):
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    embed_fn, input_ch = H.get_embedder(10, 0)
    base = dict(D=8, W=256, input_ch=input_ch, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False, ray_bender=None,
                ray_bending_latent_size=32)
    base.update(kw)
    return H.NeRF(**base)


def test_refusals_before_launch():
    from nonrigid_nerf_b200 import geometry as G, train as T
    grid = G.OccupancyGrid(torch.zeros(2, dtype=torch.int32), np.float32([-1] * 3), np.float32([1] * 3), (4, 4, 4))
    views = _nets(use_viewdirs=True, input_ch_views=27, output_ch=4)
    tc = _nets(time_conditioned_baseline=True)
    plain = _nets()
    with pytest.raises(RuntimeError, match="use_viewdirs=True"):
        G.occupancy_grid(views, [-1] * 3, [1] * 3, 8, 1.0)
    with pytest.raises(RuntimeError, match="time_conditioned_baseline=True"):
        G.occupancy_grid(tc, [-1] * 3, [1] * 3, 8, 1.0)
    with pytest.raises(RuntimeError, match="resolution"):
        G.occupancy_grid(plain, [-1] * 3, [1] * 3, 0, 1.0)
    rays_o, rays_d = torch.zeros(4, 3), torch.ones(4, 3)
    kw = dict(near=0.0, far=1.0, ndc=False, N_samples=8, N_importance=0, network_query_fn=None, perturb=0.0, white_bkgd=False,
              raw_noise_std=0.0, lindisp=False, additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="use_viewdirs=True"):
            T.render(rays_o, rays_d, use_viewdirs=True, network_fn=views, occupancy=grid, **kw)
        with pytest.raises(RuntimeError, match="time_conditioned_baseline=True"):
            T.render(rays_o, rays_d, network_fn=tc, occupancy=grid, **kw)
        with pytest.raises(RuntimeError, match="OccupancyGrid"):
            T.render(rays_o, rays_d, network_fn=plain, occupancy=grid.bits, **kw)
    with pytest.raises(RuntimeError, match="inference only"):    # parameters that require a gradient: a differentiable call
        T.render(rays_o, rays_d, network_fn=plain, occupancy=grid, **kw)
    with pytest.raises(RuntimeError, match="inference only"):
        T.render_rays(torch.zeros(4, 8), plain, None, 8, occupancy=grid,
                      additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
