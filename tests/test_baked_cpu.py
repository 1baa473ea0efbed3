"""CPU tests of baked radiance grids: the numpy restatement (tests/baked_reference.py) against fp64 trilinear
interpolation, the refusals of bake_radiance and render(..., baked=) (raised before anything reaches the device), the
workspace sizes, and the C entry points' argument checks on host pointers (no kernel is launched)."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import baked_reference as R


def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


def _trilinear64(values, points, lo, hi):
    """fp64 trilinear interpolation of values [nz, ny, nx, 4] at points [P, 3] inside the box."""
    nz, ny, nx, _ = values.shape
    n = np.array([nx, ny, nz], np.float64)
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    u = (np.asarray(points, np.float64) - lo) / (hi - lo) * (n - 1)
    c = np.minimum(np.floor(u).astype(np.int64), (n - 2).astype(np.int64))
    f = u - c
    v = values.astype(np.float64)
    out = np.zeros((u.shape[0], 4))
    for q in range(8):
        dx, dy, dz = q & 1, (q >> 1) & 1, (q >> 2) & 1
        w = (f[:, 0] if dx else 1 - f[:, 0]) * (f[:, 1] if dy else 1 - f[:, 1]) * (f[:, 2] if dz else 1 - f[:, 2])
        out += w[:, None] * v[c[:, 2] + dz, c[:, 1] + dy, c[:, 0] + dx]
    return out


@pytest.mark.parametrize("res", [(2, 2, 2), (17, 33, 9), (64, 5, 40)])
def test_restatement_against_fp64_trilinear(res):
    rs = np.random.RandomState(sum(res))
    nx, ny, nz = res
    lo, hi = np.float32([-1.5, 0.25, -0.7]), np.float32([1.0, 2.0, 0.9])
    values = rs.uniform(-1, 1, size=(nz, ny, nx, 4)).astype(np.float16)
    pts = rs.uniform(lo, hi, size=(20000, 3)).astype(np.float32)
    inside, raw = R.lookup(pts, values, lo, hi)
    assert inside.all()
    want = _trilinear64(values, pts, lo, hi)
    # fp32 rounding: u carries an error of a few ulp(n), which moves the result by up to that times the largest step
    # between neighbours (< 2), and each of the seven lerps rounds once
    assert np.abs(raw - want).max() < 4 * max(res) * 2.0 ** -23 * 2 + 8 * 2.0 ** -24
    # the vertices themselves: their stored values, up to the same rounding
    verts = R.vertex_points(lo, hi, res).reshape(-1, 3)
    inside, raw = R.lookup(verts, values, lo, hi)
    assert inside.all()
    assert np.abs(raw - values.reshape(-1, 4).astype(np.float32)).max() < 4 * max(res) * 2.0 ** -23 * 2


def test_restatement_box_faces_and_non_finite():
    lo, hi = np.float32([-1, 0, 2]), np.float32([1, 2, 5])
    values = np.arange(3 * 4 * 5 * 4, dtype=np.float32).reshape(5, 4, 3, 4).astype(np.float16)
    below, above = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
    pts = np.array([lo, hi, [below[0], 1, 3], [above[0], 1, 3], [0, below[1], 3], [0, 1, above[2]],
                    [np.nan, 1, 3], [0, np.inf, 3], [0, 1, -np.inf]], np.float32)
    inside, raw = R.lookup(pts, values, lo, hi)
    assert inside.tolist() == [True, True] + [False] * 7
    assert np.array_equal(raw[0], values[0, 0, 0].astype(np.float32))     # the first vertex exactly
    assert np.array_equal(raw[1], values[-1, -1, -1].astype(np.float32))  # the last: i = n - 2, f = 1
    assert np.isnan(raw[2:]).all()


def test_restatement_nan_corner_spreads_to_its_cells_only():
    values = np.ones((3, 3, 3, 4), np.float16)
    values[1, 1, 1, 2] = np.nan
    lo, hi = np.float32([0, 0, 0]), np.float32([2, 2, 2])
    pts = np.array([[0.5, 0.5, 0.5], [1.5, 1.5, 1.5], [0.0, 0.0, 0.0]], np.float32)
    _, raw = R.lookup(pts, values, lo, hi)
    assert np.isnan(raw[:2, 2]).all() and not np.isnan(raw[:2, [0, 1, 3]]).any()
    assert np.isnan(raw[2, 2])   # f = 0 still multiplies the NaN corner: 0 * NaN
    assert np.array_equal(raw[2, [0, 1, 3]], np.ones(3, np.float32))


def test_restatement_fp16_store():
    raw = np.array([[1.0, -2.5, 65504.0, 65519.0], [65520.0, -1e30, np.inf, -np.inf], [np.nan, 1e-8, 3.14159, -0.0],
                    [6e-5, 1e-4, 0.1, 1.0 + 2.0 ** -11]], np.float32)
    h = R.to_f16(raw)
    assert h.dtype == np.float16
    assert h[0].tolist() == [1.0, -2.5, 65504.0, 65504.0]
    assert h[1, 0] == 65504 and h[1, 1] == -65504 and h[1, 2] == np.inf and h[1, 3] == -np.inf   # saturation; inf stays
    assert np.isnan(h[2, 0]) and np.signbit(h[2, 3])
    assert np.array_equal(h[3], raw[3].astype(np.float16))        # round to nearest even inside the range
    assert h[3, 3] == np.float16(1.0)                                # a tie rounds to even


def test_vertex_points_are_the_mesh_grid():
    from tests import mesh_reference as M
    lo, hi, res = np.float32([-1, 0.5, 2]), np.float32([0.3, 0.9, 7]), (5, 3, 4)
    p = R.vertex_points(lo, hi, res)
    assert p.shape == (4, 3, 5, 3) and p.dtype == np.float32
    assert np.array_equal(p[2], M.grid_points_plane(lo, hi, res, 2))
    assert np.array_equal(p[-1, -1, -1], hi) and np.array_equal(p[0, 0, 0], lo)


def test_workspace_sizes_and_timing_kinds():
    L, lib = _lib()
    for args in ((1000, 64, 5, 1), (1000, 64, 4, 0), (1, 1, 5, 1), (0, 64, 5, 0)):
        assert lib.nrn_baked_workspace_bytes(*args) == lib.nrn_occupancy_workspace_bytes(*args) + 256
    assert lib.nrn_baked_workspace_bytes(1000, 64, 6, 0) == 0
    assert lib.nrn_baked_workspace_bytes(-1, 64, 5, 0) == 0
    assert lib.nrn_baked_workspace_bytes(1 << 20, 1 << 12, 5, 0) == 0   # more than 2^31 - 1 points
    kinds = (L.KERNEL_KINDS + L.TC_KERNEL_KINDS + L.VIEW_KERNEL_KINDS + L.VIEW_TRAIN_KERNEL_KINDS + L.DET_KERNEL_KINDS
             + L.HELD_OUT_KERNEL_KINDS + L.EVAL_KERNEL_KINDS + L.FRAME_IMAGE_KERNEL_KINDS + L.MESH_KERNEL_KINDS
             + L.LPIPS_KERNEL_KINDS + L.MATCH_KERNEL_KINDS + L.OCCUPANCY_KERNEL_KINDS + L.TERMINATION_KERNEL_KINDS
             + L.DEFORM_KERNEL_KINDS + L.NORMAL_KERNEL_KINDS + L.LPIPS_MAP_KERNEL_KINDS)
    assert len(kinds) == 45   # the baked kinds are 45 to 49
    assert L.BAKED_KERNEL_KINDS == ("baked_plane", "baked_bend", "baked_compact", "baked_field", "baked_scatter")


def _grid(L, **kw):
    g = L.NrnRadianceGrid()
    g.values, g.nx, g.ny, g.nz = kw.get("values", 4096), kw.get("nx", 4), kw.get("ny", 4), kw.get("nz", 4)
    g.min_point[:] = kw.get("lo", [-1.0, -1.0, -1.0])
    g.max_point[:] = kw.get("hi", [1.0, 1.0, 1.0])
    return g


def test_c_argument_checks():
    L, lib = _lib()
    err = lambda: lib.nrn_last_error().decode()
    buf = (C.c_float * 64)()
    plane = C.c_void_p(4096)
    # the plane store
    assert lib.nrn_radiance_plane_f16(buf, -1, 5, plane, None) == -1 and "bad sizes" in err()
    assert lib.nrn_radiance_plane_f16(buf, 4, 3, plane, None) == -1 and "bad sizes" in err()
    assert lib.nrn_radiance_plane_f16(buf, 4, 6, plane, None) == -1 and "bad sizes" in err()
    assert lib.nrn_radiance_plane_f16(None, 4, 5, plane, None) == -1 and "null" in err()
    assert lib.nrn_radiance_plane_f16(buf, 4, 5, None, None) == -1 and "null" in err()
    assert lib.nrn_radiance_plane_f16(buf, 4, 5, C.c_void_p(4100), None) == -1 and "aligned" in err()
    assert lib.nrn_radiance_plane_f16(C.c_void_p(4097), 4, 5, plane, None) == -1 and "aligned" in err()
    assert lib.nrn_radiance_plane_f16(None, 0, 5, None, None) == 0   # nothing to store
    # the render pass
    a = L.NrnFieldArgs()
    a.rays, a.z_vals, a.n_rays, a.n_samples, a.out_ch, a.nerf_packed, a.raw = 4096, 4096, 10, 64, 5, 4096, 4096
    ws = C.c_void_p(4096)
    need = lib.nrn_baked_workspace_bytes(10, 64, 5, 0)
    bad_grids = [({"nx": 1}, "out of range"), ({"nz": 1025}, "out of range"), ({"values": None}, "values"), ({"values": 4100}, "values"),
                 ({"lo": [1.0, 0.0, 0.0], "hi": [1.0, 1.0, 1.0]}, "max > min"), ({"hi": [float("nan"), 1.0, 1.0]}, "finite"),
                 ({"lo": [0.0, 0.0, 0.0], "hi": [1e-44, 1.0, 1.0]}, "fp32 range"),
                 ({"lo": [-3e38, 0.0, 0.0], "hi": [3e38, 1.0, 1.0]}, "fp32 range")]
    for kw, msg in bad_grids:
        g = _grid(L, **kw)
        assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), ws, need) == -1 and msg in err(), (kw, err())
    g = _grid(L)
    assert lib.nrn_field_forward_baked(C.byref(a), None, ws, need) == -1 and "null grid" in err()
    assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), ws, need - 1) == -1 and "workspace" in err()
    assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), C.c_void_p(4096 + 16), need) == -1 and "workspace" in err()
    assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), None, need) == -1 and "workspace" in err()
    a.bender_packed, a.latents, a.latent_stride = 4096, 4096, 32
    assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), ws, need) == -1 and "workspace" in err()   # the bend workspace too
    a.bender_packed = a.latents = None
    a.latent_stride = 0
    a.stash, a.relu_mask = 4096, 4096
    assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), ws, need) == -1 and "inference only" in err()
    a.stash = a.relu_mask = None
    a.points, a.points_stride = 4096, 3
    assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), ws, need) == -1 and "ray mode" in err()
    a.points = None
    a.raw = None
    assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), ws, need) == -1 and "raw" in err()
    a.raw, a.out_ch = 4096, 6
    assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), ws, need) == -1 and "out_ch" in err()
    a.out_ch, a.n_rays = 5, 0
    assert lib.nrn_field_forward_baked(C.byref(a), C.byref(g), None, 0) == 0   # no rays: nothing to do


def _nets(**kw):
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    embed_fn, input_ch = H.get_embedder(10, 0)
    base = dict(D=8, W=256, input_ch=input_ch, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False, ray_bender=None,
                ray_bending_latent_size=32)
    base.update(kw)
    return H.NeRF(**base)


def _grid_py(res=(4, 4, 4), dtype=torch.float16, shape=None):
    from nonrigid_nerf_b200 import geometry as G
    nx, ny, nz = res
    return G.RadianceGrid(torch.zeros(shape or (nz, ny, nx, 4), dtype=dtype), np.float32([-1] * 3), np.float32([1] * 3), res)


def test_bake_refusals_before_launch():
    from nonrigid_nerf_b200 import geometry as G
    views = _nets(use_viewdirs=True, input_ch_views=27, output_ch=4)
    tc = _nets(time_conditioned_baseline=True)
    plain = _nets()   # on the CPU: anything that reached the device would fail with another message
    with pytest.raises(RuntimeError, match="use_viewdirs=True"):
        G.bake_radiance(views, [-1] * 3, [1] * 3, 8)
    with pytest.raises(RuntimeError, match="time_conditioned_baseline=True"):
        G.bake_radiance(tc, [-1] * 3, [1] * 3, 8)
    for res in (1, 1025, (8, 8, 1), (2, 1025, 2), (8, 8), 2.0, (8, 8, True)):
        with pytest.raises(RuntimeError, match="resolution"):
            G.bake_radiance(plain, [-1] * 3, [1] * 3, res)
    for lo, hi in (([0, 0, 0], [1, 0, 1]), ([0, 2, 0], [1, 1, 1]), ([0, 0, 0], [1, 1, np.inf]), ([np.nan, 0, 0], [1, 1, 1])):
        with pytest.raises(RuntimeError, match="must exceed min_point"):
            G.bake_radiance(plain, lo, hi, 8)
    with pytest.raises(RuntimeError, match="CUDA device"):   # past the refusals, the CPU model is where the bake stops
        G.bake_radiance(plain, [-1] * 3, [1] * 3, 8)


def test_grid_struct_checks():
    g = _grid_py()
    for bad in (_grid_py(dtype=torch.float32), _grid_py(shape=(4, 4, 4, 3)), _grid_py(shape=(4, 4, 5, 4)), _grid_py(res=(4, 4, 5), shape=(4, 4, 4, 4))):
        with pytest.raises(RuntimeError, match="float16 tensor"):
            bad.c_struct("cpu")
    with pytest.raises(RuntimeError, match="is on cpu"):
        g.c_struct("cuda:0")
    s = g.c_struct("cpu")
    assert (s.nx, s.ny, s.nz) == (4, 4, 4) and list(s.min_point) == [-1.0] * 3 and s.values == g.values.data_ptr()


def test_render_refusals_before_launch():
    from nonrigid_nerf_b200 import geometry as G, train as T
    grid = _grid_py()
    scene = G.BakedScene(grid, grid)
    views = _nets(use_viewdirs=True, input_ch_views=27, output_ch=4)
    tc = _nets(time_conditioned_baseline=True)
    plain = _nets()
    rays_o, rays_d = torch.zeros(4, 3), torch.ones(4, 3)
    kw = dict(near=0.0, far=1.0, ndc=False, N_samples=8, N_importance=0, network_query_fn=None, perturb=0.0, white_bkgd=False,
              raw_noise_std=0.0, lindisp=False, additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="use_viewdirs=True"):
            T.render(rays_o, rays_d, use_viewdirs=True, network_fn=views, baked=scene, **kw)
        with pytest.raises(RuntimeError, match="time_conditioned_baseline=True"):
            T.render(rays_o, rays_d, network_fn=tc, baked=scene, **kw)
        with pytest.raises(RuntimeError, match="BakedScene"):
            T.render(rays_o, rays_d, network_fn=plain, baked=grid, **kw)
        with pytest.raises(RuntimeError, match="RadianceGrid"):
            T.render(rays_o, rays_d, network_fn=plain, baked=G.BakedScene(grid.values), **kw)
        with pytest.raises(RuntimeError, match="occupancy or early_termination"):
            T.render(rays_o, rays_d, network_fn=plain, baked=scene, early_termination=0.01, **kw)
        occ = G.OccupancyGrid(torch.zeros(2, dtype=torch.int32), np.float32([-1] * 3), np.float32([1] * 3), (4, 4, 4))
        with pytest.raises(RuntimeError, match="occupancy or early_termination"):
            T.render(rays_o, rays_d, network_fn=plain, baked=scene, occupancy=occ, **kw)
        fine_kw = dict(kw, N_importance=8)
        with pytest.raises(RuntimeError, match="needs a fine grid"):
            T.render(rays_o, rays_d, network_fn=plain, network_fine=_nets(), baked=G.BakedScene(grid), **fine_kw)
        with pytest.raises(RuntimeError, match="time_conditioned_baseline=True"):   # the fine pass's model is checked too
            T.render(rays_o, rays_d, network_fn=plain, network_fine=tc, baked=scene, **fine_kw)
        with pytest.raises(RuntimeError, match="needs a fine grid"):
            T.render_rays(torch.zeros(4, 8), plain, None, 8, N_importance=8, baked=G.BakedScene(grid),
                          additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
    with pytest.raises(RuntimeError, match="inference only"):    # parameters that require a gradient: a differentiable call
        T.render(rays_o, rays_d, network_fn=plain, baked=scene, **kw)
    with pytest.raises(RuntimeError, match="inference only"):
        T.render_rays(torch.zeros(4, 8), plain, None, 8, baked=scene,
                      additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
