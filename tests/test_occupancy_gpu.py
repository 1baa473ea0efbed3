"""Occupancy grids on the GPU: the grid build and the lookup + compaction bit for bit against tests/occupancy_reference.py,
and render(..., occupancy=grid) against render() without one: identical with an all-occupied grid, and for any grid raw =
where(kept, raw of the fused kernel on the same depths, 0) with the maps composited from that raw."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import occupancy_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _G():
    from nonrigid_nerf_b200 import geometry
    return geometry


# ---- grid build --------------------------------------------------------------------------------------------------------
def _check_build(sigma_np, threshold, dilation, lo=(-1.0, -1.0, -1.0), hi=(1.0, 1.0, 1.0)):
    g = _G().occupancy_from_sigma(torch.from_numpy(sigma_np).to(DEV), lo, hi, threshold, dilation)
    want = R.pack(R.build(sigma_np, threshold, dilation))
    got = g.bits.cpu().numpy()
    assert got.shape == want.shape and np.array_equal(got, want), (sigma_np.shape, dilation)
    return g


@pytest.mark.parametrize("n", [1, 2, 3, 7, 31, 64, 100, 257])
def test_build_random_cubes(n):
    rs = np.random.RandomState(n)
    sigma = rs.standard_exponential((n + 1,) * 3).astype(np.float32)
    t = np.float32(2.5)   # corner probability e^-2.5: about half the cells of a cube are occupied before dilation
    for d in (0, 1, 3):
        _check_build(sigma, t, d)


def test_build_box_96x112x80_ties_and_nan():
    rs = np.random.RandomState(5)
    nx, ny, nz = 96, 112, 80
    sigma = rs.standard_exponential((nz + 1, ny + 1, nx + 1)).astype(np.float32) * np.float32(0.5)
    t = np.float32(2.0)
    sigma[rs.rand(*sigma.shape) < 0.01] = t                                     # exactly at the threshold: empty
    sigma[rs.rand(*sigma.shape) < 0.002] = np.nan                               # NaN: occupied
    sigma[rs.rand(*sigma.shape) < 0.001] = np.nextafter(t, np.float32(np.inf))  # one ulp above: occupied
    for d in (0, 1, 3):
        _check_build(sigma, t, d, lo=(-1.5, -2.0, 0.25), hi=(1.5, 2.5, 3.0))


def test_build_single_voxels_at_corners_and_faces():
    n = 9
    for k in (0, n // 2, n):
        for j in (0, n // 2, n):
            for i in (0, n // 2, n):
                sigma = np.zeros((n + 1,) * 3, np.float32)
                sigma[k, j, i] = 1.0
                for d in (0, 1, 3):
                    _check_build(sigma, 0.5, d)
    empty = np.zeros((n + 1,) * 3, np.float32)
    assert _check_build(empty, 0.5, 3).occupied_fraction() == 0.0
    assert _check_build(empty + 1, 0.5, 0).occupied_fraction() == 1.0


# ---- lookup and compaction ---------------------------------------------------------------------------------------------
def _compact(points_np, occ, lo, hi, reruns=1):
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    nz, ny, nx = occ.shape
    grid = _G().OccupancyGrid(torch.from_numpy(R.pack(occ)).to(DEV), np.float32(lo), np.float32(hi), (nx, ny, nz))
    pts = torch.from_numpy(np.ascontiguousarray(points_np, np.float32)).to(DEV)
    P = pts.shape[0]
    outs = []
    for _ in range(reruns):
        xyz = torch.full((max(P, 1), 3), 7.0, device=DEV)
        idx = torch.full((max(P, 1),), -5, dtype=torch.int32, device=DEV)
        cnt = torch.full((1,), -1, dtype=torch.int32, device=DEV)
        ws = torch.empty(lib.nrn_occupancy_compact_workspace_bytes(P), dtype=torch.uint8, device=DEV)
        g = grid.c_struct(pts.device)
        _lib.check(lib.nrn_occupancy_compact(C.byref(g), pts.data_ptr(), P, 3, xyz.data_ptr(), idx.data_ptr(), cnt.data_ptr(),
                                             ws.data_ptr(), torch.cuda.current_stream().cuda_stream), "occupancy_compact")
        k = int(cnt.item())
        outs.append((xyz[:k].cpu().numpy(), idx[:k].cpu().numpy()))
    want_xyz, want_idx = R.compact(points_np, occ, lo, hi)
    for xyz, idx in outs:
        assert np.array_equal(idx, want_idx)
        assert np.array_equal(xyz.view(np.uint32), want_xyz.view(np.uint32))   # bit for bit, NaN payloads included
        assert np.all(np.diff(idx.astype(np.int64)) > 0)
    return outs[0][1]


def _face_points(lo, hi, res):
    """Points on every cell face and box face of each axis, and one ulp either side, with the other coordinates random."""
    rs = np.random.RandomState(3)
    out = []
    for ax in range(3):
        n = res[ax]
        faces = (lo[ax] + (hi[ax] - lo[ax]) * (np.arange(n + 1, dtype=np.float32) / np.float32(n))).astype(np.float32)
        vals = np.concatenate([faces, np.nextafter(faces, np.float32(-np.inf)), np.nextafter(faces, np.float32(np.inf))])
        p = rs.uniform(lo, hi, size=(vals.size, 3)).astype(np.float32)
        p[:, ax] = vals
        out.append(p)
    return np.concatenate(out)


def test_compact_faces_and_non_finite():
    lo, hi = np.float32([-1.0, -0.5, 0.1]), np.float32([1.0, 2.0, 0.9])
    res = (13, 7, 5)
    rs = np.random.RandomState(11)
    occ = rs.rand(res[2], res[1], res[0]) < 0.5
    pts = _face_points(lo, hi, res)
    special = np.array([[np.nan, 0, 0.5], [0, np.nan, 0.5], [0, 0, np.nan], [np.inf, 0, 0.5], [-np.inf, 0, 0.5],
                        [0, np.inf, 0.5], [0, 0, -np.inf], [0, 0, 0.5]], np.float32)
    kept = _compact(np.concatenate([pts, special]), occ, lo, hi, reruns=3)
    assert set(range(pts.shape[0], pts.shape[0] + 7)) <= set(kept.tolist())   # every non-finite point is kept


@pytest.mark.parametrize("P", [0, 1, 1023, 1024, 1025, 3 * 1024 + 17, 1_300_001])
def test_compact_sizes_empty_and_full(P):
    lo, hi = np.float32([-1.0] * 3), np.float32([1.0] * 3)
    rs = np.random.RandomState(P % 1000)
    pts = rs.uniform(-0.99, 0.99, size=(P, 3)).astype(np.float32)
    res = (16, 16, 16)
    empty = np.zeros(res, bool)
    assert _compact(pts, empty, lo, hi).size == 0                     # K = 0
    assert _compact(pts, ~empty, lo, hi).size == P                    # K = P
    _compact(pts, rs.rand(*res) < 0.3, lo, hi, reruns=2)              # ragged last tile, reruns identical


# ---- rendering ---------------------------------------------------------------------------------------------------------
def _models(bender):
    coarse, fine, b, _ = helpers.build_models(O, 900, DEV, with_bender=bender)
    return coarse, fine, b


def _render(coarse, fine, r, n_imp, occupancy=None, chunk=32768, detailed=True, surface=True):
    from nonrigid_nerf_b200 import train as T
    n = r["rays_o"].shape[0]
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=n_imp, network_fine=fine if n_imp else None, N_samples=64,
              network_fn=coarse, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    if occupancy is not None:
        kw["occupancy"] = occupancy
    with torch.no_grad():
        rgb, disp, acc, ex = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=chunk, near=r["near"], far=r["far"],
                                      additional_pixel_information={"ray_bending_latents": r["latents"][:n].to(DEV)},
                                      detailed_output=detailed, retraw=True, surface_output=surface, **kw)
    out = dict(ex)
    out.update(rgb_map=rgb, disp_map=disp, acc_map=acc)
    return out


def _full_grid(lo=(-4.0,) * 3, hi=(4.0,) * 3, res=(8, 8, 8)):
    occ = np.ones(res[::-1], bool)
    return _G().OccupancyGrid(torch.from_numpy(R.pack(occ)).to(DEV), np.float32(lo), np.float32(hi), tuple(res))


def _assert_same(a, b):
    assert set(a) == set(b), set(a) ^ set(b)
    for k in a:
        x, y = a[k].cpu(), b[k].cpu()
        assert x.dtype == y.dtype and x.shape == y.shape, k
        if x.is_floating_point():
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), k   # bit for bit
        else:
            assert torch.equal(x, y), k


@pytest.mark.parametrize("bender", [True, False])
@pytest.mark.parametrize("n_imp", [0, 64])
def test_all_occupied_grid_is_identical(bender, n_imp):
    coarse, fine, b = _models(bender)
    r = O.make_rays(901, 300)
    grid = _full_grid(lo=(-0.2, -0.2, -0.7), hi=(0.3, 0.2, 0.45))   # points outside this small box are kept as well
    for chunk in (32768, 100):
        _assert_same(_render(coarse, fine, r, n_imp, chunk=chunk), _render(coarse, fine, r, n_imp, grid, chunk=chunk))


@pytest.mark.parametrize("knob", ["cutoff", "scaling", "removal"])
def test_all_occupied_grid_with_test_time_knobs(knob):
    coarse, fine, b = _models(True)
    if knob == "cutoff":
        b.rigidity_test_time_cutoff = 0.5
    elif knob == "scaling":
        b.test_time_scaling = 1.7
    else:
        coarse.test_time_nonrigid_object_removal_threshold = 0.5
        fine.test_time_nonrigid_object_removal_threshold = 0.5
    r = O.make_rays(902, 257)
    _assert_same(_render(coarse, fine, r, 64), _render(coarse, fine, r, 64, _full_grid()))


def _random_grid(pts, frac, seed, res=(24, 20, 28)):
    """A grid over the box of pts whose occupied cells, taken in random order, hold about `frac` of pts."""
    lo = (pts.min(0) - np.float32(0.01)).astype(np.float32)
    hi = (pts.max(0) + np.float32(0.01)).astype(np.float32)
    per_cell = np.bincount(R.cells(pts, res, lo, hi), minlength=res[0] * res[1] * res[2])
    order = np.random.RandomState(seed).permutation(per_cell.size)
    take = order[:np.searchsorted(np.cumsum(per_cell[order]), frac * pts.shape[0]) + 1]
    occ = np.zeros(per_cell.size, bool)
    occ[take] = True
    occ = occ.reshape(res[2], res[1], res[0])
    return _G().OccupancyGrid(torch.from_numpy(R.pack(occ)).to(DEV), lo, hi, res), occ


@pytest.mark.parametrize("bender", [True, False])
@pytest.mark.parametrize("frac", [0.5, 0.05])
def test_any_grid_is_masked_full_raw(bender, frac):
    """Per pass: raw = where(kept, fused raw on the grid path's own depths, 0), kept from the numpy lookup of the kernel's
    own bent points; the maps are composite() of that raw."""
    from nonrigid_nerf_b200 import autograd as A, ops
    coarse, fine, b = _models(bender)
    if bender:
        coarse.test_time_nonrigid_object_removal_threshold = 0.6
        fine.test_time_nonrigid_object_removal_threshold = 0.6
    r = O.make_rays(903, 400)
    full = _render(coarse, fine, r, 64, surface=False)
    grid, occ = _random_grid(full["input_pts"].reshape(-1, 3).cpu().numpy(), frac, 7)
    got = _render(coarse, fine, r, 64, grid, surface=False)
    rays = helpers.rays8(r, DEV)
    lat = r["latents"].to(DEV)
    rays_d = rays[:, 3:6]
    with torch.no_grad():
        z = ops.sample_coarse(rays, 64, None, False)
        raw_c, det_c = A.field_occupancy(coarse, rays, z, lat, True, grid)
        full_c, _ = A.field_rays(coarse, rays, z, lat, False)
        c0 = A.composite(raw_c, z, rays_d, None, False, 64, None)
        z_f = c0["z_vals_out"]
        raw_f, det_f = A.field_occupancy(fine, rays, z_f, lat, True, grid)
        full_f, _ = A.field_rays(fine, rays, z_f, lat, False)
        c1 = A.composite(raw_f, z_f, rays_d, None, False)
    kept_fracs = []
    for raw, fullraw, det, pref in ((raw_c, full_c, det_c, ""), (raw_f, full_f, det_f, "fine_")):
        assert torch.equal(det["input_pts"].view(torch.int32), got[pref + "input_pts"].view(torch.int32))
        kept = R.keep(det["input_pts"].reshape(-1, 3).cpu().numpy(), occ, grid.min_point, grid.max_point)
        kept_fracs.append(kept.mean())
        want = np.where(kept[:, None], fullraw.reshape(-1, fullraw.shape[-1]).cpu().numpy(), np.float32(0))
        assert np.array_equal(raw.reshape(want.shape).cpu().numpy().view(np.uint32), want.view(np.uint32))
    assert abs(kept_fracs[0] - frac) < 0.5 * frac + 0.02, kept_fracs   # the coarse pass: the points the grid was made for
    for k, v in (("raw", raw_f), ("rgb_map", c1["rgb_map"]), ("disp_map", c1["disp_map"]), ("acc_map", c1["acc_map"]),
                 ("rgb0", c0["rgb_map"])):
        assert torch.equal(got[k].view(torch.int32), v.view(torch.int32)), k


def test_graph_replay_and_reruns():
    from nonrigid_nerf_b200 import ops
    coarse, fine, b = _models(True)
    r = {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in O.make_rays(904, 512).items()}   # no copies in capture
    full = _render(coarse, fine, r, 64, detailed=True, surface=False)
    grid, _ = _random_grid(full["input_pts"].reshape(-1, 3).cpu().numpy(), 0.3, 9)
    eager = _render(coarse, fine, r, 64, grid, detailed=False, surface=False)
    again = _render(coarse, fine, r, 64, grid, detailed=False, surface=False)
    _assert_same(eager, again)
    ops.pack_nerf(coarse), ops.pack_nerf(fine), ops.pack_bender(b)   # cached weight images, so capture launches no repack
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _render(coarse, fine, r, 64, grid, detailed=False, surface=False)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = _render(coarse, fine, r, 64, grid, detailed=False, surface=False)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        _assert_same(eager, captured)
