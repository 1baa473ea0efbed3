"""Baked radiance grids on the GPU: the bake bit for bit against the point-mode field and tests/baked_reference.py's fp16
store, the lookup bit for bit against the restatement on the kernel's own bent points and grid, render(..., baked=)
against render() where the grid's box holds no sample, and for any box raw = where(inside, lookup, fused raw) per pass."""
import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import baked_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _G():
    from nonrigid_nerf_b200 import geometry
    return geometry


def _models(bender):
    coarse, fine, b, _ = helpers.build_models(O, 900, DEV, with_bender=bender)
    return coarse, fine, b


def _bits_equal(a: np.ndarray, b: np.ndarray) -> bool:
    """Equal bit for bit, except that any NaN matches any NaN (payloads are not specified)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    u = np.uint16 if a.dtype == np.float16 else np.uint32
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(nan | (a.view(u) == b.view(u))))


def _point_raw(net, pts: torch.Tensor) -> torch.Tensor:
    """raw [P, out_ch] of the canonical model (bender off) in point mode."""
    from nonrigid_nerf_b200 import ops
    with torch.no_grad():
        raw, _ = ops.field_forward_points(pts, None, ops.pack_nerf(net), None, net.output_linear.weight.shape[0])
    return raw.reshape(pts.shape[0], -1)


# ---- the bake ----------------------------------------------------------------------------------------------------------
def _check_bake(net, lo, hi, res):
    grid = _G().bake_radiance(net, lo, hi, res)
    nx, ny, nz = res
    assert grid.values.shape == (nz, ny, nx, 4) and grid.values.dtype == torch.float16 and grid.resolution == tuple(res)
    got = grid.values.cpu().numpy()
    for k0 in range(0, nz, 32):   # 32 planes at a time
        k1 = min(k0 + 32, nz)
        pts = torch.from_numpy(np.ascontiguousarray(R.vertex_points(lo, hi, res)[k0:k1].reshape(-1, 3))).to(DEV)
        want = R.to_f16(_point_raw(net, pts).cpu().numpy()).reshape(k1 - k0, ny, nx, 4)
        assert _bits_equal(got[k0:k1], want), (res, k0)
    return grid, got


@pytest.mark.parametrize("res", [(2, 2, 2), (17, 33, 9), (257, 257, 257)])
@pytest.mark.parametrize("bender", [True, False])
def test_bake_is_point_mode_field_in_fp16(res, bender):
    coarse, fine, _ = _models(bender)
    lo, hi = np.float32([-0.9, -0.7, -1.1]), np.float32([0.8, 0.6, 0.05])
    _check_bake(coarse, lo, hi, res)
    if res == (17, 33, 9):
        _check_bake(fine, lo, hi, res)


def test_plane_store_saturation_and_nan():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(4)
    specials = np.float32([65504, 65519, 65520, 1e5, -1e30, np.inf, -np.inf, np.nan, -0.0, 6e-8, 3e-8, 1e-8, 1 + 2 ** -11, 65535])
    for out_ch in (4, 5):
        raw = (rs.randn(1000, out_ch) * 3e4).astype(np.float32)
        raw.reshape(-1)[rs.choice(raw.size, 200, replace=False)] = rs.choice(specials, 200)
        plane = torch.full((1000, 4), 7, dtype=torch.float16, device=DEV)
        t = torch.from_numpy(raw).to(DEV)
        _lib.check(lib.nrn_radiance_plane_f16(t.data_ptr(), 1000, out_ch, plane.data_ptr(), torch.cuda.current_stream().cuda_stream), "plane")
        got = plane.cpu().numpy()
        want = R.to_f16(raw)
        assert _bits_equal(got, want)
        fin = np.isfinite(raw[:, :4])
        assert np.all(np.isfinite(got[fin])) and np.all(~np.isfinite(got[~fin]))   # saturated, not inf; inf and NaN kept
        assert np.all(np.abs(got[fin & (np.abs(raw[:, :4]) >= 65520)]) == 65504)


def test_bake_saturation_and_nan_of_a_model():
    coarse, _, _ = _models(False)
    with torch.no_grad():   # the head's biases are added in fp32: raw beyond fp16's range, and NaN
        coarse.output_linear.bias[0] = 1e5
        coarse.output_linear.bias[1] = float("nan")
        coarse.output_linear.bias[2] = -1e6
    lo, hi = np.float32([-0.9, -0.7, -1.1]), np.float32([0.8, 0.6, 0.05])
    _, got = _check_bake(coarse, lo, hi, (20, 18, 16))
    assert (got[..., 0] == 65504).all() and np.isnan(got[..., 1]).all() and (got[..., 2] == -65504).all()
    assert np.isfinite(got[..., 3]).all()


# ---- the lookup --------------------------------------------------------------------------------------------------------
def _pass(net, rays, z, lat, grid):
    """(raw of the baked pass, its details, the fused pass's raw) under no_grad."""
    from nonrigid_nerf_b200 import autograd as A
    with torch.no_grad():
        raw, det = A.field_baked(net, rays, z, lat if net.ray_bender[0] is not None else None, True, grid)
        full, _ = A.field_rays(net, rays, z, lat if net.ray_bender[0] is not None else None, False)
    return raw, det, full


def _want(net, det, full, grid):
    """where(inside, lookup of the kernel's own points in its own grid (object removal applied, raw[4] = 0), fused raw)."""
    pts = det["input_pts"].reshape(-1, 3).cpu().numpy()
    inside, look = R.lookup(pts, grid.values.cpu().numpy(), grid.min_point, grid.max_point)
    thr = getattr(net, "test_time_nonrigid_object_removal_threshold", None)
    if thr is not None and "rigidity_mask" in det:
        removed = det["rigidity_mask"].reshape(-1).cpu().numpy() >= np.float32(thr)
        look[:, 3] = np.where(removed, look[:, 3] * np.float32(0), look[:, 3])
    f = full.reshape(-1, full.shape[-1]).cpu().numpy()
    if f.shape[1] == 5:
        look = np.concatenate([look, np.zeros((look.shape[0], 1), np.float32)], 1)
    return inside, np.where(inside[:, None], look, f)


def _check_pass(net, rays, z, lat, grid):
    raw, det, full = _pass(net, rays, z, lat, grid)
    inside, want = _want(net, det, full, grid)
    assert _bits_equal(raw.reshape(want.shape).cpu().numpy(), want)
    return inside


def _rays(seed, n, dev=DEV):
    r = O.make_rays(seed, n)
    return helpers.rays8(r, dev), r["latents"].to(dev)


def _depths(rays, S, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    near, far = rays[:, 6:7], rays[:, 7:8]
    return (near + (far - near) * torch.rand(rays.shape[0], S, generator=g, device=DEV)).sort(1)[0].contiguous()


def _half_box_grid(net, rays, z, lat, res=(33, 29, 31)):
    """A grid baked over the box of the pass's (bent) points, cut at the median x: about half the samples inside."""
    _, det, _ = _pass(net, rays, z, lat, _far_grid(net))
    p = det["input_pts"].reshape(-1, 3).cpu().numpy()
    lo, hi = p.min(0).astype(np.float32), p.max(0).astype(np.float32)
    hi[0] = np.float32(np.median(p[:, 0]))
    return _G().bake_radiance(net, lo, hi, res)


def _far_grid(net):
    """A grid whose box holds no sample of these tests."""
    return _G().bake_radiance(net, [50.0] * 3, [51.0] * 3, 2)


@pytest.mark.parametrize("bender", [True, False])
@pytest.mark.parametrize("n,S", [(300, 64), (37, 100), (5, 192), (1, 64), (777, 1), (1, 1)])
def test_lookup_bit_for_bit(bender, n, S):
    coarse, fine, _ = _models(bender)
    rays, lat = _rays(910 + S, n)
    z = _depths(rays, S, n)
    box_rays, box_lat = _rays(999, 300)   # the grids' boxes come from other rays of the same frustum: about half inside
    box_z = _depths(box_rays, 64, 999)
    for net in (coarse, fine):
        _check_pass(net, rays, z, lat, _half_box_grid(net, box_rays, box_z, box_lat))


@pytest.mark.parametrize("knob", ["cutoff", "scaling", "removal"])
def test_lookup_with_test_time_knobs(knob):
    coarse, fine, b = _models(True)
    if knob == "cutoff":
        b.rigidity_test_time_cutoff = 0.5
    elif knob == "scaling":
        b.test_time_scaling = 1.7
    else:
        coarse.test_time_nonrigid_object_removal_threshold = 0.5
    rays, lat = _rays(920, 257)
    z = _depths(rays, 64, 920)
    grid = _half_box_grid(coarse, rays, z, lat)
    inside = _check_pass(coarse, rays, z, lat, grid)
    assert 0.2 < inside.mean() < 0.8


def test_lookup_box_faces_ulps_and_non_finite_points():
    """Canonical model, rays with d = 0, so every sample sits exactly at its ray's origin: the box faces, vertex planes and
    one ulp either side of each, and NaN / inf coordinates."""
    coarse, _, _ = _models(False)
    lo, hi = np.float32([-0.9, -0.7, -1.1]), np.float32([0.8, 0.6, 0.05])
    res = (9, 7, 11)
    grid = _G().bake_radiance(coarse, lo, hi, res)
    rs = np.random.RandomState(3)
    pts = []
    for ax in range(3):
        planes = R.vertex_points(lo, hi, res)[..., ax]
        vals = np.unique(planes)
        vals = np.concatenate([vals, np.nextafter(vals, np.float32(-np.inf)), np.nextafter(vals, np.float32(np.inf))])
        p = rs.uniform(lo, hi, size=(vals.size, 3)).astype(np.float32)
        p[:, ax] = vals
        pts.append(p)
    pts.append(np.array([[np.nan, 0, -0.5], [0, np.nan, -0.5], [0, 0, np.nan], [np.inf, 0, -0.5], [-np.inf, 0, -0.5],
                         [0, np.inf, -0.5], [0, 0, -np.inf], lo, hi, [lo[0], hi[1], lo[2]]], np.float32))
    pts = np.concatenate(pts)
    o = torch.from_numpy(pts).to(DEV)
    rays = torch.cat([o, torch.zeros_like(o), torch.zeros(o.shape[0], 1, device=DEV), torch.ones(o.shape[0], 1, device=DEV)], 1)
    z = torch.full((o.shape[0], 1), 0.5, device=DEV)
    inside = _check_pass(coarse, rays.contiguous(), z, None, grid)
    want_inside, _ = R.lookup(pts, grid.values.cpu().numpy(), lo, hi)
    assert np.array_equal(inside, want_inside) and 0.3 < inside.mean() < 0.9
    assert not inside[-10:-3].any() and inside[-3:].all()


def test_large_grid_far_corner():
    """A grid past 2^31 bytes (1024 x 1024 x 300 vertices, 2.5 GB): lookups near its far corner bit for bit."""
    from nonrigid_nerf_b200 import autograd as A
    coarse, _, _ = _models(False)
    res = (1024, 1024, 300)
    g = torch.Generator(device=DEV).manual_seed(5)
    values = torch.randn(res[2], res[1], res[0], 4, device=DEV, generator=g).half()
    assert values.numel() * 2 > 2 ** 31
    lo, hi = np.float32([-1.0, -0.5, -2.0]), np.float32([1.0, 0.75, 0.5])
    grid = _G().RadianceGrid(values, lo, hi, res)
    rs = np.random.RandomState(6)
    step = (hi - lo) / (np.asarray(res, np.float32) - 1)
    pts = (hi - rs.uniform(0, 3, size=(5000, 3)).astype(np.float32) * step).astype(np.float32)
    pts[:3] = hi
    o = torch.from_numpy(pts).to(DEV)
    rays = torch.cat([o, torch.zeros_like(o), torch.zeros(o.shape[0], 1, device=DEV), torch.ones(o.shape[0], 1, device=DEV)], 1)
    z = torch.full((o.shape[0], 1), 0.5, device=DEV)
    with torch.no_grad():
        raw, _ = A.field_baked(coarse, rays.contiguous(), z, None, False, grid)
    inside, c, f = R.cells(pts, res, lo, hi)
    assert inside.all()
    idx = torch.from_numpy(R.corner_index(c, res)).to(DEV)
    assert int(idx.max()) * 8 > 2 ** 31
    corners = values.view(-1, 4)[idx.reshape(-1)].reshape(-1, 8, 4).cpu().numpy()
    want = R.interpolate(corners, f)
    assert _bits_equal(raw.reshape(-1, 5)[:, :4].cpu().numpy(), want)
    assert torch.count_nonzero(raw.reshape(-1, 5)[:, 4]) == 0


# ---- rendering ---------------------------------------------------------------------------------------------------------
def _render(coarse, fine, r, n_imp, baked=None, chunk=32768, detailed=True, surface=True):
    from nonrigid_nerf_b200 import train as T
    n = r["rays_o"].shape[0]
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=n_imp, network_fine=fine if n_imp else None, N_samples=64,
              network_fn=coarse, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    if baked is not None:
        kw["baked"] = baked
    with torch.no_grad():
        rgb, disp, acc, ex = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=chunk, near=r["near"], far=r["far"],
                                      additional_pixel_information={"ray_bending_latents": r["latents"][:n].to(DEV)},
                                      detailed_output=detailed, retraw=True, surface_output=surface, **kw)
    out = dict(ex)
    out.update(rgb_map=rgb, disp_map=disp, acc_map=acc)
    return out


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
def test_box_without_samples_renders_as_without_grid(bender, n_imp):
    coarse, fine, _ = _models(bender)
    r = O.make_rays(901, 300)
    scene = _G().BakedScene(_far_grid(coarse), _far_grid(fine))
    for chunk in (32768, 100):
        _assert_same(_render(coarse, fine, r, n_imp, chunk=chunk), _render(coarse, fine, r, n_imp, scene, chunk=chunk))


@pytest.mark.parametrize("bender", [True, False])
def test_half_box_is_lookup_else_fused_raw(bender):
    """Per pass: raw = where(inside, lookup, fused raw on the baked path's own depths) on the kernel's own points; the maps
    are composite() of that raw; chunk = 100 gives the same frame."""
    from nonrigid_nerf_b200 import autograd as A, ops
    coarse, fine, _ = _models(bender)
    if bender:
        coarse.test_time_nonrigid_object_removal_threshold = 0.6
        fine.test_time_nonrigid_object_removal_threshold = 0.6
    r = O.make_rays(903, 400)
    rays = helpers.rays8(r, DEV)
    lat = r["latents"].to(DEV)
    z = ops.sample_coarse(rays, 64, None, False)
    scene = _G().BakedScene(_half_box_grid(coarse, rays, z, lat), _half_box_grid(fine, rays, z, lat))
    got = _render(coarse, fine, r, 64, scene, surface=False)
    _assert_same(got, _render(coarse, fine, r, 64, scene, chunk=100, surface=False))
    rays_d = rays[:, 3:6]
    with torch.no_grad():
        raw_c, det_c, full_c = _pass(coarse, rays, z, lat, scene.coarse)
        c0 = A.composite(raw_c, z, rays_d, None, False, 64, None)
        z_f = c0["z_vals_out"]
        raw_f, det_f, full_f = _pass(fine, rays, z_f, lat, scene.fine)
        c1 = A.composite(raw_f, z_f, rays_d, None, False)
    fracs = []
    for net, raw, full, det, grid, pref in ((coarse, raw_c, full_c, det_c, scene.coarse, ""), (fine, raw_f, full_f, det_f, scene.fine, "fine_")):
        assert torch.equal(det["input_pts"].view(torch.int32), got[pref + "input_pts"].view(torch.int32))
        inside, want = _want(net, det, full, grid)
        fracs.append(inside.mean())
        assert _bits_equal(raw.reshape(want.shape).cpu().numpy(), want)
    assert 0.3 < fracs[0] < 0.7, fracs
    for k, v in (("raw", raw_f), ("rgb_map", c1["rgb_map"]), ("disp_map", c1["disp_map"]), ("acc_map", c1["acc_map"]),
                 ("rgb0", c0["rgb_map"])):
        assert torch.equal(got[k].view(torch.int32), v.view(torch.int32)), k


def test_convergence_with_resolution(capsys):
    """Baked-vs-exact rgb error of a 64 x 64 frame (init weights, with a bender) falls from 64^3 to 128^3 to 256^3."""
    coarse, fine, _ = _models(True)
    Hh = Ww = 64
    focal = 64.0
    j, i = np.meshgrid(np.arange(Hh, dtype=np.float32), np.arange(Ww, dtype=np.float32), indexing="ij")
    dirs = np.stack([(i - Ww * 0.5) / focal, -(j - Hh * 0.5) / focal, -np.ones_like(i)], -1).reshape(-1, 3).astype(np.float32)
    n = dirs.shape[0]
    lat = np.broadcast_to((np.random.RandomState(7).randn(32) * 0.1).astype(np.float32), (n, 32)).copy()
    r = {"rays_o": torch.zeros(n, 3), "rays_d": torch.from_numpy(dirs), "near": 0.0022, "far": 1.0024, "latents": torch.from_numpy(lat)}
    exact = _render(coarse, fine, r, 64, surface=False)
    pts = torch.cat([exact["input_pts"].reshape(-1, 3), exact["fine_input_pts"].reshape(-1, 3)]).cpu().numpy()
    lo, hi = pts.min(0) - np.float32(0.01), pts.max(0) + np.float32(0.01)
    errs = {}
    for res in (64, 128, 256):
        scene = _G().BakedScene(_G().bake_radiance(coarse, lo, hi, res), _G().bake_radiance(fine, lo, hi, res))
        got = _render(coarse, fine, r, 64, scene, detailed=False, surface=False)
        d = (got["rgb_map"] - exact["rgb_map"]).abs()
        errs[res] = (float(d.mean()), float(d.max()))
    with capsys.disabled():
        print("\nbaked vs exact rgb, 64 x 64 frame, init weights (mean |d|, max |d|): " +
              ", ".join(f"{k}^3: {v[0]:.3e}, {v[1]:.3e}" for k, v in errs.items()))
    assert errs[64][0] > errs[128][0] > errs[256][0], errs


def test_reruns_graph_replay_and_sharded_wrapper():
    from nonrigid_nerf_b200 import ops, parallel as Pl
    coarse, fine, b = _models(True)
    r_host = O.make_rays(904, 512)
    r = {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in r_host.items()}   # no copies in capture
    rays = helpers.rays8(r_host, DEV)
    z = ops.sample_coarse(rays, 64, None, False)
    scene = _G().BakedScene(_half_box_grid(coarse, rays, z, r["latents"]), _half_box_grid(fine, rays, z, r["latents"]))
    eager = _render(coarse, fine, r, 64, scene, detailed=False, surface=False)
    again = _render(coarse, fine, r, 64, scene, detailed=False, surface=False)
    _assert_same(eager, again)
    # the ray-sharded render wrapper at world size 1 hands the scene on whole
    fn = Pl.get_parallelized_render_function(coarse, fine, b)
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=64, N_samples=64, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0,
              ndc=False, lindisp=False, baked=scene)
    with torch.no_grad():
        sh = fn(r["rays_o"], r["rays_d"], chunk=32768, near=r["near"], far=r["far"],
                additional_pixel_information={"ray_bending_latents": r["latents"]}, retraw=True, **kw)
    assert torch.equal(sh[0].view(torch.int32), eager["rgb_map"].view(torch.int32))
    assert torch.equal(sh[3]["raw"].view(torch.int32), eager["raw"].view(torch.int32))
    # CUDA graph replay
    ops.pack_nerf(coarse), ops.pack_nerf(fine), ops.pack_bender(b)   # cached weight images, so capture launches no repack
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _render(coarse, fine, r, 64, scene, detailed=False, surface=False)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = _render(coarse, fine, r, 64, scene, detailed=False, surface=False)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        _assert_same(eager, captured)
