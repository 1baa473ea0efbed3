"""Baked deformation grids on the GPU: the bake bit for bit against the point-mode bender and the fp16 store rule, the
lookup and the knob algebra bit for bit against tests/baked_deformation_reference.py on the kernel's own sample points, the
per-ray fallback bit for bit against the baked render without a deformation grid, the error falling with resolution, a grid
past 2^32 bytes, reruns, CUDA-graph replay, the ray-sharded wrapper, and refusals that launch nothing."""
import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import baked_reference as R
from tests import baked_deformation_reference as D
from tests.test_baked_gpu import _assert_same, _bits_equal, _depths, _far_grid, _half_box_grid, _models, _point_raw, _rays, _render

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DETAILS = ("initial_input_pts", "input_pts", "unmasked_offsets", "masked_offsets", "rigidity_mask")


def _G():
    from nonrigid_nerf_b200 import geometry
    return geometry


def _np(t):
    return t.detach().cpu().numpy()


def _lats(n_frames, seed=0):
    return torch.from_numpy((np.random.RandomState(seed).randn(n_frames, 32) * 0.1).astype(np.float32)).to(DEV)


def _box(points, pad=0.01):
    p = points.reshape(-1, 3)
    return (p.min(0) - np.float32(pad)).astype(np.float32), (p.max(0) + np.float32(pad)).astype(np.float32)


def _cut_box(x, mode="exit"):
    """The padded box of samples x [N, S, 3], cut in x so that rays cross it.  The rays share an origin and fan out in x;
    `out` are the rays that move towards +x.  exit: max x is the lower quartile of their last samples' x, so the rays
    towards -x lie inside and most of `out` start inside and leave the box.  enter: min x is the lower quartile of their x
    at sample S // 2, so the rays towards -x lie outside and most of `out` enter the box partway."""
    lo, hi = _box(x)
    out = x[:, -1, 0] > x[:, 0, 0]
    if mode == "exit":
        hi[0] = np.float32(np.quantile(x[out, -1, 0], 0.25))
    else:
        lo[0] = np.float32(np.quantile(x[out, x.shape[1] // 2, 0], 0.25))
    return lo, hi


def _crossing(x, lo, hi):
    """(rays with samples both inside and outside the box [N] bool, the index of each ray's first sample on the other side
    of the box from its sample 0 [N])"""
    with np.errstate(invalid="ignore"):
        ins = np.all((x >= lo) & (x <= hi), -1)
    return ins.any(1) & ~ins.all(1), np.argmax(ins != ins[:, :1], 1)


# ---- the bake ----------------------------------------------------------------------------------------------------------
def _exact_bend(net, pts, lat):
    """(unmasked offsets [P, 3], rigidity [P]) of the full point-mode kernel with latent `lat`, knobs off."""
    from nonrigid_nerf_b200 import ops
    b = net.ray_bender[0]
    with torch.no_grad():
        _, det = ops.field_forward_points(pts, lat.reshape(1, 32).expand(pts.shape[0], 32), ops.pack_nerf(net), ops.pack_bender(b),
                                          net.output_linear.weight.shape[0], want_details=True)
    return _np(det["unmasked_offsets"]).reshape(-1, 3), _np(det["rigidity_mask"]).reshape(-1)


def _check_bake(net, lats, lo, hi, res):
    grid = _G().bake_deformation(net.ray_bender[0], lats, lo, hi, res)
    nx, ny, nz = res
    F = lats.shape[0] if lats.dim() == 2 else 1
    assert grid.values.shape == (F, nz, ny, nx, 4) and grid.values.dtype == torch.float16 and grid.resolution == tuple(res)
    assert torch.equal(grid.latents, lats.reshape(F, 32))
    got = _np(grid.values)
    pts = torch.from_numpy(np.ascontiguousarray(R.vertex_points(lo, hi, res).reshape(-1, 3))).to(DEV)
    for f in range(F):
        o, r = _exact_bend(net, pts, lats.reshape(F, 32)[f])
        assert _bits_equal(got[f], D.to_f16(o, r).reshape(nz, ny, nx, 4)), (res, f)
    return grid, got


@pytest.mark.parametrize("res", [(2, 2, 2), (17, 33, 9)])
@pytest.mark.parametrize("n_frames", [1, 3])
def test_bake_is_point_mode_bender_in_fp16(res, n_frames):
    coarse, _, b = _models(True)
    lo, hi = np.float32([-0.9, -0.7, -1.1]), np.float32([0.8, 0.6, 0.05])
    lats = _lats(n_frames, sum(res))
    _check_bake(coarse, lats if n_frames > 1 else lats[0], lo, hi, res)


def test_bake_ignores_test_time_knobs():
    coarse, _, b = _models(True)
    lo, hi = np.float32([-0.9, -0.7, -1.1]), np.float32([0.8, 0.6, 0.05])
    lats = _lats(2, 5)
    plain = _G().bake_deformation(b, lats, lo, hi, (11, 7, 5))
    b.rigidity_test_time_cutoff, b.test_time_scaling = 0.6, 1.9
    coarse.test_time_nonrigid_object_removal_threshold = 0.3
    knobs = _G().bake_deformation(b, lats, lo, hi, (11, 7, 5))
    assert torch.equal(plain.values.view(torch.int16), knobs.values.view(torch.int16))


def test_bake_saturation_and_nan():
    coarse, _, b = _models(True)
    with torch.no_grad():   # the offset head (fp16 weights, fp32 sums, no bias): offsets beyond fp16's range, and NaN
        b.network[-1].weight[0] = 1e4
        b.network[-1].weight[1] = float("nan")
        b.network[-1].weight[2] = -1e4
    from nonrigid_nerf_b200 import ops
    ops.note_parameters_changed()
    lo, hi = np.float32([-0.9, -0.7, -1.1]), np.float32([0.8, 0.6, 0.05])
    _, got = _check_bake(coarse, _lats(2, 9), lo, hi, (6, 5, 4))
    assert np.isnan(got[..., 1]).all() and np.isfinite(got[..., [0, 2, 3]]).all()   # saturated, not inf
    assert (got[..., 0] == 65504).mean() > 0.25 and (got[..., 2] == -65504).mean() > 0.25


# ---- the lookup --------------------------------------------------------------------------------------------------------
def _pass(net, rays, z, lat, rgrid, deformation):
    from nonrigid_nerf_b200 import autograd as A
    with torch.no_grad():
        return A.field_baked(net, rays, z, lat, True, rgrid, deformation)


def _check(net, rays, z, lat, rgrid, frame):
    """Deformed rays bit for bit against the restatement on the kernel's own x; fallback rays bit for bit against the baked
    pass without a deformation grid.  Returns the deformed-ray mask."""
    raw, det = _pass(net, rays, z, lat, rgrid, frame)
    base_raw, base_det = _pass(net, rays, z, lat, rgrid, None)
    g = frame.grid
    x = D.sample_points(_np(rays), _np(z))
    ok = D.deformed_rays(x, g.min_point, g.max_point)
    n_ch = raw.shape[-1]
    got = {k: _np(det[k]) for k in DETAILS}
    for k in DETAILS:
        assert _bits_equal(got[k][~ok], _np(base_det[k])[~ok]), k
    assert _bits_equal(_np(raw)[~ok], _np(base_raw)[~ok])
    if ok.any():
        b = net.ray_bender[0]
        want = D.bend(x[ok], _np(g.values[frame.index]), g.min_point, g.max_point, b.rigidity_test_time_cutoff, b.test_time_scaling)
        for k in DETAILS:
            assert _bits_equal(got[k][ok].reshape(want[k].shape), want[k]), k
        c = want["input_pts"]
        inside, look = R.lookup(c, _np(rgrid.values), rgrid.min_point, rgrid.max_point)
        if n_ch == 5:
            look = np.concatenate([look, np.zeros((look.shape[0], 1), np.float32)], 1)
        trunk = _np(_point_raw(net, torch.from_numpy(np.ascontiguousarray(c)).to(DEV)))
        w = np.where(inside[:, None], look, trunk)
        thr = getattr(net, "test_time_nonrigid_object_removal_threshold", None)
        if thr is not None:
            w[:, 3] = np.where(want["rigidity_mask"] >= np.float32(thr), w[:, 3] * np.float32(0), w[:, 3])
        assert _bits_equal(_np(raw)[ok].reshape(-1, n_ch), w)
    return ok


def _frames(b, lats, lo, hi, res=(9, 11, 13)):
    """The deformation grid of lats, and for frames 0, a middle one and the last a copy whose other frames are NaN."""
    grid = _G().bake_deformation(b, lats, lo, hi, res)
    F = lats.shape[0]
    out = []
    for i in (0, F // 2, F - 1):
        v = torch.full_like(grid.values, float("nan"))
        v[i] = grid.values[i]
        out.append(_G().DeformationGrid(v, grid.min_point, grid.max_point, grid.resolution, grid.latents).frame(i))
    return grid, out


@pytest.mark.parametrize("n,S", [(300, 64), (37, 100), (5, 192), (1, 64), (777, 1), (1, 1)])
def test_lookup_bit_for_bit(n, S):
    coarse, fine, b = _models(True)
    rays, lat = _rays(930 + S, n)
    z = _depths(rays, S, n)
    box_rays, box_lat = _rays(999, 300)
    rgrid = _half_box_grid(coarse, box_rays, _depths(box_rays, 64, 999), box_lat)
    lo, hi = _box(D.sample_points(_np(rays), _np(z)))
    _, frames = _frames(b, _lats(5, n), lo, hi)
    for frame in frames:
        ok = _check(coarse, rays, z, lat, rgrid, frame)
        assert ok.all()


@pytest.mark.parametrize("knobs", [("cutoff",), ("scaling",), ("removal",), ("cutoff", "scaling", "removal")])
def test_lookup_with_test_time_knobs(knobs):
    coarse, fine, b = _models(True)
    if "cutoff" in knobs:
        b.rigidity_test_time_cutoff = 0.5
    if "scaling" in knobs:
        b.test_time_scaling = 1.7
    if "removal" in knobs:
        coarse.test_time_nonrigid_object_removal_threshold = 0.5
    rays, lat = _rays(940, 257)
    z = _depths(rays, 64, 940)
    rgrid = _half_box_grid(coarse, rays, z, lat)
    x = D.sample_points(_np(rays), _np(z))
    lo, hi = _cut_box(x)
    _, frames = _frames(b, _lats(3, 1), lo, hi)
    ok = _check(coarse, rays, z, lat, rgrid, frames[1])
    assert 0.4 < ok.mean() < 0.85 and _crossing(x, lo, hi)[0].mean() > 0.2
    rt = _np(_pass(coarse, rays, z, lat, rgrid, frames[1])[1]["rigidity_mask"])[ok]
    if "cutoff" in knobs:
        assert (rt == 0).any() and (rt > 0.5).any()


@pytest.mark.parametrize("S", [64, 100, 192])
@pytest.mark.parametrize("mode", ["exit", "enter"])
def test_rays_crossing_the_box_fall_back_whole(mode, S):
    """Rays that leave the box partway (exit) or enter it partway (enter) fall back as a whole: raw and details bit for bit
    the baked pass's without a deformation grid.  In the kernel's warp per ray, lane l takes samples l, l + 32, ...: for
    some rays the sample where the ray crosses is a lane's second or later one, and on entering rays every lane's last
    sample can be inside while an earlier one is not."""
    coarse, fine, b = _models(True)
    rays, lat = _rays(950 + S, 300)
    z = _depths(rays, S, 950 + S)
    x = D.sample_points(_np(rays), _np(z))
    lo, hi = _cut_box(x, mode)
    cross, change = _crossing(x, lo, hi)
    assert cross.mean() > 0.2 and (change[cross] >= 32).any(), (cross.mean(), np.unique(change[cross]))
    if mode == "enter":
        assert (change[cross] <= S - 32).any()
    rgrid = _half_box_grid(coarse, rays, z, lat)
    frame = _G().bake_deformation(b, _lats(2, S), lo, hi, (19, 23, 17)).frame(1)
    ok = _check(coarse, rays, z, lat, rgrid, frame)
    assert not ok[cross].any()
    if mode == "exit":
        assert 0.4 < ok.mean() < 0.85


def test_lookup_box_faces_ulps_and_non_finite_points():
    """Rays with d = 0 and one sample, so each sample is its ray's origin: the deformation box's faces and vertex planes,
    one ulp either side of each, and NaN / inf coordinates."""
    coarse, _, b = _models(True)
    lo, hi = np.float32([-0.9, -0.7, -1.1]), np.float32([0.8, 0.6, 0.05])
    res = (9, 7, 11)
    grid = _G().bake_deformation(b, _lats(2, 3), lo, hi, res)
    rs = np.random.RandomState(3)
    pts = []
    for ax in range(3):
        vals = np.unique(R.vertex_points(lo, hi, res)[..., ax])
        vals = np.concatenate([vals, np.nextafter(vals, np.float32(-np.inf)), np.nextafter(vals, np.float32(np.inf))])
        p = rs.uniform(lo, hi, size=(vals.size, 3)).astype(np.float32)
        p[:, ax] = vals
        pts.append(p)
    pts.append(np.array([[np.nan, 0, -0.5], [0, np.nan, -0.5], [0, 0, np.nan], [np.inf, 0, -0.5], [-np.inf, 0, -0.5],
                         [0, np.inf, -0.5], [0, 0, -np.inf], lo, hi, [lo[0], hi[1], lo[2]]], np.float32))
    pts = np.concatenate(pts)
    o = torch.from_numpy(pts).to(DEV)
    rays = torch.cat([o, torch.zeros_like(o), torch.zeros(o.shape[0], 1, device=DEV), torch.ones(o.shape[0], 1, device=DEV)], 1).contiguous()
    z = torch.full((o.shape[0], 1), 0.5, device=DEV)
    lat = grid.latents[1].reshape(1, 32).expand(o.shape[0], 32)
    rgrid = _G().bake_radiance(coarse, lo * np.float32(0.5), hi * np.float32(0.5), (5, 6, 7))
    ok = _check(coarse, rays, z, lat, rgrid, grid.frame(1))
    want_ok, _ = R.lookup(pts, _np(grid.values[1]), lo, hi)
    assert np.array_equal(ok, want_ok) and 0.3 < ok.mean() < 0.9
    assert not ok[-10:-3].any() and ok[-3:].all()


def test_scale_far_corner():
    """5 frames of 512^3 vertices (5.37 GB, past 2^31 and 2^32 bytes): lookups near frame 4's far corner bit for bit."""
    coarse, _, b = _models(True)
    res, F = (512, 512, 512), 5
    g = torch.Generator(device=DEV).manual_seed(8)
    values = torch.rand(F, res[2], res[1], res[0], 4, device=DEV, generator=g, dtype=torch.float16)
    values[..., :3] -= 0.5
    assert values.numel() * 2 > 2 ** 32
    lo, hi = np.float32([-1.0, -0.5, -2.0]), np.float32([1.0, 0.75, 0.5])
    grid = _G().DeformationGrid(values, lo, hi, res, torch.zeros(F, 32, device=DEV))
    rs = np.random.RandomState(6)
    step = (hi - lo) / (np.asarray(res, np.float32) - 1)
    pts = (hi - rs.uniform(0, 3, size=(4000, 3)).astype(np.float32) * step).astype(np.float32)
    pts[:3] = hi
    o = torch.from_numpy(pts).to(DEV)
    rays = torch.cat([o, torch.zeros_like(o), torch.zeros(o.shape[0], 1, device=DEV), torch.ones(o.shape[0], 1, device=DEV)], 1).contiguous()
    z = torch.full((o.shape[0], 1), 0.5, device=DEV)
    b.test_time_scaling = 1.3
    raw, det = _pass(coarse, rays, z, torch.zeros(o.shape[0], 32, device=DEV), _far_grid(coarse), grid.frame(4))
    inside, c, f = R.cells(pts, res, lo, hi)
    assert inside.all()
    idx = torch.from_numpy(R.corner_index(c, res)).to(DEV)
    slab = values[4].view(-1, 4)
    assert (int(idx.max()) + 4 * res[0] * res[1] * res[2]) * 8 > 2 ** 32
    corners = _np(slab[idx.reshape(-1)].reshape(-1, 8, 4))
    want = D.knobs(pts, R.interpolate(corners, f), None, 1.3)
    for k in DETAILS:
        assert _bits_equal(_np(det[k]).reshape(want[k].shape), want[k]), k
    del values, grid


# ---- the per-ray fallback, and rendering -------------------------------------------------------------------------------
def _far_deformation(b):
    return _G().bake_deformation(b, _lats(2, 4), [50.0] * 3, [51.0] * 3, 2).frame(1)


@pytest.mark.parametrize("knob", [None, "cutoff", "scaling", "removal"])
@pytest.mark.parametrize("n_imp", [0, 64])
def test_box_without_samples_renders_as_baked(knob, n_imp):
    coarse, fine, b = _models(True)
    if knob == "cutoff":
        b.rigidity_test_time_cutoff = 0.5
    elif knob == "scaling":
        b.test_time_scaling = 1.7
    elif knob == "removal":
        coarse.test_time_nonrigid_object_removal_threshold = fine.test_time_nonrigid_object_removal_threshold = 0.5
    r = O.make_rays(905, 300)
    rays = helpers.rays8(r, DEV)
    z = _depths(rays, 64, 905)
    rc, rf = _half_box_grid(coarse, rays, z, r["latents"].to(DEV)), _half_box_grid(fine, rays, z, r["latents"].to(DEV))
    base = _G().BakedScene(rc, rf)
    scene = _G().BakedScene(rc, rf, _far_deformation(b))
    _assert_same(_render(coarse, fine, r, n_imp, base, chunk=100), _render(coarse, fine, r, n_imp, scene, chunk=100))


def test_half_box_per_ray_and_chunk_independent():
    """A deformation box that about half the rays leave partway: per pass, those rays equal the baked pass without it and
    the others the restatement; chunk = 100 and 2^20 render the same frame."""
    coarse, fine, b = _models(True)
    r = O.make_rays(906, 400)
    rays, lat = helpers.rays8(r, DEV), r["latents"].to(DEV)
    from nonrigid_nerf_b200 import ops
    z = ops.sample_coarse(rays, 64, None, False)
    x = D.sample_points(_np(rays), _np(z))
    lo, hi = _cut_box(x)
    assert _crossing(x, lo, hi)[0].mean() > 0.2
    frame = _G().bake_deformation(b, _lats(3, 6), lo, hi, (21, 17, 19)).frame(2)
    scene = _G().BakedScene(_half_box_grid(coarse, rays, z, lat), _half_box_grid(fine, rays, z, lat), frame)
    ok = _check(coarse, rays, z, lat, scene.coarse, frame)
    assert 0.4 < ok.mean() < 0.85, ok.mean()
    _assert_same(_render(coarse, fine, r, 64, scene, chunk=100, surface=False), _render(coarse, fine, r, 64, scene, chunk=1 << 20, surface=False))


def _bender(offset_std, seed=7):
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    embed_fn, input_ch = H.get_embedder(10, 0)
    return helpers.load_bender_module(H.ray_bending(input_ch, 32, "simple_neural", embed_fn),
                                      O.make_bender_params(seed, offset_std=offset_std)).to(DEV)


@pytest.mark.parametrize("offset_std", [0.01, 0.1])
def test_accuracy_with_resolution(offset_std, capsys):
    """max |c - exact bent point| of the coarse pass and the mean rgb difference from the radiance-only baked frame fall from
    64^3 to 128^3 to 256^3 (64 x 64 frame, init trunk weights)."""
    coarse, fine, _ = _models(True)
    b = _bender(offset_std)
    coarse.ray_bender = fine.ray_bender = (b,)
    Hh = Ww = 64
    j, i = np.meshgrid(np.arange(Hh, dtype=np.float32), np.arange(Ww, dtype=np.float32), indexing="ij")
    dirs = np.stack([(i - Ww * 0.5) / 64.0, -(j - Hh * 0.5) / 64.0, -np.ones_like(i)], -1).reshape(-1, 3).astype(np.float32)
    n = dirs.shape[0]
    latent = _lats(1, 17)
    r = {"rays_o": torch.zeros(n, 3), "rays_d": torch.from_numpy(dirs), "near": 0.0022, "far": 1.0024,
         "latents": latent.cpu().expand(n, 32).contiguous()}
    exact = _render(coarse, fine, r, 64, surface=False)
    bent = torch.cat([exact["input_pts"].reshape(-1, 3), exact["fine_input_pts"].reshape(-1, 3)]).cpu().numpy()
    obs = torch.cat([exact["initial_input_pts"].reshape(-1, 3), exact["fine_initial_input_pts"].reshape(-1, 3)]).cpu().numpy()
    rlo, rhi = _box(bent)
    base = _G().BakedScene(_G().bake_radiance(coarse, rlo, rhi, 128), _G().bake_radiance(fine, rlo, rhi, 128))
    radiance_only = _render(coarse, fine, r, 64, base, surface=False)
    rays = helpers.rays8(r, DEV)
    lat = r["latents"].to(DEV)
    from nonrigid_nerf_b200 import ops
    z = ops.sample_coarse(rays, 64, None, False)
    exact_c = _np(_pass(coarse, rays, z, lat, base.coarse, None)[1]["input_pts"])
    dlo, dhi = _box(obs)
    errs = {}
    for res in (64, 128, 256):
        frame = _G().bake_deformation(b, latent, dlo, dhi, res).frame(0)
        scene = _G().BakedScene(base.coarse, base.fine, frame)
        c = _np(_pass(coarse, rays, z, lat, base.coarse, frame)[1]["input_pts"])
        got = _render(coarse, fine, r, 64, scene, detailed=False, surface=False)
        errs[res] = (float(np.abs(c - exact_c).max()), float((got["rgb_map"] - radiance_only["rgb_map"]).abs().mean()))
    with capsys.disabled():
        print(f"\ndeformation grid, offset std {offset_std} (max |c - exact|, mean |rgb - radiance-only rgb|): " +
              ", ".join(f"{k}^3: {v[0]:.3e}, {v[1]:.3e}" for k, v in errs.items()))
    assert errs[64][0] > errs[128][0] > errs[256][0], errs
    assert errs[64][1] > errs[128][1] > errs[256][1], errs


def test_reruns_graph_replay_and_sharded_wrapper():
    from nonrigid_nerf_b200 import ops, parallel as Pl
    coarse, fine, b = _models(True)
    r_host = O.make_rays(907, 512)
    r = {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in r_host.items()}   # no copies in capture
    rays = helpers.rays8(r_host, DEV)
    z = ops.sample_coarse(rays, 64, None, False)
    x = D.sample_points(_np(rays), _np(z))
    lo, hi = _cut_box(x)   # a third of the rays leave the box partway and fall back
    frame = _G().bake_deformation(b, _lats(2, 8), lo, hi, 24).frame(1)
    scene = _G().BakedScene(_half_box_grid(coarse, rays, z, r["latents"]), _half_box_grid(fine, rays, z, r["latents"]), frame)
    eager = _render(coarse, fine, r, 64, scene, detailed=False, surface=False)
    _assert_same(eager, _render(coarse, fine, r, 64, scene, detailed=False, surface=False))
    fn = Pl.get_parallelized_render_function(coarse, fine, b)
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=64, N_samples=64, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0,
              ndc=False, lindisp=False, baked=scene)
    with torch.no_grad():
        sh = fn(r["rays_o"], r["rays_d"], chunk=32768, near=r["near"], far=r["far"],
                additional_pixel_information={"ray_bending_latents": r["latents"]}, retraw=True, **kw)
    assert torch.equal(sh[0].view(torch.int32), eager["rgb_map"].view(torch.int32))
    assert torch.equal(sh[3]["raw"].view(torch.int32), eager["raw"].view(torch.int32))
    ops.pack_nerf(coarse), ops.pack_nerf(fine), ops.pack_bender(b)
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


def test_refusals_launch_nothing():
    from nonrigid_nerf_b200 import _lib, geometry as G
    coarse, fine, b = _models(True)
    plain, _, _ = _models(False)
    r = O.make_rays(908, 64)
    rgrid = _far_grid(coarse)
    dgrid = G.bake_deformation(b, _lats(2, 1), [-1] * 3, [1] * 3, 4)
    bad_values = G.DeformationGrid(dgrid.values.float(), dgrid.min_point, dgrid.max_point, dgrid.resolution, dgrid.latents)
    elsewhere = G.DeformationGrid(dgrid.values.cpu(), dgrid.min_point, dgrid.max_point, dgrid.resolution, dgrid.latents)
    cases = [(plain, G.BakedScene(_far_grid(plain), None, dgrid.frame(0)), "ray bender"),
             (coarse, G.BakedScene(rgrid, None, dgrid), "FrameDeformation"),
             (coarse, G.BakedScene(rgrid, None, bad_values.frame(0)), "float16"),
             (coarse, G.BakedScene(rgrid, None, elsewhere.frame(0)), "is on cpu")]
    kinds = tuple(_lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + _lib.DET_KERNEL_KINDS
                  + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + _lib.MESH_KERNEL_KINDS
                  + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS + _lib.OCCUPANCY_KERNEL_KINDS + _lib.TERMINATION_KERNEL_KINDS
                  + _lib.DEFORM_KERNEL_KINDS + _lib.NORMAL_KERNEL_KINDS + _lib.LPIPS_MAP_KERNEL_KINDS + _lib.BAKED_KERNEL_KINDS
                  + _lib.DEFORMATION_KERNEL_KINDS)
    assert len(kinds) == 58
    torch.cuda.synchronize()
    _lib.timing_enable(True)
    try:
        for net, scene, msg in cases:
            with pytest.raises(RuntimeError, match=msg):
                _render(net, None, r, 0, scene, surface=False)
        with pytest.raises(RuntimeError, match="out of range"):
            dgrid.frame(2)
        with pytest.raises(RuntimeError, match="inference only"):
            from nonrigid_nerf_b200 import train as T
            T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), near=r["near"], far=r["far"], ndc=False, N_samples=64, network_fn=coarse,
                     network_query_fn=None, baked=G.BakedScene(rgrid, None, dgrid.frame(0)),
                     additional_pixel_information={"ray_bending_latents": r["latents"].to(DEV)})
    finally:
        _lib.timing_enable(False)
    counts = {k: c for k, (_, c) in _lib.timing_read(kinds).items()}
    assert all(c == 0 for c in counts.values()), {k: c for k, c in counts.items() if c}
