"""Early ray termination on the GPU: render(..., early_termination=t) against render() without it.  t = 0 is bit-identical;
for any t, per pass and on the pass's own depths, raw = where(i < termination_index (and grid-kept), fused raw, 0) bit for
bit, the maps are composite() of that raw, and termination_index equals tests/termination_reference.py restated from the
pass's own composite alphas, bit for bit.  Densities are made opaque by adding a constant to output_linear's sigma bias,
so that rays die in the first, a middle or the last segment."""
import math

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import occupancy_reference as OR
from tests import termination_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _K():
    from nonrigid_nerf_b200 import _lib
    return _lib.load().nrn_termination_segment()


def _models(bender, seed=900):
    coarse, fine, b, _ = helpers.build_models(O, seed, DEV, with_bender=bender, density_boost=0.0)
    return coarse, fine, b


def _opaque(nets, r, S, cross):
    """Add to the sigma bias the density that makes T = exp(-sigma * depth * |d|) cross 1e-4 about `cross` of the way
    along [near, far] (a median ray, S samples); cross = None: leave the model as it is."""
    if cross is None:
        return
    d = float(r["rays_d"].norm(dim=-1).median())
    sigma = math.log(1e4) / (cross * (float(r["far"]) - float(r["near"])) * d)
    with torch.no_grad():
        for net in nets:
            if net is not None:
                net.output_linear.bias[3] += sigma


def _render(coarse, fine, r, n_imp, S=64, chunk=32768, detailed=True, surface=False, white=False, noise_std=0.0, rnd=None, **kw):
    from nonrigid_nerf_b200 import train as T
    n = r["rays_o"].shape[0]
    args = dict(network_query_fn=None, perturb=0.0, N_importance=n_imp, network_fine=fine if n_imp else None, N_samples=S,
                network_fn=coarse, use_viewdirs=False, white_bkgd=white, raw_noise_std=noise_std, ndc=False, lindisp=False)
    if rnd is not None:
        args["randomness"] = rnd
    args.update(kw)
    with torch.no_grad():
        rgb, disp, acc, ex = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=chunk, near=r["near"], far=r["far"],
                                      additional_pixel_information={"ray_bending_latents": r["latents"][:n].to(DEV)},
                                      detailed_output=detailed, retraw=True, surface_output=surface, **args)
    out = dict(ex)
    out.update(rgb_map=rgb, disp_map=disp, acc_map=acc)
    return out


def _assert_same(a, b, skip=("termination_index", "termination_index0")):
    ka, kb = set(a) - set(skip), set(b) - set(skip)
    assert ka == kb, ka ^ kb
    for k in ka:
        x, y = a[k].cpu(), b[k].cpu()
        assert x.dtype == y.dtype and x.shape == y.shape, k
        if x.is_floating_point():
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), k   # bit for bit
        else:
            assert torch.equal(x, y), k


def _check_indices(out, n_imp, S, t):
    """termination_index (and termination_index0) of a render equal the restatement from its own composite alphas."""
    K = _K()
    passes = [("opacity_alpha", "termination_index0" if n_imp else "termination_index")]
    if n_imp:
        passes.append(("fine_opacity_alpha", "termination_index"))
    got = []
    for ak, tk in passes:
        idx = out[tk].cpu().numpy()
        assert out[tk].dtype == torch.int32
        want = R.termination_index(out[ak].cpu().numpy(), K, t)
        assert np.array_equal(idx, want), (tk, np.nonzero(idx != want)[0][:10])
        got.append(idx)
    return got


# ---- t = 0 is the render without termination ---------------------------------------------------------------------------
@pytest.mark.parametrize("bender", [True, False])
@pytest.mark.parametrize("n_imp", [0, 64])
def test_t0_is_identical(bender, n_imp):
    coarse, fine, b = _models(bender)
    r = O.make_rays(901, 300)
    _opaque((coarse, fine), r, 64, 0.5)
    for chunk in (32768, 100):
        base = _render(coarse, fine, r, n_imp, chunk=chunk, surface=True)
        got = _render(coarse, fine, r, n_imp, chunk=chunk, surface=True, early_termination=0.0)
        _assert_same(base, got)
        for k in ("termination_index",) + (("termination_index0",) if n_imp else ()):
            assert torch.all(got[k] == (64 + n_imp if k == "termination_index" and n_imp else 64)), k
        assert "termination_index" not in base


@pytest.mark.parametrize("knob", ["cutoff", "scaling", "removal"])
def test_t0_with_test_time_knobs(knob):
    coarse, fine, b = _models(True)
    if knob == "cutoff":
        b.rigidity_test_time_cutoff = 0.5
    elif knob == "scaling":
        b.test_time_scaling = 1.7
    else:
        coarse.test_time_nonrigid_object_removal_threshold = 0.5
        fine.test_time_nonrigid_object_removal_threshold = 0.5
    r = O.make_rays(902, 257)
    _opaque((coarse, fine), r, 64, 0.5)
    _assert_same(_render(coarse, fine, r, 64), _render(coarse, fine, r, 64, early_termination=0))


def _random_grid(pts, frac, seed, res=(24, 20, 28)):
    from nonrigid_nerf_b200 import geometry as G
    lo = (pts.min(0) - np.float32(0.01)).astype(np.float32)
    hi = (pts.max(0) + np.float32(0.01)).astype(np.float32)
    per_cell = np.bincount(OR.cells(pts, res, lo, hi), minlength=res[0] * res[1] * res[2])
    order = np.random.RandomState(seed).permutation(per_cell.size)
    take = order[:np.searchsorted(np.cumsum(per_cell[order]), frac * pts.shape[0]) + 1]
    occ = np.zeros(per_cell.size, bool)
    occ[take] = True
    occ = occ.reshape(res[2], res[1], res[0])
    return G.OccupancyGrid(torch.from_numpy(OR.pack(occ)).to(DEV), lo, hi, res), occ


def test_t0_with_grid_is_the_grid_render():
    coarse, fine, b = _models(True)
    r = O.make_rays(905, 300)
    _opaque((coarse, fine), r, 64, 0.5)
    full = _render(coarse, fine, r, 64)
    grid, _ = _random_grid(full["input_pts"].reshape(-1, 3).cpu().numpy(), 0.2, 3)
    _assert_same(_render(coarse, fine, r, 64, occupancy=grid), _render(coarse, fine, r, 64, occupancy=grid, early_termination=0.0))


# ---- per pass: masked raw, composited maps, exact termination_index -----------------------------------------------------
def _check_pass(net, rays, z, lat, t, noise=None, grid=None, occ=None, removal_ws=None):
    """One pass through field_terminate against the fused field on the same depths; returns (raw, composite, index)."""
    from nonrigid_nerf_b200 import autograd as A
    raw, det, idx = A.field_terminate(net, rays, z, lat, True, t, grid, noise)
    full, det_full = A.field_rays(net, rays, z, lat, True)
    n, S = z.shape
    alive = np.arange(S)[None, :] < idx.cpu().numpy()[:, None]
    keep = alive.reshape(-1)
    if grid is not None:
        kept = OR.keep(det["input_pts"].reshape(-1, 3).cpu().numpy(), occ, grid.min_point, grid.max_point)
        keep = keep & kept
    want = np.where(keep[:, None], full.reshape(-1, full.shape[-1]).cpu().numpy(), np.float32(0))
    assert np.array_equal(raw.reshape(want.shape).cpu().numpy().view(np.uint32), want.view(np.uint32))
    for k in det_full:   # the details cover every sample
        assert torch.equal(det[k].view(torch.int32), det_full[k].view(torch.int32)), k
    c = A.composite(raw, z, rays[:, 3:6], noise, False)
    assert np.array_equal(idx.cpu().numpy(), R.termination_index(c["alpha"].cpu().numpy(), _K(), t))
    return raw, idx


@pytest.mark.parametrize("bender", [True, False])
@pytest.mark.parametrize("cross", [0.02, 0.5, 0.97, None])
def test_per_pass_masked_raw_and_exact_index(bender, cross):
    from nonrigid_nerf_b200 import autograd as A, ops
    coarse, fine, b = _models(bender)
    if bender:
        coarse.test_time_nonrigid_object_removal_threshold = 0.6
        fine.test_time_nonrigid_object_removal_threshold = 0.6
    r = O.make_rays(903, 400)
    _opaque((coarse, fine), r, 64, cross)
    t = 1e-4
    got = _render(coarse, fine, r, 64, early_termination=t)
    rays = helpers.rays8(r, DEV)
    lat = r["latents"].to(DEV)
    with torch.no_grad():
        z = ops.sample_coarse(rays, 64, None, False)
        raw_c, idx_c = _check_pass(coarse, rays, z, lat, t)
        c0 = A.composite(raw_c, z, rays[:, 3:6], None, False, 64, None)
        z_f = c0["z_vals_out"]
        raw_f, idx_f = _check_pass(fine, rays, z_f, lat, t)
        c1 = A.composite(raw_f, z_f, rays[:, 3:6], None, False)
    for k, v in (("raw", raw_f), ("rgb_map", c1["rgb_map"]), ("disp_map", c1["disp_map"]), ("acc_map", c1["acc_map"]),
                 ("rgb0", c0["rgb_map"]), ("termination_index0", idx_c), ("termination_index", idx_f)):
        assert torch.equal(got[k].view(torch.int32), v.view(torch.int32)), k
    _check_indices(got, 64, 64, t)
    died = (idx_c < 64).float().mean().item()
    K = _K()
    if cross is None:
        assert died < 0.5
    elif cross < 0.05:
        assert (idx_c == K).float().mean().item() > 0.5      # most rays die in the first segment
    elif cross > 0.9:
        assert died < 0.9 or (idx_c >= 64 - K).float().mean().item() > 0.5
    else:
        assert died > 0.5


def test_grid_and_termination_together():
    from nonrigid_nerf_b200 import autograd as A, ops
    coarse, fine, b = _models(True)
    r = O.make_rays(906, 400)
    _opaque((coarse, fine), r, 64, 0.5)
    full = _render(coarse, fine, r, 64)
    grid, occ = _random_grid(full["input_pts"].reshape(-1, 3).cpu().numpy(), 0.2, 7)
    t = 1e-4
    got = _render(coarse, fine, r, 64, occupancy=grid, early_termination=t)
    rays = helpers.rays8(r, DEV)
    lat = r["latents"].to(DEV)
    with torch.no_grad():
        z = ops.sample_coarse(rays, 64, None, False)
        raw_c, idx_c = _check_pass(coarse, rays, z, lat, t, grid=grid, occ=occ)
        c0 = A.composite(raw_c, z, rays[:, 3:6], None, False, 64, None)
        raw_f, idx_f = _check_pass(fine, rays, c0["z_vals_out"], lat, t, grid=grid, occ=occ)
    assert torch.equal(got["raw"].view(torch.int32), raw_f.view(torch.int32))
    assert torch.equal(got["termination_index0"], idx_c) and torch.equal(got["termination_index"], idx_f)
    _check_indices(got, 64, 64, t)


# ---- the error bound against the render without termination at the same depths ----------------------------------------
@pytest.mark.parametrize("white", [False, True])
def test_rgb_and_acc_bounds(white):
    coarse, fine, b = _models(True)
    r = O.make_rays(907, 500)
    _opaque((coarse,), r, 64, 0.4)
    for t in (1e-4, 1e-2, 0.2):
        full = _render(coarse, None, r, 0, white=white)
        got = _render(coarse, None, r, 0, white=white, early_termination=t)
        (idx,) = _check_indices(got, 0, 64, t)
        T_term = R.transmittance_at_death(got["opacity_alpha"].cpu().numpy(), _K(), t)
        T_term = np.where(idx < 64, T_term, 0.0)   # rays that never died are unchanged
        d_rgb = (got["rgb_map"] - full["rgb_map"]).abs().max(-1).values.cpu().numpy()
        d_acc = (got["acc_map"] - full["acc_map"]).abs().cpu().numpy()
        assert np.all(d_acc <= T_term + 1e-5), float((d_acc - T_term).max())
        assert np.all(d_rgb <= (2 if white else 1) * T_term + 1e-5), float((d_rgb - T_term).max())
        assert (idx < 64).mean() > 0.5


# ---- segment edge cases ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 5, 19, 100, 192])
def test_sample_counts(S):
    coarse, fine, b = _models(True)
    r = O.make_rays(908, 257)   # ragged tiles
    _opaque((coarse,), r, S, 0.5)
    for t in (1e-4, 0.3):
        got = _render(coarse, None, r, 0, S=S, early_termination=t)
        _check_indices(got, 0, S, t)
        full = _render(coarse, None, r, 0, S=S)
        idx = got["termination_index"].cpu().numpy()
        mask = np.arange(S)[None, :] < idx[:, None]
        want = np.where(mask[..., None], full["raw"].cpu().numpy(), np.float32(0))
        assert np.array_equal(got["raw"].cpu().numpy().view(np.uint32), want.view(np.uint32))


def test_one_ray_and_all_dead_after_round_0_and_none_dying():
    coarse, fine, b = _models(True)
    r = O.make_rays(909, 1)
    got = _render(coarse, fine, r, 64, early_termination=1e-4)
    _check_indices(got, 64, 64, 1e-4)
    r = O.make_rays(910, 300)
    _opaque((coarse, fine), r, 64, 0.001)
    got = _render(coarse, fine, r, 64, early_termination=1.0)       # every ray dies after round 0
    K = _K()
    assert torch.all(got["termination_index0"] == K) and torch.all(got["termination_index"] == K)
    assert torch.all(got["raw"][:, K:] == 0)
    _check_indices(got, 64, 64, 1.0)
    coarse, fine, b = _models(True, seed=911)
    got = _render(coarse, fine, r, 64, early_termination=1e-30)     # no ray ever dies
    assert torch.all(got["termination_index0"] == 64) and torch.all(got["termination_index"] == 128)
    _assert_same(_render(coarse, fine, r, 64), got)


@pytest.mark.parametrize("value", [float("nan"), float("inf")])
def test_nan_and_inf_sigma(value):
    coarse, fine, b = _models(True)
    r = O.make_rays(912, 200)
    with torch.no_grad():
        coarse.output_linear.weight[3, ::2] = 0.0
        coarse.output_linear.bias[3] = value
    got = _render(coarse, None, r, 0, early_termination=1e-4)
    (idx,) = _check_indices(got, 0, 64, 1e-4)
    if value != value:
        assert np.all(idx == 64)                  # relu(NaN) = 0 in compositing: alpha 0, nothing dies
    else:
        assert np.all(idx == _K())                # alpha 1: T = 1e-10 after the first sample


def test_noise_from_randomness():
    coarse, fine, b = _models(True)
    n = 300
    r = O.make_rays(913, n)
    _opaque((coarse, fine), r, 64, 0.5)
    rnd = O.make_randomness(913, n, 64, 64)
    t = 1e-3
    got = _render(coarse, fine, r, 64, noise_std=2.0, rnd=rnd, early_termination=t, perturb=1.0)
    _check_indices(got, 64, 64, t)
    again = _render(coarse, fine, r, 64, noise_std=2.0, rnd=rnd, early_termination=t, perturb=1.0)
    _assert_same(got, again, skip=())
    base = _render(coarse, fine, r, 64, noise_std=2.0, rnd=rnd, perturb=1.0)
    _assert_same(base, _render(coarse, fine, r, 64, noise_std=2.0, rnd=rnd, early_termination=0.0, perturb=1.0))


# ---- outputs, reruns, graphs, the ray-sharded wrapper ------------------------------------------------------------------
def test_surface_output_and_chunking():
    coarse, fine, b = _models(True)
    r = O.make_rays(914, 333)
    _opaque((coarse, fine), r, 64, 0.5)
    a = _render(coarse, fine, r, 64, surface=True, early_termination=1e-4)
    c = _render(coarse, fine, r, 64, surface=True, early_termination=1e-4, chunk=100)
    _assert_same(a, c, skip=())
    assert "surface_pts" in a and "median_indices" in a
    _check_indices(a, 64, 64, 1e-4)


def test_graph_replay_and_reruns():
    from nonrigid_nerf_b200 import ops
    coarse, fine, b = _models(True)
    r = {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in O.make_rays(915, 512).items()}   # no copies in capture
    _opaque((coarse, fine), r, 64, 0.5)
    full = _render(coarse, fine, r, 64)
    grid, _ = _random_grid(full["input_pts"].reshape(-1, 3).cpu().numpy(), 0.3, 9)
    for kw in ({"early_termination": 1e-4}, {"early_termination": 1e-4, "occupancy": grid}):
        eager = _render(coarse, fine, r, 64, detailed=False, **kw)
        _assert_same(eager, _render(coarse, fine, r, 64, detailed=False, **kw), skip=())
        ops.pack_nerf(coarse), ops.pack_nerf(fine), ops.pack_bender(b)   # cached weight images, so capture launches no repack
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            _render(coarse, fine, r, 64, detailed=False, **kw)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            captured = _render(coarse, fine, r, 64, detailed=False, **kw)
        for _ in range(2):
            g.replay()
            torch.cuda.synchronize()
            _assert_same(eager, captured, skip=())


def test_parallelized_render_function_on_one_gpu():
    from nonrigid_nerf_b200 import parallel as Pl, train as T
    coarse, fine, b = _models(True)
    r = O.make_rays(916, 300)
    _opaque((coarse, fine), r, 64, 0.5)
    fn = Pl.get_parallelized_render_function(coarse, fine, b)
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=64, N_samples=64, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0,
              ndc=False, lindisp=False, early_termination=1e-4)
    with torch.no_grad():
        got = fn(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=32768, near=r["near"], far=r["far"],
                 additional_pixel_information={"ray_bending_latents": r["latents"].to(DEV)}, detailed_output=True, **kw)
    want = _render(coarse, fine, r, 64, early_termination=1e-4)
    for k in ("termination_index", "termination_index0", "rgb0", "opacity_alpha"):
        assert torch.equal(got[3][k], want[k]), k
    assert torch.equal(got[0], want["rgb_map"])
