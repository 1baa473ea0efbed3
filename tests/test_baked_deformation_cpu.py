"""CPU tests of baked deformation grids: the numpy restatement (tests/baked_deformation_reference.py) against fp64 trilinear
interpolation and the knob algebra, the fp16 store rule, the workspace sizes, the C entry points' argument checks on host
pointers (no kernel is launched) and the Python refusals, raised before anything reaches the device."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import baked_deformation_reference as D
from tests.test_baked_cpu import _trilinear64


def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


@pytest.mark.parametrize("cutoff,scaling", [(None, None), (0.5, None), (None, 1.7), (0.3, 0.25)])
def test_bend_restatement_against_fp64(cutoff, scaling):
    rs = np.random.RandomState(11)
    nx, ny, nz = 9, 13, 7
    lo, hi = np.float32([-1.0, -0.5, -2.0]), np.float32([0.5, 1.0, -0.25])
    values = np.concatenate([rs.uniform(-0.2, 0.2, (nz, ny, nx, 3)), rs.uniform(0, 1, (nz, ny, nx, 1))], -1).astype(np.float16)
    x = rs.uniform(lo, hi, size=(5000, 3)).astype(np.float32)
    got = D.bend(x, values, lo, hi, cutoff, scaling)
    v64 = _trilinear64(values, x, lo, hi)
    o64, r64 = v64[:, :3], v64[:, 3]
    tol = 4 * max(nx, ny, nz) * 2.0 ** -23 * 2 + 8 * 2.0 ** -24
    assert np.abs(got["unmasked_offsets"] - o64).max() < tol
    r = got["rigidity_mask"]
    if cutoff is not None:   # the cut-off acts on the fp32 lookup, so compare where fp64 agrees on the side
        far = np.abs(r64 - cutoff) > tol
        assert np.all((r[far] == 0) == (r64[far] <= cutoff))
        keep = far & (r64 > cutoff)
        assert np.abs(r[keep] - r64[keep]).max() < tol
    else:
        assert np.abs(r - r64).max() < tol
    m64 = r.astype(np.float64)[:, None] * got["unmasked_offsets"].astype(np.float64) * (1.0 if scaling is None else scaling)
    assert np.abs(got["masked_offsets"] - m64).max() <= 2 * 2.0 ** -24 * np.abs(m64).max() + 1e-30
    c64 = x.astype(np.float64) + got["masked_offsets"].astype(np.float64)
    assert np.abs(got["input_pts"] - c64).max() <= 2.0 ** -24 * np.abs(c64).max()
    assert np.array_equal(got["initial_input_pts"], x)


def test_bend_restatement_rounds_each_operation():
    values = np.zeros((2, 2, 2, 4), np.float16)
    values[..., :3] = np.float16(0.1)
    values[..., 3] = np.float16(0.7)
    lo, hi = np.float32([0, 0, 0]), np.float32([1, 1, 1])
    x = np.float32([[0.3, 0.6, 0.9]])
    got = D.bend(x, values, lo, hi, None, 1.3)
    o, r = np.float32(np.float16(0.1)), np.float32(np.float16(0.7))
    m = np.float32(np.float32(r * o) * np.float32(1.3))
    assert got["masked_offsets"][0, 0] == m and got["input_pts"][0, 0] == np.float32(x[0, 0] + m)


def test_store_rule():
    o = np.float32([[1.0, 65519.0, 65520.0], [np.nan, -np.inf, -1e30], [1 + 2 ** -11, 3e-8, -0.0]])
    r = np.float32([0.25, np.inf, 1e6])
    h = D.to_f16(o, r)
    assert h.dtype == np.float16 and h.shape == (3, 4)
    assert h[0].tolist() == [1.0, 65504.0, 65504.0, 0.25]
    assert np.isnan(h[1, 0]) and h[1, 1] == -np.inf and h[1, 2] == -65504 and h[1, 3] == np.inf
    assert h[2, 0] == 1.0 and h[2, 3] == 65504 and np.signbit(h[2, 2])


def test_per_ray_rule():
    lo, hi = np.float32([-1, -1, -1]), np.float32([1, 1, 1])
    rays = np.float32([[0, 0, 0, 0, 0, 1, 0, 1], [0, 0, 0, 0, 0, 1, 0, 1], [0, 0, 0, np.nan, 0, 1, 0, 1]])
    z = np.float32([[0.0, 0.5, 1.0], [0.0, 0.5, np.nextafter(np.float32(1), np.float32(2))], [0.0, 0.0, 0.0]])
    x = D.sample_points(rays, z)
    assert D.deformed_rays(x, lo, hi).tolist() == [True, False, False]


def test_workspace_sizes_and_timing_kinds():
    L, lib = _lib()
    a256 = lambda n: (n + 255) // 256 * 256
    for n, s, ch, det in ((1000, 64, 5, 1), (1000, 64, 4, 0), (1, 1, 5, 1), (3000, 192, 5, 0)):
        p = n * s
        want = (lib.nrn_baked_workspace_bytes(n, s, ch, 1) + a256(n) + a256(4 * ((n + 1023) // 1024 + 1)) + 256 + a256(4 * n)
                + a256(32 * n) + a256(128 * n) + a256(4 * p) + a256(16 * p) + (4 * a256(12 * p) + a256(4 * p) if det else 0))
        assert lib.nrn_deformed_workspace_bytes(n, s, ch, det) == want
    assert lib.nrn_deformed_workspace_bytes(1000, 64, 6, 0) == 0
    assert lib.nrn_deformed_workspace_bytes(-1, 64, 5, 0) == 0
    assert lib.nrn_deformed_workspace_bytes(1 << 20, 1 << 12, 5, 0) == 0   # more than 2^31 - 1 points
    assert L.DEFORMATION_KERNEL_KINDS == ("deformation_plane", "deformed_rays", "deformed_fallback", "deformed_bend",
                                          "deformed_bend_scatter", "deformed_compact", "deformed_field", "deformed_scatter")
    assert L.BAKED_KERNEL_KINDS[-1] == "baked_scatter"   # kinds 45 to 49 stay; these are 50 to 57


def _grids(L, **kw):
    g = L.NrnRadianceGrid()
    g.values, g.nx, g.ny, g.nz = 4096, 4, 4, 4
    g.min_point[:] = [-1.0] * 3
    g.max_point[:] = [1.0] * 3
    d = L.NrnDeformGrid()
    d.values, d.nx, d.ny, d.nz = kw.get("values", 8192), kw.get("nx", 4), kw.get("ny", 4), kw.get("nz", 4)
    d.min_point[:] = kw.get("lo", [-1.0, -1.0, -1.0])
    d.max_point[:] = kw.get("hi", [1.0, 1.0, 1.0])
    d.n_frames, d.frame = kw.get("n_frames", 3), kw.get("frame", 2)
    return g, d


def test_c_argument_checks():
    L, lib = _lib()
    err = lambda: lib.nrn_last_error().decode()
    buf = (C.c_float * 64)()
    plane = C.c_void_p(4096)
    # the plane store
    assert lib.nrn_deformation_plane_f16(buf, buf, -1, plane, None) == -1 and "bad size" in err()
    assert lib.nrn_deformation_plane_f16(None, buf, 4, plane, None) == -1 and "null" in err()
    assert lib.nrn_deformation_plane_f16(buf, None, 4, plane, None) == -1 and "null" in err()
    assert lib.nrn_deformation_plane_f16(buf, buf, 4, None, None) == -1 and "null" in err()
    assert lib.nrn_deformation_plane_f16(buf, buf, 4, C.c_void_p(4100), None) == -1 and "aligned" in err()
    assert lib.nrn_deformation_plane_f16(C.c_void_p(4097), buf, 4, plane, None) == -1 and "aligned" in err()
    assert lib.nrn_deformation_plane_f16(buf, C.c_void_p(4098), 4, plane, None) == -1 and "aligned" in err()
    assert lib.nrn_deformation_plane_f16(None, None, 0, None, None) == 0   # nothing to store
    # the render pass
    a = L.NrnFieldArgs()
    a.rays, a.z_vals, a.n_rays, a.n_samples, a.out_ch, a.nerf_packed, a.raw = 4096, 4096, 10, 64, 5, 4096, 4096
    a.bender_packed, a.latents, a.latent_stride = 4096, 4096, 32
    ws = C.c_void_p(4096)
    need = lib.nrn_deformed_workspace_bytes(10, 64, 5, 0)
    run = lambda g, d, w=ws, nb=need: lib.nrn_field_forward_deformed(C.byref(a), C.byref(g) if g is not None else None,
                                                                     C.byref(d) if d is not None else None, w, nb)
    bad = [({"frame": 3}, "frame 3 out of range"), ({"frame": -1}, "out of range"), ({"n_frames": 0, "frame": 0}, "out of range"),
           ({"nx": 1}, "out of range"), ({"nz": 1025}, "out of range"), ({"values": None}, "values"), ({"values": 8196}, "values"),
           ({"lo": [1.0, 0.0, 0.0], "hi": [1.0, 1.0, 1.0]}, "max > min"), ({"hi": [float("nan"), 1.0, 1.0]}, "finite"),
           ({"lo": [-3e38, 0.0, 0.0], "hi": [3e38, 1.0, 1.0]}, "fp32 range")]
    for kw, msg in bad:
        g, d = _grids(L, **kw)
        assert run(g, d) == -1 and msg in err() and "deformation grid" in err(), (kw, err())
    g, d = _grids(L)
    assert run(g, None) == -1 and "deformation grid: null" in err()
    assert run(None, d) == -1 and "null grid" in err()
    assert run(g, d, nb=need - 1) == -1 and "workspace" in err()
    assert run(g, d, w=C.c_void_p(4096 + 16)) == -1 and "workspace" in err()
    assert run(g, d, w=None) == -1 and "workspace" in err()
    a.input_pts = 4096
    assert run(g, d) == -1 and "workspace" in err()   # details need their gathered rows too
    a.input_pts = None
    a.z_vals = 4098
    assert run(g, d) == -1 and "aligned" in err()
    a.z_vals = 4096
    a.n_rays, a.n_samples = 1 << 17, 1 << 15
    assert run(g, d, nb=1 << 40) == -1 and "2^31 - 1" in err()
    a.n_rays, a.n_samples = 10, 64
    a.bender_packed = None
    assert run(g, d) == -1 and "ray bender" in err()
    a.bender_packed = 4096
    a.latents = None
    assert run(g, d) == -1 and "latents" in err()
    a.latents = 4096
    a.stash, a.relu_mask = 4096, 4096
    assert run(g, d) == -1 and "inference only" in err()
    a.stash = a.relu_mask = None
    a.points, a.points_stride = 4096, 3
    assert run(g, d) == -1 and "ray mode" in err()
    a.points = None
    a.raw = None
    assert run(g, d) == -1 and "raw" in err()
    a.raw, a.out_ch = 4096, 6
    assert run(g, d) == -1 and "out_ch" in err()
    a.out_ch, a.n_rays = 5, 0
    assert run(g, d, w=None, nb=0) == 0   # no rays: nothing to do


def _nets(bender=True, **kw):
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    embed_fn, input_ch = H.get_embedder(10, 0)
    b = H.ray_bending(input_ch, 32, "simple_neural", embed_fn) if bender else None
    base = dict(D=8, W=256, input_ch=input_ch, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False, ray_bender=b,
                ray_bending_latent_size=32)
    base.update(kw)
    return H.NeRF(**base)


def _deform(frames=3, res=(4, 4, 4), dtype=torch.float16, shape=None, lo=(-1, -1, -1), hi=(1, 1, 1)):
    from nonrigid_nerf_b200 import geometry as G
    nx, ny, nz = res
    return G.DeformationGrid(torch.zeros(shape or (frames, nz, ny, nx, 4), dtype=dtype), np.float32(lo), np.float32(hi), res,
                             torch.zeros(frames, 32))


def test_frame_checks_and_struct():
    from nonrigid_nerf_b200 import geometry as G
    grid = _deform()
    for i in (3, -1, True, 1.0, "0"):
        with pytest.raises(RuntimeError, match="out of range"):
            grid.frame(i)
    with pytest.raises(RuntimeError, match="DeformationGrid"):
        G.FrameDeformation(grid.values, 0)
    for values in (torch.zeros(4, 4, 4, 4, dtype=torch.float16), torch.zeros(1, 3, 4, 4, 4, 4, dtype=torch.float16), None):
        flat = G.DeformationGrid(values, grid.min_point, grid.max_point, grid.resolution, grid.latents)
        with pytest.raises(RuntimeError, match=r"values must be a contiguous \[F, nz, ny, nx, 4\] float16 tensor"):
            flat.frame(0)   # a values tensor of the wrong rank is named as such, not as a frame out of range
    f = grid.frame(np.int64(2))
    s = f.c_struct("cpu")
    assert (s.nx, s.ny, s.nz, s.n_frames, s.frame) == (4, 4, 4, 3, 2) and s.values == grid.values.data_ptr()
    for bad in (_deform(dtype=torch.float32), _deform(shape=(3, 4, 4, 4, 3)), _deform(shape=(3, 4, 4, 5, 4)),
                _deform(res=(4, 4, 5), shape=(3, 4, 4, 4, 4))):
        with pytest.raises(RuntimeError, match="float16"):
            bad.frame(0).c_struct("cpu")
    for res in ((1, 4, 4), (4, 1025, 4)):
        with pytest.raises(RuntimeError, match="deformation grid resolution must be 2..1024"):
            _deform(res=res, shape=(3, 4, 4, 4, 4)).frame(0).c_struct("cpu")
    with pytest.raises(RuntimeError, match="must exceed min_point"):
        _deform(lo=(0, 0, 0), hi=(1, 0, 1)).frame(0).c_struct("cpu")
    with pytest.raises(RuntimeError, match="is on cpu"):
        f.c_struct("cuda:0")


def test_bake_refusals_before_launch():
    from nonrigid_nerf_b200 import geometry as G, run_nerf_helpers as H
    embed_fn, input_ch = H.get_embedder(10, 0)
    b = H.ray_bending(input_ch, 32, "simple_neural", embed_fn)   # on the CPU: anything that reached the device would fail
    for res in (1, 1025, (8, 8, 1), (8, 8), 2.0):
        with pytest.raises(RuntimeError, match="resolution"):
            G.bake_deformation(b, torch.zeros(2, 32), [-1] * 3, [1] * 3, res)
    with pytest.raises(RuntimeError, match="must exceed min_point"):
        G.bake_deformation(b, torch.zeros(2, 32), [0, 0, 0], [1, 1, 0], 8)
    with pytest.raises(RuntimeError, match="CUDA device"):
        G.bake_deformation(b, torch.zeros(2, 32), [-1] * 3, [1] * 3, 8)


def test_render_refusals_before_launch():
    from nonrigid_nerf_b200 import geometry as G, train as T
    rgrid = G.RadianceGrid(torch.zeros(4, 4, 4, 4, dtype=torch.float16), np.float32([-1] * 3), np.float32([1] * 3), (4, 4, 4))
    dgrid = _deform()
    bent, plain = _nets(), _nets(bender=False)
    views = _nets(bender=False, use_viewdirs=True, input_ch_views=27, output_ch=4)
    tc = _nets(bender=False, time_conditioned_baseline=True)
    rays_o, rays_d = torch.zeros(4, 3), torch.ones(4, 3)
    kw = dict(near=0.0, far=1.0, ndc=False, N_samples=8, N_importance=0, network_query_fn=None, perturb=0.0, white_bkgd=False,
              raw_noise_std=0.0, lindisp=False, additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
    scene = lambda d, fine=None: G.BakedScene(rgrid, fine, d)
    cases = [
        (plain, scene(dgrid.frame(0)), {}, "needs a model with a ray bender"),
        (bent, scene(dgrid), {}, "must be a geometry.FrameDeformation"),
        (bent, scene(_deform(dtype=torch.float32).frame(0)), {}, "float16"),
        (bent, scene(_deform(res=(4, 4, 5), shape=(3, 4, 4, 4, 4)).frame(0)), {}, "float16"),
        (bent, scene(_deform(res=(1, 4, 4), shape=(3, 4, 4, 1, 4)).frame(0)), {}, "2..1024"),
        (bent, scene(_deform(lo=(0, 0, 0), hi=(1, 1, -1)).frame(0)), {}, "must exceed min_point"),
        (views, scene(dgrid.frame(0)), {"use_viewdirs": True}, "use_viewdirs=True"),
        (tc, scene(dgrid.frame(0)), {}, "time_conditioned_baseline=True"),
        (bent, scene(dgrid.frame(0)), {"early_termination": 0.01}, "occupancy or early_termination"),
        (bent, scene(dgrid.frame(0)), {"N_importance": 8, "network_fine": _nets()}, "needs a fine grid"),
        (bent, scene(dgrid.frame(0), rgrid), {"N_importance": 8, "network_fine": plain}, "needs a model with a ray bender"),
    ]
    with torch.no_grad():
        for net, sc, extra, msg in cases:
            with pytest.raises(RuntimeError, match=msg):
                T.render(rays_o, rays_d, network_fn=net, baked=sc, **dict(kw, **extra))
        with pytest.raises(RuntimeError, match="must be a geometry.FrameDeformation"):
            T.render_rays(torch.zeros(4, 8), bent, None, 8, baked=scene(rgrid),
                          additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
    with pytest.raises(RuntimeError, match="inference only"):
        T.render(rays_o, rays_d, network_fn=bent, baked=scene(dgrid.frame(0)), **kw)
