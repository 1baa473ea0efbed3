"""GPU tests of the meshes (geometry.py, csrc/mesh.cu).

Marching cubes is compared with the numpy restatement tests/mesh_reference.py bit for bit (vertices, faces, their order and
the per-plane offsets).  Topology is checked on analytic fields the test first shows to have no ambiguous face and no
occupied boundary point; the 1024^3 case has more than 2^31 grid edges.  The density equals NeRF.forward in point mode bit
for bit and the fp32 oracle within the forward tolerance of tests/test_field_forward_gpu.py."""
import math

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import mesh_reference as M

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _np_mesh(sigma, lo, hi, t):
    return M.marching_cubes(sigma.cpu().numpy() if isinstance(sigma, torch.Tensor) else sigma, lo, hi, t)


def _assert_same(mesh, ref):
    v, f, vo, fo = ref
    got_v = mesh.vertices.cpu().numpy()
    assert got_v.shape == v.shape and mesh.faces.shape == f.shape, (got_v.shape, v.shape, tuple(mesh.faces.shape), f.shape)
    assert got_v.view(np.int32).tolist() == v.astype(np.float32).view(np.int32).tolist()
    np.testing.assert_array_equal(mesh.faces.cpu().numpy(), f)
    assert mesh.faces.dtype == torch.int32 and mesh.vertices.dtype == torch.float32
    np.testing.assert_array_equal(mesh.vertex_offsets, vo)
    np.testing.assert_array_equal(mesh.face_offsets, fo)


def _mc(sigma, lo, hi, t):
    from nonrigid_nerf_b200 import geometry as G
    return G.marching_cubes(sigma if isinstance(sigma, torch.Tensor) else torch.from_numpy(sigma).to(DEV), lo, hi, t)


def test_all_single_cell_cases_match_the_restatement():
    for case in range(256):
        for pad in (0, 1):
            n = 2 + 2 * pad
            s = np.zeros((n, n, n), dtype=np.float32)
            for c, (dx, dy, dz) in enumerate(M.CORNERS):
                s[pad + dz, pad + dy, pad + dx] = 0.25 + 0.5 * ((case >> c) & 1) + 0.01 * c
            lo, hi = [-0.5, 0.25, 1.0], [0.75, 1.5, 2.0]
            _assert_same(_mc(s, lo, hi, 0.5), _np_mesh(s, lo, hi, 0.5))


@pytest.mark.parametrize("shape", [(2, 2, 2), (3, 5, 7), (65, 33, 17), (257, 257, 257)])
def test_random_fields_match_the_restatement(shape):
    nx, ny, nz = shape
    g = torch.Generator(device=DEV).manual_seed(nx * 7 + ny)
    s = torch.rand(nz, ny, nx, generator=g, device=DEV) * 2.0
    lo, hi = [-1.0, -0.3, 0.1], [1.0, 2.7, 0.4]
    _assert_same(_mc(s, lo, hi, 1.0), _np_mesh(s, lo, hi, 1.0))


def test_threshold_ties_nan_empty_and_full():
    g = torch.Generator(device=DEV).manual_seed(5)
    s = torch.randint(0, 4, (9, 11, 13), generator=g, device=DEV).float() * 0.25      # many values exactly at 0.5
    s[torch.rand(s.shape, generator=g, device=DEV) < 0.1] = float("nan")
    lo, hi = [0, 0, 0], [1, 1, 1]
    _assert_same(_mc(s, lo, hi, 0.5), _np_mesh(s, lo, hi, 0.5))
    for fill in (0.0, 1.0, float("nan")):
        m = _mc(torch.full((6, 5, 4), fill, device=DEV), lo, hi, 0.5)
        assert m.vertices.shape == (0, 3) and m.faces.shape == (0, 3) and m.colors is None and m.rigidity is None
        assert m.vertex_offsets.tolist() == [0] * 7 and m.face_offsets.tolist() == [0] * 6


# ---- topology ---------------------------------------------------------------------------------------------------------
def _axes_t(lo, hi, shape_xyz):
    return [torch.from_numpy(M.grid_axis(lo[a], hi[a], n)).to(DEV) for a, n in enumerate(shape_xyz)]


def _field(kind, shape_xyz, lo, hi):
    """sigma [nz, ny, nx] (positive inside), and the enclosed volume."""
    xs, ys, zs = _axes_t(lo, hi, shape_xyz)
    z, y, x = torch.meshgrid(zs, ys, xs, indexing="ij")
    if kind == "sphere":
        return 0.6 - torch.sqrt(x * x + y * y + z * z), 4 / 3 * math.pi * 0.6 ** 3
    if kind == "torus":
        q = torch.sqrt(x * x + y * y) - 0.5
        return 0.2 - torch.sqrt(q * q + z * z), 2 * math.pi ** 2 * 0.5 * 0.2 ** 2
    a = 0.35 - torch.sqrt((x - 0.45) ** 2 + y * y + z * z)
    b = 0.3 - torch.sqrt((x + 0.45) ** 2 + (y - 0.1) ** 2 + z * z)
    return torch.maximum(a, b), 4 / 3 * math.pi * (0.35 ** 3 + 0.3 ** 3)


def _ambiguous_faces(occ):
    """Number of cell faces whose occupied corners are exactly one diagonal."""
    n = 0
    for d in range(3):
        o = occ.movedim(d, 0)                       # faces perpendicular to axis d: the two other axes vary
        a, b, c, e = o[:, :-1, :-1], o[:, :-1, 1:], o[:, 1:, :-1], o[:, 1:, 1:]
        n += int(((a == e) & (b == c) & (a != b)).sum())
    return n


def _boundary_occupied(occ):
    return bool(occ[0].any() or occ[-1].any() or occ[:, 0].any() or occ[:, -1].any() or occ[:, :, 0].any() or occ[:, :, -1].any())


def _topology(mesh):
    """(every edge in exactly two faces and each directed edge once, Euler characteristic, signed volume) on the GPU."""
    f = mesh.faces.long()
    v = mesh.vertices.double()
    nv = v.shape[0]
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    und = torch.minimum(e[:, 0], e[:, 1]) * nv + torch.maximum(e[:, 0], e[:, 1])
    uniq, cnt = torch.unique(und, return_counts=True)
    directed = torch.unique(e[:, 0] * nv + e[:, 1]).numel() == e.shape[0]
    manifold = bool((cnt == 2).all()) and directed
    euler = nv - uniq.numel() + f.shape[0]
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    vol = float((a * torch.cross(b, c, dim=1)).sum() / 6.0)
    area = float(torch.linalg.norm(torch.cross(b - a, c - a, dim=1), dim=1).sum() / 2.0)
    return manifold, euler, vol, area


@pytest.mark.parametrize("shape", [(128, 128, 128), (96, 112, 80)])
@pytest.mark.parametrize("kind,euler", [("sphere", 2), ("torus", 0), ("two_spheres", 4)])
def test_closed_surfaces_of_analytic_fields(kind, euler, shape):
    lo, hi = [-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]
    s, volume = _field(kind, shape, lo, hi)
    occ = s > 0
    assert _ambiguous_faces(occ) == 0 and not _boundary_occupied(occ)
    m = _mc(s, lo, hi, 0.0)
    manifold, chi, vol, area = _topology(m)
    assert manifold and chi == euler, (manifold, chi)
    h = max((hi[a] - lo[a]) / (shape[a] - 1) for a in range(3))
    assert vol > 0 and abs(vol - volume) <= area * h, (vol, volume, area * h)
    _assert_same(m, _np_mesh(s, lo, hi, 0.0))


def test_1024_cubed_past_2_31_edges():
    n = 1024
    lo, hi = [-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]
    assert 3 * (n - 1) * n * n > 2 ** 31
    xs, ys, zs = _axes_t(lo, hi, (n, n, n))
    sigma = torch.empty(n, n, n, device=DEV)
    r2 = (xs[None, :] ** 2 + ys[:, None] ** 2)
    for k in range(n):      # an ellipsoid, one plane at a time
        sigma[k] = 0.8 - torch.sqrt(r2 + (1.3 * zs[k]) ** 2)
    amb = sum(_ambiguous_faces(sigma[k0:k0 + 129] > 0) for k0 in range(0, n - 1, 128))
    assert amb == 0 and not _boundary_occupied(sigma > 0)
    # independent per-plane counts: crossed edges owned by each plane, and the table's triangles of each cell layer
    table = torch.from_numpy(M.TRI_COUNT).to(DEV)
    v_count, f_count = [], []
    for k in range(n):
        o0 = sigma[k] > 0
        cnt = (o0[:, 1:] != o0[:, :-1]).sum() + (o0[1:] != o0[:-1]).sum()
        if k + 1 < n:
            o1 = sigma[k + 1] > 0
            cnt = cnt + (o0 != o1).sum()
            case = sum((o1 if dz else o0)[dy:dy + n - 1, dx:dx + n - 1].long() << c for c, (dx, dy, dz) in enumerate(M.CORNERS))
            f_count.append(table[case].sum())
        v_count.append(cnt)
    v_count, f_count = torch.stack(v_count).tolist(), torch.stack(f_count).tolist()
    m = _mc(sigma, lo, hi, 0.0)
    assert np.diff(m.vertex_offsets).tolist() == v_count
    assert np.diff(m.face_offsets).tolist() == f_count
    manifold, chi, vol, _ = _topology(m)
    assert manifold and chi == 2 and vol > 0, (manifold, chi, vol)
    axes = [M.grid_axis(lo[a], hi[a], n) for a in range(3)]
    for k in (0, 517, n - 3, n - 1):
        planes = sigma[k:k + 3].cpu().numpy()
        v, f, nv = M.slab(planes, k, axes, np.float32(0.0), int(m.vertex_offsets[k]))
        vo, fo = m.vertex_offsets, np.append(m.face_offsets, m.faces.shape[0])
        assert nv == vo[k + 1] - vo[k]
        assert m.vertices[vo[k]:vo[k + 1]].cpu().numpy().view(np.int32).tolist() == v.view(np.int32).tolist()
        np.testing.assert_array_equal(m.faces[fo[k]:fo[k + 1]].cpu().numpy(), f)


# ---- the model ----------------------------------------------------------------------------------------------------------
LO_M, HI_M = [-1.2, -0.9, -1.0], [1.1, 1.0, 0.8]
RES = (21, 18, 15)


def _grid_points(res):
    nx, ny, nz = res
    return torch.from_numpy(np.concatenate([M.grid_points_plane(LO_M, HI_M, res, k).reshape(-1, 3) for k in range(nz)])).to(DEV)


def _point_mode(net, pts, latent, detailed=False):
    """NeRF.forward(x) on run_network's layout: [xyz | embedding | latent]."""
    x = torch.cat([pts, torch.zeros(pts.shape[0], 60, device=DEV)] + ([latent.reshape(1, 32).expand(pts.shape[0], 32)] if latent is not None else []), 1)
    with torch.no_grad():
        return net(x, detailed_output=detailed)


def _bending_model(seed=31):
    coarse, _, bender, (cp, _, bp) = helpers.build_models(O, seed, DEV, True)
    lat = O.make_rays(seed, 4)["latents"][1].to(DEV)
    return coarse, bender, cp, bp, lat


def _set_knobs(net, bender, knob):
    bender.rigidity_test_time_cutoff = 0.5 if knob == "cutoff" else None
    bender.test_time_scaling = 2.5 if knob == "scaling" else None
    net.test_time_nonrigid_object_removal_threshold = 0.5 if knob == "removal" else None


@pytest.mark.parametrize("knob", [None, "cutoff", "scaling", "removal"])
def test_density_grid_equals_point_mode_and_the_oracle(knob):
    from nonrigid_nerf_b200 import geometry as G
    net, bender, cp, bp, lat = _bending_model()
    _set_knobs(net, bender, knob)
    pts = _grid_points(RES)
    sig = G.density_grid(net, LO_M, HI_M, RES, latent=lat)
    assert sig.shape == (RES[2], RES[1], RES[0]) and sig.dtype == torch.float32
    ref = torch.relu(_point_mode(net, pts, lat)[:, 3])
    assert torch.equal(sig.reshape(-1), ref)
    raw_o, _ = O.query_field(cp, bp, pts.cpu()[None], lat.cpu()[None])
    sig_o = torch.relu(raw_o[0, :, 3])
    if knob is None:      # a knob that cuts at a rigidity value can flip points whose rigidity sits within rounding of it
        assert bool(((sig.reshape(-1).cpu() - sig_o).abs() <= 2e-2 + 1e-2 * sig_o.abs()).all())
    if knob is None:      # the canonical grid: the bender is off
        can = G.density_grid(net, LO_M, HI_M, RES)
        net.ray_bender = (None,)
        try:
            assert torch.equal(can.reshape(-1), torch.relu(_point_mode(net, pts, None)[:, 3]))
        finally:
            net.ray_bender = (bender,)
        sig_c = torch.relu(O.query_field(cp, None, pts.cpu()[None], None)[0][0, :, 3])
        assert bool(((can.reshape(-1).cpu() - sig_c).abs() <= 2e-2 + 1e-2 * sig_c.abs()).all())
        assert not torch.equal(can, sig)


def test_density_grid_of_the_time_conditioned_baseline():
    from nonrigid_nerf_b200 import geometry as G
    coarse, _, _ = helpers.tc_models(17, DEV)
    lat = torch.randn(32, generator=torch.Generator().manual_seed(3)).to(DEV)
    sig = G.density_grid(coarse, LO_M, HI_M, RES, latent=lat)
    assert torch.equal(sig.reshape(-1), torch.relu(_point_mode(coarse, _grid_points(RES), lat)[:, 3]))


def _threshold(sig):
    return float(sig.flatten().median())


@pytest.mark.parametrize("canonical", [False, True])
def test_extract_mesh_equals_marching_cubes_of_the_density_grid(canonical):
    from nonrigid_nerf_b200 import geometry as G
    net, bender, cp, bp, lat = _bending_model()
    latent = None if canonical else lat
    sig = G.density_grid(net, LO_M, HI_M, RES, latent=latent)
    t = _threshold(sig)
    m = G.extract_mesh(net, LO_M, HI_M, RES, t, latent=latent)
    ref = G.marching_cubes(sig, LO_M, HI_M, t)
    assert m.faces.shape[0] > 100
    _assert_same(m, (ref.vertices.cpu().numpy(), ref.faces.cpu().numpy(), ref.vertex_offsets, ref.face_offsets))
    _assert_same(m, _np_mesh(sig, LO_M, HI_M, t))
    # colours (and with a latent the rigidity) are point mode at the vertices
    if canonical:
        net.ray_bender = (None,)
    try:
        raw, det = _point_mode(net, m.vertices, latent, detailed=True)
    finally:
        net.ray_bender = (bender,)
    col = (255.0 * torch.clamp(1.0 / (1.0 + torch.exp(-raw[:, :3])), 0.0, 1.0)).to(torch.uint8)
    assert m.colors.dtype == torch.uint8 and torch.equal(m.colors, col)
    if canonical:
        assert m.rigidity is None
    else:
        assert torch.equal(m.rigidity, det["rigidity_mask"].reshape(-1))
    bare = G.extract_mesh(net, LO_M, HI_M, RES, t, latent=latent, colors=False, rigidity=False)
    assert bare.colors is None and bare.rigidity is None and torch.equal(bare.vertices, m.vertices)
    again = G.extract_mesh(net, LO_M, HI_M, RES, t, latent=latent)
    for a, b in zip(again[:4], m[:4]):
        assert (a is None and b is None) or torch.equal(a, b)


def test_fresh_bender_gives_the_canonical_mesh():
    from nonrigid_nerf_b200 import geometry as G, run_nerf_helpers as H
    net, bender, cp, bp, lat = _bending_model()
    embed_fn, ch = H.get_embedder(10, 0)
    fresh = H.ray_bending(ch, 32, "simple_neural", embed_fn).to(DEV)     # zero output layer: straight rays
    net.ray_bender = (fresh,)
    sig = G.density_grid(net, LO_M, HI_M, RES)
    t = _threshold(sig)
    bent = G.extract_mesh(net, LO_M, HI_M, RES, t, latent=lat)
    can = G.extract_mesh(net, LO_M, HI_M, RES, t)
    assert bent.faces.shape[0] > 100
    for a, b in zip(bent[:3], can[:3]):
        assert torch.equal(a, b)
    assert bent.rigidity is not None and can.rigidity is None


def test_model_without_bender_and_writers(tmp_path):
    from nonrigid_nerf_b200 import geometry as G
    net, _, _, _ = helpers.build_models(O, 44, DEV, False)
    sig = G.density_grid(net, LO_M, HI_M, RES)
    t = _threshold(sig)
    m = G.extract_mesh(net, LO_M, HI_M, RES, t)
    assert m.rigidity is None and m.colors is not None
    _assert_same(m, _np_mesh(sig, LO_M, HI_M, t))
    G.write_ply(tmp_path / "m.ply", m)
    G.write_obj(tmp_path / "m.obj", m)
    assert (tmp_path / "m.ply").stat().st_size > 15 * m.vertices.shape[0]
