"""CPU tests of the meshes (geometry.py, csrc/mesh.cu): the numpy restatement tests/mesh_reference.py on hand-checked cases
and on all 256 cube configurations, the library's cube table against the restatement's, the PLY / OBJ writers, and every
argument check of the new entry points and of the Python API.  No kernel is launched here."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from tests import mesh_reference as M

LO, HI = [-1.0, -2.0, 0.5], [1.0, 3.0, 2.0]


def _case_grid(case, pad):
    """sigma [nz, ny, nx] holding one cell's configuration (1 occupied, 0 not) at offset `pad` in a grid of 2 + 2 pad points."""
    n = 2 + 2 * pad
    s = np.zeros((n, n, n), dtype=np.float32)
    for c, (dx, dy, dz) in enumerate(M.CORNERS):
        s[pad + dz, pad + dy, pad + dx] = (case >> c) & 1
    return s


def _edges_of(faces):
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    return e


def _signed_volume(v, f):
    a, b, c = (v[f[:, i]].astype(np.float64) for i in range(3))
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


def test_table_matches_the_library():
    from nonrigid_nerf_b200 import _lib
    counts = np.zeros(256, dtype=np.int32)
    edges = np.zeros((256, 5, 3), dtype=np.int8)
    assert _lib.load().nrn_mesh_cube_table(counts.ctypes.data, edges.ctypes.data) == 0
    assert M.TRI_EDGES.shape == (256, 5, 3)
    np.testing.assert_array_equal(counts, M.TRI_COUNT)
    np.testing.assert_array_equal(edges, M.TRI_EDGES)


def test_hand_checked_cases():
    # numbering: corner c at (c & 1, c >> 1 & 1, c >> 2 & 1); edge 4 * axis + r from the corner with offsets (r & 1, r >> 1)
    assert M.EDGES[0] == (0, 0) and M.EDGES[3] == (0, 6) and M.EDGES[5] == (1, 1) and M.EDGES[6] == (1, 4) and M.EDGES[11] == (2, 3)
    # corner 0 alone: the triangle on its three edges, normal towards (1, 1, 1) (out of the occupied corner)
    assert M.TRI_COUNT[1] == 1 and M.TRI_EDGES[1, 0].tolist() == [0, 4, 8]
    # corners 0 and 1 (the x edge at y = z = 0): a quad of the y and z edges of both corners
    assert M.TRI_COUNT[0b11] == 2 and sorted(set(M.TRI_EDGES[0b11, :2].ravel())) == [4, 5, 8, 9]
    # the bottom face: a quad on the four z edges
    assert M.TRI_COUNT[0x0F] == 2 and sorted(set(M.TRI_EDGES[0x0F, :2].ravel())) == [8, 9, 10, 11]
    # three corners of the bottom face: a pentagon
    assert M.TRI_COUNT[0b0111] == 3
    # checkerboards: every face ambiguous; the segments cut off each occupied corner, so four separate triangles
    for cs in (0x69, 0x96):
        assert M.TRI_COUNT[cs] == 4
        assert len(set(M.TRI_EDGES[cs, :4].ravel())) == 12
    # two diagonal corners of one face (0 and 3): the face is ambiguous, the occupied corners are cut off separately
    assert M.TRI_COUNT[0b1001] == 2
    # ... and its complement joins the two unoccupied corners' regions through the face: one loop of six edges
    assert M.TRI_COUNT[0xFF ^ 0b1001] == 4
    assert M.TRI_COUNT[0] == 0 and M.TRI_COUNT[255] == 0


@pytest.mark.parametrize("case", range(256))
def test_every_single_cell_configuration(case):
    """One cell: a vertex at the midpoint of each crossed edge, in edge-key order; faces only on those vertices, with the
    table's count.  Embedded in unoccupied space the cell's surface is closed: every edge in exactly two faces, each in both
    directions, and a positive signed volume (normals point out of the occupied region)."""
    t = 0.5
    v, f, vo, fo = M.marching_cubes(_case_grid(case, 0), [0, 0, 0], [1, 1, 1], t)
    crossed = []
    for k, j, i, a in itertools.product(range(2), range(2), range(2), range(3)):
        p = np.array([i, j, k])
        q = p + np.eye(3, dtype=int)[a]
        if q.max() > 1:
            continue
        oa = (case >> (p[0] | p[1] << 1 | p[2] << 2)) & 1
        ob = (case >> (q[0] | q[1] << 1 | q[2] << 2)) & 1
        if oa != ob:
            crossed.append((p + q) / 2.0)
    assert len(v) == len(crossed)
    np.testing.assert_array_equal(v, np.array(crossed, dtype=np.float32).reshape(-1, 3))
    assert len(f) == M.TRI_COUNT[case] and vo[0] == 0 and vo[-1] == len(v) and fo.tolist() == [0, len(f)]
    assert len(f) == 0 or (f.min() >= 0 and f.max() < len(v))
    if case == 0:
        return
    v, f, _, _ = M.marching_cubes(_case_grid(case, 1), [0, 0, 0], [3, 3, 3], t)
    e = _edges_of(f)
    key = np.minimum(e[:, 0], e[:, 1]) * len(v) + np.maximum(e[:, 0], e[:, 1])
    _, cnt = np.unique(key, return_counts=True)
    assert (cnt == 2).all(), case
    directed = e[:, 0] * len(v) + e[:, 1]
    assert len(np.unique(directed)) == len(directed), case          # consistent orientation
    assert _signed_volume(v, f) > 0, case


def test_grid_point_formula():
    lo, hi = np.float32(-1.3), np.float32(0.7)
    for n in (2, 3, 17, 256, 1024):
        x = M.grid_axis(-1.3, 0.7, n)
        assert x.dtype == np.float32 and x[0] == lo and x[-1] == hi
        for i in range(n - 1):   # each operation rounded in fp32, in this order
            assert x[i] == np.float32(lo + np.float32(np.float32(hi - lo) * np.float32(np.float32(i) / np.float32(n - 1)))), (n, i)
        np.testing.assert_allclose(x, -1.3 + 2.0 * np.arange(n) / (n - 1), rtol=0, atol=4e-7)
    np.testing.assert_array_equal(M.grid_axis(-1, 1, 3), np.array([-1, 0, 1], dtype=np.float32))
    p = M.grid_points_plane(LO, HI, (4, 3, 5), 4)
    assert p.shape == (3, 4, 3) and (p[..., 2] == np.float32(2.0)).all() and p[2, 3, 1] == np.float32(3.0)


def test_restatement_threshold_nan_and_empty_cases():
    s = np.zeros((3, 3, 3), dtype=np.float32)
    assert [len(x) for x in M.marching_cubes(s, LO, HI, 0.0)[:2]] == [0, 0]            # nothing above the threshold
    assert [len(x) for x in M.marching_cubes(s + 1, LO, HI, 0.5)[:2]] == [0, 0]        # everything above
    s[1, 1, 1] = 0.5
    assert len(M.marching_cubes(s, LO, HI, 0.5)[0]) == 0                             # exactly at the threshold: unoccupied
    s[:] = 1
    s[1, 1, 1] = np.nan
    v, f, _, _ = M.marching_cubes(s, [0, 0, 0], [2, 2, 2], 0.5)
    # NaN is not occupied, and counts as 0 where the six vertices around it are placed: the edge midpoints
    expect = [[1, 1, 0.5], [1, 0.5, 1], [0.5, 1, 1], [1.5, 1, 1], [1, 1.5, 1], [1, 1, 1.5]]
    np.testing.assert_array_equal(v, np.array(expect, dtype=np.float32))
    assert len(f) == 8 and _signed_volume(v, f) < 0     # a cavity: its faces point into the hole, away from the occupied space


def test_writers_round_trip(tmp_path):
    from nonrigid_nerf_b200 import geometry as G
    rng = np.random.default_rng(3)
    v = torch.from_numpy(rng.standard_normal((7, 3)).astype(np.float32))
    f = torch.from_numpy(rng.integers(0, 7, (5, 3)).astype(np.int32))
    col = torch.from_numpy(rng.integers(0, 256, (7, 3)).astype(np.uint8))
    rig = torch.from_numpy(rng.random(7).astype(np.float32))
    off = np.zeros(1, dtype=np.int64)
    for mesh in (G.Mesh(v, f, col, rig, off, off), G.Mesh(v, f, None, None, off, off), G.Mesh(v, f, col, None, off, off)):
        p = tmp_path / "m.ply"
        G.write_ply(p, mesh)
        data = p.read_bytes()
        head, body = data.split(b"end_header\n", 1)
        lines = head.decode().splitlines()
        assert lines[:3] == ["ply", "format binary_little_endian 1.0", "element vertex 7"] and "element face 5" in lines
        props = [ln.split()[-1] for ln in lines if ln.startswith("property") and "list" not in ln]
        dt = [(n, "<f4" if n in ("x", "y", "z", "rigidity") else "u1") for n in props]
        vert = np.frombuffer(body, dtype=dt, count=7)
        face = np.frombuffer(body[vert.nbytes:], dtype=[("n", "u1"), ("v", "<i4", (3,))])
        np.testing.assert_array_equal(np.stack([vert["x"], vert["y"], vert["z"]], 1), v.numpy())
        np.testing.assert_array_equal(face["v"], f.numpy())
        assert (face["n"] == 3).all() and len(face) == 5
        if mesh.colors is not None:
            np.testing.assert_array_equal(np.stack([vert["red"], vert["green"], vert["blue"]], 1), col.numpy())
        assert ("rigidity" in props) == (mesh.rigidity is not None)
        if mesh.rigidity is not None:
            np.testing.assert_array_equal(vert["rigidity"], rig.numpy())
        o = tmp_path / "m.obj"
        G.write_obj(o, mesh)
        rows = [ln.split() for ln in o.read_text().splitlines()]
        vs = np.array([[float(x) for x in r[1:]] for r in rows if r[0] == "v"])
        fs = np.array([[int(x) for x in r[1:]] for r in rows if r[0] == "f"])
        np.testing.assert_array_equal(vs[:, :3].astype(np.float32), v.numpy())
        np.testing.assert_array_equal(fs - 1, f.numpy())
        if mesh.colors is not None:
            np.testing.assert_array_equal(np.rint(vs[:, 3:] * 255).astype(np.uint8), col.numpy())


def test_entry_points_validate_before_touching_the_device():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    lo, hi = (np.array(x, dtype=np.float32) for x in (LO, HI))
    buf = ctypes.c_void_p(16)      # never dereferenced: every call below fails validation or returns before any CUDA call
    bad = {
        "points nx": lambda: lib.nrn_mesh_grid_points(lo.ctypes.data, hi.ctypes.data, 1, 4, 4, 0, buf, None),
        "points k": lambda: lib.nrn_mesh_grid_points(lo.ctypes.data, hi.ctypes.data, 4, 4, 4, 4, buf, None),
        "points k<0": lambda: lib.nrn_mesh_grid_points(lo.ctypes.data, hi.ctypes.data, 4, 4, 4, -1, buf, None),
        "points plane": lambda: lib.nrn_mesh_grid_points(lo.ctypes.data, hi.ctypes.data, 1 << 15, 1 << 14, 4, 0, buf, None),
        "points extent": lambda: lib.nrn_mesh_grid_points(hi.ctypes.data, lo.ctypes.data, 4, 4, 4, 0, buf, None),
        "points null extent": lambda: lib.nrn_mesh_grid_points(None, hi.ctypes.data, 4, 4, 4, 0, buf, None),
        "points null": lambda: lib.nrn_mesh_grid_points(lo.ctypes.data, hi.ctypes.data, 4, 4, 4, 0, None, None),
        "points align": lambda: lib.nrn_mesh_grid_points(lo.ctypes.data, hi.ctypes.data, 4, 4, 4, 0, ctypes.c_void_p(18), None),
        "sigma n": lambda: lib.nrn_mesh_sigma(buf, -1, 5, buf, None),
        "sigma out_ch": lambda: lib.nrn_mesh_sigma(buf, 4, 3, buf, None),
        "sigma null": lambda: lib.nrn_mesh_sigma(None, 4, 5, buf, None),
        "sigma align": lambda: lib.nrn_mesh_sigma(buf, 4, 5, ctypes.c_void_p(17), None),
        "colors n": lambda: lib.nrn_mesh_colors(buf, -2, 5, buf, None),
        "colors out_ch": lambda: lib.nrn_mesh_colors(buf, 2, 6, buf, None),
        "colors null": lambda: lib.nrn_mesh_colors(buf, 2, 5, None, None),
        "count null": lambda: lib.nrn_mesh_count(None),
        "emit null": lambda: lib.nrn_mesh_emit(None),
    }
    for what, call in bad.items():
        assert call() == -1, what
        assert len(lib.nrn_last_error()) > 0, what
    assert lib.nrn_mesh_sigma(None, 0, 5, None, None) == 0 and lib.nrn_mesh_colors(None, 0, 4, None, None) == 0

    def slab(**kw):
        a = _lib.NrnMeshSlabArgs()
        a.sigma0, a.sigma1, a.min_point, a.max_point = 256, 512, lo.ctypes.data, hi.ctypes.data
        a.threshold, a.nx, a.ny, a.nz, a.k = 0.5, 8, 8, 4, 0
        a.workspace, a.totals, a.vertices, a.faces = 1024, 2048, 4096, 8192
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for fn, kw, msg in [
        ("count", dict(nx=1), b"bad sizes"), ("count", dict(nz=1), b"bad sizes"), ("count", dict(k=4), b"bad sizes"),
        ("count", dict(sigma0=None), b"null sigma0"), ("count", dict(workspace=None), b"null sigma0"),
        ("count", dict(sigma1=None), b"sigma1"), ("count", dict(k=3), b"sigma1"), ("count", dict(threshold=float("nan")), b"NaN"),
        ("count", dict(workspace=1040), b"aligned"), ("count", dict(sigma0=258), b"aligned"), ("count", dict(totals=None), b"totals"),
        ("emit", dict(min_point=None), b"null min_point"), ("emit", dict(max_point=lo.ctypes.data), b"exceed"),
        ("emit", dict(vertices=None), b"null vertices"), ("emit", dict(k=1, faces=None), b"null vertices"),
        ("emit", dict(faces=8194), b"aligned"), ("emit", dict(vertex_base=-1), b"bases"), ("emit", dict(face_base=1 << 31), b"bases"),
        ("emit", dict(k=1, vertex_base_prev=10, vertex_base=5), b"bases"),
    ]:
        a = slab(**kw)
        assert getattr(lib, "nrn_mesh_" + fn)(ctypes.byref(a)) == -1, (fn, kw)
        assert msg in lib.nrn_last_error(), (fn, kw, lib.nrn_last_error())
    assert lib.nrn_mesh_workspace_bytes(1, 8) == 0 and lib.nrn_mesh_workspace_bytes(1 << 15, 1 << 14) == 0
    assert lib.nrn_mesh_workspace_bytes(8, 8) > 3 * (64 + 4 * 65 + 49 + 4 * 50)
    assert lib.nrn_mesh_cube_table(None, None) == 0


def _models(**kw):
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    embed_fn, ch = H.get_embedder(10, 0)
    bender = H.ray_bending(ch, 32, "simple_neural", embed_fn) if kw.pop("bender", False) else None
    return H.NeRF(D=8, W=256, input_ch=ch, output_ch=5, skips=[4], ray_bender=bender, ray_bending_latent_size=32, **kw)


def test_api_refusals_raise_before_any_launch():
    from nonrigid_nerf_b200 import geometry as G
    net = _models(input_ch_views=0)
    views = _models(input_ch_views=27, use_viewdirs=True)
    tc = _models(input_ch_views=0, time_conditioned_baseline=True)
    with pytest.raises(RuntimeError, match="use_viewdirs"):
        G.density_grid(views, LO, HI, 4)
    with pytest.raises(RuntimeError, match="use_viewdirs"):
        G.extract_mesh(views, LO, HI, 4, 1.0)
    for res in (1, (4, 1, 4), (4, 4, 0), (4, 4), "8"):
        with pytest.raises(RuntimeError, match="resolution"):
            G.density_grid(net, LO, HI, res)
        with pytest.raises(RuntimeError, match="resolution"):
            G.extract_mesh(net, LO, HI, res, 1.0)
    for lo, hi in ((HI, LO), (LO, LO), ([0, 0, 0], [1, 1, float("nan")]), ([0, 0], [1, 1])):
        with pytest.raises(RuntimeError, match="min_point|max_point"):
            G.density_grid(net, lo, hi, 4)
        with pytest.raises(RuntimeError, match="min_point|max_point"):
            G.extract_mesh(net, lo, hi, 4, 1.0)
    with pytest.raises(RuntimeError, match="time_conditioned_baseline"):
        G.density_grid(tc, LO, HI, 4)
    with pytest.raises(RuntimeError, match="time_conditioned_baseline"):
        G.extract_mesh(tc, LO, HI, 4, 1.0)
    with pytest.raises(RuntimeError, match="no ray bender"):
        G.density_grid(net, LO, HI, 4, latent=torch.zeros(32))
    with pytest.raises(RuntimeError, match="CUDA"):
        G.density_grid(net, LO, HI, 4)                   # a CPU model: there is no CPU path
    with pytest.raises(RuntimeError, match="CUDA"):
        G.marching_cubes(torch.zeros(4, 4, 4), LO, HI, 0.5)
