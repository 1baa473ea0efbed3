"""The density gradient without a GPU: the fp64 restatement against finite differences, the C ABI's argument checks and
workspace sizes, the Python refusals, the writers' normals and the normal images' rounding."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from nonrigid_nerf_b200 import _lib, geometry
from tests import helpers, normals_reference as R


def _models(with_bender=True):
    coarse, _, bender, _ = helpers.build_models(O, 7, "cpu", with_bender=with_bender)
    return coarse


@pytest.mark.parametrize("kind", ["canonical", "bender", "bender_knobs", "tc"])
def test_reference_matches_central_differences(kind):
    torch.manual_seed(0)
    if kind == "tc":
        net = helpers.tc_models(5, "cpu")[0]
    else:
        net = _models(kind != "canonical")
    npar, bp = R.params(net)
    x = torch.rand(64, 3, dtype=torch.float64) * 2 - 1
    z = None if kind == "canonical" else torch.randn(32, dtype=torch.float64) * 0.1
    knobs = dict(cutoff=0.3, scaling=1.5) if kind == "bender_knobs" else {}
    g = R.density_gradient(npar, bp, x, z, tc=kind == "tc", **knobs)
    fd = R.central_differences(npar, bp, x, z, tc=kind == "tc", h=1e-8, **knobs)
    err = (g - fd).norm(dim=1) / fd.norm(dim=1).clamp_min(1e-3)
    # ReLU kinks within h of a point break the finite difference for a few points
    assert float((err < 1e-4).double().mean()) >= 0.9, err


@pytest.mark.parametrize("kind", ["canonical", "bender", "bender_knobs", "tc"])
def test_fixed_mask_chain_equals_autograd_on_its_own_masks(kind):
    """R.fixed_mask_chain, fed the fp64 forward's own masks, encoding, offsets and rigidity, is the autograd gradient;
    rounding_bound covers a rounding of one stage."""
    import torch.nn.functional as F
    torch.manual_seed(1)
    net = helpers.tc_models(5, "cpu")[0] if kind == "tc" else _models(kind != "canonical")
    npar, bp = R.params(net)
    P = 200
    x = torch.rand(P, 3, dtype=torch.float64) * 2 - 1
    z = None if kind == "canonical" else (torch.randn(32, dtype=torch.float64) * 0.3).expand(P, 32)
    knobs = dict(cutoff=0.5, scaling=1.5, removal=0.6) if kind == "bender_knobs" else {}
    masks, un, rig, bent = {}, None, None, x
    if bp is not None and z is not None:
        h, r = torch.cat([x, z], -1), x
        for i in range(4):
            h = F.relu(F.linear(h, bp["net_w"][i], bp["net_b"][i]))
            if i < 2:
                r = F.relu(F.linear(r, bp["rig_w"][i], bp["rig_b"][i]))
                masks[f"Hb{i + 1}"] = torch.cat([h > 0, r > 0], 1)
            else:
                masks[f"Hb{i + 1}"] = h > 0
        out = O.bender_forward(bp, x, z, knobs.get("cutoff"), knobs.get("scaling"))
        un, rig, bent = out["unmasked_offsets"], out["rigidity_mask"][:, 0], out["bent"]
    pe = O.positional_encoding(bent)
    emb = torch.cat([pe, z], -1) if kind == "tc" else pe
    h = emb
    for i in range(8):
        h = F.relu(F.linear(h, npar["pts_w"][i], npar["pts_b"][i]))
        masks[f"H{i + 1}"] = h > 0
        if i == 4:
            h = torch.cat([emb, h], -1)
    E = torch.cat([pe, torch.ones(P, 1, dtype=torch.float64)], 1)
    chain = R.fixed_mask_chain(npar, bp if z is not None else None, masks, E, un, rig, **knobs)
    want = R.density_gradient(npar, bp, x, None if z is None else z[0], tc=kind == "tc", **knobs)
    assert torch.allclose(chain, want, rtol=1e-10, atol=1e-12)
    g, bound, _ = R.rounding_bound(npar, bp if z is not None else None, masks, E, un, rig, **knobs)
    assert torch.equal(g, chain) and bool((bound >= 0).all()) and bool(torch.isfinite(bound).all())
    # the bound is first order: it covers a U16 relative rounding of every stage, here of dY3 alone
    eps = {"Y3": None}
    cap = {}
    R.fixed_mask_chain(npar, bp if z is not None else None, masks, E, un, rig, capture=cap, **knobs)
    eps["Y3"] = cap["Y3"][0] * R.U16
    moved = R.fixed_mask_chain(npar, bp if z is not None else None, masks, E, un, rig, eps=eps, **knobs)
    assert bool(((moved - chain).abs() <= bound * (1 + 1e-9) + 1e-15).all())


def test_normals_reference_convention():
    g = torch.tensor([[0.0, 0.0, -2.0], [0.0, 0.0, 0.0], [float("nan"), 0.0, 1.0]], dtype=torch.float64)
    n = R.normals(g)
    assert n[0].tolist() == [0.0, 0.0, 1.0] and n[1].tolist() == [0.0, 0.0, 0.0] and n[2].tolist() == [0.0, 0.0, 0.0]


def _args():
    a = _lib.NrnDensityGradArgs()
    buf = (C.c_float * 64)()
    a.points, a.n_points, a.points_stride = C.addressof(buf), 4, 3
    a.nerf_packed = 1024
    a.grad = C.addressof(buf)
    return a, buf


def test_abi_argument_checks_return_errors_before_any_cuda_call():
    lib = _lib.load()
    assert lib.nrn_field_density_gradient(None) == -1
    cases = []
    a, keep = _args(); a.points = None; cases.append((a, b"null argument"))
    a, keep2 = _args(); a.n_points = -1; cases.append((a, b"n_points"))
    a, keep3 = _args(); a.points_stride = 2; cases.append((a, b"points_stride"))
    a, keep4 = _args(); a.bender_packed = 2048; cases.append((a, b"latents"))
    a, keep5 = _args(); a.latents = C.addressof(keep5); cases.append((a, b"latents"))
    a, keep6 = _args(); a.tc_w0 = C.addressof(keep6); cases.append((a, b"tc_w0"))
    a, keep7 = _args(); a.bender_packed = 2048; a.latents = C.addressof(keep7); a.latent_stride = 16; cases.append((a, b"latent_stride"))
    a, keep8 = _args(); a.bender_packed = 2048; a.latents = C.addressof(keep8); a.use_scaling, a.scaling = 1, float("inf")
    cases.append((a, b"knob"))
    a, keep9 = _args(); a.nerf_packed = 1028; cases.append((a, b"16-byte aligned"))
    a, keep10 = _args(); a.workspace, a.workspace_bytes = 4096, 16; cases.append((a, b"workspace"))
    a, keep11 = _args(); a.points = C.addressof(keep11) + 2; cases.append((a, b"4-byte aligned"))
    for a, msg in cases:
        assert lib.nrn_field_density_gradient(C.byref(a)) == -1
        assert msg in lib.nrn_last_error(), (msg, lib.nrn_last_error())
    a, keep12 = _args(); a.n_points = 0
    assert lib.nrn_field_density_gradient(C.byref(a)) == 0   # nothing to launch


def test_workspace_size_is_one_chunk():
    lib = _lib.load()
    chunk = lib.nrn_density_gradient_chunk()
    assert chunk == 65536
    per_tile = 40960 + 16384                                  # ReLU mask bits + E
    one = lib.nrn_density_gradient_workspace_bytes(chunk, 0)
    assert one == 512 * per_tile + chunk * 12 + chunk * 4 + 2048
    assert lib.nrn_density_gradient_workspace_bytes(10 ** 9, 0) == one       # bounded: does not grow with P
    assert lib.nrn_density_gradient_workspace_bytes(10 ** 9, 1) == one - 2048 + chunk * 2048
    assert lib.nrn_density_gradient_workspace_bytes(1, 0) == 2 * per_tile + 256 + 256 + 2048
    assert lib.nrn_density_gradient_workspace_bytes(-1, 0) == 0


def test_python_refusals():
    net = _models(True)
    with pytest.raises(RuntimeError, match="CUDA"):
        geometry.density_gradient(net, torch.zeros(4, 3))
    with pytest.raises(RuntimeError, match=r"\[P, 3\]"):
        geometry.density_gradient(net, torch.zeros(4, 2))
    canon = _models(False)
    with pytest.raises(RuntimeError, match="CUDA"):
        geometry.density_gradient(canon, torch.zeros(4, 3), torch.zeros(32))


def _mesh():
    v = torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=torch.float32) * 0.5
    f = torch.tensor([[0, 2, 1], [0, 1, 3]], dtype=torch.int32)
    return geometry.Mesh(v, f, torch.tensor([[255, 0, 0]] * 4, dtype=torch.uint8), None, np.array([0, 4]), np.array([0, 2]))


def test_writers_with_and_without_normals(tmp_path):
    m = _mesh()
    nrm = torch.tensor([[0, 0, 1], [1, 0, 0], [0, 1, 0], [0.6, 0.8, 0]], dtype=torch.float32)
    geometry.write_ply(tmp_path / "a.ply", m)
    geometry.write_ply(tmp_path / "b.ply", m, normals=None)
    assert (tmp_path / "a.ply").read_bytes() == (tmp_path / "b.ply").read_bytes()
    assert b"property float nx" not in (tmp_path / "a.ply").read_bytes()
    geometry.write_ply(tmp_path / "n.ply", m, normals=nrm)
    data = (tmp_path / "n.ply").read_bytes()
    head, body = data.split(b"end_header\n")
    assert b"property float nx\nproperty float ny\nproperty float nz\nproperty uchar red" in head
    vert = np.frombuffer(body[:4 * 27], dtype=[("xyz", "<f4", 3), ("n", "<f4", 3), ("c", "u1", 3)])
    assert np.array_equal(vert["n"], nrm.numpy()) and np.array_equal(vert["xyz"], m.vertices.numpy())
    geometry.write_obj(tmp_path / "a.obj", m)
    geometry.write_obj(tmp_path / "b.obj", m, normals=None)
    assert (tmp_path / "a.obj").read_bytes() == (tmp_path / "b.obj").read_bytes()
    geometry.write_obj(tmp_path / "n.obj", m, normals=nrm)
    lines = (tmp_path / "n.obj").read_text().splitlines()
    vn = np.array([[float(t) for t in l.split()[1:]] for l in lines if l.startswith("vn ")], dtype=np.float32)
    assert np.array_equal(vn, nrm.numpy())
    assert [l for l in lines if l.startswith("f ")] == ["f 1//1 3//3 2//2", "f 1//1 2//2 4//4"]
    with pytest.raises(RuntimeError, match="normals must be"):
        geometry.write_obj(tmp_path / "x.obj", m, normals=nrm[:3])
