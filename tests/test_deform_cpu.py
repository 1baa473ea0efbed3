"""CPU tests of the inverse ray bender: the fp64 restatement (tests/deform_reference.py) against a direct fp64 check of
b(x) = c and its Jacobian against finite differences, the argument checks of nrn_deform_points (on host pointers, before
any CUDA call) and the refusals of geometry.deform_points / deform_mesh."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import deform_reference as R

LO, HI = np.array([-1.2, -1.0, -1.4]), np.array([1.1, 1.0, 0.6])   # about the example sequence's volume


def _points(seed, n):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.uniform(LO, HI, size=(n, 3)))


def _latents(seed, f):
    return torch.from_numpy(np.random.RandomState(seed).randn(f, 32) * 0.1)


@pytest.mark.parametrize("offset_std", [0.01, 0.05])
def test_restatement_solves_the_bend(offset_std):
    bp = R.params64(O.make_bender_params(3, offset_std=offset_std))
    c, z = _points(1, 400), _latents(2, 3)
    x, res, conv, rig, its = R.deform(bp, c, z, iterations=20, tol=0.0)
    for f in range(3):
        b, r, _ = R.bend(bp, x[f], z[f].expand(400, 32))
        assert float((b - c).norm(dim=1).max()) <= 1e-12
        torch.testing.assert_close(r, rig[f], rtol=0, atol=0)
    assert torch.equal(res <= 1e-12, torch.ones_like(conv))
    # with a tolerance every point freezes after a few steps, and its residual is within it
    x8, res8, conv8, _, its8 = R.deform(bp, c, z, iterations=8, tol=1e-5)
    assert bool(conv8.all()) and float(res8.max()) <= 1e-5 and int(its8.max()) <= 4
    assert float((x8 - x).abs().max()) <= 1e-4


@pytest.mark.parametrize("knobs", [(None, None), (0.5, None), (None, 0.3), (0.45, 1.7)])
def test_restatement_jacobian_against_finite_differences(knobs):
    bp = R.params64(O.make_bender_params(5, offset_std=0.1))
    x, z = _points(6, 64), _latents(7, 1).expand(64, 32)
    J = R.jacobian(bp, x, z, *knobs)
    h = 1e-6
    for a in range(3):
        e = torch.zeros(3, dtype=torch.float64)
        e[a] = h
        fd = (R.bend(bp, x + e, z, *knobs)[0] - R.bend(bp, x - e, z, *knobs)[0]) / (2 * h)
        # points within h of a ReLU kink or of the cutoff have a one-sided derivative; there are none at this seed
        torch.testing.assert_close(J[:, :, a], fd, rtol=1e-6, atol=1e-7)


def test_restatement_fallback_and_non_finite():
    bp = R.params64(O.make_bender_params(3))
    c = _points(1, 4)
    c[1, 2] = float("nan")
    z = _latents(2, 2)
    z[1, 5] = float("inf")
    x, res, conv, rig, _ = R.deform(bp, c, z, iterations=4, tol=1e-5)
    assert torch.isnan(x[0, 1]).all() and torch.isnan(res[0, 1]) and not conv[0, 1] and torch.isnan(rig[0, 1])
    assert torch.isnan(x[1]).all() and torch.isnan(res[1]).all() and not conv[1].any()
    assert conv[0, [0, 2, 3]].all()
    # a singular J takes the fixed-point step
    J = torch.zeros(2, 3, 3, dtype=torch.float64)
    J[1] = torch.eye(3, dtype=torch.float64) * 2
    g = torch.tensor([[1.0, 2.0, 3.0], [1.0, 2.0, 3.0]], dtype=torch.float64)
    st = R.newton_step(J, g)
    assert torch.equal(st[0], g[0]) and torch.equal(st[1], g[1] / 2)


# ---- the C entry point's argument checks -------------------------------------------------------------------------------
def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


def _args(L, bufs):
    a = L.NrnDeformArgs()
    a.points, a.n_points = C.addressof(bufs["pts"]), 4
    a.latents, a.n_latents, a.latent_stride = C.addressof(bufs["lat"]), 2, 32
    a.bender_packed = C.addressof(bufs["pack"])
    a.use_cutoff, a.rigidity_cutoff, a.use_scaling, a.scaling = 0, 0.0, 0, 1.0
    a.iterations, a.tol = 8, 1e-5
    a.out, a.residual, a.converged, a.rigidity = (C.addressof(bufs[k]) for k in ("out", "res", "conv", "rig"))
    return a


def _bufs():
    return {"pts": (C.c_float * 12)(), "lat": (C.c_float * 64)(), "pack": (C.c_longlong * 4)(), "out": (C.c_float * 24)(),
            "res": (C.c_float * 8)(), "conv": (C.c_uint8 * 8)(), "rig": (C.c_float * 8)()}


_BAD = {
    "null points": lambda a: setattr(a, "points", None),
    "null latents": lambda a: setattr(a, "latents", None),
    "null bender": lambda a: setattr(a, "bender_packed", None),
    "null out": lambda a: setattr(a, "out", None),
    "negative points": lambda a: setattr(a, "n_points", -1),
    "negative latents": lambda a: setattr(a, "n_latents", -1),
    "short stride": lambda a: setattr(a, "latent_stride", 31),
    "zero iterations": lambda a: setattr(a, "iterations", 0),
    "65 iterations": lambda a: setattr(a, "iterations", 65),
    "nan tol": lambda a: setattr(a, "tol", float("nan")),
    "inf tol": lambda a: setattr(a, "tol", float("inf")),
    "negative tol": lambda a: setattr(a, "tol", -1e-6),
    "inf scaling": lambda a: (setattr(a, "use_scaling", 1), setattr(a, "scaling", float("inf"))),
    "nan scaling": lambda a: (setattr(a, "use_scaling", 1), setattr(a, "scaling", float("nan"))),
    "nan cutoff": lambda a: (setattr(a, "use_cutoff", 1), setattr(a, "rigidity_cutoff", float("nan"))),
    "misaligned points": lambda a: setattr(a, "points", a.points + 2),
    "misaligned out": lambda a: setattr(a, "out", a.out + 1),
    "misaligned residual": lambda a: setattr(a, "residual", a.residual + 2),
    "misaligned rigidity": lambda a: setattr(a, "rigidity", a.rigidity + 3),
    "misaligned bender": lambda a: setattr(a, "bender_packed", a.bender_packed + 4),
}


@pytest.mark.parametrize("case", sorted(_BAD))
def test_c_argument_checks(case):
    L, lib = _lib()
    bufs = _bufs()
    a = _args(L, bufs)
    _BAD[case](a)
    assert lib.nrn_deform_points(C.byref(a)) == -1
    assert lib.nrn_last_error().decode().startswith("nrn_deform_points")
    assert lib.nrn_deform_points(None) == -1


@pytest.mark.parametrize("empty", ["n_points", "n_latents"])
def test_c_empty_call_launches_nothing(empty):
    L, lib = _lib()
    bufs = _bufs()
    a = _args(L, bufs)
    setattr(a, empty, 0)
    a.use_scaling, a.scaling = 1, 0.0      # knobs that are finite are accepted
    a.use_cutoff, a.rigidity_cutoff = 1, 2.0
    assert lib.nrn_deform_points(C.byref(a)) == 0


def test_abi_and_timing_kind():
    L, lib = _lib()
    assert lib.nrn_abi_version() == 4
    assert L.DEFORM_KERNEL_KINDS == ("deform",)


# ---- the Python refusals -----------------------------------------------------------------------------------------------
def _bender():
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    embed_fn, ch = H.get_embedder(10, 0)
    return H.ray_bending(ch, 32, "simple_neural", embed_fn)


@pytest.mark.parametrize("case,match", [
    ("none", "ray_bending module"), ("linear", "ray_bending module"), ("cpu", "CUDA tensors"), ("lat31", "latents must be"),
    ("lat3d", "latents must be"), ("pts4", "points must be"), ("it0", "iterations"), ("it65", "iterations"),
    ("itbool", "iterations"), ("itfloat", "iterations"), ("tolnan", "tol"), ("tolneg", "tol"), ("tolinf", "tol"),
    ("notensor", "must be tensors"),
])
def test_deform_points_refuses(case, match):
    from nonrigid_nerf_b200 import geometry as G
    b = _bender()
    pts, lat = torch.zeros(5, 3), torch.zeros(32)
    kw = {}
    if case == "none":
        b = None
    elif case == "linear":
        b = torch.nn.Linear(3, 3)
    elif case == "lat31":
        lat = torch.zeros(2, 31)
    elif case == "lat3d":
        lat = torch.zeros(1, 2, 32)
    elif case == "pts4":
        pts = torch.zeros(5, 4)
    elif case == "notensor":
        pts = [[0.0, 0.0, 0.0]]
    elif case.startswith("it"):
        kw["iterations"] = {"it0": 0, "it65": 65, "itbool": True, "itfloat": 4.0}[case]
    elif case.startswith("tol"):
        kw["tol"] = {"tolnan": float("nan"), "tolneg": -1.0, "tolinf": float("inf")}[case]
    with pytest.raises(RuntimeError, match=match):
        G.deform_points(b, pts, lat, **kw)


def test_deform_mesh_refuses():
    from nonrigid_nerf_b200 import geometry as G
    mesh = G.Mesh(torch.zeros(3, 3), torch.zeros(1, 3, dtype=torch.int32), None, None, np.zeros(2, np.int64), np.zeros(1, np.int64))
    with pytest.raises(RuntimeError, match="one latent code"):
        G.deform_mesh(_bender(), mesh, torch.zeros(2, 32))
    with pytest.raises(RuntimeError, match="one latent code"):
        G.deform_mesh(_bender(), mesh, None)
    with pytest.raises(RuntimeError, match="ray_bending module"):
        G.deform_mesh(None, mesh, torch.zeros(32))
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        G.deform_mesh(_bender(), mesh, torch.zeros(32))


def test_restatement_kink_margin():
    bp = R.params64(O.make_bender_params(3, offset_std=0.1))
    x, z = _points(40, 50), _latents(41, 1).expand(50, 32)
    m = R.kink_margin(bp, x, z)
    assert bool((m > 0).all()) and bool((m < 1).all())
    # moving a point onto the kink of one first-layer unit gives margin 0 there
    w, b0 = bp["net_w"][0][0], bp["net_b"][0][0]
    pre = x @ w[:3] + z @ w[3:] + b0
    x0 = x - (pre / (w[:3] @ w[:3])).unsqueeze(1) * w[:3]
    assert float(R.kink_margin(bp, x0, z).max()) <= 1e-12
    # one step: J is taken once, at x_0 = c - s r~ o (tol 0: no point is frozen)
    _, _, _, _, _, mg = R.deform(bp, x, z[:1], 1, 0.0, with_margin=True)
    x_0 = x - R.bend(bp, x, z)[2]
    torch.testing.assert_close(mg[0], R.kink_margin(bp, x_0, z), rtol=0, atol=0)
