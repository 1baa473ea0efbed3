"""GPU tests of the inverse ray bender (geometry.deform_points / deform_mesh, csrc/deform.cu) against the fp64 restatement
tests/deform_reference.py: exact identities bit for bit, accuracy on benders with offsets of 0.01 and 0.1, the round trip
through the production field kernel, the test-time knobs, non-convergence and non-finite inputs, shapes, determinism,
CUDA-graph replay, an output past 2^31 bytes, and meshes."""
import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import deform_reference as R
from tests import helpers

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
LO, HI = np.array([-1.2, -1.0, -1.4]), np.array([1.1, 1.0, 0.6])   # about the example sequence's volume
TOL = 1e-5


def _bender(bp=None, cutoff=None, scaling=None):
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    embed_fn, ch = H.get_embedder(10, 0)
    b = H.ray_bending(ch, 32, "simple_neural", embed_fn)
    if bp is not None:
        helpers.load_bender_module(b, bp)
    b.rigidity_test_time_cutoff, b.test_time_scaling = cutoff, scaling
    return b.to(DEV)


def _points(seed, n):
    return torch.from_numpy(np.random.RandomState(seed).uniform(LO, HI, size=(n, 3)).astype(np.float32)).to(DEV)


def _latents(seed, f, std=0.1):
    return torch.from_numpy((np.random.RandomState(seed).randn(f, 32) * std).astype(np.float32)).to(DEV)


def _deform(b, c, z, **kw):
    from nonrigid_nerf_b200 import geometry as G
    d = G.deform_points(b, c, z, **kw)
    torch.cuda.synchronize()
    return d


def _near(res64):
    """Points whose fp64 residual lies within a factor of 2 of tol, either way: fp32 and fp64 may judge them differently."""
    return (res64 >= TOL / 2) & (res64 <= 2 * TOL)


KINK = 1e-6   # fp32 and fp64 iterates differ by ~1e-7, so their ReLU pre-activations may differ in sign within this margin


def _same_steps(b, bp64, c, z, steps, cutoff=None, scaling=None):
    """The converged sets after 1, 2, ... Newton steps equal the fp64 restatement's outside the near band, and away from
    ReLU kinks (a point whose J was taken within KINK of one may get the other one-sided derivative in fp32): the kernel
    takes the restatement's steps, which a wrong Jacobian (or the fixed-point step) would not.  Returns per step the
    converged counts (kernel, fp64) and the number of points excluded at kinks."""
    counts = []
    for k in steps:
        dk = _deform(b, c, z, iterations=k, tol=TOL)
        _, resk, convk, _, _, mk = R.deform(bp64, c, z, k, TOL, cutoff, scaling, with_margin=True)
        skip = _near(resk) | (mk <= KINK)
        assert torch.equal(dk.converged & ~skip, convk & ~skip), (k, int(dk.converged.sum()), int(convk.sum()))
        counts.append((int(dk.converged.sum()), int(convk.sum()), int((mk <= KINK).sum())))
    return counts


def _res64(bp64, x, c, z, cutoff=None, scaling=None):
    """|b64(x) - c| [F, P] of fp32 results x [F, P, 3]."""
    return torch.stack([(R.bend(bp64, x[f].double(), z[f].double().expand(c.shape[0], 32), cutoff, scaling)[0] - c.double()).norm(dim=1)
                        for f in range(z.shape[0])])


# ---- exact identities -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knob", ["fresh", "scaling0", "cutoff1"])
def test_identities_bit_for_bit(knob):
    c, z = _points(1, 1000), _latents(2, 3)
    if knob == "fresh":
        b = _bender()                       # zero last layers: straight rays
    elif knob == "scaling0":
        b = _bender(O.make_bender_params(3, offset_std=0.1), scaling=0.0)
    else:
        b = _bender(O.make_bender_params(3, offset_std=0.1), cutoff=1.0)
    d = _deform(b, c, z)
    assert torch.equal(d.points, c.expand(3, -1, -1))
    assert torch.equal(d.residual, torch.zeros_like(d.residual)) and bool(d.converged.all())
    if knob == "fresh":
        assert torch.equal(d.rigidity, torch.full_like(d.rigidity, 0.5))
    if knob == "cutoff1":
        assert torch.equal(d.rigidity, torch.zeros_like(d.rigidity))


@pytest.mark.parametrize("scaling", [None, 1.7])
def test_constant_rigidity_offset_of_the_latent_only(scaling):
    bp = O.make_bender_params(4, offset_std=0.1)
    bp["net_w"][0][:, :3] = 0.0          # o depends on z only
    for w in bp["rig_w"][:2]:
        w.zero_()                        # r = (tanh(rig_b2) + 1) / 2, a constant
    bp["rig_b"][2].fill_(0.3)
    b = _bender(bp, scaling=scaling)
    c, z = _points(5, 2000), _latents(6, 4)
    d = _deform(b, c, z)
    bp64 = R.params64(bp, DEV)
    s = 1.0 if scaling is None else scaling
    for f in range(4):
        _, r, m = R.bend(bp64, c.double(), z[f].double().expand(2000, 32), None, scaling)
        x64 = c.double() - m
        # fp32 rounding of c - m, plus the fp32-accuracy evaluation of o (its 64-term sums carry ~2^-22 of their terms,
        # measured 2.5e-8 absolute on an H100)
        err = (d.points[f].double() - x64).abs()
        assert bool((err <= 2.0 ** -23 * c.double().abs() + 1e-7).all()), (f, float(err.max()))
        torch.testing.assert_close(d.rigidity[f].double(), r, rtol=1e-6, atol=0)
    assert bool(d.converged.all()) and float(d.residual.max()) <= 1e-6 * s


# ---- accuracy against fp64 ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset_std", [0.01, 0.1])
def test_accuracy_against_fp64(offset_std):
    bp = O.make_bender_params(7, offset_std=offset_std)
    b = _bender(bp)
    c, z = _points(8, 100_000), _latents(9, 8)
    d = _deform(b, c, z, iterations=8, tol=TOL)
    bp64 = R.params64(bp, DEV)
    x64, res64, conv64, rig64, its = R.deform(bp64, c, z, 8, TOL)
    near = _near(res64)
    assert torch.equal(d.converged & ~near, conv64 & ~near)
    steps = _same_steps(b, bp64, c, z, (1, 2, 3))
    r64 = _res64(bp64, d.points, c, z)
    assert float(r64[d.converged].max()) <= 2 * TOL
    err = (d.points.double() - x64).norm(dim=2) / (1 + c.double().norm(dim=1))
    assert float(err[d.converged & conv64].max()) <= 1e-5
    torch.testing.assert_close(d.rigidity.double()[d.converged], rig64[d.converged], rtol=0, atol=1e-5)
    hist = torch.bincount(its[its >= 0].flatten().cpu(), minlength=9)
    print(f"offset_std {offset_std}: converged {int(d.converged.sum())}/{d.converged.numel()} (fp64 {int(conv64.sum())}), "
          f"fp64 steps to converge {hist.tolist()}, max |x - x64| / (1 + |c|) {float(err[d.converged & conv64].max()):.3e}, "
          f"max fp64 residual {float(r64[d.converged].max()):.3e}, converged after 1 / 2 / 3 steps (kernel, fp64, at kinks) {steps}")


def test_round_trip_through_the_field_kernel():
    from nonrigid_nerf_b200 import ops
    coarse, _, bender, (cp, fp, bp) = helpers.build_models(O, 11, DEV)
    c, z = _points(12, 20_000), _latents(13, 3)
    d = _deform(bender, c, z)
    assert bool(d.converged.all())
    pack_n, pack_b = ops.pack_nerf(coarse), ops.pack_bender(bender)
    for f in range(3):
        _, det = ops.field_forward_points(d.points[f].contiguous(), z[f].expand(c.shape[0], 32).contiguous(), pack_n, pack_b, 5,
                                          want_details=True)
        torch.testing.assert_close(det["input_pts"].view(-1, 3), c, rtol=0, atol=1e-4)
        torch.testing.assert_close(det["rigidity_mask"].view(-1), d.rigidity[f], rtol=0, atol=1e-3)


@pytest.mark.parametrize("cutoff,scaling", [(0.5, None), (None, 0.4), (0.47, 2.0)])
def test_knobs_against_fp64(cutoff, scaling):
    from nonrigid_nerf_b200 import ops
    bp = O.make_bender_params(14, offset_std=0.1)
    b = _bender(bp, cutoff, scaling)
    c, z = _points(15, 20_000), _latents(16, 2)
    d = _deform(b, c, z)
    bp64 = R.params64(bp, DEV)
    x64, res64, conv64, rig64, _ = R.deform(bp64, c, z, 8, TOL, cutoff, scaling)
    # with a cutoff b jumps where r crosses it: points whose preimage would straddle that surface have none, and neither
    # solver converges there; the converged sets agree, after the full schedule and after 1 and 2 steps
    ok = d.converged & conv64
    near = _near(res64)
    assert torch.equal(d.converged & ~near, conv64 & ~near)
    steps = _same_steps(b, bp64, c, z, (1, 2), cutoff, scaling)
    print(f"cutoff {cutoff} scaling {scaling}: converged {float(d.converged.float().mean()):.4f} (fp64 "
          f"{float(conv64.float().mean()):.4f}), after 1 / 2 steps (kernel, fp64, at kinks) {steps}")
    err = (d.points.double() - x64).norm(dim=2) / (1 + c.double().norm(dim=1))
    assert float(err[ok].max()) <= 1e-5
    assert float(_res64(bp64, d.points, c, z, cutoff, scaling)[d.converged].max()) <= 2 * TOL
    # rigidity = point mode's rigidity_mask at the result (fp16 tolerance of the field kernel)
    _, det = ops.field_forward_points(d.points[0].contiguous(), z[0].expand(c.shape[0], 32).contiguous(),
                                      ops.pack_nerf(helpers.build_models(O, 1, DEV, False)[0]), ops.pack_bender(b), 5,
                                      cutoff, scaling, want_details=True)
    mask = det["rigidity_mask"].view(-1)
    away = torch.ones_like(mask, dtype=torch.bool)
    if cutoff is not None:   # r within the field kernel's fp16 tolerance of the cutoff may be cut by one and not the other
        rig = d.rigidity[0]
        away = ~(((mask == 0) & ((rig - cutoff).abs() <= 2e-3)) | ((rig == 0) & ((mask - cutoff).abs() <= 2e-3)))
    torch.testing.assert_close(mask[away], d.rigidity[0][away], rtol=0, atol=1e-3)


# ---- non-convergence and non-finite inputs ------------------------------------------------------------------------------
def test_folding_field_reports_non_convergence():
    bp = O.make_bender_params(17, offset_std=1.0)
    b = _bender(bp)
    c, z = _points(18, 50_000), _latents(19, 2)
    d = _deform(b, c, z, iterations=4)
    bad = ~d.converged
    assert int(bad.sum()) > 0
    assert bool(torch.isfinite(d.residual[bad]).all()) and bool((d.residual[bad] > TOL).all())
    assert bool(torch.isfinite(d.points).all())


def test_non_finite_points_and_latents():
    bp = O.make_bender_params(20, offset_std=0.1)
    b = _bender(bp)
    c, z = _points(21, 300), _latents(22, 3)
    c[5, 0], c[77, 2], c[200, 1] = float("nan"), float("inf"), float("-inf")
    z[1, 9] = float("nan")
    z[2, 31] = float("inf")
    d = _deform(b, c, z)
    badp = torch.zeros(300, dtype=torch.bool, device=DEV)
    badp[[5, 77, 200]] = True
    for f in range(3):
        bad = badp if f == 0 else torch.ones_like(badp)
        assert bool(torch.isnan(d.points[f][bad]).all()) and bool(torch.isnan(d.residual[f][bad]).all())
        assert not bool(d.converged[f][bad].any()) and bool(torch.isnan(d.rigidity[f][bad]).all())
    assert bool(d.converged[0][~badp].all())


# ---- shapes and determinism ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 127, 128, 129])
def test_frames_alone_equal_frames_in_a_batch(P):
    bp = O.make_bender_params(23, offset_std=0.1)
    b = _bender(bp)
    c = _points(24, P)
    for F in (1, 5, 86):
        z = _latents(25 + F, F)
        d = _deform(b, c, z)
        assert d.points.shape == (F, P, 3) and d.residual.shape == (F, P) and d.converged.dtype == torch.bool
        for f in sorted({0, F // 2, F - 1}):
            one = _deform(b, c, z[f])
            assert one.points.shape == (P, 3)
            for a, e in zip(one, d):
                assert torch.equal(a, e[f])
    x64 = R.deform(R.params64(bp, DEV), c, z[:2], 8, TOL)[0]
    assert float((d.points[:2].double() - x64).abs().max()) <= 1e-4


def test_reruns_and_graph_replay_are_bit_identical():
    from nonrigid_nerf_b200 import geometry as G
    b = _bender(O.make_bender_params(26, offset_std=0.1))
    c, z = _points(27, 30_000), _latents(28, 5)
    ref = _deform(b, c, z)
    again = _deform(b, c, z)
    for a, e in zip(again, ref):
        assert torch.equal(a, e)
    G.deform_points(b, c, z)   # pack cached before the capture
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = G.deform_points(b, c, z)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for a, e in zip(out, ref):
            assert torch.equal(a, e)


def test_output_past_2_to_the_31_bytes():
    bp = O.make_bender_params(29, offset_std=0.1)
    b = _bender(bp)
    P, F = 2_100_000, 86
    c, z = _points(30, P), _latents(31, F)
    d = _deform(b, c, z)
    assert d.points.numel() * 4 > 2 ** 31
    rows = torch.tensor([0, 1, 777_777, P - 129, P - 1], device=DEV)
    frames = [0, 41, 85]
    x64, _, conv64, _, _ = R.deform(R.params64(bp, DEV), c[rows], z[frames], 8, TOL)
    got = d.points[frames][:, rows]
    assert torch.equal(d.converged[frames][:, rows], conv64)
    assert float(((got.double() - x64).norm(dim=2) / (1 + c[rows].double().norm(dim=1))).max()) <= 1e-5
    print(f"output {d.points.numel() * 4 / 2 ** 30:.2f} GiB, converged {float(d.converged.float().mean()):.6f}")


# ---- meshes -------------------------------------------------------------------------------------------------------------
def test_deform_mesh_of_a_canonical_sphere():
    from nonrigid_nerf_b200 import geometry as G
    n = 48
    lo, hi = [-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]
    ax = torch.linspace(-1.0, 1.0, n, device=DEV)
    zz, yy, xx = torch.meshgrid(ax, ax, ax, indexing="ij")
    sigma = (0.7 - (xx * xx + yy * yy + zz * zz).sqrt()).contiguous()
    mesh = G.marching_cubes(sigma, lo, hi, 0.0)
    V = mesh.vertices.shape[0]
    col = torch.randint(0, 255, (V, 3), dtype=torch.uint8, device=DEV)
    mesh = mesh._replace(colors=col)
    bp = O.make_bender_params(32, offset_std=0.1)
    b = _bender(bp)
    z = _latents(33, 1)[0]
    dm = G.deform_mesh(b, mesh, z)
    m = dm.mesh
    assert torch.equal(m.faces, mesh.faces) and torch.equal(m.colors, mesh.colors)
    assert np.array_equal(m.vertex_offsets, mesh.vertex_offsets) and np.array_equal(m.face_offsets, mesh.face_offsets)
    d = _deform(b, mesh.vertices, z)
    assert torch.equal(m.vertices, d.points) and torch.equal(m.rigidity, d.rigidity)
    assert torch.equal(dm.residual, d.residual) and torch.equal(dm.converged, d.converged)
    assert bool(dm.converged.all())
    bp64 = R.params64(bp, DEV)
    r64 = _res64(bp64, m.vertices[None], mesh.vertices, z[None])
    assert float(r64.max()) <= 2 * TOL
    x64 = R.deform(bp64, mesh.vertices, z[None], 8, TOL)[0][0]
    assert float(((m.vertices.double() - x64).norm(dim=1) / (1 + mesh.vertices.double().norm(dim=1))).max()) <= 1e-5


def test_timing_kind():
    from nonrigid_nerf_b200 import _lib
    kinds = (_lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + _lib.DET_KERNEL_KINDS
             + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + _lib.MESH_KERNEL_KINDS
             + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS + _lib.OCCUPANCY_KERNEL_KINDS + _lib.TERMINATION_KERNEL_KINDS
             + _lib.DEFORM_KERNEL_KINDS)
    assert kinds.index("deform") == 41
    b = _bender(O.make_bender_params(34, offset_std=0.1))
    c, z = _points(35, 5000), _latents(36, 2)
    _deform(b, c, z)                   # pack outside the timed session
    _lib.timing_enable(True)
    try:
        _deform(b, c, z)
    finally:
        _lib.timing_enable(False)
    t = _lib.timing_read(kinds)
    assert t["deform"][1] == 1 and t["deform"][0] > 0
    assert all(n == 0 for k, (_, n) in t.items() if k != "deform")
