"""Every forward variant of the fused field kernel tied bit for bit to the training kernel, whose stages
tests/test_stage_parity_gpu.py checks against fp64 references.

The inference instantiations (render(), chunked rendering), the object-removal switch, point mode (NeRF.forward(x)) and a
batch's position inside the tile grid change only what a kernel stores or where a row sits, never its arithmetic.  So each
is compared with the verified kernel bit for bit, through the C ABI with outputs filled with NaN beforehand:

  * inference vs training kernel: raw and the per-point details, with and without a bender, with cut-off and scaling,
    the time-conditioned baseline (TC) with explicit latent rows and with latent stride 0, out_ch 4 and 5;
  * use_removal: channel 3 exactly 0 where rigidity >= the threshold (one of the run's own values), all else unchanged;
  * point mode vs ray mode with rays_o = x, rays_d = 0, z > 0, S = 1 (the ray path's point o + 0 * z is exactly x),
    points_stride 3 and 95 (the latent read in place from columns 63:95, as run_network passes it);
  * a subset of rays run on its own vs inside a larger batch, where its rows sit at other tiles and row offsets.
"""
import copy

import pytest
import torch

from tests import test_stage_parity_gpu as SP
from tests.parity import DEV

pytestmark = pytest.mark.gpu
N, S = 37, 29                 # 1073 points: 9 tiles, the last one ragged, rays straddle tiles
OUTPUTS = ("raw", "init", "bent", "un", "masked", "rig")


def case(mode, n, s, **kw):
    """mode: bender, nobender, tc (explicit latent rows) or tc_stride0 (one latent row for every ray)."""
    if mode.startswith("tc"):
        return SP.Case(n, s, bender=False, tc=True, lat_stride0=mode == "tc_stride0", **kw)
    return SP.Case(n, s, bender=mode == "bender", **kw)


def assert_same(a, b, what, rows=slice(None)):
    """Every output a holds equals b's (rows `rows` of b) bit for bit; a NaN (a slot no kernel wrote) never does."""
    for k in OUTPUTS:
        if k in a:
            got, ref = a[k], b[k][rows]
            assert torch.equal(got, ref), f"{what}: {k} differs in {int((got != ref).sum())} of {got.numel()} elements"


VARIANTS = {
    "bender": dict(mode="bender"),
    "nobender": dict(mode="nobender"),
    "bender_cutoff_scaling": dict(mode="bender", cutoff="median", scaling=0.7),
    "tc": dict(mode="tc"),
    "tc_stride0": dict(mode="tc_stride0"),
    "bender_out4": dict(mode="bender", out_ch=4),
    "nobender_out4": dict(mode="nobender", out_ch=4),
    "tc_out4": dict(mode="tc", out_ch=4),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_inference_kernel_matches_the_training_kernel(name):
    kw = dict(VARIANTS[name])
    mode = kw.pop("mode")
    if kw.get("cutoff") == "median":
        # a cut-off that removes about half of the points
        kw["cutoff"] = float(SP.run_forward(case(mode, N, S))["rig"].median())
    cs = case(mode, N, S, **kw)
    assert_same(SP.run_forward(cs, train=False), SP.run_forward(cs), f"{name}: inference vs training")


def test_object_removal_zeroes_channel_3_exactly_from_the_threshold_up():
    cs = case("bender", N, S)
    ref = SP.run_forward(cs, train=False)
    rig = ref["rig"]
    thr = float(rig.median())                  # one of the run's own rigidity values: the >= edge is hit
    cut = rig >= thr
    assert bool((rig == thr).any()) and bool(cut.any()) and bool((~cut).any())
    got = SP.run_forward(cs, train=False, removal=thr)
    exp = dict(ref)
    exp["raw"] = ref["raw"].clone()
    exp["raw"][cut, 3] = 0.0
    assert_same(got, exp, "use_removal")
    assert bool((got["raw"][cut, 3] == 0).all()) and bool((got["raw"][~cut, 3] != 0).all())


@pytest.mark.parametrize("stride", [3, 95])
@pytest.mark.parametrize("mode", ["bender", "nobender", "tc"])
def test_point_mode_matches_ray_mode(mode, stride):
    cs = case(mode, 300, 1)
    assert bool((cs.z > 0).all())
    x = cs.rays[:, :3] + cs.rays[:, 3:6] * cs.z         # distinct points along the rays
    cs.rays[:, :3], cs.rays[:, 3:6] = x, 0.0            # rays_o = x, rays_d = 0: the ray path's point is exactly x
    pts = torch.zeros(cs.n, stride, device=DEV)
    pts[:, :3] = x
    if stride == 95:
        pts[:, 63:] = cs.lat
        cs.lat = pts[:, 63:]                            # [xyz | PE columns | latent], the latent read in place
    assert_same(SP.run_forward(cs, train=False, points=pts), SP.run_forward(cs, train=False), f"{mode} stride {stride}: point mode vs ray mode")


@pytest.mark.parametrize("mode", ["bender", "nobender", "tc"])
def test_a_ray_subset_computes_what_it_computes_inside_a_larger_batch(mode):
    cs = case(mode, 1031, 7)
    full = SP.run_forward(cs, train=False)
    for first, last in ((100, cs.n), (0, 1)):
        sub = copy.copy(cs)
        sub.rays, sub.z, sub.lat = (t[first:last].contiguous() for t in (cs.rays, cs.z, cs.lat))
        sub.n, sub.P = last - first, (last - first) * cs.s
        assert_same(SP.run_forward(sub, train=False), full, f"{mode} rays[{first}:{last}] alone vs in the batch",
                    slice(first * cs.s, last * cs.s))
