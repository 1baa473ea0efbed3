"""The launch sequence of one call of each render pass that runs the trunk on some samples only: the launches the kernel
timing records per kind, with and without a ray bender (the deformed pass, which needs one: with and without details)."""
import numpy as np
import pytest
import torch

from tests import occupancy_reference as OR
from tests.test_baked_gpu import _depths, _far_grid, _models, _rays

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N, S = 300, 40   # S not a multiple of the termination segment: a ragged last round


def _kinds():
    from nonrigid_nerf_b200 import _lib as L
    kinds = tuple(L.KERNEL_KINDS + L.TC_KERNEL_KINDS + L.VIEW_KERNEL_KINDS + L.VIEW_TRAIN_KERNEL_KINDS + L.DET_KERNEL_KINDS
                  + L.HELD_OUT_KERNEL_KINDS + L.EVAL_KERNEL_KINDS + L.FRAME_IMAGE_KERNEL_KINDS + L.MESH_KERNEL_KINDS
                  + L.LPIPS_KERNEL_KINDS + L.MATCH_KERNEL_KINDS + L.OCCUPANCY_KERNEL_KINDS + L.TERMINATION_KERNEL_KINDS
                  + L.DEFORM_KERNEL_KINDS + L.NORMAL_KERNEL_KINDS + L.LPIPS_MAP_KERNEL_KINDS + L.BAKED_KERNEL_KINDS
                  + L.DEFORMATION_KERNEL_KINDS)
    assert len(kinds) == 58
    return kinds


def _launches(call):
    """{kind: launches} of one call(), after an untimed one that packs the weights."""
    from nonrigid_nerf_b200 import _lib
    with torch.no_grad():
        call()
        torch.cuda.synchronize()
        _lib.timing_enable(True)
        try:
            call()
            torch.cuda.synchronize()
        finally:
            _lib.timing_enable(False)
    return {k: c for k, (_, c) in _lib.timing_read(_kinds()).items() if c}


def _occupancy_grid():
    from nonrigid_nerf_b200 import geometry as G
    occ = np.random.RandomState(7).rand(8, 8, 8) < 0.5
    return G.OccupancyGrid(torch.from_numpy(OR.pack(occ)).to(DEV), np.float32([-1.0] * 3), np.float32([1.0] * 3), (8, 8, 8))


def _inputs(bender):
    coarse, _, b = _models(bender)
    rays, lat = _rays(930, N)
    return coarse, b, rays, _depths(rays, S, 930), (lat if bender else None)


@pytest.mark.parametrize("bender", [True, False])
def test_occupancy_launches(bender):
    from nonrigid_nerf_b200 import autograd as A
    net, _, rays, z, lat = _inputs(bender)
    grid = _occupancy_grid()
    got = _launches(lambda: A.field_occupancy(net, rays, z, lat, True, grid))
    want = {"occupancy_compact": 1, "occupancy_field": 1, "occupancy_scatter": 1}
    if bender:
        want["occupancy_bend"] = 1
    assert got == want


@pytest.mark.parametrize("with_grid", [True, False])
@pytest.mark.parametrize("bender", [True, False])
def test_termination_launches(bender, with_grid):
    from nonrigid_nerf_b200 import _lib, autograd as A
    seg = _lib.load().nrn_termination_segment()
    assert S % seg
    R = -(-S // seg)
    net, _, rays, z, lat = _inputs(bender)
    grid = _occupancy_grid() if with_grid else None
    got = _launches(lambda: A.field_terminate(net, rays, z, lat, True, 1e-3, grid))
    want = {"termination_compact": R, "termination_field": R, "termination_scatter": R + 1, "termination_transmittance": R + 1}
    if bender:
        want["termination_bend"] = 1
    assert got == want


@pytest.mark.parametrize("bender", [True, False])
def test_baked_launches(bender):
    from nonrigid_nerf_b200 import autograd as A
    net, _, rays, z, lat = _inputs(bender)
    grid = _far_grid(net)
    got = _launches(lambda: A.field_baked(net, rays, z, lat, True, grid))
    assert got == {"baked_bend": 1, "baked_compact": 1, "baked_field": 1, "baked_scatter": 1}


@pytest.mark.parametrize("details", [True, False])
def test_deformed_launches(details):
    from nonrigid_nerf_b200 import _lib, autograd as A, geometry as G
    net, b, rays, z, lat = _inputs(True)
    lats = torch.from_numpy((np.random.RandomState(1).randn(2, 32) * 0.1).astype(np.float32)).to(DEV)
    frame = G.bake_deformation(b, lats, [-1] * 3, [1] * 3, 4).frame(0)
    grid = _far_grid(net)
    got = _launches(lambda: A.field_baked(net, rays, z, lat, details, grid, frame))
    assert got == {k: 1 for k in _lib.DEFORMATION_KERNEL_KINDS[1:]}
