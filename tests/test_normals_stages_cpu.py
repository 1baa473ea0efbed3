"""The density gradient's stage-test helpers without a GPU (tests/normals_stages.py, tests/normals_reference.py): the
exact 2^k equivariance of the fp64 chain and its bound, the encoding's stage of the bound, the launch-size and chunk
planner, the restated bent point against numpy fp32, and the fp64 trunk forward at a point against autograd."""
import math

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers, normals_reference as R, normals_stages as NS
from tests.parity import half_ulp


def _params(kind):
    if kind == "tc":
        net = helpers.tc_models(5, "cpu")[0]
    else:
        net = helpers.build_models(O, 7, "cpu", with_bender=kind != "canonical")[0]
    npar, bp = R.params(net, fp16=True)
    return npar, (bp if kind.startswith("bender") else None)


def _path(P, bent, seed=0):
    """A random path: ReLU masks, an fp16 encoding, offsets and rigidity (the chain is linear for any of them)."""
    g = torch.Generator().manual_seed(seed)
    masks = {f"H{l + 1}": torch.rand(P, 256, generator=g) < 0.5 for l in range(8)}
    for name, cols in (("Hb1", 96), ("Hb2", 96), ("Hb3", 64), ("Hb4", 64)):
        masks[name] = torch.rand(P, cols, generator=g) < 0.5
    E = (torch.rand(P, 64, generator=g) * 2 - 1).half().double()
    E[:, 63] = 1.0
    un = (torch.randn(P, 3, generator=g) * 0.1).float() if bent else None
    rig = torch.rand(P, generator=g).float() if bent else None
    return masks, E, un, rig


def _scale_head(npar, k):
    out = dict(npar)
    out["out_w"] = npar["out_w"].clone()
    out["out_w"][3] *= 2.0 ** k
    return out


@pytest.mark.parametrize("kind", ["canonical", "bender", "bender_knobs", "tc"])
def test_chain_and_bound_scale_exactly_with_the_head_row(kind):
    """fixed_mask_chain, rounding_bound and the captured trunk operands are linear in the head row: 2^k on it scales g,
    the bound, sigma and every trunk operand by exactly 2^k in fp64, and the saturation step drops by k."""
    npar, bp = _params(kind)
    kn = dict(cutoff=0.3, scaling=2.5, removal=0.8) if kind == "bender_knobs" else {}
    masks, E, un, rig = _path(40, bp is not None)
    g, bound, sigma = R.rounding_bound(npar, bp, masks, E, un, rig, e_term=True, **kn)
    trunk = NS.trunk_capture(npar, bp, masks, E, un, rig, **kn)
    amax = max(float(y.abs().max()) for y in trunk.values())
    k_sat = NS.saturation_step(amax)
    assert amax * NS.TRUNK_SCALE * 2.0 ** (k_sat - 1) <= NS.F16_MAX < amax * NS.TRUNK_SCALE * 2.0 ** k_sat
    for k in (1, 4, 13):
        s = 2.0 ** k
        gk, bk, sk = R.rounding_bound(_scale_head(npar, k), bp, masks, E, un, rig, e_term=True, **kn)
        assert torch.equal(gk, g * s) and torch.equal(bk, bound * s) and torch.equal(sk, sigma * s)
        tk = NS.trunk_capture(_scale_head(npar, k), bp, masks, E, un, rig, **kn)
        assert all(torch.equal(tk[n], trunk[n] * s) for n in NS.TRUNK_STAGES)
        assert NS.saturation_step(amax * s) == max(k_sat - k, 0)


@pytest.mark.parametrize("kind", ["canonical", "bender_knobs", "tc"])
def test_the_encoding_stage_of_the_bound(kind):
    """e_term adds sum_j |d g_i / d E_j| (half_ulp(E_j) + E_PE) over the sin / cos columns and nothing else; the
    derivatives are the chain's exact differences in E (it is linear in E), and the worst-case encoding error moves each
    component by exactly that term."""
    npar, bp = _params(kind)
    kn = dict(cutoff=0.3, scaling=2.5) if kind == "bender_knobs" else {}
    P = 12
    masks, E, un, rig = _path(P, bp is not None, seed=3)
    g0, b0, s0 = R.rounding_bound(npar, bp, masks, E, un, rig, **kn)
    g1, b1, s1 = R.rounding_bound(npar, bp, masks, E, un, rig, e_term=True, **kn)
    assert torch.equal(g0, g1) and torch.equal(s0, s1)
    J = torch.zeros(P, 3, 64, dtype=torch.float64)
    for j in range(3, 63):
        Ej = E.clone()
        Ej[:, j] += 1.0
        J[:, :, j] = R.fixed_mask_chain(npar, bp, masks, Ej, un, rig, **kn) - g0
    r = half_ulp(E) + R.E_PE
    r[:, :3] = 0.0
    r[:, 63] = 0.0
    term = (J.abs() * r[:, None, :]).sum(2)
    assert torch.allclose(b1 - b0, term, rtol=1e-9, atol=1e-18)
    for i in range(3):
        moved = R.fixed_mask_chain(npar, bp, masks, E + torch.sign(J[:, i]) * r, un, rig, **kn)
        assert torch.allclose((moved - g0)[:, i], term[:, i], rtol=1e-9, atol=1e-18)


@pytest.mark.parametrize("num_sms", [132, 114, 78])
def test_launch_sizes_make_ctas_run_several_tiles(num_sms):
    chunk = 65536
    full, one_extra, one_row, less = NS.wave_sizes(num_sms, chunk)
    assert NS.tiles(full) == 512 and NS.tiles(less) == 512 and less % 128 == 127
    lo, hi = NS.tiles_per_cta(full, num_sms)
    assert lo == 512 // num_sms and hi == -(-512 // num_sms) and lo >= 3
    assert NS.tiles(one_extra) == num_sms + 1 and NS.tiles_per_cta(one_extra, num_sms) == (1, 2) and one_extra % 128 == 0
    assert NS.tiles(one_row) == 2 * num_sms + 1 and one_row - (NS.tiles(one_row) - 1) * 128 == 1
    assert NS.tiles_per_cta(one_row, num_sms) == (2, 3)
    if num_sms == 132:
        assert (lo, hi) == (3, 4)


def test_chunk_plan_and_the_chunks_past_2_31_bytes():
    chunk = 65536
    assert NS.chunks(3 * chunk + 77, chunk) == [(0, chunk), (chunk, chunk), (2 * chunk, chunk), (3 * chunk, 77)]
    assert NS.chunks(chunk, chunk) == [(0, chunk)] and NS.chunks(1, chunk) == [(0, 1)]
    # bender, latents per point: 128 B per point, byte 2^31 opens chunk 256, the last (300 points)
    n = 2 ** 24 + 300
    c = NS.chunk_of_byte(2 ** 31, 128, chunk)
    assert c == 256 and NS.chunks(n, chunk)[-1] == (256 * chunk, 300)
    assert c * chunk * 128 <= 2 ** 31 < (c * chunk + 300) * 128
    # canonical: points and output at 12 B per point; byte 2^31 lies in the last chunk
    n = math.ceil(2 ** 31 / 12) + 300
    c = NS.chunk_of_byte(2 ** 31, 12, chunk)
    c0, m = NS.chunks(n, chunk)[-1]
    assert c == c0 // chunk and c0 * 12 <= 2 ** 31 < (c0 + m) * 12 and n * 12 > 2 ** 31


@pytest.mark.parametrize("scaling", [None, 2.5, 0.7])
def test_bent_point_restatement_against_numpy_fp32(scaling):
    g = torch.Generator().manual_seed(9)
    P = 4096
    x = (torch.rand(P, 3, generator=g) * 2.4 - 1.2).float()
    un = (torch.randn(P, 3, generator=g) * 0.3).float()
    rig = torch.rand(P, generator=g).float()
    rig[:64] = 0.0
    got = NS.bent_point(x, un, rig, scaling).numpy()
    xn, un_n, rn = x.numpy(), un.numpy(), rig.numpy()
    m = np.multiply(rn[:, None], un_n, dtype=np.float32)
    if scaling is not None:
        m = np.multiply(m, np.float32(scaling), dtype=np.float32)
    want = np.add(xn, m, dtype=np.float32)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), want.view(np.int32))
    assert np.array_equal(got[:64], xn[:64])
    # one rounding per operation: the exact value of the same operations differs from it
    exact = x.double() + rig.double()[:, None] * un.double() * (scaling if scaling is not None else 1.0)
    assert not torch.equal(torch.from_numpy(got).double(), exact)


@pytest.mark.parametrize("kind", ["canonical", "tc"])
def test_trunk_forward64_masks_give_the_free_running_gradient(kind):
    """The fixed-mask chain fed trunk_forward64's masks and exact encoding at a point is R.density_gradient there."""
    npar, _ = _params(kind)
    P = 64
    x = torch.rand(P, 3, generator=torch.Generator().manual_seed(2), dtype=torch.float64) * 2 - 1
    z = torch.randn(32, dtype=torch.float64, generator=torch.Generator().manual_seed(3)).expand(P, 32) * 0.3 if kind == "tc" else None
    E, masks, pre, mag = NS.trunk_forward64(npar, x, z, tc=kind == "tc")
    assert all(torch.equal(masks[f"H{l + 1}"], pre[l] > 0) for l in range(8))
    assert all(bool((pre[l].abs() <= mag[l] + npar["pts_b"][l].abs() + 1e-12).all()) for l in range(8))
    g = R.fixed_mask_chain(npar, None, masks, E)
    want = R.density_gradient(npar, None, x, z, tc=kind == "tc")
    assert torch.allclose(g, want, rtol=1e-10, atol=1e-12)
