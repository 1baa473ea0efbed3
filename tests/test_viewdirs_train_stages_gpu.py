"""Training the view-dependent head without a bender (NeRF(use_viewdirs=True), rigid scenes), stage by stage: every
caller-owned buffer is filled with NaN first, then nrn_field_forward_views_train and nrn_field_backward_views run, and
every stage is checked against fp64 of the kernel's own fp16 operands read back from its stashes (tests/stage_reference.py,
Case(views=True)), with the per-element bound 0.5 ulp_fp16 (where stored as fp16) + c 2^-24 (|A| |W|), c = K + 2:

    forward  H1 .. H8 and the trunk's mask bits as the trunk kernel's; Dir (the direction encoding) within 0.5 ulp +
             E_DIR_ENC of fp64 of the fp32 direction's encoding; F (K = 256); Hv = relu(F WvF^T + Dir WvE^T + bv) (K = 288,
             one accumulator); raw rgb from Hv (K = 128) and raw alpha from H8 (K = 256); the Hv mask bits == Hv > 0
    DGRAD    dYv = fp16(d_raw . rgb_linear) * [hv > 0] (K = 16); dF = fp16(dYv . views_linears.0[:, :256]) (K = 128);
             dY7 = fp16(dF . feature_linear + d_alpha alpha_linear) * [h8 > 0] (K = 256 + 16); then dY6 .. dY0 from the
             kernel's own dY7 (K = 256), with L5's embedding columns skipped
    WGRAD    every tensor of the 595,844-float flat layout, per element at c_wgrad(T) and at relative L2 1.5e-4: the trunk
             W0 b0 .. W7 b7, then views_linears.0 (feature and direction columns), feature_linear, alpha_linear (row 3 of
             the trunk's head job), rgb_linear; into one flat buffer, and into a trunk and a separate head destination,
             which must give the same bits (and leave the trunk buffer's head slot untouched), and added in place

Which wrong implementation each check catches: the stash written from the wrong registers or rows (H1 .. H8, F, Hv: DGRAD
and WGRAD consume the stash, so the gradients alone would stay self-consistent), the direction encoding rounded toward
zero or of the wrong ray (Dir), feature and direction columns of views_linears.0 swapped (Hv, raw rgb, WGRAD), the Hv
mask not applied (dYv), ViewsF^T reading the direction columns (dF), the alpha term dropped (dY7), the register flow
around dY5 of the chain without L5e^T (dY5 .. dY0), a head block in the wrong order or a wrong partial layout in the
reduce (the flat gradient), a row of a ragged tile left unwritten or non-finite (rows past P are checked with the rest).
Shapes: a ragged single tile, 1023 x 64, S = 100, 1024 x 128, and 25 x 64, whose 13 tiles leave an empty trailing split
in views_linears.0's feature-column job at this device's CTA budget; the loss-scale edges (upstream 0, 1e-15, 1e10).
"""
import pytest
import torch

from tests import stash_layout as SL
from tests.parity import DEV, Report, poison_f32
from tests.stage_reference import (VIEW_HEAD_JOBS, Case, _lib, check_forward, check_wgrad, dgrad_reference, empty_splits,
                                   expected_scale, grad_stash_images, run_backward, run_forward, wgrad_plan)

pytestmark = pytest.mark.gpu

# (n, s, upstream factor): a ragged single tile (64 of 128 rows), several tiles per CTA (ragged), rays straddling tiles,
# the benchmark's fine pass at 1,024 rays, the loss-scale edges, and 25 x 64 (13 tiles: an empty trailing split in a head
# job, see below)
SHAPES = [(1, 64, 1.0), (1023, 64, 1.0), (40, 100, 1.0), (1024, 128, 1.0), (1023, 64, 0.0), (1023, 64, 1e-15),
          (1023, 64, 1e10), (25, 64, 1.0)]


def run_views(cs, tag):
    rep = Report(tag)
    o = run_forward(cs)
    check_forward(cs, o, rep)
    b = run_backward(cs, o)
    scale = expected_scale(cs)
    imgs = dgrad_reference(cs, o, b, rep, scale)
    check_wgrad(cs, b, imgs, rep, scale)
    return o, b, imgs, rep, scale


@pytest.mark.parametrize("n,s,factor", SHAPES)
def test_stages_against_fp64_of_their_own_operands(n, s, factor):
    cs = Case(n, s, views=True, draw_mag=factor)
    o, b, imgs, rep, scale = run_views(cs, f"{n}x{s} |d_raw| x {factor:g}")
    flat = b["nerf_grad"]
    if factor == 0.0:
        assert bool((flat == 0).all()), "a zero upstream gives zero gradients"
        assert bool((grad_stash_images(cs, b) == 0).all()), "gradient stash"
        vg = SL.image(b["vgstash"], SL.V_GRAD_TILE, 0, SL.V_GRAD_TILE // SL.CHUNK, cs.T)
        assert bool((vg == 0).all()), "view gradient stash"
    # the trunk and the head block to two destinations: the same bits; the trunk buffer's head slot stays untouched
    lib = _lib().load()
    n_all = lib.nrn_nerf_views_grad_floats()
    trunk, head = poison_f32(n_all), poison_f32(n_all - SL.TRUNK_FLOATS)
    run_backward(cs, o, nerf_grad=trunk, nerf_head=head)
    assert bool(torch.isnan(trunk[SL.TRUNK_FLOATS:]).all()), "the head's slot of nerf_grad was written despite nerf_grad_head"
    assert torch.equal(trunk[:SL.TRUNK_FLOATS], flat[:SL.TRUNK_FLOATS]) and torch.equal(head, flat[SL.TRUNK_FLOATS:])
    # accumulation into both destinations: fp32(base + gradient), bit for bit
    g = torch.Generator(device=DEV).manual_seed(7)
    base_t, base_h = torch.randn(n_all, generator=g, device=DEV), torch.randn(n_all - SL.TRUNK_FLOATS, generator=g, device=DEV)
    base_t[SL.TRUNK_FLOATS:] = float("nan")
    trunk, head = base_t.clone(), base_h.clone()
    run_backward(cs, o, nerf_grad=trunk, nerf_head=head, accumulate=True)
    assert torch.equal(trunk[:SL.TRUNK_FLOATS], base_t[:SL.TRUNK_FLOATS] + flat[:SL.TRUNK_FLOATS])
    assert torch.equal(head, base_h + flat[SL.TRUNK_FLOATS:])
    assert bool(torch.isnan(trunk[SL.TRUNK_FLOATS:]).all())
    if cs.T >= 500:
        gs = grad_stash_images(cs, b).float().abs()
        assert float(gs.max()) < 65504.0, f"gradient stash saturates: max {float(gs.max())}"


def test_the_13_tile_shape_has_an_empty_trailing_split_in_a_head_job():
    """wgrad_views_reduce_kernel skips splits that own no tiles.  25 x 64 covers that path in a head job (12-15) only if
    the views plan for this device leaves such a split there; a cluster-limited device runs fewer CTAs than SMs, so every
    even CTA budget down to 13/16 of the SMs (108 of 132) is checked."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    n_tiles = -(-25 * 64 // SL.TILE_M)
    assert n_tiles == 13
    for max_ctas in range(sms & ~1, (13 * sms // 16) & ~1, -2):
        empty = empty_splits(n_tiles, wgrad_plan(n_tiles, max_ctas, views=True))
        assert any(j in VIEW_HEAD_JOBS for j in empty), (max_ctas, empty)
