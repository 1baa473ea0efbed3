"""Every stage of the fused training kernels against an fp64 reference of that one stage, fed with the kernel's own
fp16 operands read back from the stashes (tests/stash_layout.py) and the packed weights' own rounding fp16(w).

What is left between kernel and reference is fp32 accumulation and one final rounding, bounded per element by

    |kernel - exact| <= 0.5 ulp_fp16(kernel)        (only where the output is stored as fp16)
                        + c * 2^-24 * (|A| @ |W|)   (the same product on absolute values)

c is the accumulation depth of the step: K + 2 for one tensor-core GEMM of depth K (K products, the bias add and the
final fp32 rounding).  Where a check spans several fp32 stages (PE backward, bend, latent reduction) the absolute-value
product is propagated through those stages and c is the sum of their depths.  The weight gradients use c = 16 T + 64
(8 wgmma k-steps per tile over T tiles, plus the split reduction) and, because that per-element bound grows with the batch,
also a relative L2 bound of 1.5e-4 per tensor (the worst measured, 3.5e-5, is L0's at 1024 x 128, whose sin / cos inputs
cancel strongly); a weight gradient missing one tile of 1024 moves by about 1e-3.
The divergence kernels are checked against the full tangent / adjoint chains in fp64 with the UNROUNDED fp32 bender
weights, from the kernel's own hi + lo probe operand (itself within 2^-22 |e| + 2^-25 of e), at c = 64 (eta = 2^-18):
their hi/lo split is meant to be fp32-accurate, and plain fp16 operands (about 4e-4) fail this by orders of magnitude.

The time-conditioned baseline (TC: no bender, the latent z enters L0 and L5 as a per-ray bias) adds these checks:
  ray bias rb[ray][l] = b_l + W_l[:, 63:95] z    fp32 weights and latents, c = 34 on |b| + |W||z|
  H1, H6 (L0, L5)      each accumulator row adds rb of its own ray, min(row, P - 1) // S; c_mma(K) on |A||W| + |rb|
  per-ray sums         sum of the decoded dY0 / dY5 over the ray's samples / loss scale, c = S + 2
  d z                  from the kernel's own sums and the fp32 W0 / W5 latent columns, c = 514
  dW0 / dW5[:, 63:95]  from the kernel's own sums, c = 4 (n + 2): n fp32 FMAs, whose worst case few rays nearly reach
and WGRAD checks the whole TC gradient layout (W0 [256][95], W5 [256][351]) as above.

Measured on one H100 80GB HBM3 (700 W power limit): the worst observed ratio of each stage (|kernel - exact| - rounding)
/ (2^-24 |A||W|) is printed with `pytest -s` ("c_obs"); every c above has at least 4x margin over the largest c_obs of its
stage.  The worst TC c_obs: ray bias 4.48 (1023 x 64), H1 1.55 and H6 8.30 (1024 x 128), per-ray sums 0.69 (37 x 3),
d z 6.49 (1024 x 128), latent columns 2.24 of c = 20 (3 x 100); H2 .. H8, raw and dY0 .. dY6 at most 3.70 of c = 258,
dY7 1.99 of 18, the other weight gradients 5.43 of 80 (37 x 3).

Every caller-owned buffer (stashes, masks, scratch, outputs) is filled with 0xFF (fp16 / fp32 NaN) before the calls, so a
read of memory no kernel wrote shows up as a NaN in a checked value.
"""
import ctypes as C

import pytest
import torch

from tests import stash_layout as SL
from tests.parity import DEV, Report, poison_f32
from tests.stage_reference import (Case, _lib, check_wgrad, dgrad_reference, empty_splits, expected_scale, grad_stash_images,
                                   models, pack_nerf, run_all, run_backward, run_forward, wgrad_plan)

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------------------------
# shapes
# ----------------------------------------------------------------------------------------------------------------------
SHAPES = {
    "1x7": dict(n=1, s=7),                     # one ragged tile, odd tile count
    "2x64": dict(n=2, s=64),                   # exactly one tile
    "3x100": dict(n=3, s=100),                 # rays straddle tiles
    "11x100": dict(n=11, s=100),               # 9 tiles: WGRAD plan with empty trailing splits (see below)
    "1023x64": dict(n=1023, s=64),             # several tiles per CTA everywhere, ragged
    "1024x128": dict(n=1024, s=128),           # the benchmark's fine pass, full WGRAD plan
    "3x100_nobender": dict(n=3, s=100, bender=False),
    "2x64_out4": dict(n=2, s=64, out_ch=4),
    "3x100_out4_nobender": dict(n=3, s=100, out_ch=4, bender=False),
    "3x100_cutoff_scaling": dict(n=3, s=100, cutoff="median", scaling=0.7),
    # time-conditioned baseline: L0 / L5 take each accumulator row's bias from its own ray
    "37x3_tc": dict(n=37, s=3, bender=False, tc=True),          # rows r0 and r0 + 8 on different rays; one ragged tile
    "5x1_tc": dict(n=5, s=1, bender=False, tc=True),            # every row its own ray
    "1x7_tc": dict(n=1, s=7, bender=False, tc=True),            # one ray, rows past P
    "3x100_tc": dict(n=3, s=100, bender=False, tc=True),        # rays straddle tiles
    "3x100_tc_stride0": dict(n=3, s=100, bender=False, tc=True, lat_stride0=True),   # one latent row for every ray
    "3x100_out4_tc": dict(n=3, s=100, out_ch=4, bender=False, tc=True),
    "11x100_tc": dict(n=11, s=100, bender=False, tc=True),      # 9 tiles: empty trailing WGRAD splits without a bender
    "1023x64_tc": dict(n=1023, s=64, bender=False, tc=True),
    "1024x128_tc": dict(n=1024, s=128, bender=False, tc=True),
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_every_stage_matches_its_fp64_reference(name):
    kw = dict(SHAPES[name])
    if kw.get("cutoff") == "median":
        # a cut-off that removes about half of the points: the median rigidity of the same points without one
        kw["cutoff"] = float(run_forward(Case(**dict(kw, cutoff=None)))["rig"].median())
    cs = Case(**kw)
    o, b, _ = run_all(cs, name)
    if kw.get("lat_stride0"):
        # a broadcast latent row computes exactly what the same row repeated for every ray does
        ex = Case(**kw)
        ex.lat = cs.lat.contiguous()
        oe = run_forward(ex)
        for k in ("stash", "mask", "raw"):
            assert torch.equal(o[k], oe[k]), f"latent stride 0 vs repeated rows: {k} differs"
    if cs.T >= 500:
        # the fp16 gradient chain must not saturate at the benchmark's shapes
        g = grad_stash_images(cs, b).float().abs()
        assert float(g.max()) < 65504.0, f"gradient stash saturates: max {float(g.max())}"
        print(f"  [{name}] max |gradient stash| {float(g.max()):.1f}")


# ---- WGRAD's split plan (wgrad.cu, launch_wgrad; replicated in tests/stage_reference.py) ----
def test_the_9_tile_shape_has_an_empty_trailing_wgrad_split():
    """wgrad_reduce_kernel skips splits that own no tiles (n_valid).  The 11 x 100 shape above covers that path only if
    the plan for this device leaves such a split; a cluster-limited device can run fewer CTAs than SMs, so every even
    CTA budget down to 3/4 of the SMs is checked.  The same holds for the bender-less plan of 11 x 100_tc."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    for name, has_bender in (("11x100", True), ("11x100_tc", False)):
        n_tiles = SHAPES[name]["n"] * SHAPES[name]["s"] // SL.TILE_M + 1
        assert n_tiles == 9
        for max_ctas in range(sms & ~1, (3 * sms // 4) & ~1, -2):
            assert empty_splits(n_tiles, wgrad_plan(n_tiles, max_ctas, has_bender)), (name, max_ctas)


# ---- loss-scale edges: the bending model and the time-conditioned baseline (TC) ----
def edge_case(mode, **kw):
    return Case(3, 100, bender=False, tc=True, **kw) if mode == "tc" else Case(3, 100, **kw)


MODES = ["bender", "tc"]


def test_zero_upstream_gives_exactly_zero_gradients():
    for mode in MODES:
        cs = edge_case(mode, draw_mag=0.0, reg_mag=0.0)
        o = run_forward(cs)
        b = run_backward(cs, o)
        # every float of each buffer (nerf_grad: the TC layout's full length), the TC per-ray sums and latent columns included
        for k in ("nerf_grad", "d_lat") + (("tc_ws",) if cs.tc else ("bender_grad",)):
            assert bool((b[k] == 0).all()), (mode, k)
        assert bool((grad_stash_images(cs, b) == 0).all()), (mode, "gradient stash")


@pytest.mark.parametrize("mag", [1e-15, 1e10])
def test_extreme_upstream_magnitudes_keep_every_stage_bound(mag):
    for mode in MODES:
        cs = edge_case(mode, draw_mag=mag, reg_mag=0.05 * mag)
        run_all(cs, f"{mode} |d_raw| x {mag:g}", divergence=False)


def test_regulariser_upstream_sets_the_loss_scale():
    cs = Case(3, 100, draw_mag=1e-3, reg_mag=40.0)
    assert float(cs.d_un_up.abs().max()) > 100 * float(cs.d_raw[:, :4].abs().max())
    run_all(cs, "regulariser-dominated", divergence=False)


def test_channel_4_of_d_raw_changes_nothing():
    """Channel 4 never reaches the loss (the head's row 4 gets a zero gradient), so a large d_raw[..., 4] must not move
    the loss scale: every gradient equals the channel-4-zero run bit for bit (the bender's latent gradient up to the order
    of its fp32 atomics; the TC latent sums run in a fixed order, so there the latent gradient too)."""
    for mode in MODES:
        cs = edge_case(mode)
        o = run_forward(cs)
        b0 = run_backward(cs, o)
        d4 = cs.d_raw.clone()
        d4[:, 4] = 3.0e4 * torch.sign(torch.randn(cs.P, device=DEV))
        b4 = run_backward(cs, o, d_raw=d4)
        assert torch.equal(b0["gstash"], b4["gstash"]), f"{mode}: gradient stash differs"
        assert torch.equal(b0["nerf_grad"], b4["nerf_grad"]), f"{mode}: NeRF weight gradients differ"
        if cs.tc:
            assert torch.equal(b0["tc_ws"], b4["tc_ws"]), "tc: per-ray sums or latent weight columns differ"
            assert torch.equal(b0["d_lat"], b4["d_lat"]), "tc: latent gradients differ"
        else:
            assert torch.equal(b0["bender_grad"], b4["bender_grad"]), "bender weight gradients differ"
            # the latent gradient's fp32 atomics add in no fixed order: equal up to that rounding
            torch.testing.assert_close(b0["d_lat"], b4["d_lat"], rtol=0.0, atol=1e-5 * float(b0["d_lat"].abs().max()))


def test_head_redirection_and_accumulation():
    """nerf_grad_head puts the output layer's gradient in its own buffer; accumulate_nerf / accumulate_bender add the
    gradients onto what the destination holds (optim.Adam's gradient arena)."""
    lib = _lib().load()
    for mode in MODES:
        cs = edge_case(mode)
        rep = Report(f"{mode} accumulate + head redirect")
        o = run_forward(cs)
        g = torch.Generator(device=DEV).manual_seed(3)
        n_head = cs.out_ch * 257
        pre_n = torch.randn(lib.nrn_nerf_tc_grad_floats(cs.out_ch) if cs.tc else lib.nrn_nerf_grad_floats(cs.out_ch),
                            generator=g, device=DEV)
        pre_n[-n_head:] = float("nan")        # the head part lives elsewhere: this tail must stay untouched
        pre_h = torch.randn(n_head, generator=g, device=DEV)
        pre_b = torch.randn(lib.nrn_bender_grad_floats(), generator=g, device=DEV)
        nerf, head, bend = pre_n.clone(), pre_h.clone(), pre_b.clone()
        b = run_backward(cs, o, nerf_grad=nerf, nerf_head=head, bender_grad=bend, accumulate=True)
        assert bool(torch.isnan(nerf[-n_head:]).all()), f"{mode}: the head's slot of nerf_grad was written despite nerf_grad_head"
        imgs = dgrad_reference(cs, o, b, rep, expected_scale(cs))
        full = torch.cat([nerf[:-n_head], head])
        base = torch.cat([pre_n[:-n_head], pre_h])
        b["nerf_head"] = None
        check_wgrad(cs, b, imgs, rep, expected_scale(cs), nerf_flat=full, bend_flat=bend, base_nerf=base, base_bend=pre_b)


@pytest.mark.parametrize("head", [False, True])
def test_empty_tc_batch_zeroes_the_whole_gradient_layout(head):
    """n_rays = 0 (an empty shard) contributes zero gradients: every float of the time-conditioned layout, the latent
    columns of W0 / W5 included, is overwritten with 0; with nerf_grad_head the head's slot of nerf_grad stays untouched."""
    from nonrigid_nerf_b200 import ops
    L = _lib()
    lib = L.load()
    npk, _, _ = pack_nerf(*ops.nerf_param_list(models(False, tc=True)[0]), 5, 95)
    n_nerf, n_head = lib.nrn_nerf_tc_grad_floats(5), 5 * 257
    grad, head_buf = poison_f32(n_nerf), poison_f32(n_head)
    a, t = L.NrnFieldBwdArgs(), L.NrnTcBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = 0, 64, 5
    a.nerf_packed, a.nerf_grad = npk.data_ptr(), grad.data_ptr()
    if head:
        a.nerf_grad_head = head_buf.data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    L.check(lib.nrn_field_backward_tc(C.byref(a), C.byref(t)), "field_backward_tc")
    L.device_error_check()
    if head:
        assert bool((grad[:-n_head] == 0).all()) and bool((head_buf == 0).all())
        assert bool(torch.isnan(grad[-n_head:]).all()), "the head's slot of nerf_grad was written despite nerf_grad_head"
    else:
        assert bool((grad == 0).all())


def test_forward_is_deterministic_past_p():
    """Rows past P of a ragged last tile are computed from x = 0 and a zero latent: finite (checked with the stages) and
    the same on every run, masks included."""
    cs = Case(1, 7)
    o1, o2 = run_forward(cs), run_forward(cs)
    n = cs.T
    assert torch.equal(o1["stash"][:n * SL.STASH_TILE], o2["stash"][:n * SL.STASH_TILE])
    assert torch.equal(o1["mask"][:n * SL.MASK_TILE], o2["mask"][:n * SL.MASK_TILE])
