"""The fused training kernels at the benchmark's cfg4 batch (8192 rays: 4,096 coarse and 8,192 fine tiles, stashes past
2^31 and 2^32 bytes), at 53,248 x 128 points (ReLU masks past 2^31 bytes, divergence stashes past 2^32) and at
52,480 x 128 (DGRAD and WGRAD on masks past 2^31), stage by stage against the fp64 references of
tests/stage_reference.py, with the bounds of tests/test_stage_parity_gpu.py.  The cfg4 passes, the coverage sweep, the
52,480 x 128 case and the render chunk run for the bending model and for the time-conditioned baseline (the latent as a
per-ray bias of L0 / L5; its per-ray sums of dY0 / dY5, d z and the latent columns of W0 / W5 are checked too, and
WGRAD runs the bender-less plan and wgrad_reduce_tc_kernel).

Every stage is row-local, so it is checked on sampled tiles: 0 and T - 1, the tiles whose byte range in some buffer holds
byte 2^31 or 2^32 and their neighbours (from the library's per-tile sizes), and the tiles of the persistent CTAs' first
and last grid sweep.  WGRAD sums over every tile; it is checked twice:
  dense     against an fp64 sum streamed over blocks of 256 tiles, at c_wgrad(T) and at the relative L2 of
            wgrad_rel_l2 for the deepest split of the replicated plan.  The fixed 1.5e-4 of the stage test does not hold
            here: W0's error grows in step with the tiles one split accumulates (relative L2 3.5e-5, 1.44e-4 and
            2.84e-4 at 256, 1,024 and 2,048 tiles per split: 1,024, 4,096 and 8,192 tiles, W0's job in 4 splits each
            time), as fp32 accumulation of a sum that grows with every tile does; the per-element bound c_wgrad(T) holds
            with c_obs far below it.  The plan is replicated with one CTA per SM; launch_wgrad caps it at the resident
            2-CTA clusters, so on a device with fewer of those the real splits are deeper and this bound tighter than
            it should be (a spurious failure, never a false pass);
  coverage  m = 97 backward passes on one forward stash, pass j with upstreams only on the tiles t = j (mod m).  Zero
            upstream gives exactly zero gradient rows, so each pass's WGRAD is the sum over its own ~T / m tiles, checked
            per element at c_wgrad(T / m).  One tile is then about 1 % of sum |terms| against a bound of about 1e-4 of
            it: a tile dropped, repeated or read from the wrong address fails by two orders of magnitude, where the
            dense check's relative L2 cannot see it (one tile of 8,192 moves a gradient by about 1.2e-4).
The divergence kernels' compact WGRAD gets the same sweep, with g_ray non-zero only on the rays of the pass's tiles.
  52,480 x 128  the smallest shape whose masks pass 2^31 bytes (51 of its 52,480 tiles lie past tile 52,428, which holds
            byte 2^31); stash 33.3 GB, gradient stash 32.5 GB, masks 2.15 GB, 63.3 GiB in all, skipped with the GiB it
            needs when the device has less free.  Forward, DGRAD and the gradient-stash statistics on the tiles at the
            2^31 .. 2^34 boundaries of all three buffers, dense WGRAD, then a second backward on the same forward stash
            with upstreams only on those tiles, every WGRAD element at c_wgrad(len(tiles)): the dense relative L2 moves
            by about 2e-5 for one misaddressed tile of 52,480, this check by orders of magnitude.
The latent columns of W0 / W5 (tc_dw_lat_kernel, one fp32 FMA per ray) are held per element to c_latent_columns(n) and,
in the dense checks, to the relative L2 bound of the plan: one ray left out stays inside the per-element worst case at
8,192 rays but moves the columns by about 1 / sqrt(n).

Beyond single kernels:
  render chunk   render() at 65,536 rays (64 + 64 samples, the render workload's settings): 40 sampled rays equal a
                 separate call on just those rays bit for bit in every output, and their fine compositing holds the fp64
                 bounds of tests/ray_reference.py on the kernel's own raw and alpha;
  cfg4 step      training_wrapper_class at 8,192 rays against the fp32 oracle on the GPU with TF32 off: the per-ray
                 loss and every parameter gradient within DESIGN section 2's bounds for 1,024 rays;
  graph replay   the same step under GraphedStep (plain Adam, set_lr between replays, one replay at lr = 0) against
                 eager steps 4..6.

Every caller-owned buffer is filled with 0xFF before the calls, as in the stage test.

Measured on one H100 80GB HBM3 (700 W power limit, 132 SMs), printed with `pytest -s`; the file runs in about 45 s, the
52,480 x 128 cases in 4 to 6 s each (two runs), with 80 GB on the card.
  worst c_obs   forward H1 .. H8 and raw at most 6.32 of c = 322 (H6); bender steps 0.92 of 98; DGRAD dY0 .. dY7 4.94 of
                258, dY7 2.41 of 18; bender DGRAD 2.56 of 82; divergence chains at most 9.7 of 64 (t2), closed forms
                4.0 of 16; WGRAD dense 61.6 of c = 131,136 (W0, 8,192 tiles), swept 8.06 of 1,424, divergence compact
                WGRAD swept 10.6 of 8,848; render compositing 13.3 of 592
  tangent t1    3.71 of 64.  Checked against the exact probe e it reached 36.3 over the 6.8 M points of 53,248 x 128:
                the probe enters as fp16(e) + fp16(e - fp16(e)), whose residual is an fp16 subnormal below |e| of about
                2^-3 and so resolved to 2^-25 absolute only.  The chain now starts from that operand, and the operand is
                held to |hi + lo - e| <= 2^-22 |e| + 2^-25, as the bender input's hi / lo columns are
  dense WGRAD   relative L2 at 8,192 tiles: W0 2.84e-4, W5 2.95e-4, W1 1.55e-4; at 4,096: W0 1.44e-4
  fp16 flush    where the ReLU mask is on, 1.0e-7 of dY0 .. dY7 are fp16 zero and 2.0e-4 subnormal (8192 x 128); the
                largest |gradient stash| value is 44,928 of 65,504 (24,656 at 1024 x 128)
  cfg4 step     per-ray loss 2.3e-6 L-inf, 3.0e-6 relative L2; gradients at most 1.64e-2 (coarse W0) for the NeRF
                layers, 2.5e-4 for the heads, 3.0e-2 for the bender, 4.1e-2 for the latent table
  graph replay  relative L2 to eager 0 to 3.2e-7 per step; two eager runs differ by 3.2e-7
  52,480 x 128  worst c_obs H1 .. H8 5.62 of 322 (H6), dY0 .. dY7 3.02 of 258, dY7 1.67 of 18, bender DGRAD 1.07 of 82;
                WGRAD dense 134.5 of c = 839,744 (W0), on the boundary tiles only 7.43 of 592; dense relative L2 at most
                1.86e-3 (W0, bending; deepest split 13,120 tiles, bound 7.8e-3) and 1.55e-3 (W5, time-conditioned;
                10,496 tiles, bound 6.3e-3)
  time-cond.    at 8,192 x 64 / 128 worst c_obs ray bias 4.48 of 34, H1 .. H8 4.67 of 322, dY0 .. dY7 2.45 of 258,
                per-ray sums 0.69 of 130, d z 7.81 of 514, dense WGRAD 44.9 of 131,136, swept 6.39 of 1,424; the latent
                columns of W0 / W5 3.56 of c_latent_columns(8,192) = 32,776 (5.83 swept) and 3.98 of 209,928 at 52,480
                rays, relative L2 1.6e-6 and 4.1e-6; the render chunk's compositing 13.0 of 592
"""
import copy
import time

import pytest
import torch

from tests import stash_layout as SL
from tests.parity import DEV, Report
from tests.stage_reference import (Case, Tiles, _lib, check_divergence, check_forward, check_wgrad, dgrad_reference,
                                   expected_scale, run_backward, run_divergence_backward, run_divergence_forward,
                                   run_forward, split_ranges, wgrad_images, wgrad_plan, wgrad_reference, wgrad_rel_l2)

pytestmark = pytest.mark.gpu
M_SWEEP = 97          # prime: the tile sets line up with neither the split boundaries nor the even-tile padding
BLOCK = 256           # tiles per block of the streamed fp64 WGRAD sum
LIMITS = (2 ** 31, 2 ** 32, 2 ** 33, 2 ** 34)


def tile_bytes(lib, n, s):
    """Per-tile bytes of every buffer a pass writes, from the library's sizes: the field stashes and masks (the view
    head's included) hold an even tile count, the divergence stashes the point tiles."""
    T = -(-n * s // SL.TILE_M)
    even = T + (T & 1)
    return {"stash": lib.nrn_stash_bytes(n, s) // even, "grad stash": lib.nrn_grad_stash_bytes(n, s) // even,
            "masks": lib.nrn_relu_mask_bytes(n, s) // even, "tangent": lib.nrn_div_stash_bytes(n, s) // T,
            "adjoint": lib.nrn_div_grad_stash_bytes(n, s) // T, "views stash": lib.nrn_views_stash_bytes(n, s) // even,
            "views grad stash": lib.nrn_views_grad_stash_bytes(n, s) // even, "hv mask": lib.nrn_hv_mask_bytes(n, s) // even}


def sample_tiles(cs, buffers):
    """0 and T - 1, the tiles at every 2^31 .. 2^34 byte boundary of the named buffers and their neighbours, and the
    first / last grid sweep of the persistent kernels (one tile per CTA and step of multi_processor_count)."""
    lib = _lib().load()
    sizes = tile_bytes(lib, cs.n, cs.s)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    out = {0, cs.T - 1, sms - 1, sms, cs.T - sms - 1, cs.T - sms}
    for name in buffers:
        found = SL.boundary_tiles(sizes[name], cs.T, LIMITS)
        assert found, f"{name}: no tile of {cs.T} reaches 2^31 bytes"
        out.update(found)
    return sorted(t for t in out if 0 <= t < cs.T)


def tile_set(cs, m, j):
    return [t for t in range(j, cs.T, m)]


def only_on_tiles(cs, tiles):
    """cs with d_raw and the regulariser upstreams zero on every point outside the listed tiles, and g_ray zero on every
    ray that does not lie inside one of them."""
    on = torch.zeros(cs.T, dtype=torch.bool, device=DEV)
    on[torch.tensor(tiles, dtype=torch.long, device=DEV)] = True
    keep = on[torch.arange(cs.P, device=DEV) // SL.TILE_M]
    c = copy.copy(cs)
    c.d_raw = cs.d_raw * keep[:, None]
    c.d_un_up = None if cs.d_un_up is None else cs.d_un_up * keep[:, None]
    c.d_rig_up = None if cs.d_rig_up is None else cs.d_rig_up * keep
    ray = torch.arange(cs.n, device=DEV)
    first, last = ray * cs.s // SL.TILE_M, ((ray + 1) * cs.s - 1) // SL.TILE_M
    c.g_ray = cs.g_ray * (on[first] & (first == last))
    return c


def grad_stash_stats(cs, o, b, tag):
    """Saturation of every gradient-stash image, and the share of the trunk's gradients dY0 .. dY7 that flush to fp16 zero
    or subnormal where their ReLU mask bit is set (a zero there is not the mask's)."""
    g_max, n_on, n_zero, n_sub = 0.0, 0, 0, 0
    chunks = (SL.GRAD_TILE if cs.bender else SL.GS_YB4[0]) // SL.CHUNK    # without a bender no dYb image is written
    for t0 in range(0, cs.T, BLOCK):
        sub = Tiles(cs, range(t0, min(t0 + BLOCK, cs.T)))
        g_max = max(g_max, float(sub.img(b["gstash"], SL.GRAD_TILE, (0, chunks)).float().abs().max()))
        for l in range(8):
            y = sub.img(b["gstash"], SL.GRAD_TILE, SL.GS_Y[l])[:sub.n].float().abs()
            on = sub.bits(o["mask"], SL.MK_H[l])[:sub.n]
            n_on += int(on.sum())
            n_zero += int(((y == 0) & on).sum())
            n_sub += int(((y > 0) & (y < 2.0 ** -14) & on).sum())
    print(f"  [{tag}] max |gradient stash| {g_max:.1f}; dY0..dY7 where the mask is on: {n_zero / n_on:.3e} fp16 zero, "
          f"{n_sub / n_on:.3e} subnormal")
    assert g_max < 65504.0, f"gradient stash saturates: max {g_max}"


def dense_wgrad(cs, o, b, rep, scale):
    """WGRAD against the fp64 sum over every tile, streamed over blocks of BLOCK tiles."""
    tot = None
    for t0 in range(0, cs.T, BLOCK):
        sub = Tiles(cs, range(t0, min(t0 + BLOCK, cs.T)))
        imgs = wgrad_images(cs, o, b, sub)
        imgs["sub"] = sub
        refs = wgrad_reference(cs, imgs)
        if tot is None:
            tot = refs
        else:
            for d, r in zip(tot, refs):
                for k, (v, a) in (r or {}).items():          # no bender: no bender sums
                    d[k] = (d[k][0] + v, d[k][1] + a)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    plan = wgrad_plan(cs.T, sms & ~1, cs.bender)
    depth = {j: max(e - s for s, e in split_ranges(cs.T, n)) for j, n in plan.items()}
    rel = wgrad_rel_l2(max(depth.values()))
    print(f"  [{rep.tag}] WGRAD plan at {sms} CTAs: splits {plan}; tiles per split {depth}; rel L2 bound {rel:.2e}")
    check_wgrad(cs, b, None, rep, scale, refs=tot, n_tiles=cs.T, rel_l2=rel)


SHAPES = {
    "8192x64_div": dict(n=8192, s=64),       # cfg4's coarse pass: stash and gradient stash past 2^31
    "8192x128": dict(n=8192, s=128),         # cfg4's fine pass: both past 2^32
    # the time-conditioned baseline's passes: every sampled tile holds whole rays, so their per-ray sums are checked
    "8192x64_tc": dict(n=8192, s=64, bender=False, tc=True),
    "8192x128_tc": dict(n=8192, s=128, bender=False, tc=True),
}
MODELS = {"bender": dict(), "tc": dict(bender=False, tc=True)}   # the bending model and the time-conditioned baseline


@pytest.mark.parametrize("name", list(SHAPES))
def test_cfg4_pass_every_stage_on_sampled_tiles_and_dense_wgrad(name):
    cs = Case(**SHAPES[name])
    div = name.endswith("_div")
    tiles = sample_tiles(cs, ("stash", "grad stash"))
    rep = Report(name)
    print(f"  [{name}] {cs.T} tiles; sampled {tiles}")
    o = run_forward(cs)
    check_forward(cs, o, rep, tiles)
    b = run_backward(cs, o)
    scale = expected_scale(cs)
    dgrad_reference(cs, o, b, rep, scale, tiles)
    grad_stash_stats(cs, o, b, name)
    dense_wgrad(cs, o, b, Report(f"{name} dense"), scale)
    if div:
        d = run_divergence_backward(cs, o, run_divergence_forward(cs, o))
        check_divergence(cs, o, d, rep, tiles, wgrad=False)


def wgrad_sweep(model):
    """cfg4's fine pass of `model` (a key of MODELS): M_SWEEP backward passes on one forward stash, each with upstreams on
    one residue class of tiles."""
    cs = Case(8192, 128, **MODELS[model])
    o = run_forward(cs)
    rep = Report(f"{model} 8192x128 sweep m={M_SWEEP}", quiet=True)
    for j in range(M_SWEEP):
        cj = only_on_tiles(cs, tile_set(cs, M_SWEEP, j))
        b = run_backward(cj, o)
        imgs = dgrad_reference(cj, o, b, rep, expected_scale(cj), tile_set(cs, M_SWEEP, j))
        check_wgrad(cj, b, imgs, rep, expected_scale(cj))
    rep.worst()


def test_every_tile_enters_every_wgrad_job_exactly_once():
    """The bending model's fine pass at cfg4: every WGRAD job of the plan with a bender."""
    wgrad_sweep("bender")


def test_every_tile_enters_every_tc_wgrad_job_exactly_once():
    """The time-conditioned baseline's fine pass at cfg4: the bender-less plan and wgrad_reduce_tc_kernel, the latent
    columns of W0 / W5 from the pass's rays only."""
    wgrad_sweep("tc")


def divergence_sweep(cs, o, d, m, tag):
    rep = Report(tag, quiet=True)
    for j in range(m):
        cj = only_on_tiles(cs, tile_set(cs, m, j))
        run_divergence_backward(cj, o, d)
        check_divergence(cj, o, d, rep, tile_set(cs, m, j))
    rep.worst()


def test_divergence_compact_wgrad_sees_every_tile_exactly_once():
    """cfg4's coarse pass: the divergence backward M_SWEEP times on one divergence forward."""
    cs = Case(8192, 64)
    o = run_forward(cs)
    divergence_sweep(cs, o, run_divergence_forward(cs, o), M_SWEEP, f"8192x64 divergence sweep m={M_SWEEP}")


def test_masks_past_2_31_and_divergence_stashes_past_2_32():
    """53,248 x 128 points: the forward's stash (33.8 GB) and masks (2.2 GB, past 2^31), then, with the stash freed, the
    divergence forward / backward (tangent 5.0 GB and adjoint 4.8 GB, past 2^32) and the compact WGRAD sweep."""
    n, s = 53248, 128
    lib = _lib().load()
    need = lib.nrn_stash_bytes(n, s) + lib.nrn_relu_mask_bytes(n, s) + (3 << 30)
    torch.cuda.empty_cache()      # what earlier tests left in the caching allocator is free for this case
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of device memory, {free / 2 ** 30:.1f} GiB free")
    cs = Case(n, s)
    assert lib.nrn_relu_mask_bytes(n, s) > 2 ** 31 and lib.nrn_div_stash_bytes(n, s) > 2 ** 32
    assert lib.nrn_div_grad_stash_bytes(n, s) > 2 ** 32
    tag = f"{n}x{s}"
    rep = Report(tag)
    tiles = sample_tiles(cs, ("stash", "masks"))
    print(f"  [{tag}] {cs.T} tiles; forward sampled {tiles}")
    o = run_forward(cs)
    check_forward(cs, o, rep, tiles)
    del o["stash"]        # the divergence kernels read the masks, not the stash
    d = run_divergence_forward(cs, o)
    run_divergence_backward(cs, o, d)
    tiles = sample_tiles(cs, ("masks", "tangent", "adjoint"))
    print(f"  [{tag}] divergence sampled {tiles}")
    check_divergence(cs, o, d, rep, tiles, wgrad=False)
    divergence_sweep(cs, o, d, M_SWEEP, f"{tag} divergence sweep m={M_SWEEP}")
    print(f"  [{tag}] ran: masks {lib.nrn_relu_mask_bytes(n, s)} B, tangent {lib.nrn_div_stash_bytes(n, s)} B, "
          f"adjoint {lib.nrn_div_grad_stash_bytes(n, s)} B")


@pytest.mark.parametrize("model", list(MODELS))
def test_dgrad_and_wgrad_on_masks_past_2_31(model):
    """52,480 x 128 points, the smallest shape whose ReLU masks (2.15 GB) pass 2^31 bytes, forward and backward: the stash
    (33.3 GB) and gradient stash (32.5 GB) past 2^34.  Every stage on the tiles at the byte boundaries of all three
    buffers (and the persistent CTAs' last sweep, which straddles the masks' 2^31); dense WGRAD; then a second backward
    on the same forward stash with upstreams only on those tiles, whose WGRAD is checked per element at
    c_wgrad(len(tiles)): one tile read from the wrong place fails it by orders of magnitude, where the dense relative L2
    moves by about 2e-5."""
    n, s = 52480, 128
    lib = _lib().load()
    need = lib.nrn_stash_bytes(n, s) + lib.nrn_relu_mask_bytes(n, s) + lib.nrn_grad_stash_bytes(n, s) + (3 << 30)
    torch.cuda.empty_cache()      # what earlier tests left in the caching allocator is free for this case
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of device memory, {free / 2 ** 30:.1f} GiB free")
    assert lib.nrn_relu_mask_bytes(n, s) > 2 ** 31 and lib.nrn_grad_stash_bytes(n, s) > 2 ** 34
    t_start = time.perf_counter()
    cs = Case(n, s, **MODELS[model])
    tag = f"{model} {n}x{s}"
    rep = Report(tag)
    tiles = sample_tiles(cs, ("stash", "masks", "grad stash"))
    print(f"  [{tag}] {cs.T} tiles; sampled {tiles}")
    o = run_forward(cs)
    check_forward(cs, o, rep, tiles)
    b = run_backward(cs, o)
    scale = expected_scale(cs)
    dgrad_reference(cs, o, b, rep, scale, tiles)
    grad_stash_stats(cs, o, b, tag)
    dense_wgrad(cs, o, b, Report(f"{tag} dense"), scale)
    del b
    cj = only_on_tiles(cs, tiles)
    b = run_backward(cj, o)
    rep = Report(f"{tag} upstream on the sampled tiles only")
    scale = expected_scale(cj)
    check_wgrad(cj, b, dgrad_reference(cj, o, b, rep, scale, tiles), rep, scale)
    torch.cuda.synchronize()
    print(f"  [{tag}] ran: stash {lib.nrn_stash_bytes(n, s)} B, masks {lib.nrn_relu_mask_bytes(n, s)} B, gradient stash "
          f"{lib.nrn_grad_stash_bytes(n, s)} B; {time.perf_counter() - t_start:.1f} s")


# ----------------------------------------------------------------------------------------------------------------------
# inference at the render chunk, and the whole cfg4 training step
# ----------------------------------------------------------------------------------------------------------------------
SEED_STEP = 8192


def f32_bits_equal(a, b):
    """bit-for-bit equality of float32 tensors, NaN included"""
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def render_chunk(model):
    """render() of `model` (a key of MODELS) at one 65,536-ray chunk as the render workload runs it (64 coarse + 64
    importance samples, perturb 0, no noise, one latent row for every ray, detailed output): 98,304 fine tiles per field
    launch; for the time-conditioned baseline that broadcast latent is a single ray-bias row for every ray.  Sampled rays
    (the first, the last, those of the persistent CTAs' first and last sweep, and random ones) equal a separate call on
    just those
    rays bit for bit, every per-ray and per-sample output included; and the fine compositing of those rays holds the fp64
    bounds of tests/test_ray_kernels_parity_gpu.py on the kernel's own raw and alpha."""
    import oracle.nrnerf_oracle as O
    from nonrigid_nerf_b200 import _lib as L, train as T
    from tests import helpers, ray_reference as RR
    from tests.test_ray_kernels_parity_gpu import UNDERFLOW, c_scan
    n, S = 65536, 128
    if model == "tc":
        coarse, fine, _ = helpers.tc_models(SEED_STEP, DEV)
        bender = None
    else:
        coarse, fine, bender, _ = helpers.build_models(O, SEED_STEP, DEV)
    r = O.make_rays(SEED_STEP, n)
    ro, rd = r["rays_o"].to(DEV), r["rays_d"].to(DEV)
    lat = r["latents"][0].to(DEV)
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=64, network_fine=fine, N_samples=64, network_fn=coarse,
              ray_bender=bender, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False,
              near=r["near"], far=r["far"])

    def call(sel):
        m = sel.shape[0]
        with torch.no_grad():
            rgb, disp, acc, ex = T.render(ro[sel], rd[sel], chunk=65536, detailed_output=True, retraw=True,
                                          additional_pixel_information={"ray_bending_latents": lat[None].expand(m, 32)}, **kw)
        L.device_error_check()
        return dict(ex, rgb_map=rgb, disp_map=disp, acc_map=acc)

    full = call(torch.arange(n, device=DEV))
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    rays = {0, 1, n - 2, n - 1}
    for s_pass in (64, S + 64):                       # the coarse and the fine field launch: tiles of 128 samples
        T_pass = n * s_pass // SL.TILE_M
        for t in (sms - 1, sms, T_pass - sms - 1, T_pass - sms):
            rays.update({t * SL.TILE_M // s_pass, (t * SL.TILE_M + SL.TILE_M - 1) // s_pass})
    rays.update(torch.randint(0, n, (24,), generator=torch.Generator().manual_seed(3)).tolist())
    sel = torch.tensor(sorted(rays), device=DEV)
    small = call(sel)
    assert set(small) == set(full)
    for k, v in full.items():
        if v.is_floating_point() and v.shape[0] == n:
            assert f32_bits_equal(v[sel], small[k]), f"{k}: the {n}-ray chunk differs from a {sel.shape[0]}-ray call"
    print(f"  [{model} render {n} rays] {sel.shape[0]} sampled rays equal a separate call bit for bit in {len(full)} outputs")
    rep = Report(f"{model} render {n} rays, sampled")
    raw, alpha = small["raw"], small["fine_opacity_alpha"]
    ref = RR.composite_ref(alpha, raw, torch.zeros_like(alpha))          # depth and disp need z, which render() keeps
    for k, got in (("weights", small["fine_visibility_weights"]), ("rgb", small["rgb_map"]), ("acc", small["acc_map"])):
        rep.check(f"fine {k}", got, *ref[k], c_scan(S + 64), floor=UNDERFLOW)


def test_render_chunk_rays_equal_a_small_call_and_composite_within_fp64_bounds():
    """The bending model's render chunk (render_chunk)."""
    render_chunk("bender")


def test_tc_render_chunk_rays_equal_a_small_call_and_composite_within_fp64_bounds():
    """The time-conditioned baseline's render chunk (render_chunk): one ray-bias row serves all 65,536 rays."""
    render_chunk("tc")


def cfg4_setup(seed, n, n_iters):
    """bench.py --workload cfg4's step inputs at n rays: models, an 86-row latent table, (image, y, x) pixel indices, and
    every random draw injected (render_rays' four and the divergence probes)."""
    import types
    import oracle.nrnerf_oracle as O
    from nonrigid_nerf_b200 import optim
    from tests import helpers
    n_images = 86
    coarse, fine, bender, params = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    g = torch.Generator().manual_seed(seed)
    rnd = {k: v.to(DEV) for k, v in O.make_randomness(seed, n, 64, 64).items()}
    rnd["e"] = torch.randn(n, 64, 3, generator=g).to(DEV)
    table = (torch.randn(n_images, 32, generator=g) * 0.1).to(DEV)
    pix = torch.stack([torch.randint(0, n_images, (n,), generator=g), torch.randint(0, 384, (n,), generator=g),
                       torch.randint(0, 512, (n,), generator=g)], 1).to(DEV)
    latents = [table[i].clone().requires_grad_(True) for i in range(n_images)]
    opt = optim.Adam(latents + list(bender.parameters()) + list(coarse.parameters()) + list(fine.parameters()), lr=5e-4)
    targs = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=n_iters, offsets_loss_weight=60.0,
                                  divergence_loss_weight=3.0, rigidity_loss_weight=0.0005, ray_bending_latent_size=32)
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64,
          "network_fn": coarse, "ray_bender": bender, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": 1.0,
          "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"], "randomness": rnd}
    inputs = [r["rays_o"].to(DEV), r["rays_d"].to(DEV), r["target"].to(DEV), pix]
    extras = {"imageid_to_timestepid": list(range(n_images))}
    return dict(models=(coarse, fine, bender), params=params, r=r, rnd=rnd, table=table, latents=latents, opt=opt,
                targs=targs, kw=kw, inputs=inputs, extras=extras)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def test_cfg4_training_step_matches_the_fp32_oracle():
    """training_wrapper_class at 8,192 rays (64 + 64 samples, offsets, rigidity and divergence terms) against the fp32
    oracle's training_wrapper_loss run on the GPU with TF32 off, in chunks of 1,024 rays whose gradients add up: the
    per-ray loss and every parameter gradient within DESIGN section 2's bounds for 1,024 rays."""
    import oracle.nrnerf_oracle as O
    from nonrigid_nerf_b200 import _lib as L, parallel
    n, global_step = 8192, 1000
    st = cfg4_setup(SEED_STEP, n, 200000)
    coarse, fine, bender = st["models"]
    ro, rd, target, pix = st["inputs"]
    wrapper = parallel.training_wrapper_class(coarse, st["latents"], fine_model=fine, ray_bender=bender)
    loss = wrapper(st["targs"], ro, rd, 100, st["kw"], target, global_step, 0, st["extras"], pix)
    loss.mean().backward()
    L.device_error_check()

    def dev_params(p):
        return {k: [t.to(DEV).requires_grad_(True) for t in v] if isinstance(v, list) else v.to(DEV).requires_grad_(True)
                for k, v in p.items()}

    cpo, fpo, bpo = (dev_params(p) for p in st["params"])
    table = st["table"].clone().requires_grad_(True)
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        ref = []
        for a in range(0, n, 1024):
            sl = slice(a, a + 1024)
            rays = {"rays_o": ro[sl], "rays_d": rd[sl], "near": st["r"]["near"], "far": st["r"]["far"], "target": target[sl]}
            rnd = {k: v[sl] for k, v in st["rnd"].items() if k != "e"}
            lo, _ = O.training_wrapper_loss(cpo, fpo, bpo, rays, table, st["extras"]["imageid_to_timestepid"], pix[sl], rnd,
                                            st["rnd"]["e"][sl].reshape(-1, 3), global_step, st["targs"].N_iters, 60.0, 3.0,
                                            0.0005)
            (lo.sum() / n).backward()
            ref.append(lo.detach())
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    ref = torch.cat(ref)
    d, rel = float((loss.detach() - ref).abs().max()), _rel(loss.detach(), ref)
    print(f"  [cfg4 step] per-ray loss vs fp32 oracle: L-inf {d:.3e}, rel L2 {rel:.3e}")
    assert d <= 2e-3 and rel <= 2e-3, (d, rel)
    worst = {}
    checks = []
    for net, po, nm in ((coarse, cpo, "coarse"), (fine, fpo, "fine")):
        for i in range(8):
            checks += [(f"{nm} W{i}", net.pts_linears[i].weight.grad, po["pts_w"][i].grad, 5e-2),
                       (f"{nm} b{i}", net.pts_linears[i].bias.grad, po["pts_b"][i].grad, 5e-2)]
        checks.append((f"{nm} head", net.output_linear.weight.grad, po["out_w"].grad, 2e-2))
    for i in range(5):
        checks.append((f"bender net W{i}", bender.network[i].weight.grad, bpo["net_w"][i].grad, 8e-2))
    for i in range(3):
        checks.append((f"bender rigidity W{i}", bender.rigidity_network[i].weight.grad, bpo["rig_w"][i].grad, 8e-2))
    checks.append(("latent table", torch.stack([l.grad for l in st["latents"]]), table.grad, 8e-2))
    for nm, got, exp, tol in checks:
        e = _rel(got, exp)
        worst[nm] = e
        assert e <= tol, (nm, e, tol)
    print("  [cfg4 step] gradient rel L2 vs fp32 oracle: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


LRS_STEP = [5e-4, 5e-4, 5e-4, 2e-3, 0.0, 1e-3]   # steps 1..6; the graph's 3 warm-up steps run at the first value
LOSS_REL_STEP = 1e-5


def _cfg4_run(graph):
    """Six steps of bench.py's local_step at 8,192 rays (Adam, a device-scalar global_step, N_iters = 8 so that the
    regularisers' weights change strongly per step): eagerly, or 3 warm-up steps inside GraphedStep and 3 replays.
    Returns per step (losses, parameters before, parameters after) for the steps run after the warm-up."""
    from nonrigid_nerf_b200 import _lib as L, parallel
    from nonrigid_nerf_b200.graphs import GraphedStep
    st = cfg4_setup(SEED_STEP, 8192, 8)
    coarse, fine, bender = st["models"]
    opt, inputs = st["opt"], st["inputs"]
    wrapper = parallel.training_wrapper_class(coarse, st["latents"], fine_model=fine, ray_bender=bender)
    global_step = torch.zeros((), dtype=torch.float32, device=DEV)
    n = inputs[0].shape[0]

    def local_step(rays_o, rays_d, target, pix):
        opt.zero_grad()
        losses = wrapper(st["targs"], rays_o, rays_d, 100, st["kw"], target, global_step, 0, st["extras"], pix)
        (losses.sum() / n).backward()
        opt.step()
        global_step.add_(1.0)
        return losses.detach()

    first = 3 if graph else 0
    if graph:
        opt.set_lr(LRS_STEP[0])
        run = GraphedStep(local_step, inputs, warmup=3)
    else:
        run = local_step
    out = []
    for i in range(first, 6):
        opt.set_lr(LRS_STEP[i])
        p0 = opt._flat.clone()
        losses = run(*inputs)
        torch.cuda.synchronize()
        out.append((losses.clone(), p0, opt._flat.clone()))
    L.device_error_check()
    assert float(global_step) == 6
    return out[-3:]


def test_cfg4_graphed_step_matches_eager():
    """bench.py --workload cfg4's step replayed from a CUDA graph (GraphedStep, plain Adam), set_lr between replays and
    one replay at lr = 0, against eager steps 4..6 from the same initial state; two eager runs bound the spread that the
    fp32 atomics of the latent gradient and the divergence loss leave."""
    eager, eager2, graph = _cfg4_run(False), _cfg4_run(False), _cfg4_run(True)
    spread = max(_rel(a[0], b[0]) for a, b in zip(eager2, eager))
    print(f"  [cfg4 graph] eager vs eager, steps 4..6: max rel L2 {spread:.3e}")
    assert spread <= LOSS_REL_STEP, spread
    for j, ((le, pe0, pe1), (lg, pg0, pg1)) in enumerate(zip(eager, graph)):
        step = 4 + j
        d = _rel(lg, le)
        print(f"  [cfg4 graph] step {step} lr {LRS_STEP[step - 1]:g}: replay vs eager per-ray loss rel L2 {d:.3e}")
        assert d <= LOSS_REL_STEP, (step, d)
        if LRS_STEP[step - 1] == 0.0:
            assert f32_bits_equal(pg1, pg0) and f32_bits_equal(pe1, pe0), f"step {step}: lr = 0 moved the parameters"
        else:
            assert not f32_bits_equal(pg1, pg0), f"step {step}: the replay did not move the parameters"
