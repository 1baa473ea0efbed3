"""Training the view-dependent head without a bender (NeRF(use_viewdirs=True), rigid scenes) at the benchmark's cfg4
batch and past 2^31 / 2^32 bytes of its stashes, stage by stage against the fp64 references of tests/stage_reference.py
(Case(views=True); bounds as in tests/test_viewdirs_train_stages_gpu.py), with the sampled-tile rule of
tests/test_scale_gpu.py: 0 and T - 1, the tiles at each 2^31 .. 2^34 byte boundary of the named buffers and their
neighbours, and the persistent CTAs' first and last grid sweep.  Every caller-owned buffer is filled with 0xFF first.

  cfg4 passes   8192 x 64 and 8192 x 128: every stage on sampled tiles (the trunk's stash and gradient stash past 2^31 /
                2^32), and WGRAD dense over every tile against an fp64 sum streamed in blocks of 256 tiles, at c_wgrad(T)
                and at wgrad_rel_l2 of the deepest split of the replicated views plan
  coverage      8192 x 128: 97 backward passes on one forward stash, pass j with d_raw only on the tiles t = j (mod 97),
                every trunk and head element at c_wgrad(T / 97): a tile dropped, repeated or misaddressed in the head jobs
                12-15 or in wgrad_views_reduce_kernel fails its bound by about two orders of magnitude
  22,528 x 128  forward and backward: the view stash (2.40 GB) and view gradient stash (2.21 GB) past 2^31, the trunk's
                stash (14.3 GB) and gradient stash (13.9 GB) past 2^33; every stage on the boundary tiles, then dense
                WGRAD.  About 34 GB; skipped with the GiB it needs when the device has less free
  40,960 x 128  forward only: the view stash (4.36 GB) past 2^32; about 32 GB.  Its backward would need about 30 GB more
                (gradient stashes of 25.2 and 4.0 GB) and is not run
  cfg4 step     training_wrapper_class at 8,192 rays (64 + 64 samples, perturb 1, noise 1, injected randomness) against
                the fp32 oracle on the GPU with TF32 off, in 1,024-ray chunks: per-ray loss and every gradient; the
                latents get no gradient, as in the reference
  graph replay  that step under GraphedStep (plain Adam, set_lr between replays, one at lr = 0): this path has no fp32
                atomics (no latent gradient, a deterministic WGRAD reduce), so two eager runs must be bit-identical, and
                the replay must equal them bit for bit

Faults these checks are meant to catch: a 32-bit byte offset into the view stash, the view gradient stash or the Hv
masks (the boundary tiles), a head job's split reading the wrong tiles or none (the sweep, and the dense relative L2),
wrong stash rows at the CTAs' last sweep, and anything the graph capture changes (replay vs eager).

Measured on one H100 80GB HBM3 (700 W power limit, 132 SMs), printed with `pytest -s`; the file's tests run in about
15 s, and both large cases ran (80 GB free).
  worst c_obs   H1 .. H8 2.7 of 258 (22,528 x 128), Hv 6.3 of 290, DGRAD dY0 .. dY7 4.0 of 258, WGRAD swept 8.2 of 1,424,
                dense 82.8 of 360,512 (W0, 22,528 tiles)
  dense WGRAD   relative L2, deepest split of the views plan 2,731 / 7,510 tiles: at 8,192 tiles at most 4.6e-4
                (rgb_linear), W0 2.9e-4; at 22,528 tiles at most 9.9e-4 (alpha_linear), W0 8.0e-4
  cfg4 step     per-ray loss 1.0e-5 relative; gradients at most 9.7e-3 (coarse W0)
  graph replay  two eager runs and the replay bit-identical
"""
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import stash_layout as SL
from tests.parity import DEV, Report
from tests.stage_reference import (Case, Tiles, _lib, check_forward, check_wgrad, dgrad_reference, expected_scale,
                                   run_backward, run_forward, split_ranges, wgrad_images, wgrad_plan, wgrad_reference,
                                   wgrad_rel_l2)
from tests.test_scale_gpu import BLOCK, M_SWEEP, f32_bits_equal, only_on_tiles, sample_tiles, tile_set

pytestmark = pytest.mark.gpu


def dense_wgrad_views(cs, o, b, rep, scale):
    """WGRAD against the fp64 sum over every tile, streamed over blocks of BLOCK tiles."""
    tot = None
    for t0 in range(0, cs.T, BLOCK):
        sub = Tiles(cs, range(t0, min(t0 + BLOCK, cs.T)))
        imgs = wgrad_images(cs, o, b, sub)
        imgs["sub"] = sub
        ref, _ = wgrad_reference(cs, imgs)
        if tot is None:
            tot = ref
        else:
            for k, (v, a) in ref.items():
                tot[k] = (tot[k][0] + v, tot[k][1] + a)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    plan = wgrad_plan(cs.T, sms & ~1, views=True)
    depth = {j: max(e - s for s, e in split_ranges(cs.T, n)) for j, n in plan.items()}
    rel = wgrad_rel_l2(max(depth.values()))
    print(f"  [{rep.tag}] views WGRAD plan at {sms} CTAs: splits {plan}; tiles per split {depth}; rel L2 bound {rel:.2e}")
    check_wgrad(cs, b, None, rep, scale, refs=(tot, None), n_tiles=cs.T, rel_l2=rel)


def _free_gib_or_skip(need):
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of device memory, {free / 2 ** 30:.1f} GiB free")


def _fwd_bytes(lib, n, s):
    return sum(f(n, s) for f in (lib.nrn_stash_bytes, lib.nrn_relu_mask_bytes, lib.nrn_views_stash_bytes, lib.nrn_hv_mask_bytes))


def _bwd_bytes(lib, n, s):
    return lib.nrn_grad_stash_bytes(n, s) + lib.nrn_views_grad_stash_bytes(n, s)


@pytest.mark.parametrize("n,s", [(8192, 64), (8192, 128)])
def test_cfg4_views_pass_every_stage_on_sampled_tiles_and_dense_wgrad(n, s):
    cs = Case(n, s, views=True)
    tag = f"views {n}x{s}"
    tiles = sample_tiles(cs, ("stash", "grad stash"))
    rep = Report(tag)
    print(f"  [{tag}] {cs.T} tiles; sampled {tiles}")
    o = run_forward(cs)
    check_forward(cs, o, rep, tiles)
    b = run_backward(cs, o)
    scale = expected_scale(cs)
    dgrad_reference(cs, o, b, rep, scale, tiles)
    dense_wgrad_views(cs, o, b, Report(f"{tag} dense"), scale)


def test_every_tile_enters_every_views_wgrad_job_exactly_once():
    """8192 x 128: M_SWEEP backward passes on one forward stash, each with d_raw on one residue class of tiles."""
    cs = Case(8192, 128, views=True)
    o = run_forward(cs)
    rep = Report(f"views 8192x128 sweep m={M_SWEEP}", quiet=True)
    for j in range(M_SWEEP):
        cj = only_on_tiles(cs, tile_set(cs, M_SWEEP, j))
        b = run_backward(cj, o)
        scale = expected_scale(cj)
        imgs = dgrad_reference(cj, o, b, rep, scale, tile_set(cs, M_SWEEP, j))
        check_wgrad(cj, b, imgs, rep, scale)
        del b, imgs
    rep.worst()


def test_views_stashes_past_2_31_forward_and_backward():
    """22,528 x 128: the view stash and view gradient stash past 2^31 bytes, the trunk's stashes past 2^33."""
    n, s = 22528, 128
    lib = _lib().load()
    _free_gib_or_skip(_fwd_bytes(lib, n, s) + _bwd_bytes(lib, n, s) + (3 << 30))
    assert lib.nrn_views_stash_bytes(n, s) > 2 ** 31 and lib.nrn_views_grad_stash_bytes(n, s) > 2 ** 31
    assert lib.nrn_stash_bytes(n, s) > 2 ** 33 and lib.nrn_grad_stash_bytes(n, s) > 2 ** 33
    cs = Case(n, s, views=True)
    tag = f"views {n}x{s}"
    rep = Report(tag)
    tiles = sample_tiles(cs, ("views stash", "views grad stash", "stash", "grad stash"))
    print(f"  [{tag}] {cs.T} tiles; sampled {tiles}")
    o = run_forward(cs)
    check_forward(cs, o, rep, tiles)
    b = run_backward(cs, o)
    scale = expected_scale(cs)
    dgrad_reference(cs, o, b, rep, scale, tiles)
    dense_wgrad_views(cs, o, b, Report(f"{tag} dense"), scale)


def test_views_stash_past_2_32_forward():
    """40,960 x 128, forward only: the view stash past 2^32 bytes (and the trunk's stash past 2^34).  The backward at this
    size would need its gradient stashes, about 30 GB more, and is not run; the 22,528 x 128 case covers the view
    gradient stash past 2^31."""
    n, s = 40960, 128
    lib = _lib().load()
    _free_gib_or_skip(_fwd_bytes(lib, n, s) + (3 << 30))
    assert lib.nrn_views_stash_bytes(n, s) > 2 ** 32 and lib.nrn_stash_bytes(n, s) > 2 ** 34
    cs = Case(n, s, views=True)
    tag = f"views {n}x{s}"
    tiles = sample_tiles(cs, ("views stash", "stash"))
    print(f"  [{tag}] {cs.T} tiles; sampled {tiles}")
    o = run_forward(cs)
    check_forward(cs, o, Report(tag), tiles)


# ----------------------------------------------------------------------------------------------------------------------
# the whole cfg4 training step
# ----------------------------------------------------------------------------------------------------------------------
SEED_STEP = 8193
N_IMAGES = 86


def views_setup(seed, n, n_iters):
    """cfg4's step inputs for a rigid scene with the view-dependent head: coarse and fine NeRF(use_viewdirs=True), no
    bender, an 86-row latent table (which gets no gradient), (image, y, x) pixel indices and injected random draws."""
    import types
    from nonrigid_nerf_b200 import optim
    from tests.viewdirs_reference import build_view_models
    coarse, fine, _, (cp, fp, _, vc, vf) = build_view_models(O, seed, DEV, with_bender=False)
    r = O.make_rays(seed, n)
    g = torch.Generator().manual_seed(seed)
    rnd = {k: v.to(DEV) for k, v in O.make_randomness(seed, n, 64, 64).items()}
    table = (torch.randn(N_IMAGES, 32, generator=g) * 0.1).to(DEV)
    pix = torch.stack([torch.randint(0, N_IMAGES, (n,), generator=g), torch.randint(0, 384, (n,), generator=g),
                       torch.randint(0, 512, (n,), generator=g)], 1).to(DEV)
    latents = [table[i].clone().requires_grad_(True) for i in range(N_IMAGES)]
    opt = optim.Adam(latents + list(coarse.parameters()) + list(fine.parameters()), lr=5e-4)
    targs = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=n_iters, offsets_loss_weight=0.0,
                                  divergence_loss_weight=0.0, rigidity_loss_weight=0.0, ray_bending_latent_size=32)
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64,
          "network_fn": coarse, "ray_bender": None, "use_viewdirs": True, "white_bkgd": False, "raw_noise_std": 1.0,
          "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"], "randomness": rnd}
    inputs = [r["rays_o"].to(DEV), r["rays_d"].to(DEV), r["target"].to(DEV), pix]
    extras = {"imageid_to_timestepid": list(range(N_IMAGES))}
    return dict(models=(coarse, fine), params=(cp, fp, vc, vf), r=r, rnd=rnd, table=table, latents=latents, opt=opt,
                targs=targs, kw=kw, inputs=inputs, extras=extras)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


HEAD_MODULES = (("views_linears.0", "views"), ("feature_linear", "feature"), ("alpha_linear", "alpha"), ("rgb_linear", "rgb"))


def grads_against_oracle(coarse, fine, po, tag, tol=8e-2):
    """Every parameter gradient of the two models against the oracle's (po: (cp, fp, vc, vf) with .grad), relative L2
    per tensor within DESIGN section 2's 5-8 % bound; returns the worst."""
    cp, fp, vc, vf = po
    worst = {}
    for net, p, v, nm in ((coarse, cp, vc, "coarse"), (fine, fp, vf, "fine")):
        checks = []
        for i in range(8):
            checks += [(f"{nm} W{i}", net.pts_linears[i].weight.grad, p["pts_w"][i].grad),
                       (f"{nm} b{i}", net.pts_linears[i].bias.grad, p["pts_b"][i].grad)]
        for mod, key in HEAD_MODULES:
            m = net.get_submodule(mod)
            checks += [(f"{nm} {mod}.weight", m.weight.grad, v[key + "_w"].grad), (f"{nm} {mod}.bias", m.bias.grad, v[key + "_b"].grad)]
        for k, got, exp in checks:
            assert got is not None and exp is not None, k
            assert bool(torch.isfinite(got).all()), k
            worst[k] = _rel(got, exp)
            assert worst[k] <= tol, (k, worst[k], tol)
    print(f"  [{tag}] gradient rel L2 vs fp32 oracle: worst {max(worst.values()):.2e} ({max(worst, key=worst.get)}); " +
          ", ".join(f"{k} {e:.1e}" for k, e in worst.items()))
    return worst


def test_cfg4_views_training_step_matches_the_fp32_oracle():
    """training_wrapper_class at 8,192 rays against the oracle's training_wrapper_loss (vpar_c / vpar_f) on the GPU with
    TF32 off, in chunks of 1,024 rays whose gradients add up."""
    from nonrigid_nerf_b200 import _lib as L, parallel
    n, global_step = 8192, 1000
    st = views_setup(SEED_STEP, n, 200000)
    coarse, fine = st["models"]
    ro, rd, target, pix = st["inputs"]
    wrapper = parallel.training_wrapper_class(coarse, st["latents"], fine_model=fine)
    loss = wrapper(st["targs"], ro, rd, 100, st["kw"], target, global_step, 0, st["extras"], pix)
    loss.mean().backward()
    L.device_error_check()
    assert all(l.grad is None or not bool(l.grad.any()) for l in st["latents"]), "the latents got a gradient"

    def dev_params(p):
        return {k: [t.to(DEV).requires_grad_(True) for t in v] if isinstance(v, list) else v.to(DEV).requires_grad_(True)
                for k, v in p.items()}

    po = tuple(dev_params(O.clone_params(p)) for p in st["params"])
    table = st["table"].clone().requires_grad_(True)
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        ref = []
        for a in range(0, n, 1024):
            sl = slice(a, a + 1024)
            rays = {"rays_o": ro[sl], "rays_d": rd[sl], "near": st["r"]["near"], "far": st["r"]["far"], "target": target[sl]}
            rnd = {k: v[sl] for k, v in st["rnd"].items()}
            lo, _ = O.training_wrapper_loss(po[0], po[1], None, rays, table, st["extras"]["imageid_to_timestepid"], pix[sl], rnd,
                                            None, global_step, st["targs"].N_iters, 0.0, 0.0, 0.0, vpar_c=po[2], vpar_f=po[3])
            (lo.sum() / n).backward()
            ref.append(lo.detach())
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    ref = torch.cat(ref)
    d, rel = float((loss.detach() - ref).abs().max()), _rel(loss.detach(), ref)
    print(f"  [views cfg4 step] per-ray loss vs fp32 oracle: L-inf {d:.3e}, rel L2 {rel:.3e}")
    assert d <= 2e-3 and rel <= 2e-3, (d, rel)
    assert table.grad is None or not bool(table.grad.any()), "the oracle's latents got a gradient"
    grads_against_oracle(coarse, fine, po, "views cfg4 step")


LRS_STEP = [5e-4, 5e-4, 5e-4, 2e-3, 0.0, 1e-3]   # steps 1..6; the graph's 3 warm-up steps run at the first value


def _views_run(graph):
    """Six steps at 8,192 rays (Adam, a device-scalar global_step): eagerly, or 3 warm-up steps inside GraphedStep and 3
    replays.  Returns per step (losses, parameters before, parameters after) for the steps run after the warm-up."""
    from nonrigid_nerf_b200 import _lib as L, parallel
    from nonrigid_nerf_b200.graphs import GraphedStep
    st = views_setup(SEED_STEP, 8192, 8)
    coarse, fine = st["models"]
    opt, inputs = st["opt"], st["inputs"]
    wrapper = parallel.training_wrapper_class(coarse, st["latents"], fine_model=fine)
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


def test_cfg4_views_graphed_step_equals_eager_bit_for_bit():
    """Two eager runs of steps 1..6 are bit-identical (no fp32 atomics on this path), and GraphedStep's replays of steps
    4..6 equal them bit for bit: losses and every parameter; lr = 0 leaves the parameters untouched."""
    eager, eager2, graph = _views_run(False), _views_run(False), _views_run(True)
    for j, ((le, pe0, pe1), (le2, _, pe12), (lg, pg0, pg1)) in enumerate(zip(eager, eager2, graph)):
        step = 4 + j
        assert f32_bits_equal(le, le2) and f32_bits_equal(pe1, pe12), f"step {step}: two eager runs differ"
        assert f32_bits_equal(lg, le), f"step {step}: replay vs eager per-ray loss differs, rel L2 {_rel(lg, le):.3e}"
        assert f32_bits_equal(pg0, pe0) and f32_bits_equal(pg1, pe1), f"step {step}: replay vs eager parameters differ"
        if LRS_STEP[step - 1] == 0.0:
            assert f32_bits_equal(pg1, pg0), f"step {step}: lr = 0 moved the parameters"
        else:
            assert not f32_bits_equal(pg1, pg0), f"step {step}: the replay did not move the parameters"
    print("  [views cfg4 graph] steps 4..6: two eager runs and the replay are bit-identical in losses and parameters")
