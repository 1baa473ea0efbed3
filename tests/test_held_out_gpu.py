"""Held-out rays (render(..., held_out=)) on the GPU.

One backward of ((train + test) * loss).mean() with held_out=test must give the gradients of the reference loop's two
backward passes (train.py:1595-1608): test rays reach their latent codes only, with a bender; without one they add nothing.
Checked end to end against the port's own two-pass loop at 96, 1,024 and 8,192 rays, and stage by stage: the held-out
DGRAD and divergence backward write the gradient-stash / adjoint-stash rows of training rays bit for bit as the ordinary
kernels do and those of held-out rays as zeros."""
import ctypes as C

import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_FRAMES, HELD_FRAMES = 7, (2, 5)   # about 2/7 of the images held out, as with test_block_size / train_block_size


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _targs():
    import types
    # example_sequence's regularisers: offsets 60 (rigidity 0.0005), divergence 3
    return types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=200000, offsets_loss_weight=60.0,
                                 divergence_loss_weight=3.0, rigidity_loss_weight=0.0005, ray_bending_latent_size=32)


def _setup(seed, n, with_bender=True, tc=False, views=False):
    if tc:
        coarse, fine, _ = helpers.tc_models(seed, DEV)
        bender = None
    elif views:
        from tests.viewdirs_reference import build_view_models
        coarse, fine, bender, _ = build_view_models(O, seed, DEV, with_bender=False)
    else:
        coarse, fine, bender, _ = helpers.build_models(O, seed, DEV, with_bender=with_bender)
    r = O.make_rays(seed, n)
    rnd = dict(O.make_randomness(seed, n, 64, 64))
    g = torch.Generator().manual_seed(seed + 9)
    rnd["e"] = torch.randn(n * 64, 3, generator=g)
    latents = [(0.1 * torch.randn(32, generator=g)).to(DEV).requires_grad_(True) for _ in range(N_FRAMES)]
    pix = torch.stack([torch.randint(N_FRAMES, (n,), generator=g), torch.zeros(n, dtype=torch.long),
                       torch.zeros(n, dtype=torch.long)], -1).to(DEV)
    test = torch.isin(pix[:, 0], torch.tensor(HELD_FRAMES, device=DEV))
    return coarse, fine, bender, r, rnd, latents, pix, test


def _loss(coarse, fine, bender, r, rnd, latents, pix, held_out=None):
    from nonrigid_nerf_b200 import parallel
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64,
          "network_fn": coarse, "ray_bender": bender, "use_viewdirs": bool(getattr(coarse, "use_viewdirs", False)),
          "white_bkgd": False, "raw_noise_std": 1.0,
          "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"], "randomness": rnd}
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
    return wrapper(_targs(), r["rays_o"].to(DEV), r["rays_d"].to(DEV), 100, kw, r["target"].to(DEV), 1000, 0,
                   {"imageid_to_timestepid": list(range(N_FRAMES))}, pix, held_out=held_out)


def _weights(coarse, fine, bender):
    named = [("coarse." + k, v) for k, v in coarse.named_parameters()] + [("fine." + k, v) for k, v in fine.named_parameters()]
    if bender is not None:
        named += [("bender." + k, v) for k, v in bender.named_parameters()]
    return named


def _clear(named, latents):
    for _, p in named:
        p.grad = None
    for l in latents:
        l.grad = None


def _grads(named, latents):
    out = {k: (None if p.grad is None else p.grad.detach().clone()) for k, p in named}
    out["latents"] = torch.stack([l.grad if l.grad is not None else torch.zeros_like(l) for l in latents]).detach().clone()
    return out


def _two_pass(models, r, rnd, latents, pix, test):
    """The reference loop: mean(test * L).backward(retain_graph=True), the network gradients dropped, mean(train * L)."""
    named = _weights(*models)
    _clear(named, latents)
    loss = _loss(*models, r, rnd, latents, pix)
    train = (~test).float()
    if bool(test.any()) and models[2] is not None:
        (test.float() * loss).mean().backward(retain_graph=True)
        for _, p in named:
            p.grad = None
    (train * loss).mean().backward()
    return loss.detach(), _grads(named, latents)


def _one_pass(models, r, rnd, latents, pix, test, held=True):
    named = _weights(*models)
    _clear(named, latents)
    loss = _loss(*models, r, rnd, latents, pix, held_out=test if held else None)
    ((~test).float() + test.float()).mul(loss).mean().backward()
    return loss.detach(), _grads(named, latents)


@pytest.mark.parametrize("n", [96, 1024, 8192])
def test_one_backward_matches_the_two_pass_loop(n):
    from nonrigid_nerf_b200 import _lib
    coarse, fine, bender, r, rnd, latents, pix, test = _setup(1234 + n, n)
    models = (coarse, fine, bender)
    l2, g2 = _two_pass(models, r, rnd, latents, pix, test)
    l1, g1 = _one_pass(models, r, rnd, latents, pix, test)
    _lib.device_error_check()
    assert torch.equal(l1, l2)   # the same forward
    frames = torch.arange(N_FRAMES)
    held = torch.isin(frames, torch.tensor(HELD_FRAMES))
    worst = 0.0
    for k, a in g2.items():
        if k == "latents":
            continue
        if a is None:
            assert g1[k] is None, k
            continue
        e = _rel(g1[k], a)
        worst = max(worst, e)
        assert e <= 1e-2, (k, e)
    e_test, e_train = _rel(g1["latents"][held], g2["latents"][held]), _rel(g1["latents"][~held], g2["latents"][~held])
    print(f"n={n}: worst parameter gradient rel err {worst:.2e}; latents of held-out frames {e_test:.2e}, "
          f"of training frames {e_train:.2e}")
    assert float(g2["latents"][held].abs().max()) > 0 and e_test <= 1e-2 and e_train <= 1e-2


def test_all_zero_mask_is_bit_identical_and_none_runs_todays_kernels():
    from nonrigid_nerf_b200 import _lib
    coarse, fine, bender, r, rnd, latents, pix, test = _setup(77, 1024)
    models = (coarse, fine, bender)
    none = torch.zeros_like(test)
    kinds = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + \
        _lib.DET_KERNEL_KINDS + _lib.HELD_OUT_KERNEL_KINDS
    torch.use_deterministic_algorithms(True)   # fixed-order latent sums: the comparison is bitwise
    try:
        counts, grads = {}, {}
        for label, held in (("none", False), ("zero-mask", True)):
            _lib.timing_enable(True)
            _, grads[label] = _one_pass(models, r, rnd, latents, pix, none, held=held)
            torch.cuda.synchronize()
            counts[label] = {k: c for k, (_, c) in _lib.timing_read(kinds).items()}
            _lib.timing_enable(False)
    finally:
        torch.use_deterministic_algorithms(False)
    for k, a in grads["none"].items():
        if a is not None:
            assert torch.equal(a, grads["zero-mask"][k]), k
    c0, c1 = counts["none"], counts["zero-mask"]
    assert c0["field_dgrad_held_out"] == 0 and c0["div_bwd_held_out"] == 0 and c0["field_dgrad"] == 2
    assert c1["field_dgrad_held_out"] == 2 and c1["div_bwd_held_out"] == 1 and c1["field_dgrad"] == 0
    assert c1["divergence"] == c0["divergence"] - 1
    for k in kinds:
        if k not in ("field_dgrad", "field_dgrad_held_out", "divergence", "div_bwd_held_out"):
            assert c0[k] == c1[k], k


def test_deterministic_one_pass_is_bit_reproducible():
    coarse, fine, bender, r, rnd, latents, pix, test = _setup(5, 1024)
    torch.use_deterministic_algorithms(True)
    try:
        runs = [_one_pass((coarse, fine, bender), r, rnd, latents, pix, test)[1] for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(False)
    for k, a in runs[0].items():
        if a is not None:
            assert torch.equal(a, runs[1][k]), k


@pytest.mark.parametrize("kind", ["rigid", "time_conditioned", "views"])
def test_without_a_bender_held_out_rays_add_nothing(kind):
    """Bit for bit the backward of mean(train * L): the reference skips its second pass without a bender.  "views": the
    view-dependent head of a rigid scene (use_viewdirs=True)."""
    coarse, fine, bender, r, rnd, latents, pix, test = _setup(31, 1024, with_bender=False, tc=kind == "time_conditioned",
                                                              views=kind == "views")
    models = (coarse, fine, None)
    torch.use_deterministic_algorithms(True)   # the latent table's index_add_ in a fixed order: the comparison is bitwise
    try:
        _, g1 = _one_pass(models, r, rnd, latents, pix, test)
        _, g2 = _two_pass(models, r, rnd, latents, pix, test)
    finally:
        torch.use_deterministic_algorithms(False)
    for k, a in g2.items():
        if a is None:
            assert g1[k] is None, k
        else:
            assert torch.equal(g1[k], a), k
    if kind == "time_conditioned":
        frames = torch.isin(torch.arange(N_FRAMES), torch.tensor(HELD_FRAMES))
        assert float(g1["latents"][frames].abs().max()) == 0 and float(g1["latents"][~frames].abs().max()) > 0


# ---- stage tests: the held-out kernels against the ordinary ones on the same upstream gradients ----------------------
def _field_ctx(n, s, with_div):
    """A differentiable coarse pass (n rays x s samples, bender) and its autograd node, which holds the forward's stash."""
    from nonrigid_nerf_b200 import autograd as ag, ops
    coarse, _, bender, _ = helpers.build_models(O, 3, DEV)
    coarse.ray_bender = (bender,)
    r = O.make_rays(3, n)
    rays = helpers.rays8(r, DEV)
    z = ops.sample_coarse(rays, s, torch.rand(n, s, device=DEV), False)
    lat = (0.1 * torch.randn(n, 32, device=DEV)).requires_grad_(True)
    raw, det = ag.field(coarse, rays, z, lat, True)
    div = None
    if with_div:
        c = ag.composite(raw, z, rays[:, 3:6])
        div = ag.divergence_loss(det["unmasked_offsets"], det["rigidity_mask"], None, bender, opacity_alpha=c["alpha"])
    return raw, det, div


def _bwd_args(ctx, d_raw, d_un, d_rig, gstash, scratch, nerf_grad, bend_grad, d_lat):
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    n, s, out_ch = ctx.shape
    un, rig = ctx.saved_tensors
    a = _lib.NrnFieldBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = n, s, out_ch
    a.d_raw, a.stash, a.relu_mask = d_raw.data_ptr(), ctx.stash.data_ptr(), ctx.relu_mask.data_ptr()
    a.grad_stash, a.wgrad_scratch = gstash.data_ptr(), scratch.data_ptr()
    a.nerf_packed, a.bender_packed = ctx.packs[0].data_ptr(), ctx.packs[1].data_ptr()
    a.unmasked_offsets, a.rigidity_mask = un.data_ptr(), rig.data_ptr()
    a.d_unmasked_offsets, a.d_rigidity_mask = d_un.data_ptr(), d_rig.data_ptr()
    a.nerf_grad, a.bender_grad, a.d_latents = nerf_grad.data_ptr(), bend_grad.data_ptr(), d_lat.data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    return a, lib


def _check_rows(base, held_run, pt_held, n_tiles, label):
    """Chunk-major images of 128 rows x 16 bytes: rows of training points bit-identical, rows of held-out points zero in
    every chunk the ordinary kernel wrote (buffers start as 0xff bytes, fp16 NaN)."""
    chunk_rows = lambda t: t[: n_tiles * (t.numel() // n_tiles)].view(n_tiles, -1, 128, 16)
    b, h = chunk_rows(base), chunk_rows(held_run)
    rows = torch.zeros(n_tiles * 128, dtype=torch.bool, device=DEV)
    rows[: pt_held.numel()] = pt_held
    rows = rows.view(n_tiles, 1, 128)
    written = (b != 0xFF).any(-1)
    keep = ~rows.expand_as(written)
    assert torch.equal(b[keep], h[keep]), f"{label}: training rows differ"
    # zero as fp16 values (a zero upstream times a negative operand leaves -0, which adds nothing to WGRAD's sums)
    assert int((h[~keep & written].view(torch.float16) != 0).sum()) == 0, f"{label}: held-out rows not zero"
    assert bool(written.any())


@pytest.mark.parametrize("n,s,mode", [(1, 100, "some"), (5, 100, "some"), (1023, 64, "some"), (300, 64, "all"),
                                      (300, 64, "none")])
def test_dgrad_stash_rows_of_held_out_rays_are_zero(n, s, mode):
    from nonrigid_nerf_b200 import _lib
    raw, det, _ = _field_ctx(n, s, False)
    ctx = raw.grad_fn
    lib = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(n)
    d_raw = torch.randn(n, s, 5, device=DEV, generator=g) * 1e-3
    d_un = torch.randn(n, s, 3, device=DEV, generator=g) * 1e-3
    d_rig = torch.randn(n, s, 1, device=DEV, generator=g) * 1e-3
    held = {"some": torch.arange(n, device=DEV) % 3 == 1, "all": torch.ones(n, dtype=torch.bool, device=DEV),
            "none": torch.zeros(n, dtype=torch.bool, device=DEV)}[mode]
    tiles = (n * s + 127) // 128
    outs = {}
    for det_mode in (False, True):
        for label in ("base", "held"):
            gstash = torch.full((lib.nrn_grad_stash_bytes(n, s),), 0xFF, dtype=torch.uint8, device=DEV)
            scratch = torch.full((lib.nrn_wgrad_scratch_bytes(),), 0xFF, dtype=torch.uint8, device=DEV)
            nerf_grad = torch.full((lib.nrn_nerf_grad_floats(5),), float("nan"), device=DEV)
            bend_grad = torch.full((lib.nrn_bender_grad_floats(),), float("nan"), device=DEV)
            d_lat = torch.full((n, 32), float("nan"), device=DEV)
            rows = torch.full((lib.nrn_latent_rows_bytes(n, s) // 4,), float("nan"), device=DEV)
            a, lib = _bwd_args(ctx, d_raw, d_un, d_rig, gstash, scratch, nerf_grad, bend_grad, d_lat)
            h8 = held.to(torch.uint8)
            if det_mode:
                rc = lib.nrn_field_backward_det_held_out(C.byref(a), rows.data_ptr(), h8.data_ptr()) if label == "held" else \
                    lib.nrn_field_backward_det(C.byref(a), rows.data_ptr())
            else:
                rc = lib.nrn_field_backward_held_out(C.byref(a), h8.data_ptr()) if label == "held" else lib.nrn_field_backward(C.byref(a))
            _lib.check(rc, label)
            torch.cuda.synchronize()
            outs[(det_mode, label)] = (gstash, nerf_grad, bend_grad, d_lat)
        _lib.device_error_check()
        (gs0, ng0, bg0, dl0), (gs1, ng1, bg1, dl1) = outs[(det_mode, "base")], outs[(det_mode, "held")]
        pt_held = held.repeat_interleave(s)
        _check_rows(gs0, gs1, pt_held, tiles, f"n={n} S={s} {mode} det={det_mode}")
        if det_mode:
            assert torch.equal(dl0, dl1)   # the latent gradient of every ray, held out or not
        else:
            assert _rel(dl1, dl0) <= 1e-6
        if mode == "none":
            assert torch.equal(ng0, ng1) and torch.equal(bg0, bg1) and torch.equal(gs0, gs1)
        if mode == "all":
            assert float(ng1.abs().max()) == 0 and float(bg1.abs().max()) == 0


@pytest.mark.parametrize("n,s,mode", [(5, 100, "some"), (1023, 64, "some"), (300, 64, "all"), (300, 64, "none")])
def test_divergence_adjoint_rows_of_held_out_rays_are_zero(n, s, mode):
    from nonrigid_nerf_b200 import _lib, autograd as ag
    lib = _lib.load()
    _, _, div = _field_ctx(n, s, True)
    ctx = div.grad_fn
    held = {"some": torch.arange(n, device=DEV) % 3 == 1, "all": torch.ones(n, dtype=torch.bool, device=DEV),
            "none": torch.zeros(n, dtype=torch.bool, device=DEV)}[mode]
    g_ray = torch.rand(n, device=DEV) + 0.5
    tiles = (n * s + 127) // 128
    outs = {}
    for label in ("base", "held"):
        a = ag._div_args(ctx)
        G = torch.empty(n * s, device=DEV)
        adj = torch.full((lib.nrn_div_grad_stash_bytes(n, s),), 0xFF, dtype=torch.uint8, device=DEV)
        scratch = torch.empty(lib.nrn_wgrad_scratch_bytes(), dtype=torch.uint8, device=DEV)
        d_un = torch.full((n * s, 3), float("nan"), device=DEV)
        d_rg = torch.full((n * s,), float("nan"), device=DEV)
        bg = torch.full((lib.nrn_bender_grad_floats(),), float("nan"), device=DEV)
        a.g_ray, a.G_workspace, a.adjoint_stash, a.wgrad_scratch = g_ray.data_ptr(), G.data_ptr(), adj.data_ptr(), scratch.data_ptr()
        a.d_unmasked_offsets, a.d_rigidity_mask, a.bender_grad = d_un.data_ptr(), d_rg.data_ptr(), bg.data_ptr()
        h8 = held.to(torch.uint8)
        rc = lib.nrn_divergence_backward_held_out(C.byref(a), h8.data_ptr()) if label == "held" else lib.nrn_divergence_backward(C.byref(a))
        _lib.check(rc, label)
        torch.cuda.synchronize()
        outs[label] = (adj, d_un, d_rg, bg)
    _lib.device_error_check()
    (a0, u0, r0, b0), (a1, u1, r1, b1) = outs["base"], outs["held"]
    _check_rows(a0, a1, held.repeat_interleave(s), tiles, f"divergence n={n} S={s} {mode}")
    assert torch.equal(u0, u1) and torch.equal(r0, r1)   # the latent path into DGRAD is unchanged
    if mode == "none":
        assert torch.equal(b0, b1) and torch.equal(a0, a1)
    if mode == "all":
        assert float(b1.abs().max()) == 0
