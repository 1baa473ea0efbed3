"""Training the view-dependent head without a bender (NeRF(use_viewdirs=True), rigid scenes): the training forward against
the inference kernel and its own view stash, the training step against the fp32 oracle on the GPU (TF32 off), and the
determinism of the gradients and of the optimizer arena path.

Which wrong implementation each check catches:
- raw not bit-equal to field_views_kernel: any change of the forward arithmetic by the stash writes (the E / direction
  encoding hazard included);
- Hv mask bits != encoding of the stashed Hv > 0: mask words written to the wrong rows or columns;
- per-ray loss and per-tensor gradients against the oracle: the Hv mask not applied in DGRAD, the alpha term dropped from
  dY7 (alpha_linear's and the trunk's gradients), ViewsF^T reading the direction columns (feature_linear's and the trunk's),
  a wrong block order of the head in the flat layout (every head tensor), rgb_linear's gradient from the wrong A columns;
- two runs bit-identical, arena == fresh buffers: a non-deterministic reduce or a wrong in-place destination;
- a separate head destination (trunk and head apart in the arena), a second backward without zero_grad (g1 + g2) and one
  over a retained graph (2 g): the head block written behind the trunk instead of to nerf_grad_head, accumulation that
  overwrites, stashes freed after the first backward;
- a frozen trunk: the in-place path taken for a partly trainable model (the frozen slots would be written);
- n_rays = 0: destinations not zeroed, an accumulating arena cleared, a kernel launched on an empty batch;
- golden case M: the whole wrapper against the executed reference."""
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import stash_layout as SL
from tests.parity import DEV
from tests.viewdirs_reference import build_view_models

pytestmark = pytest.mark.gpu

V_STASH_TILE, V_DIR, V_F, V_HV = 106496, (0, 4), (4 * SL.CHUNK, 32), (36 * SL.CHUNK, 16)


def _rays_z(seed, n, s):
    r = O.make_rays(seed, n)
    g = torch.Generator().manual_seed(seed)
    t = torch.sort(torch.rand(n, s, generator=g), -1).values
    z = r["near"] * (1.0 - t) + r["far"] * t
    return r, helpers.rays8(r, DEV), z.float().to(DEV)


@pytest.mark.parametrize("n,s", [(7, 64), (1023, 64), (64, 100)])
def test_training_forward_equals_inference_and_keeps_its_view_stash(n, s):
    from nonrigid_nerf_b200 import _lib, ops, autograd as ag
    coarse, _, _, _ = build_view_models(O, 5100 + s, DEV, with_bender=False, s_coarse=s)
    _, rays, z = _rays_z(5100 + s, n, s)
    vd = torch.nn.functional.normalize(rays[:, 3:6], dim=-1)
    with torch.no_grad():
        raw_i, _ = ag.field_views(coarse, rays, z, None, None, vd, False)
        raw_t, _, bufs = ops.field_forward_views_train(rays, z, vd, ops.pack_nerf(coarse), ops.pack_views(coarse))
    _lib.device_error_check()
    assert torch.equal(raw_i, raw_t), float((raw_i - raw_t).abs().max())
    P, T = n * s, (n * s + 127) // 128
    dirs = SL.image(bufs["views_stash"], V_STASH_TILE, V_DIR[0], V_DIR[1], T)[:P].float().cpu()
    ref = O.direction_encoding(vd.cpu()[:, None].expand(n, s, 3).reshape(-1, 3))
    assert float((dirs[:, :27] - ref).abs().max()) <= 2e-3 and bool((dirs[:, 27:] == 0).all())
    hv = SL.image(bufs["views_stash"], V_STASH_TILE, V_HV[0], V_HV[1], T)[:P]
    bits = SL.relu_bits(bufs["hv_mask"], 0, 128, T, tile_bytes=2048)[:P]
    assert torch.equal(bits, hv > 0)
    # F against fp64 from the stashed h8 and the fp16 weights
    h8 = SL.image(bufs["stash"], SL.STASH_TILE, *SL.ST_H[7], T)[:P].double().cpu()
    F = SL.image(bufs["views_stash"], V_STASH_TILE, V_F[0], V_F[1], T)[:P].double().cpu()
    wf = coarse.feature_linear.weight.detach().half().double().cpu()
    Fx = h8 @ wf.T + coarse.feature_linear.bias.detach().double().cpu()
    bound = 258 * 2.0 ** -24 * (h8.abs() @ wf.abs().T + 1) + Fx.abs() * 2.0 ** -11 + 2.0 ** -25
    assert bool(((F - Fx).abs() <= bound).all())


def _train_grads(coarse, fine, r, n_imp=64):
    from nonrigid_nerf_b200 import train as T
    for m in (coarse, fine):
        m.zero_grad(set_to_none=True)
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=n_imp, network_fine=fine, N_samples=64, network_fn=coarse,
              white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    rgb, _, _, ex = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=1 << 20, near=r["near"], far=r["far"], use_viewdirs=True,
                             additional_pixel_information={"ray_bending_latents": r["latents"].to(DEV)}, retraw=True, **kw)
    tgt = r["target"].to(DEV)
    loss = ((rgb - tgt) ** 2).mean(-1) + ((ex["rgb0"] - tgt) ** 2).mean(-1)
    loss.sum().backward()
    return loss.detach(), {k: p.grad.detach().clone() for m, pre in ((coarse, "c."), (fine, "f.")) for k, p in
                           ((pre + k, p) for k, p in m.named_parameters()) if p.grad is not None}


def _oracle_grads(cp, fp, vc, vf, r, n_imp=64):
    cp_, fp_ = O.clone_params(cp, True), O.clone_params(fp, True)
    vc_, vf_ = O.clone_params(vc, True), O.clone_params(vf, True)
    to = lambda d: {k: ([t.to(DEV).detach().requires_grad_(True) for t in v] if isinstance(v, list) else v.to(DEV).detach().requires_grad_(True))
                    for k, v in d.items()}
    cp_, fp_, vc_, vf_ = to(cp_), to(fp_), to(vc_), to(vf_)
    ret = O.render_rays(cp_, fp_, None, r["rays_o"].to(DEV), r["rays_d"].to(DEV), r["near"], r["far"], r["latents"].to(DEV), 64, n_imp,
                        vpar_c=vc_, vpar_f=vf_)
    loss = O.training_loss(ret, r["target"].to(DEV))
    loss.sum().backward()
    out = {}
    for pre, p, v in (("c.", cp_, vc_), ("f.", fp_, vf_)):
        for i in range(8):
            out[f"{pre}pts_linears.{i}.weight"] = p["pts_w"][i].grad
            out[f"{pre}pts_linears.{i}.bias"] = p["pts_b"][i].grad
        for mod, key in (("views_linears.0", "views"), ("feature_linear", "feature"), ("alpha_linear", "alpha"), ("rgb_linear", "rgb")):
            out[f"{pre}{mod}.weight"] = v[key + "_w"].grad
            out[f"{pre}{mod}.bias"] = v[key + "_b"].grad
    return loss.detach(), out


@pytest.mark.parametrize("n", [1, 3, 1024, 8192])
def test_training_step_matches_the_fp32_oracle(n):
    """1 ray: the coarse pass is one ragged tile (64 of 128 rows); 3 rays: its second tile is ragged and the first tile
    of its CTA.  The gradients must be finite and match."""
    from nonrigid_nerf_b200 import _lib
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    seed = 6200
    coarse, fine, _, (cp, fp, _, vc, vf) = build_view_models(O, seed, DEV, with_bender=False)
    r = O.make_rays(seed, n)
    loss, grads = _train_grads(coarse, fine, r)
    _lib.device_error_check()
    loss_o, grads_o = _oracle_grads(cp, fp, vc, vf, r)
    rel_loss = float((loss - loss_o).norm() / loss_o.norm())
    print(f"n={n}: per-ray loss relative L2 {rel_loss:.3e}")
    assert rel_loss <= 2e-3
    assert set(grads) == set(grads_o), set(grads) ^ set(grads_o)
    worst = 0.0
    for k, g in grads.items():
        go = grads_o[k]
        assert g.shape == go.shape, k
        assert bool(torch.isfinite(g).all()), k
        rel = float((g - go).norm() / go.norm().clamp_min(1e-30))
        worst = max(worst, rel)
        assert rel <= 8e-2, (k, rel)
    print(f"n={n}: worst per-tensor gradient relative L2 {worst:.3e}")


def test_gradients_deterministic_and_arena_equals_fresh_buffers():
    from nonrigid_nerf_b200 import _lib, optim
    seed = 6300
    coarse, fine, _, _ = build_view_models(O, seed, DEV, with_bender=False)
    r = O.make_rays(seed, 512)
    _, g1 = _train_grads(coarse, fine, r)
    _, g2 = _train_grads(coarse, fine, r)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
    # optim.Adam seats every .grad in one arena: the backward then accumulates in place; from zero it must give the same bits
    params = list(coarse.parameters()) + list(fine.parameters())
    opt = optim.Adam(params, lr=1e-3)
    opt.zero_grad()
    for p in params:
        if p.grad is not None:
            p.grad.zero_()
    from nonrigid_nerf_b200 import train as T
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=64, network_fine=fine, N_samples=64, network_fn=coarse,
              white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    rgb, _, _, ex = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=1 << 20, near=r["near"], far=r["far"], use_viewdirs=True,
                             additional_pixel_information={"ray_bending_latents": r["latents"].to(DEV)}, retraw=True, **kw)
    tgt = r["target"].to(DEV)
    (((rgb - tgt) ** 2).mean(-1) + ((ex["rgb0"] - tgt) ** 2).mean(-1)).sum().backward()
    _lib.device_error_check()
    # the in-place path runs: the trunk's and the head block's .grad tensors lay back to back in the arena
    from nonrigid_nerf_b200.autograd import _arena_destination, _views_flat_params
    for m in (coarse, fine):
        trunk, head = _views_flat_params(m)
        assert _arena_destination(trunk) is not None and _arena_destination(head) is not None
    for m, pre in ((coarse, "c."), (fine, "f.")):
        for k, p in m.named_parameters():
            if pre + k in g1:
                assert torch.equal(p.grad, g1[pre + k]), pre + k


def test_bender_training_still_raises_before_any_launch():
    """A view model without a bender, trained through training_wrapper_class with a bender to seat: refused first."""
    from nonrigid_nerf_b200 import _lib, parallel
    seed = 6400
    coarse, fine, _, _ = build_view_models(O, seed, DEV, with_bender=False)
    _, _, bender, _ = build_view_models(O, seed, DEV, with_bender=True)
    lat = [torch.zeros(32, device=DEV, requires_grad=True)]
    wrapper = parallel.training_wrapper_class(coarse, lat, fine_model=fine, ray_bender=bender)
    kinds = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS
    _lib.timing_enable(True)
    try:
        with pytest.raises(RuntimeError, match="training with the view-dependent head is not implemented"):
            wrapper.forward(None, None, None, 0, {}, torch.zeros(4, 3, device=DEV), 0, 0, {"imageid_to_timestepid": [0]},
                            torch.zeros(4, 3, device=DEV))
    finally:
        _lib.timing_enable(False)
    counts = {k: c for k, (_, c) in _lib.timing_read(kinds).items()}
    assert sum(counts.values()) == 0, counts


# ----------------------------------------------------------------------------------------------------------------------
# gradient destinations and edges
# ----------------------------------------------------------------------------------------------------------------------
def _render_loss(coarse, fine, r):
    from nonrigid_nerf_b200 import train as T
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=64, network_fine=fine, N_samples=64, network_fn=coarse,
              white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    rgb, _, _, ex = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=1 << 20, near=r["near"], far=r["far"], use_viewdirs=True,
                             additional_pixel_information={"ray_bending_latents": r["latents"].to(DEV)}, retraw=True, **kw)
    tgt = r["target"].to(DEV)
    return (((rgb - tgt) ** 2).mean(-1) + ((ex["rgb0"] - tgt) ** 2).mean(-1)).sum()


def _grads_equal(models, expect, what):
    for m, pre in zip(models, ("c.", "f.")):
        for k, p in m.named_parameters():
            if pre + k in expect:
                assert torch.equal(p.grad, expect[pre + k]), (what, pre + k)


@pytest.mark.parametrize("layout", ["adjacent", "separate"])
def test_arena_destinations_and_accumulation_equal_fresh_buffers(layout):
    """optim.Adam's arena with each model's trunk and head block back to back ("adjacent": one flat destination) or each
    contiguous but apart ("separate": [*heads, *latents, *trunks], nerf_grad_head set): the in-place backward equals the
    fresh-buffer path bit for bit, and a second backward without zero_grad gives fp32(g1 + g2) bit for bit."""
    from nonrigid_nerf_b200 import _lib, optim
    from nonrigid_nerf_b200.autograd import _arena_destination, _views_flat_params
    seed = 6500
    coarse, fine, _, _ = build_view_models(O, seed, DEV, with_bender=False)
    r1, r2 = O.make_rays(seed, 512), O.make_rays(seed + 1, 512)
    _, g1 = _train_grads(coarse, fine, r1)
    _, g2 = _train_grads(coarse, fine, r2)
    split = {id(m): _views_flat_params(m) for m in (coarse, fine)}
    lat = [torch.zeros(32, device=DEV, requires_grad=True) for _ in range(3)]
    if layout == "adjacent":
        params = [p for m in (coarse, fine) for part in split[id(m)] for p in part] + lat
    else:
        params = [p for m in (coarse, fine) for p in split[id(m)][1]] + lat + [p for m in (coarse, fine) for p in split[id(m)][0]]
    opt = optim.Adam(params, lr=1e-3)
    opt.zero_grad()
    _render_loss(coarse, fine, r1).backward()
    _lib.device_error_check()
    for m in (coarse, fine):
        trunk, head = split[id(m)]
        t_dst, h_dst = _arena_destination(trunk), _arena_destination(head)
        assert t_dst is not None and h_dst is not None
        adjacent = h_dst == t_dst + 4 * SL.TRUNK_FLOATS
        assert adjacent == (layout == "adjacent"), (layout, t_dst, h_dst)
    _grads_equal((coarse, fine), g1, "arena from zero")
    _render_loss(coarse, fine, r2).backward()
    _lib.device_error_check()
    _grads_equal((coarse, fine), {k: g1[k] + g2[k] for k in g1}, "second backward without zero_grad")


def test_backward_twice_over_a_retained_graph():
    """The stashes live as long as the autograd node: a second backward reads them again, so .grad = g + g = 2 g."""
    from nonrigid_nerf_b200 import _lib
    seed = 6600
    coarse, fine, _, _ = build_view_models(O, seed, DEV, with_bender=False)
    r = O.make_rays(seed, 256)
    _, g1 = _train_grads(coarse, fine, r)
    for m in (coarse, fine):
        m.zero_grad(set_to_none=True)
    loss = _render_loss(coarse, fine, r)
    loss.backward(retain_graph=True)
    loss.backward()
    _lib.device_error_check()
    _grads_equal((coarse, fine), {k: g1[k] + g1[k] for k in g1}, "retain_graph")


def test_frozen_trunk_trains_the_head_through_fresh_buffers():
    """Trunk frozen, head trained: the head's gradients equal the fully trainable run's bit for bit and the trunk's
    .grad stays None; with optim.Adam's arena seated, the partly frozen model takes the fresh-buffer path, so the frozen
    trunk's arena slots (preset to NaN) are never written."""
    from nonrigid_nerf_b200 import _lib, optim
    from nonrigid_nerf_b200.autograd import _views_flat_params
    seed = 6700
    coarse, fine, _, _ = build_view_models(O, seed, DEV, with_bender=False)
    r = O.make_rays(seed, 256)
    _, g_all = _train_grads(coarse, fine, r)
    trunks = [p for m in (coarse, fine) for p in _views_flat_params(m)[0]]
    for p in trunks:
        p.requires_grad_(False)
    _, g = _train_grads(coarse, fine, r)
    _lib.device_error_check()
    assert all(p.grad is None for p in trunks)
    head_keys = {k for k in g_all if not k[2:].startswith("pts_linears")}
    assert set(g) == head_keys, set(g) ^ head_keys
    for k in head_keys:
        assert torch.equal(g[k], g_all[k]), k
    params = [p for m in (coarse, fine) for part in _views_flat_params(m) for p in part]
    opt = optim.Adam(params, lr=1e-3)
    opt.zero_grad()
    for p in trunks:
        p.grad.fill_(float("nan"))
    _render_loss(coarse, fine, r).backward()
    _lib.device_error_check()
    assert all(bool(torch.isnan(p.grad).all()) for p in trunks), "a frozen trunk's arena slot was written"
    _grads_equal((coarse, fine), {k: g_all[k] for k in head_keys}, "frozen trunk, arena")


@pytest.mark.parametrize("dest", ["flat", "separate", "accumulate"])
def test_empty_batch_zeroes_the_destinations_and_launches_nothing(dest):
    """nrn_field_backward_views at n_rays = 0 (an empty shard): the flat buffer, or both destinations, are zeroed when not
    accumulating; an accumulating arena is left as it was; no kernel runs."""
    import ctypes as C
    from nonrigid_nerf_b200 import _lib
    from tests.parity import poison_f32
    lib = _lib.load()
    n_all = lib.nrn_nerf_views_grad_floats()
    n_head = n_all - SL.TRUNK_FLOATS
    g = torch.Generator(device=DEV).manual_seed(11)
    if dest == "accumulate":
        trunk, head = torch.randn(n_all, generator=g, device=DEV), torch.randn(n_head, generator=g, device=DEV)
    else:
        trunk, head = poison_f32(n_all), poison_f32(n_head)
    before = (trunk.clone(), head.clone())
    a, v = _lib.NrnFieldBwdArgs(), _lib.NrnViewBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = 0, 64, 4
    a.nerf_grad = trunk.data_ptr()
    if dest != "flat":
        a.nerf_grad_head = head.data_ptr()
    a.accumulate_nerf = 1 if dest == "accumulate" else 0
    a.stream = torch.cuda.current_stream().cuda_stream
    _lib.timing_enable(True)
    try:
        _lib.check(lib.nrn_field_backward_views(C.byref(a), C.byref(v)), "field_backward_views")
        torch.cuda.synchronize()
    finally:
        _lib.timing_enable(False)
    _lib.device_error_check()
    counts = {k: c for k, (_, c) in _lib.timing_read(_lib.VIEW_TRAIN_KERNEL_KINDS).items()}
    assert sum(counts.values()) == 0, counts
    if dest == "accumulate":
        assert torch.equal(trunk, before[0]) and torch.equal(head, before[1])
    elif dest == "separate":
        assert bool((trunk[:SL.TRUNK_FLOATS] == 0).all()) and bool((head == 0).all())
        assert bool(torch.isnan(trunk[SL.TRUNK_FLOATS:]).all()), "the head's slot of nerf_grad was written despite nerf_grad_head"
    else:
        assert bool((trunk == 0).all()) and bool(torch.isnan(head).all())


def test_training_wrapper_matches_the_executed_reference_caseM():
    """training_wrapper_class with the view-dependent head and no bender (perturb 1, noise 1, the reference's random
    draws injected) against golden case M from the executed reference: per-ray loss and every coarse and fine
    parameter's sampled gradient and norm within DESIGN section 2's bounds; the latents get no gradient."""
    import os
    import types
    import numpy as np
    from nonrigid_nerf_b200 import _lib, parallel
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "caseM_viewdirs_train.npz"))
    seed, n = int(g["seed"]), int(g["n"])
    coarse, fine, _, _ = build_view_models(O, seed, DEV, with_bender=False)
    r = O.make_rays(seed, n)
    rnd = {k: v.to(DEV) for k, v in O.make_randomness(seed, n, 64, 64).items()}
    latents = [torch.from_numpy(row.copy()).to(DEV).requires_grad_(True) for row in g["latent_table"]]
    targs = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=int(g["N_iters"]), offsets_loss_weight=0.0,
                                  divergence_loss_weight=0.0, rigidity_loss_weight=0.0, ray_bending_latent_size=32)
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64,
          "network_fn": coarse, "ray_bender": None, "use_viewdirs": True, "white_bkgd": False, "raw_noise_std": 1.0,
          "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"], "randomness": rnd}
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine)
    loss = wrapper(targs, r["rays_o"].to(DEV), r["rays_d"].to(DEV), 100, kw, r["target"].to(DEV), int(g["global_step"]), 0,
                   {"imageid_to_timestepid": [int(v) for v in g["i2t"]]}, torch.from_numpy(g["pix"]).to(DEV))
    loss.mean().backward()
    _lib.device_error_check()
    ref = torch.from_numpy(g["loss"])
    d = float((loss.detach().cpu() - ref).abs().max())
    rel = float((loss.detach().cpu().double() - ref.double()).norm() / ref.double().norm())
    print(f"case M: per-ray loss vs executed reference: L-inf {d:.3e}, rel L2 {rel:.3e}")
    assert d <= 2e-3 and rel <= 2e-3, (d, rel)
    assert not bool(g["latents_got_grad"]) and all(l.grad is None or not bool(l.grad.any()) for l in latents)
    named = dict([("coarse." + k, p) for k, p in coarse.named_parameters() if p.grad is not None] +
                 [("fine." + k, p) for k, p in fine.named_parameters() if p.grad is not None])
    assert set(named) == set(str(k) for k in g["grad_names"]), set(named) ^ set(str(k) for k in g["grad_names"])
    worst = {}
    for nm, p in named.items():
        idx = torch.from_numpy(g[nm + ".idx"])
        ours = p.grad.reshape(-1).cpu()[idx].double().numpy()
        exp = g[nm + ".val"].astype(np.float64)
        err = float(np.linalg.norm(ours - exp) / (np.linalg.norm(exp) + 1e-30))
        nrm = abs(float(p.grad.norm()) - float(g[nm + ".norm"][0])) / (float(g[nm + ".norm"][0]) + 1e-30)
        worst[nm] = max(err, nrm)
        assert bool(torch.isfinite(p.grad).all()) and err <= 8e-2 and nrm <= 8e-2, (nm, err, nrm)
    print(f"case M: worst sampled-gradient / norm relative error {max(worst.values()):.3e} ({max(worst, key=worst.get)})")
