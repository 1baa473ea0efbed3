"""GPU parity of what bench.py times and what the reference's training loop calls:

  * parallel.training_wrapper_class.forward (the module DataParallel wrapped, train.py:140-287) against the per-ray loss
    [N] and the gradients of the EXECUTED reference (golden case H) -- through autograd-owned gradients and through the
    optimizer's in-place gradient arena (both must agree with each other bit for bit up to accumulation order);
  * the fused divergence regulariser against the executed reference's compute_divergence_loss (golden case G);
  * backward(retain_graph=True) followed by a second backward() (train.py:1595-1606);
  * the point-wise entries run_network / NeRF.forward(x), the public sample_pdf / raw2outputs wrappers;
  * full gradient parity at the benchmark batch (N_rand = 1024, 64c + 128f): WGRAD split-K over 1,536 tiles;
  * the default-config regulariser weights with a vanishing data term (shared fp16 loss scale).

Tolerances are ~10x the errors measured on the GPU (printed by the tests; fp16 tensor-core operands vs the fp32 reference).
"""
import os

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda:0"


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _targs(g=None, **over):
    import types
    a = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=200000, offsets_loss_weight=60.0,
                              divergence_loss_weight=3.0, rigidity_loss_weight=0.0005, ray_bending_latent_size=32)
    if g is not None:
        a.N_iters, a.offsets_loss_weight = int(g["N_iters"]), float(g["offsets_w"])
        a.divergence_loss_weight, a.rigidity_loss_weight = float(g["divergence_w"]), float(g["rigidity_w"])
    for k, v in over.items():
        setattr(a, k, v)
    return a


def _kwargs(coarse, fine, bender, r, rnd, perturb=1.0, noise=1.0):
    return {"network_query_fn": None, "perturb": perturb, "N_importance": 64, "network_fine": fine, "N_samples": 64,
            "network_fn": coarse, "ray_bender": bender, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": noise,
            "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"], "randomness": rnd}


def _golden_grad_check(g, named, rtol, label):
    worst = 0.0
    for nm, t in named:
        if nm + ".val" not in g.files or t.grad is None:
            continue
        idx = torch.from_numpy(g[nm + ".idx"])
        ours = t.grad.reshape(-1).cpu()[idx].double().numpy()
        ref = g[nm + ".val"].astype(np.float64)
        err = np.linalg.norm(ours - ref) / (np.linalg.norm(ref) + 1e-30)
        nrm = abs(float(t.grad.norm()) - float(g[nm + ".norm"][0])) / (float(g[nm + ".norm"][0]) + 1e-30)
        worst = max(worst, err)
        if err > rtol or nrm > rtol:
            raise AssertionError(f"{label}: {nm}: sample rel err {err:.3e}, norm rel err {nrm:.3e} (tol {rtol})")
    return worst


def _run_wrapper(g, use_arena):
    from nonrigid_nerf_b200 import _lib, optim, parallel
    seed, n = int(g["seed"]), int(g["n"])
    coarse, fine, bender, _ = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    rnd = dict(O.make_randomness(seed, n, 64, 64))
    rnd["e"] = torch.from_numpy(g["e"])
    latents = [torch.from_numpy(row.copy()).to(DEV).requires_grad_(True) for row in g["latent_table"]]
    params = latents + list(bender.parameters()) + list(coarse.parameters()) + list(fine.parameters())
    opt = optim.Adam(params, lr=5e-4) if use_arena else None
    if opt is not None:
        opt.zero_grad()
        assert opt.grads_in_arena
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
    loss = wrapper(_targs(g), r["rays_o"].to(DEV), r["rays_d"].to(DEV), 100, _kwargs(coarse, fine, bender, r, rnd),
                   r["target"].to(DEV), int(g["global_step"]), 0, {"imageid_to_timestepid": [int(v) for v in g["i2t"]]},
                   torch.from_numpy(g["pix"]).to(DEV))
    loss.mean().backward()
    _lib.device_error_check()
    if opt is not None:
        assert opt.grads_in_arena, "the backward must accumulate into the arena, not re-bind .grad"
    return loss.detach().cpu(), coarse, fine, bender, latents, opt


def test_training_wrapper_loss_and_gradients_match_executed_reference():
    g = np.load(os.path.join(GOLD, "caseH_training_wrapper.npz"))
    results = {}
    for use_arena in (False, True):
        loss, coarse, fine, bender, latents, opt = _run_wrapper(g, use_arena)
        d = float(np.abs(loss.numpy() - g["loss"]).max())
        rel = _rel(loss, torch.from_numpy(g["loss"]))
        print(f"[arena={use_arena}] per-ray loss vs executed reference: L-inf {d:.3e}, rel L2 {rel:.3e}")
        assert d <= 2e-3 and rel <= 2e-3, (d, rel)
        named = [("coarse." + k, v) for k, v in coarse.named_parameters()] + [("fine." + k, v) for k, v in fine.named_parameters()] + \
                [("bender." + k, v) for k, v in bender.named_parameters()]
        worst = _golden_grad_check(g, named, 1.2e-1, f"arena={use_arena}")   # 64-entry samples of each gradient tensor
        lg = torch.stack([l.grad for l in latents]).cpu()
        e_lat = _rel(lg, torch.from_numpy(g["latent_grads"]))
        print(f"[arena={use_arena}] worst sampled gradient error {worst:.3e}; latent table gradient {e_lat:.3e}")
        assert e_lat <= 8e-2, e_lat
        results[use_arena] = [None if p.grad is None else p.grad.detach().clone() for _, p in named] + [lg]
        if use_arena:
            assert coarse.views_linears[0].weight.grad.abs().max() == 0   # dead weight: zero gradient in the arena
        else:
            assert coarse.views_linears[0].weight.grad is None          # dead weight keeps grad=None (SURVEY.md 7.3-6)
    # both gradient routes come from the same kernels: identical up to the order of the bender's three accumulations
    for a, b in zip(results[False], results[True]):
        if a is None:
            continue
        assert _rel(b, a) <= 1e-5, _rel(b, a)


def test_fused_divergence_matches_executed_reference_caseG():
    from nonrigid_nerf_b200 import _lib, autograd as ag, train as T
    g = np.load(os.path.join(GOLD, "caseG_divergence.npz"))
    seed, n = int(g["seed"]), int(g["n"])
    coarse, fine, bender, _ = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    lat = torch.from_numpy(g["latents"]).to(DEV).requires_grad_(True)
    kw = _kwargs(coarse, fine, bender, r, None, perturb=0.0, noise=0.0)
    kw.pop("randomness")
    rgb, disp, acc, extras = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=32768, retraw=True,
                                      additional_pixel_information={"ray_bending_latents": lat}, detailed_output=True, **kw)
    div = ag.divergence_loss(extras["unmasked_offsets"], extras["rigidity_mask"], None, bender, torch.from_numpy(g["e"]).to(DEV),
                             opacity_alpha=extras["opacity_alpha"])
    div.mean().backward()
    _lib.device_error_check()
    rel = _rel(div.detach().cpu(), torch.from_numpy(g["div"]))
    print(f"divergence term per ray vs executed reference: rel L2 {rel:.3e} (mean {float(g['div'].mean()):.3e})")
    assert rel <= 3e-2, rel
    worst = _golden_grad_check(g, [("bender." + k, v) for k, v in bender.named_parameters()], 1.5e-1, "caseG")
    e_lat = _rel(lat.grad.cpu(), torch.from_numpy(g["latents_grad"]))
    print(f"worst sampled bender gradient error {worst:.3e}; latents {e_lat:.3e}")
    assert e_lat <= 8e-2, e_lat


def test_second_backward_over_a_retained_graph():
    """train.py:1595-1606: masked_loss.backward(retain_graph=True), weights.grad = None, then backward() again."""
    from nonrigid_nerf_b200 import _lib, parallel
    g = np.load(os.path.join(GOLD, "caseH_training_wrapper.npz"))
    seed, n = int(g["seed"]), int(g["n"])
    coarse, fine, bender, _ = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    rnd = dict(O.make_randomness(seed, n, 64, 64)); rnd["e"] = torch.from_numpy(g["e"])
    latents = [torch.from_numpy(row.copy()).to(DEV).requires_grad_(True) for row in g["latent_table"]]
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
    loss = wrapper(_targs(g), r["rays_o"].to(DEV), r["rays_d"].to(DEV), 100, _kwargs(coarse, fine, bender, r, rnd),
                   r["target"].to(DEV), int(g["global_step"]), 0, {"imageid_to_timestepid": [int(v) for v in g["i2t"]]},
                   torch.from_numpy(g["pix"]).to(DEV))
    mask = (torch.arange(n, device=DEV) % 3 == 0).float()
    (mask * loss).mean().backward(retain_graph=True)
    lat_first = torch.stack([l.grad.clone() for l in latents])
    for w in list(coarse.parameters()) + list(fine.parameters()) + list(bender.parameters()):
        w.grad = None
    ((1 - mask) * loss).mean().backward()
    _lib.device_error_check()
    # latents accumulated both passes = gradient of the full mean; the weights hold the second pass only
    e_lat = _rel(torch.stack([l.grad for l in latents]).cpu(), torch.from_numpy(g["latent_grads"]))
    print(f"two-pass latent gradient vs executed reference: {e_lat:.3e}")
    assert e_lat <= 8e-2 and float(lat_first.abs().max()) > 0
    assert fine.pts_linears[3].weight.grad is not None and torch.isfinite(fine.pts_linears[3].weight.grad).all()


def test_point_mode_entries_run_network_and_nerf_forward():
    from nonrigid_nerf_b200 import _lib, train as T
    seed, n, s = 812, 40, 7
    coarse, fine, bender, (cp, fp, bp) = helpers.build_models(O, seed, DEV)
    rs = np.random.RandomState(seed)
    pts = torch.from_numpy(rs.uniform(-1, 1, size=(n, s, 3)).astype(np.float32))
    lat = torch.from_numpy((rs.randn(n, 32) * 0.1).astype(np.float32))
    with torch.no_grad():
        out, det = T.run_network(pts.to(DEV), None, {"ray_bending_latents": lat.to(DEV)}, coarse, None, None, detailed_output=True)
        lat_pts = lat[:, None].expand(n, s, 32).reshape(-1, 32)
        ref_raw, ref_det = O.query_field(cp, bp, pts, lat)
        ref_raw = ref_raw.reshape(-1, 5)
        ref_det = {k: v.reshape(n * s, -1) for k, v in ref_det.items()}
        # NeRF.forward(x): x = [embedded points (63, only xyz read) | latents] as run_network builds it (train.py:84-96)
        x = torch.zeros(n * s, 63 + 32)
        x[:, :3] = pts.reshape(-1, 3)
        x[:, 63:] = lat_pts
        raw2, det2 = coarse(x.to(DEV), detailed_output=True)
    _lib.device_error_check()
    assert out.shape == (n, s, 5) and raw2.shape == (n * s, 5)
    d = float((out.reshape(-1, 5).cpu() - ref_raw).abs().max())
    print(f"run_network raw vs oracle: L-inf {d:.3e}")
    assert d <= 3e-2 * max(1.0, float(ref_raw.abs().max())), d
    assert torch.equal(out.reshape(-1, 5), raw2)
    np.testing.assert_allclose(det["unmasked_offsets"].reshape(-1, 3).cpu().numpy(), ref_det["unmasked_offsets"].numpy(), atol=1e-4)
    np.testing.assert_allclose(det["rigidity_mask"].reshape(-1).cpu().numpy(), ref_det["rigidity_mask"].reshape(-1).numpy(), atol=3e-4)
    np.testing.assert_allclose(det2["input_pts"].cpu().numpy(), ref_det["input_pts"].numpy(), atol=1e-4)
    with pytest.raises(RuntimeError):
        coarse(x.to(DEV).requires_grad_(True))   # the point-wise entry is inference-only: differentiable use fails loudly


def test_public_sample_pdf_and_raw2outputs_wrappers_match_golden_caseE():
    from nonrigid_nerf_b200 import run_nerf_helpers as H, train as T
    g = np.load(os.path.join(GOLD, "caseE_ops.npz"))
    bins, w = torch.from_numpy(g["bins"]).to(DEV), torch.from_numpy(g["weights"]).to(DEV)
    det = H.sample_pdf(bins, w, 64, det=True).cpu().numpy()
    bad = np.abs(det - g["samples_det"]) > 1e-5
    assert bad.mean() <= 5e-3, bad.mean()          # flat-CDF samples depend on cumsum order (DESIGN.md section 2)
    rnd = H.sample_pdf(bins, w, 64, det=False)
    assert rnd.shape == (bins.shape[0], 64) and bool((rnd >= bins.min()).all()) and bool((rnd <= bins.max()).all())
    raw, z, rd = (torch.from_numpy(g[k]).to(DEV) for k in ("raw", "z", "rays_d"))
    o = T.raw2outputs(raw, z, rd, 0, False)
    for a, k in zip(o, ("rgb_map", "disp_map", "acc_map", "alpha", "weights_out", "depth_map")):
        np.testing.assert_allclose(a.cpu().numpy(), g[k], rtol=2e-5, atol=2e-6, equal_nan=True, err_msg=k)
    np.testing.assert_allclose(T.raw2outputs(raw, z, rd, 0, True)[0].cpu().numpy(), g["rgb_map_white"], atol=2e-6)


def test_gradient_parity_at_the_benchmark_batch_1024_rays():
    """N_rand = 1024, 64c + 128f: WGRAD split-K over 1,536 tiles / one CTA per SM against the oracle's autograd."""
    from nonrigid_nerf_b200 import _lib, train as T
    seed, n = 1024, 1024
    coarse, fine, bender, (cp, fp, bp) = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    rnd = O.make_randomness(seed, n, 64, 64)
    lat = r["latents"].clone().to(DEV).requires_grad_(True)
    kw = _kwargs(coarse, fine, bender, r, rnd)
    rgb, disp, acc, extras = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=32768, retraw=True,
                                      additional_pixel_information={"ray_bending_latents": lat}, detailed_output=True, **kw)
    ret = {"rgb_map": rgb, "rgb0": extras["rgb0"], "visibility_weights": extras["visibility_weights"],
           "unmasked_offsets": extras["unmasked_offsets"], "rigidity_mask": extras["rigidity_mask"]}
    O.training_loss(ret, r["target"].to(DEV), 60.0, 5e-4, 0.05).mean().backward()
    _lib.device_error_check()
    cpo, fpo, bpo = O.clone_params(cp, True), O.clone_params(fp, True), O.clone_params(bp, True)
    lat_o = r["latents"].clone().requires_grad_(True)
    ret_o = O.render_rays(cpo, fpo, bpo, r["rays_o"], r["rays_d"], r["near"], r["far"], lat_o, 64, 64, perturb=True,
                          raw_noise_std=1.0, rnd=rnd)
    O.training_loss(ret_o, r["target"], 60.0, 5e-4, 0.05).mean().backward()
    d = float((rgb.detach().cpu() - ret_o["rgb_map"].detach()).abs().max())
    print(f"rgb L-inf vs oracle at N=1024: {d:.3e}")
    assert d <= 2e-3, d
    worst = 0.0
    for net, po, nm in ((coarse, cpo, "coarse"), (fine, fpo, "fine")):
        for i in range(8):
            e = _rel(net.pts_linears[i].weight.grad.cpu(), po["pts_w"][i].grad)
            eb = _rel(net.pts_linears[i].bias.grad.cpu(), po["pts_b"][i].grad)
            worst = max(worst, e, eb)
            print(f"  {nm} layer {i}: W {e:.3e}  b {eb:.3e}")
            assert e <= 5e-2 and eb <= 5e-2, (nm, i, e, eb)
        e = _rel(net.output_linear.weight.grad.cpu(), po["out_w"].grad)
        assert e <= 2e-2, (nm, "head", e)
    for i in range(5):
        e = _rel(bender.network[i].weight.grad.cpu(), bpo["net_w"][i].grad)
        worst = max(worst, e)
        print(f"  bender net {i}: W {e:.3e}")
        assert e <= 8e-2, ("bender", i, e)
    for i in range(3):
        e = _rel(bender.rigidity_network[i].weight.grad.cpu(), bpo["rig_w"][i].grad)
        worst = max(worst, e)
        print(f"  bender rigidity {i}: W {e:.3e}")
        assert e <= 8e-2, ("rigidity", i, e)
    e = _rel(lat.grad.cpu(), lat_o.grad)
    print(f"  latents: {e:.3e}; worst {worst:.3e}")
    assert e <= 8e-2, e


def test_large_regulariser_weight_with_vanishing_data_term():
    """offsets_loss_weight = 600 (the reference's default, train.py config_parser) while the data term's gradient is ~0:
    the regularisers' upstream gradients take part in the fp16 loss scale, so the bender gradients stay accurate."""
    from nonrigid_nerf_b200 import _lib, train as T
    seed, n = 77, 128
    coarse, fine, bender, (cp, fp, bp) = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    rnd = O.make_randomness(seed, n, 64, 64)
    lat = r["latents"].clone().to(DEV).requires_grad_(True)
    kw = _kwargs(coarse, fine, bender, r, rnd)
    rgb, disp, acc, extras = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=32768, retraw=True,
                                      additional_pixel_information={"ray_bending_latents": lat}, detailed_output=True, **kw)
    ret = {"rgb_map": rgb, "rgb0": extras["rgb0"], "visibility_weights": extras["visibility_weights"],
           "unmasked_offsets": extras["unmasked_offsets"], "rigidity_mask": extras["rigidity_mask"]}
    cpo, fpo, bpo = O.clone_params(cp, True), O.clone_params(fp, True), O.clone_params(bp, True)
    lat_o = r["latents"].clone().requires_grad_(True)
    ret_o = O.render_rays(cpo, fpo, bpo, r["rays_o"], r["rays_d"], r["near"], r["far"], lat_o, 64, 64, perturb=True,
                          raw_noise_std=1.0, rnd=rnd)
    # data term scaled to (almost) nothing: the regulariser dominates the gradient by orders of magnitude
    for rr, tgt in ((ret, r["target"].to(DEV)), (ret_o, r["target"])):
        (1e-6 * O.training_loss({k: v for k, v in rr.items() if k in ("rgb_map", "rgb0")}, tgt).mean()
         + (O.training_loss(rr, tgt, 600.0, 5e-4, 1.0) - O.training_loss({k: v for k, v in rr.items() if k in ("rgb_map", "rgb0")}, tgt)).mean()).backward()
    _lib.device_error_check()
    for i in range(5):
        e = _rel(bender.network[i].weight.grad.cpu(), bpo["net_w"][i].grad)
        print(f"  bender net {i}: W {e:.3e}")
        assert e <= 8e-2 and torch.isfinite(bender.network[i].weight.grad).all(), (i, e)
    e = _rel(lat.grad.cpu(), lat_o.grad)
    print(f"  latents: {e:.3e}")
    assert e <= 8e-2, e


def test_device_scalar_schedule_equals_the_host_schedule():
    """global_step as a 0-dim CUDA tensor (what a captured CUDA graph replays): the regularisers' schedule is evaluated inside
    the loss kernel and must give the per-ray loss and gradients of the host-side float schedule (train.py:229, :281)."""
    from nonrigid_nerf_b200 import _lib, parallel
    g = np.load(os.path.join(GOLD, "caseH_training_wrapper.npz"))
    seed, n = int(g["seed"]), int(g["n"])
    out = {}
    for mode in ("host", "device"):
        coarse, fine, bender, _ = helpers.build_models(O, seed, DEV)
        r = O.make_rays(seed, n)
        rnd = dict(O.make_randomness(seed, n, 64, 64)); rnd["e"] = torch.from_numpy(g["e"])
        latents = [torch.from_numpy(row.copy()).to(DEV).requires_grad_(True) for row in g["latent_table"]]
        wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
        step = int(g["global_step"]) if mode == "host" else torch.full((), float(g["global_step"]), device=DEV)
        loss = wrapper(_targs(g), r["rays_o"].to(DEV), r["rays_d"].to(DEV), 100, _kwargs(coarse, fine, bender, r, rnd), r["target"].to(DEV),
                       step, 0, {"imageid_to_timestepid": [int(v) for v in g["i2t"]]}, torch.from_numpy(g["pix"]).to(DEV))
        loss.mean().backward()
        _lib.device_error_check()
        out[mode] = (loss.detach().cpu(), bender.network[0].weight.grad.cpu().clone(), torch.stack([l.grad for l in latents]).cpu())
    for a, b in zip(out["host"], out["device"]):
        assert _rel(b, a) <= 2e-5, _rel(b, a)
