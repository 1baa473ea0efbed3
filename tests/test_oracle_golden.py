"""Pins oracle/nrnerf_oracle.py against the golden vectors produced by executing the unmodified
reference (tests/golden/make_golden.py).  CPU only."""
import os

import numpy as np
import torch

import oracle.nrnerf_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    return np.load(os.path.join(GOLD, name), allow_pickle=False)


def close(a, b, atol, rtol=0.0, name=""):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = np.asarray(b)
    assert a.shape == b.shape, (name, a.shape, b.shape)
    np.testing.assert_allclose(a, b, atol=atol, rtol=rtol, equal_nan=True, err_msg=name)


def models(seed, with_bender=True):
    return (O.make_nerf_params(seed, 5, 30.0), O.make_nerf_params(seed + 1, 5, 30.0),
            O.make_bender_params(seed + 2) if with_bender else None)


def test_caseA_coarse_only():
    g = load("caseA_coarse_only.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, bp = models(seed)
    r = O.make_rays(seed, n)
    with torch.no_grad():
        ret = O.render_rays(cp, None, bp, r["rays_o"], r["rays_d"], r["near"], r["far"], r["latents"], 64, 0)
    close(ret["rgb_map"], g["rgb_map"], 2e-6, name="rgb")
    close(ret["acc_map"], g["acc_map"], 2e-6, name="acc")
    close(ret["disp_map"], g["disp_map"], 0, 2e-5, name="disp")
    close(ret["raw"][:32], g["raw"], 2e-5, name="raw")


def test_caseB_coarse_fine_det():
    g = load("caseB_coarse_fine_det.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, bp = models(seed)
    r = O.make_rays(seed, n)
    with torch.no_grad():
        ret = O.render_rays(cp, fp, bp, r["rays_o"], r["rays_d"], r["near"], r["far"], r["latents"], 64, 64)
    ref_keys = set(str(k) for k in g["keys"])
    ours = set(ret.keys()) - {"z_vals_fine", "z_vals_coarse", "rgb_map", "disp_map", "acc_map"}
    assert ref_keys == ours, (ref_keys ^ ours)
    for k in ("rgb_map", "acc_map", "rgb0", "acc0", "z_std"):
        close(ret[k], g[k], 5e-6, name=k)
    for k in ("disp_map", "disp0"):
        close(ret[k], g[k], 0, 5e-5, name=k)
    close(ret["raw"][:16], g["raw"], 5e-5, name="raw")
    for k in ("fine_visibility_weights", "fine_opacity_alpha", "visibility_weights", "opacity_alpha", "fine_input_pts",
              "fine_unmasked_offsets", "fine_masked_offsets", "fine_rigidity_mask", "fine_initial_input_pts",
              "input_pts", "unmasked_offsets", "masked_offsets", "rigidity_mask", "initial_input_pts"):
        close(ret[k][:16], g[k], 5e-6, name=k)


def test_caseC_train_forward_and_grads():
    g = load("caseC_train.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, bp = models(seed)
    cp, fp, bp = O.clone_params(cp, True), O.clone_params(fp, True), O.clone_params(bp, True)
    r = O.make_rays(seed, n)
    rnd = O.make_randomness(seed, n, 64, 64)
    lat = r["latents"].clone().requires_grad_(True)
    ret = O.render_rays(cp, fp, bp, r["rays_o"], r["rays_d"], r["near"], r["far"], lat, 64, 64, perturb=True,
                        raw_noise_std=1.0, rnd=rnd)
    for k in ("rgb_map", "acc_map", "rgb0", "z_std"):
        close(ret[k], g[k], 1e-5, name=k)
    loss = O.training_loss(ret, r["target"], float(g["offsets_w"]), float(g["rigidity_w"]), float(g["sched"]))
    close(loss, g["loss"], 1e-5, name="loss")
    loss.mean().backward()
    close(lat.grad, g["latents_grad"], 1e-7, 1e-3, name="latents_grad")
    names = {"coarse": cp, "fine": fp}
    for net, p in names.items():
        for i in range(8):
            for kind, key in (("weight", "pts_w"), ("bias", "pts_b")):
                nm = f"{net}.pts_linears.{i}.{kind}"
                gr = p[key][i].grad.reshape(-1)
                idx = torch.from_numpy(g[nm + ".idx"])
                close(gr[idx], g[nm + ".val"], 1e-7, 2e-3, name=nm)
                assert abs(float(gr.norm()) - float(g[nm + ".norm"][0])) <= 1e-3 * float(g[nm + ".norm"][0]) + 1e-9
        nm = f"{net}.output_linear.weight"
        gr = p["out_w"].grad.reshape(-1)
        close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, 2e-3, name=nm)
    for i in range(5):
        nm = f"bender.network.{i}.weight"
        gr = bp["net_w"][i].grad.reshape(-1)
        close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, 2e-3, name=nm)
    for i in range(3):
        nm = f"bender.rigidity_network.{i}.weight"
        gr = bp["rig_w"][i].grad.reshape(-1)
        close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, 2e-3, name=nm)


def test_caseD_test_time_knobs():
    g = load("caseD_knobs.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, bp = models(seed)
    r = O.make_rays(seed, n)
    with torch.no_grad():
        ret = O.render_rays(cp, fp, bp, r["rays_o"], r["rays_d"], r["near"], r["far"], r["latents"], 64, 64,
                            rigidity_cutoff=float(g["cutoff"]), scaling=float(g["scaling"]),
                            removal_threshold=float(g["removal"]))
    for k in ("rgb_map", "acc_map", "rgb0"):
        close(ret[k], g[k], 5e-6, name=k)
    close(ret["rigidity_mask"][:16], g["rigidity_mask"], 1e-6, name="rigidity")
    close(ret["masked_offsets"][:16], g["masked_offsets"], 1e-6, name="masked")
    close(ret["raw"][:8], g["raw"], 5e-5, name="raw")


def test_caseE_ops():
    g = load("caseE_ops.npz")
    bins, w = torch.from_numpy(g["bins"]), torch.from_numpy(g["weights"])
    close(O.sample_pdf(bins, w, O.det_u(bins.shape[0], 64)), g["samples_det"], 1e-6, name="det")
    close(O.sample_pdf(bins, w, torch.from_numpy(g["u_rand"])), g["samples_rand"], 1e-6, name="rand")
    raw, z, rd = torch.from_numpy(g["raw"]), torch.from_numpy(g["z"]), torch.from_numpy(g["rays_d"])
    o = O.raw2outputs(raw, z, rd)
    for a, k in zip(o, ("rgb_map", "disp_map", "acc_map", "alpha", "weights_out", "depth_map")):
        close(a, g[k], 1e-6, 1e-5, name=k)
    assert np.isnan(g["disp_map"][3])  # all-transparent ray: 0/0 (train.py:781-784)
    close(O.raw2outputs(raw, z, rd, None, True)[0], g["rgb_map_white"], 1e-6, name="white")


def test_caseF_canonical():
    g = load("caseF_canonical.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, _ = models(seed, with_bender=False)
    r = O.make_rays(seed, n)
    with torch.no_grad():
        ret = O.render_rays(cp, fp, None, r["rays_o"], r["rays_d"], r["near"], r["far"], r["latents"], 64, 64)
    for k in ("rgb_map", "acc_map", "rgb0"):
        close(ret[k], g[k], 5e-6, name=k)
    ref_keys = set(str(k) for k in g["keys"])
    ours = set(ret.keys()) - {"z_vals_fine", "z_vals_coarse", "rgb_map", "disp_map", "acc_map"}
    assert ref_keys == ours, (ref_keys ^ ours)


def _bender_grad_checks(g, bp, rtol):
    for i in range(5):
        nm = f"bender.network.{i}.weight"
        gr = bp["net_w"][i].grad.reshape(-1)
        close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, rtol, name=nm)
        assert abs(float(gr.norm()) - float(g[nm + ".norm"][0])) <= rtol * float(g[nm + ".norm"][0]) + 1e-9, nm
    for i in range(3):
        nm = f"bender.rigidity_network.{i}.weight"
        gr = bp["rig_w"][i].grad.reshape(-1)
        close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, rtol, name=nm)


def test_caseG_divergence_regulariser():
    """compute_divergence_loss / divergence_approx (run_nerf_helpers.py:22-116) with the probes the reference drew."""
    g = load("caseG_divergence.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, bp = models(seed)
    bp = O.clone_params(bp, True)
    r = O.make_rays(seed, n)
    lat = torch.from_numpy(g["latents"]).clone().requires_grad_(True)
    ret = O.render_rays(cp, fp, bp, r["rays_o"], r["rays_d"], r["near"], r["far"], lat, 64, 64)
    div = O.divergence_loss(bp, ret, lat, n, 64, torch.from_numpy(g["e"]))
    close(div, g["div"], 1e-9, 2e-4, name="div")
    div.mean().backward()
    close(lat.grad, g["latents_grad"], 1e-9, 2e-3, name="latents_grad")
    _bender_grad_checks(g, bp, 2e-3)


def test_caseH_training_wrapper_loss_and_grads():
    """The per-ray loss [N] DataParallel gathers (training_wrapper_class.forward, train.py:152-287), all regularisers on."""
    g = load("caseH_training_wrapper.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, bp = models(seed)
    cp, fp, bp = O.clone_params(cp, True), O.clone_params(fp, True), O.clone_params(bp, True)
    r = O.make_rays(seed, n)
    rnd = O.make_randomness(seed, n, 64, 64)
    table = torch.from_numpy(g["latent_table"]).clone().requires_grad_(True)
    loss, _ = O.training_wrapper_loss(cp, fp, bp, r, table, g["i2t"], torch.from_numpy(g["pix"]), rnd, torch.from_numpy(g["e"]),
                                      int(g["global_step"]), int(g["N_iters"]), float(g["offsets_w"]), float(g["divergence_w"]),
                                      float(g["rigidity_w"]))
    close(loss, g["loss"], 2e-6, 2e-5, name="loss")
    loss.mean().backward()
    close(table.grad, g["latent_grads"], 1e-8, 2e-3, name="latent_grads")
    for net, p in {"coarse": cp, "fine": fp}.items():
        for i in (0, 4, 5, 7):
            nm = f"{net}.pts_linears.{i}.weight"
            gr = p["pts_w"][i].grad.reshape(-1)
            close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, 2e-3, name=nm)
    _bender_grad_checks(g, bp, 2e-3)


def test_caseI_get_rays_bit_exact():
    g = load("caseI_get_rays.npz")
    intrin = {k: float(g[k]) for k in ("height", "width", "focal_x", "focal_y", "center_x", "center_y")}
    ro, rd = O.get_rays(torch.from_numpy(g["c2w"]), intrin)
    assert np.array_equal(rd.numpy(), g["rays_d"]) and np.array_equal(ro.numpy(), g["rays_o"])


def test_caseJ_surface_selection():
    g = load("caseJ_surface.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, bp = models(seed)
    r = O.make_rays(seed, n)
    with torch.no_grad():
        ret = O.render_rays(cp, fp, bp, r["rays_o"], r["rays_d"], r["near"], r["far"], r["latents"][:1].expand(n, 32), 64, 64)
    idx, pts, rig = O.surface_selection(ret["fine_visibility_weights"], ret["fine_input_pts"], ret["fine_rigidity_mask"])
    same = (idx.numpy() == g["median_indices"])
    assert same.mean() >= 0.99, same.mean()        # a near-tie of |acc - 0.5| may flip under 1-ulp differences of the weights
    close(pts[torch.from_numpy(same)], g["surface_pts"][same], 5e-6, name="surface_pts")
    close(rig[torch.from_numpy(same)], g["surface_rigidity"][same], 5e-6, name="surface_rigidity")
    # and on the reference's own weights the selection is exact
    idx2, _, _ = O.surface_selection(torch.from_numpy(g["fine_visibility_weights"]), ret["fine_input_pts"], None)
    assert np.array_equal(idx2.numpy(), g["median_indices"])


def test_caseK_view_dependent_head_and_finite_difference_viewdirs():
    """Row f1's oracle: use_viewdirs=True with approx_nonrigid_viewdirs=True, against the executed reference."""
    g = load("caseK_viewdirs.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, bp = models(seed)
    vc, vf = O.make_view_params(seed + 10, 30.0), O.make_view_params(seed + 11, 30.0)
    cp, fp, bp, vc, vf = (O.clone_params(q, True) for q in (cp, fp, bp, vc, vf))
    r = O.make_rays(seed, n)
    lat = r["latents"].clone().requires_grad_(True)
    ret = O.render_rays(cp, fp, bp, r["rays_o"], r["rays_d"], r["near"], r["far"], lat, 64, 64, vpar_c=vc, vpar_f=vf)
    for k in ("rgb_map", "acc_map", "rgb0"):
        close(ret[k], g[k], 5e-6, name=k)
    assert ret["raw"].shape[-1] == 4
    close(ret["raw"][:8], g["raw"], 5e-5, name="raw")
    loss = O.training_loss(ret, r["target"], 0.0, 0.0, 0.0)
    close(loss, g["loss"], 1e-5, name="loss")
    loss.mean().backward()
    close(lat.grad, g["latents_grad"], 1e-7, 2e-3, name="latents_grad")
    for net, p, v in (("coarse", cp, vc), ("fine", fp, vf)):
        for nm, t in ((f"{net}.views_linears.0.weight", v["views_w"]), (f"{net}.feature_linear.weight", v["feature_w"]),
                      (f"{net}.alpha_linear.weight", v["alpha_w"]), (f"{net}.rgb_linear.weight", v["rgb_w"]),
                      (f"{net}.pts_linears.0.weight", p["pts_w"][0]), (f"{net}.pts_linears.7.weight", p["pts_w"][7])):
            gr = t.grad.reshape(-1)
            close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, 2e-3, name=nm)
            assert abs(float(gr.norm()) - float(g[nm + ".norm"][0])) <= 1e-3 * float(g[nm + ".norm"][0]) + 1e-9, nm
        assert p["out_w"].grad is None       # output_linear is dead with use_viewdirs=True
    with torch.no_grad():                # static scene: the view direction is the ray's own
        st = O.render_rays(cp, fp, None, r["rays_o"], r["rays_d"], r["near"], r["far"], r["latents"], 64, 64, vpar_c=vc, vpar_f=vf)
    close(st["rgb_map"], g["static_rgb_map"], 5e-6, name="static rgb")
    close(st["rgb0"], g["static_rgb0"], 5e-6, name="static rgb0")
    close(st["raw"][:8], g["static_raw"], 5e-5, name="static raw")
    nm = "bender.network.0.weight"       # the view directions depend on the bent points: the bender sees that gradient too
    gr = bp["net_w"][0].grad.reshape(-1)
    close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, 2e-3, name=nm)


VIEW_HEAD_KEYS = (("views_linears.0", "views"), ("feature_linear", "feature"), ("alpha_linear", "alpha"), ("rgb_linear", "rgb"))


def view_model_tensors(p, v):
    """{reference parameter name: oracle tensor} of one NeRF(use_viewdirs=True) (make_nerf_params / make_view_params)."""
    out = {}
    for i in range(8):
        out[f"pts_linears.{i}.weight"], out[f"pts_linears.{i}.bias"] = p["pts_w"][i], p["pts_b"][i]
    for mod, key in VIEW_HEAD_KEYS:
        out[f"{mod}.weight"], out[f"{mod}.bias"] = v[key + "_w"], v[key + "_b"]
    return out


def test_caseM_training_wrapper_with_the_view_dependent_head():
    """Training the view-dependent head without a bender: the oracle's training_wrapper_loss (vpar_c / vpar_f) against
    the executed training_wrapper_class, per-ray loss and every coarse and fine parameter's gradient; the latents get
    no gradient in the reference."""
    g = load("caseM_viewdirs_train.npz")
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp, _ = models(seed, with_bender=False)
    vc, vf = O.make_view_params(seed + 10, 30.0), O.make_view_params(seed + 11, 30.0)
    cp, fp, vc, vf = (O.clone_params(q, True) for q in (cp, fp, vc, vf))
    r = O.make_rays(seed, n)
    rnd = O.make_randomness(seed, n, 64, 64)
    table = torch.from_numpy(g["latent_table"]).clone().requires_grad_(True)
    loss, _ = O.training_wrapper_loss(cp, fp, None, r, table, g["i2t"], torch.from_numpy(g["pix"]), rnd, None,
                                      int(g["global_step"]), int(g["N_iters"]), 0.0, 0.0, 0.0, vpar_c=vc, vpar_f=vf)
    close(loss, g["loss"], 5e-6, name="loss")
    loss.mean().backward()
    assert not bool(g["latents_got_grad"]) and (table.grad is None or not bool(table.grad.any()))
    tensors = {f"coarse.{k}": t for k, t in view_model_tensors(cp, vc).items()}
    tensors.update({f"fine.{k}": t for k, t in view_model_tensors(fp, vf).items()})
    assert set(str(k) for k in g["grad_names"]) == set(tensors)
    for nm, t in tensors.items():
        gr = t.grad.reshape(-1)
        close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, 2e-3, name=nm)
        assert abs(float(gr.norm()) - float(g[nm + ".norm"][0])) <= 2e-3 * float(g[nm + ".norm"][0]) + 1e-9, nm


def test_flop_ledger():
    cp = O.make_nerf_params(0)
    bp = O.make_bender_params(0)
    macs = sum(w.numel() for w in cp["pts_w"]) + cp["out_w"].numel()
    bmacs = sum(w.numel() for w in bp["net_w"]) + sum(w.numel() for w in bp["rig_w"])
    assert 2 * (macs + bmacs) == O.FLOP_PER_POINT
