#!/usr/bin/env python3
"""Golden case M: training the view-dependent head in a rigid scene (NeRF(use_viewdirs=True), ray_bender=None), generated
by EXECUTING THE UNMODIFIED REFERENCE on CPU, with the imports and shims of make_golden.py (cases A-L are untouched):
    python tests/golden/make_golden_views.py
Writes tests/golden/caseM_viewdirs_train.npz: the per-ray loss of training_wrapper_class.forward, a grad_summary of every
coarse and fine parameter, and whether the latents got a gradient.  The embedders and head weights are case K's
(get_embedder(10) / get_embedder(4), make_view_params(seed + 10 + k, 30)); perturb, noise and the seeding of the global
RNG are case H's / L's, so the oracle's make_randomness(seed) reproduces the reference's draws (asserted below).
"""
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402

SEED, N, N_IMG, LAT_STD = 1100, 96, 7, 0.1


def build_view_models(rt, rh, O, seed):
    """Coarse and fine NeRF(use_viewdirs=True) without a bender, loaded as case K's, and the reference's network_query_fn."""
    embed_fn, input_ch = rh.get_embedder(10, 0)
    embeddirs_fn, input_ch_views = rh.get_embedder(4, 0)
    mods = []
    for k, ns in ((0, 64), (1, 128)):
        cp, vp = O.make_nerf_params(seed + k, 5, 30.0), O.make_view_params(seed + 10 + k, 30.0)
        m = rh.NeRF(D=8, W=256, input_ch=input_ch, output_ch=5, skips=[4], input_ch_views=input_ch_views, use_viewdirs=True,
                    ray_bender=None, ray_bending_latent_size=32, embeddirs_fn=embeddirs_fn, num_ray_samples=ns,
                    approx_nonrigid_viewdirs=True, time_conditioned_baseline=False)
        with torch.no_grad():
            for i in range(8):
                m.pts_linears[i].weight.copy_(cp["pts_w"][i]); m.pts_linears[i].bias.copy_(cp["pts_b"][i])
            m.alpha_linear.weight.copy_(vp["alpha_w"]); m.alpha_linear.bias.copy_(vp["alpha_b"])
            m.feature_linear.weight.copy_(vp["feature_w"]); m.feature_linear.bias.copy_(vp["feature_b"])
            m.views_linears[0].weight.copy_(vp["views_w"]); m.views_linears[0].bias.copy_(vp["views_b"])
            m.rgb_linear.weight.copy_(vp["rgb_w"]); m.rgb_linear.bias.copy_(vp["rgb_b"])
        mods.append(m)
    coarse, fine = mods

    def network_query_fn(inputs, viewdirs, additional_pixel_information, network_fn, detailed_output=False):
        return rt.run_network(inputs, viewdirs, additional_pixel_information, network_fn, embed_fn=embed_fn,
                              embeddirs_fn=embeddirs_fn, netchunk=65536, detailed_output=detailed_output)

    kwargs = {"network_query_fn": network_query_fn, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64,
              "network_fn": coarse, "ray_bender": None, "use_viewdirs": True, "white_bkgd": False, "raw_noise_std": 1.0,
              "ndc": False, "lindisp": False}
    return coarse, fine, kwargs


def main():
    import oracle.nrnerf_oracle as O
    rt, rh = G.import_reference()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    outdir = os.path.dirname(os.path.abspath(__file__))
    seed, n = SEED, N
    coarse, fine, kw = build_view_models(rt, rh, O, seed)
    rays = O.make_rays(seed, n)
    lat_rs = np.random.RandomState(seed + 11)
    # training_wrapper_class.forward (train.py:152-287) without a bender and without regularisers, perturb = 1,
    # raw_noise_std = 1; the global-RNG stream is the one the oracle's Generator(seed) reproduces
    latent_list = [torch.from_numpy((lat_rs.randn(32) * LAT_STD).astype(np.float32)).requires_grad_(True) for _ in range(N_IMG)]
    pix = np.stack([lat_rs.randint(0, N_IMG, size=n), lat_rs.randint(0, 384, size=n), lat_rs.randint(0, 512, size=n)], -1)
    pix = torch.from_numpy(pix.astype(np.int64))
    i2t = [int(v) for v in lat_rs.permutation(N_IMG)]
    targs = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=200000, offsets_loss_weight=0.0,
                                  divergence_loss_weight=0.0, rigidity_loss_weight=0.0, ray_bending_latent_size=32)
    kw["near"], kw["far"] = rays["near"], rays["far"]
    global_step = 50000
    wrapper = rt.training_wrapper_class(coarse, latent_list, fine_model=fine, ray_bender=None)
    torch.manual_seed(seed)
    loss = wrapper(targs, rays["rays_o"], rays["rays_d"], 100, kw, rays["target"], global_step, 0, {"imageid_to_timestepid": i2t}, pix)
    torch.manual_seed(seed)
    chk = [torch.rand(n, 64), torch.randn(n, 64), torch.rand(n, 64), torch.randn(n, 128)]
    rnd = O.make_randomness(seed, n, 64, 64)
    for a, b in zip(chk, (rnd["t_rand"], rnd["noise_c"], rnd["u"], rnd["noise_f"])):
        assert torch.equal(a, b), "Generator stream mismatch"
    loss.mean().backward()
    latents_got_grad = any(l.grad is not None and bool(l.grad.any()) for l in latent_list)
    named = [("coarse." + k, v) for k, v in coarse.named_parameters()] + [("fine." + k, v) for k, v in fine.named_parameters()]
    save = dict(seed=seed, n=n, n_img=N_IMG, pix=pix.numpy(), i2t=np.asarray(i2t, dtype=np.int64), global_step=global_step,
                N_iters=targs.N_iters, loss=G.np32(loss), latent_table=np.stack([G.np32(l) for l in latent_list]),
                latents_got_grad=np.bool_(latents_got_grad),
                grad_names=np.array(sorted(k for k, v in named if v.grad is not None)))
    save.update(G.grad_summary(named))
    np.savez_compressed(os.path.join(outdir, "caseM_viewdirs_train.npz"), **save)
    print("case M written to", outdir, "; latents got a gradient:", latents_got_grad)


if __name__ == "__main__":
    main()
