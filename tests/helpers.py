"""Shared test helpers: build the package's modules from the oracle's seeded parameter dicts."""
import torch


def load_nerf_module(module, p):
    with torch.no_grad():
        for i in range(8):
            module.pts_linears[i].weight.copy_(p["pts_w"][i])
            module.pts_linears[i].bias.copy_(p["pts_b"][i])
        module.output_linear.weight.copy_(p["out_w"])
        module.output_linear.bias.copy_(p["out_b"])
    return module


def load_bender_module(module, p):
    with torch.no_grad():
        for i in range(5):
            module.network[i].weight.copy_(p["net_w"][i])
            if i < 4:
                module.network[i].bias.copy_(p["net_b"][i])
        for i in range(3):
            module.rigidity_network[i].weight.copy_(p["rig_w"][i])
            module.rigidity_network[i].bias.copy_(p["rig_b"][i])
    return module


def build_models(O, seed, device, with_bender=True, density_boost=30.0):
    """(coarse, fine, bender) modules of the package + the oracle parameter dicts they were loaded from."""
    from nonrigid_nerf_b200 import run_nerf_helpers as H

    embed_fn, input_ch = H.get_embedder(10, 0)
    bp = O.make_bender_params(seed + 2) if with_bender else None
    bender = None
    if with_bender:
        bender = load_bender_module(H.ray_bending(input_ch, 32, "simple_neural", embed_fn), bp).to(device)
    cp = O.make_nerf_params(seed, 5, density_boost)
    fp = O.make_nerf_params(seed + 1, 5, density_boost)
    kw = dict(D=8, W=256, input_ch=input_ch, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False,
              ray_bender=bender, ray_bending_latent_size=32)
    coarse = load_nerf_module(H.NeRF(num_ray_samples=64, **kw), cp).to(device)
    fine = load_nerf_module(H.NeRF(num_ray_samples=128, **kw), fp).to(device)
    return coarse, fine, bender, (cp, fp, bp)


def rays8(r, device):
    n = r["rays_o"].shape[0]
    near = torch.full((n, 1), float(r["near"]))
    far = torch.full((n, 1), float(r["far"]))
    return torch.cat([r["rays_o"], r["rays_d"], near, far], -1).to(device)


def tc_models(seed, device):
    """(coarse, fine) NeRF(time_conditioned_baseline=True) modules with tests/tc_reference's case-L parameters (W0 [256][95],
    W5 [256][351]), and those parameter dicts (cp, fp)."""
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    from tests import tc_reference as R
    cp, fp = R.make_params(seed)
    kw = dict(D=8, W=256, input_ch=63, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False, ray_bender=None,
              ray_bending_latent_size=32, time_conditioned_baseline=True)
    coarse = load_nerf_module(H.NeRF(num_ray_samples=64, **kw), cp).to(device)
    fine = load_nerf_module(H.NeRF(num_ray_samples=128, **kw), fp).to(device)
    return coarse, fine, (cp, fp)
