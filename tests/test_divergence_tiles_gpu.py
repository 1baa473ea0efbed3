"""The tensor-core divergence kernels (csrc/div.cu) at a size where every CTA of the persistent grid runs more than one
tile and the last tile is ragged: 1023 rays x 64 coarse samples = 511.5 tiles of 128 points.  Compared with the fp32
oracle at the bounds of test_render_gpu.py (per-ray value 2e-2, gradients 8e-2, relative L2):
  * the per-ray divergence term;
  * the gradients it hands to the coarse field backward, w.r.t. unmasked_offsets and rigidity_mask, against the closed
    form  G tau_r e  and  G (alpha + 2 beta tau_c (1 - 2 r))  evaluated in fp32 with a forward-mode derivative;
  * the bender weight and latent gradients against the oracle's double backward.
"""
import pytest
import torch
import torch.nn.functional as F

import oracle.nrnerf_oracle as O
from tests import helpers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_RAYS, S = 1023, 64


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-30))


def _closed_form_upstream_grads(bp, pts, lat, e, w, coef):
    """fp32 reference of the gradients w.r.t. the primal offsets and rigidity, for loss = coef * sum_rays div."""
    def bender(x):
        h = torch.cat([x, lat], -1)
        for i in range(5):
            h = F.linear(h, bp["net_w"][i], bp["net_b"][i] if i < 4 else None)
            if i != 4:
                h = F.relu(h)
        c = x
        for i in range(3):
            c = F.linear(c, bp["rig_w"][i], bp["rig_b"][i])
            if i != 2:
                c = F.relu(c)
        return h, c[:, 0]

    (off, c), (tau_off, tau_c) = torch.func.jvp(bender, (pts,), (e,))
    r = (torch.tanh(c) + 1.0) / 2.0
    alpha, beta = (e * tau_off).sum(-1), (e * off).sum(-1)
    tau_r = 2.0 * r * (1.0 - r) * tau_c
    d = r * alpha + beta * tau_r
    G = coef * 2.0 * w * d / S
    return G[:, None] * tau_r[:, None] * e, G * (alpha + 2.0 * beta * tau_c * (1.0 - 2.0 * r))


def test_divergence_over_many_tiles_matches_oracle():
    from nonrigid_nerf_b200 import _lib, autograd as ag
    from nonrigid_nerf_b200 import train as T
    seed = 733
    coarse, _, bender, (_, _, bp) = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, N_RAYS)
    e = torch.randn(N_RAYS * S, 3, generator=torch.Generator().manual_seed(9))
    lat = r["latents"].clone().to(DEV).requires_grad_(True)
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=0, network_fine=None, N_samples=S, network_fn=coarse,
              ray_bender=bender, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    _, _, _, extras = T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=32768, near=r["near"], far=r["far"],
                               additional_pixel_information={"ray_bending_latents": lat}, detailed_output=True, retraw=True, **kw)
    got = {}
    extras["unmasked_offsets"].register_hook(lambda g: got.__setitem__("d_un", g.detach().reshape(-1, 3).cpu()))
    extras["rigidity_mask"].register_hook(lambda g: got.__setitem__("d_rig", g.detach().reshape(-1).cpu()))
    w = 1.0 - torch.exp(-torch.relu(extras["opacity_alpha"].detach()))
    div = ag.divergence_loss(extras["unmasked_offsets"], extras["rigidity_mask"], w, bender, e.to(DEV))
    assert div.shape == (N_RAYS,)
    coef = 1e3 / N_RAYS
    (div.sum() * coef).backward()
    _lib.device_error_check()

    # oracle: the same points, weights and probes; the autograd.grad(create_graph=True) restatement of the reference
    pts = extras["initial_input_pts"].detach().reshape(-1, 3).cpu()
    ret_o = {"initial_input_pts": pts, "opacity_alpha": extras["opacity_alpha"].detach().cpu()}
    bpo = O.clone_params(bp, True)
    lat_o = r["latents"].clone().requires_grad_(True)
    div_o = O.divergence_loss(bpo, ret_o, lat_o, N_RAYS, S, e)
    (div_o.sum() * coef).backward()

    rel_v = _rel(div.detach().cpu(), div_o.detach())
    print(f"divergence per ray ({N_RAYS} rays x {S}): rel err {rel_v:.3e} (mean {float(div_o.detach().mean()):.3e})")
    assert rel_v <= 2e-2

    lat_p = r["latents"][:, None, :].expand(N_RAYS, S, r["latents"].shape[-1]).reshape(N_RAYS * S, -1)
    ref_un, ref_rig = _closed_form_upstream_grads(O.clone_params(bp), pts, lat_p, e, w.reshape(-1).cpu(), coef)
    e_un, e_rig = _rel(got["d_un"], ref_un), _rel(got["d_rig"], ref_rig)
    print(f"  d_unmasked_offsets: {e_un:.3e}   d_rigidity_mask: {e_rig:.3e}")
    assert e_un <= 8e-2 and e_rig <= 8e-2, (e_un, e_rig)

    for i in range(5):
        e_w = _rel(bender.network[i].weight.grad.cpu(), bpo["net_w"][i].grad)
        print(f"  net {i} W: {e_w:.3e}")
        assert e_w <= 8e-2, (i, e_w)
        if i < 4:
            assert _rel(bender.network[i].bias.grad.cpu(), bpo["net_b"][i].grad) <= 8e-2, i
    for i in range(3):
        e_w = _rel(bender.rigidity_network[i].weight.grad.cpu(), bpo["rig_w"][i].grad)
        print(f"  rigidity {i} W: {e_w:.3e}")
        assert e_w <= 8e-2, (i, e_w)
        assert _rel(bender.rigidity_network[i].bias.grad.cpu(), bpo["rig_b"][i].grad) <= 8e-2, i
    e_l = _rel(lat.grad.cpu(), lat_o.grad)
    print(f"  latents: {e_l:.3e}")
    assert e_l <= 8e-2
