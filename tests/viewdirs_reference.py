"""fp64 reference of the view-dependent head (NeRF(use_viewdirs=True)) for the GPU tests, and model builders.

The head is evaluated from the kernel's own inputs: h8 (the fp16 trunk output, read back from the training kernel's stash on
the same points) and the bent points (the bend pass's input_pts).  Per element the kernel may differ from it by

    alpha   c_K U (|h8| |Wa| + |ba|)
    feature c_K U (|h8| |Wf| + |bf|) + 0.5 ulp_fp16                          (stored as fp16: e_F)
    enc     0.5 ulp_fp16 + 2e-6                                             (MUFU sin / cos after an exact turn reduction: e_E)
    hv      e_F |WvF| + e_E |WvE| + c_K U (|F| |WvF| + |E| |WvE| + |bv|) + 0.5 ulp_fp16   (ReLU is 1-Lipschitz: e_V)
    rgb     e_V |Wr| + c_K U (|hv| |Wr| + |br|)

with c_K = K + 2 for a GEMM of depth K (fp32 accumulation of exact fp16 products) and U = 2^-24.  The weights are their fp16
images, the biases fp32, as the kernels use them.
"""
import torch

from tests import helpers
from tests.parity import F64, U, half_ulp


def view_params_into(module, vp):
    with torch.no_grad():
        module.alpha_linear.weight.copy_(vp["alpha_w"])
        module.alpha_linear.bias.copy_(vp["alpha_b"])
        module.feature_linear.weight.copy_(vp["feature_w"])
        module.feature_linear.bias.copy_(vp["feature_b"])
        module.views_linears[0].weight.copy_(vp["views_w"])
        module.views_linears[0].bias.copy_(vp["views_b"])
        module.rgb_linear.weight.copy_(vp["rgb_w"])
        module.rgb_linear.bias.copy_(vp["rgb_b"])
    return module


def build_view_models(O, seed, device, with_bender=True, s_coarse=64, s_fine=128):
    """Coarse and fine NeRF(use_viewdirs=True) loaded like golden case K: trunks make_nerf_params(seed / seed + 1, 5, 30),
    heads make_view_params(seed + 10 / seed + 11, 30), bender make_bender_params(seed + 2)."""
    from nonrigid_nerf_b200 import run_nerf_helpers as H

    embed_fn, input_ch = H.get_embedder(10, 0)
    _, input_ch_views = H.get_embedder(4, 0)
    bp = O.make_bender_params(seed + 2) if with_bender else None
    bender = helpers.load_bender_module(H.ray_bending(input_ch, 32, "simple_neural", embed_fn), bp).to(device) if with_bender else None
    cp, fp = O.make_nerf_params(seed, 5, 30.0), O.make_nerf_params(seed + 1, 5, 30.0)
    vc, vf = O.make_view_params(seed + 10, 30.0), O.make_view_params(seed + 11, 30.0)
    kw = dict(D=8, W=256, input_ch=input_ch, output_ch=5, skips=[4], input_ch_views=input_ch_views, use_viewdirs=True,
              ray_bender=bender, ray_bending_latent_size=32, approx_nonrigid_viewdirs=True)
    nets = []
    for p, v, s in ((cp, vc, s_coarse), (fp, vf, s_fine)):
        m = H.NeRF(num_ray_samples=s, **kw)
        with torch.no_grad():
            for i in range(8):
                m.pts_linears[i].weight.copy_(p["pts_w"][i])
                m.pts_linears[i].bias.copy_(p["pts_b"][i])
        nets.append(view_params_into(m, v).to(device))
    return nets[0], nets[1], bender, (cp, fp, bp, vc, vf)


def h16(t):
    return t.detach().to(torch.float16).to(F64).cpu()


def directions_fp32(bent, s):
    """The kernel's view directions from its bent points [P, 3] (fp32, the same rounding steps): backward differences
    along each ray of s points, sample 0 taking sample 1's."""
    p = bent.reshape(-1, s, 3).float()
    diff = p[:, 1:] - p[:, :-1]
    dx, dy, dz = diff[..., 0], diff[..., 1], diff[..., 2]
    nrm = torch.sqrt((dx * dx + dy * dy) + dz * dz) + 1e-6
    d = diff / nrm[..., None]
    return torch.cat([d[:, :1], d], 1).reshape(-1, 3)


def head_reference(net, h8, dirs):
    """raw [P, 4] in fp64 and its per-element bound, from h8 [P, 256] (fp16 values) and the directions [P, 3]."""
    import oracle.nrnerf_oracle as O

    h8 = h8.to(F64).cpu()
    wa, ba = h16(net.alpha_linear.weight), net.alpha_linear.bias.detach().to(F64).cpu()
    wf, bf = h16(net.feature_linear.weight), net.feature_linear.bias.detach().to(F64).cpu()
    wv, bv = h16(net.views_linears[0].weight), net.views_linears[0].bias.detach().to(F64).cpu()
    wr, br = h16(net.rgb_linear.weight), net.rgb_linear.bias.detach().to(F64).cpu()
    wvf, wve = wv[:, :256], wv[:, 256:]
    c = lambda k: (k + 2) * U
    alpha = h8 @ wa.T + ba
    e_a = c(256) * (h8.abs() @ wa.abs().T + ba.abs())
    F = h8 @ wf.T + bf
    e_F = c(256) * (h8.abs() @ wf.abs().T + bf.abs())
    e_F = e_F + half_ulp(F.abs() + e_F)
    E = O.direction_encoding(dirs.to(F64).cpu())
    e_E = half_ulp(E.abs()) + 2e-6
    V = F @ wvf.T + E @ wve.T + bv
    e_V = e_F @ wvf.abs().T + e_E @ wve.abs().T + c(256 + 32) * (F.abs() @ wvf.abs().T + E.abs() @ wve.abs().T + bv.abs())
    hv = torch.relu(V)
    e_V = e_V + half_ulp(hv.abs() + e_V)
    rgb = hv @ wr.T + br
    e_r = e_V @ wr.abs().T + c(128) * ((hv.abs() + e_V) @ wr.abs().T + br.abs())
    return torch.cat([rgb, alpha], -1), torch.cat([e_r, e_a], -1)
