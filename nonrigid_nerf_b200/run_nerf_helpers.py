"""Host-side mirror of the reference's run_nerf_helpers.py hot-path entry points.

Same names, constructor/forward signatures, attribute names and state_dict keys as the reference
(so `logs/*.tar` checkpoints interchange: pts_linears.N.{weight,bias}, views_linears.0.*,
output_linear.*, network.N.*, rigidity_network.N.*), but every forward dispatches to the fused
sm_90a kernels through the C ABI.  There is no PyTorch fallback: unsupported configurations raise.

Reference: run_nerf_helpers.py:10-19 (misc), :120-168 (Embedder), :172-385 (NeRF), :388-584
(ray_bending), :651-698 (sample_pdf), :701-793 (disparity visualisation).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import ops
from . import autograd as _ag

# ---- misc (run_nerf_helpers.py:10-19) ---------------------------------------------------------


def img2mse(x, y, N_rays):
    # per-ray mean squared error, shape [N_rays]
    return torch.mean(((x - y) ** 2).view(N_rays, -1), dim=1)


def mse2psnr(x):
    return -10.0 * torch.log(x) / np.log(10.0)


def to8b(x):
    return (255 * np.clip(x, 0, 1)).astype(np.uint8)


# ---- positional encoding (run_nerf_helpers.py:120-168) ----------------------------------------
class Embedder:
    """Bookkeeping object for the sinusoidal encoding.  The encoding itself is evaluated inside the
    fused field kernel (csrc/field_fwd.cu: write_pe); `embed` is kept for API compatibility and is
    used only to carry raw xyz through run_network's [P, 63(+27)+32] interface."""

    def __init__(self, **kwargs):
        self.kwargs = kwargs
        d = kwargs["input_dims"]
        self.out_dim = (d if kwargs["include_input"] else 0) + 2 * d * kwargs["num_freqs"]
        if not kwargs.get("log_sampling", True) or not kwargs["include_input"]:
            raise RuntimeError("nonrigid_nerf_b200: only include_input=True, log_sampling=True is implemented")
        self.num_freqs = kwargs["num_freqs"]

    def embed(self, inputs):
        # the kernels re-derive every feature from the first three entries (raw xyz), exactly like the
        # reference's ray bender does (run_nerf_helpers.py:517-521); the remaining slots stay zero.
        out = inputs.new_zeros(inputs.shape[:-1] + (self.out_dim,))
        out[..., : inputs.shape[-1]] = inputs
        return out


def get_embedder(multires, i=0):
    if i == -1:
        raise RuntimeError("nonrigid_nerf_b200: i_embed=-1 (no positional encoding) is not implemented")
    embed_kwargs = {"include_input": True, "input_dims": 3, "max_freq_log2": multires - 1, "num_freqs": multires,
                    "log_sampling": True, "periodic_fns": [torch.sin, torch.cos]}
    embedder_obj = Embedder(**embed_kwargs)
    embed = lambda x, eo=embedder_obj: eo.embed(x)  # noqa: E731
    return embed, embedder_obj.out_dim


# ---- models -------------------------------------------------------------------------------------
class ray_bending(nn.Module):
    """Parameters of the ray-bending deformation network (run_nerf_helpers.py:388-505).  Stays an
    ordinary nn.Module so the optimizer, checkpoints and the PyTorch-side divergence regulariser
    (which needs double backward, SURVEY.md 7.3-1) keep working on the same tensors."""

    def __init__(self, input_ch, ray_bending_latent_size, ray_bending_mode, embed_fn):
        super().__init__()
        if ray_bending_mode != "simple_neural":
            raise RuntimeError(f"nonrigid_nerf_b200: ray_bending_mode={ray_bending_mode!r} is not implemented")
        self.use_positionally_encoded_input = False
        self.input_ch = 3
        self.output_ch = 3
        self.ray_bending_latent_size = ray_bending_latent_size
        self.ray_bending_mode = ray_bending_mode
        self.embed_fn = embed_fn
        self.use_rigidity_network = True
        self.rigidity_test_time_cutoff = None   # test-time editing knobs, read at every call
        self.test_time_scaling = None
        hid, rhid = 64, 32
        self.network = nn.ModuleList([nn.Linear(3 + ray_bending_latent_size, hid)] + [nn.Linear(hid, hid) for _ in range(3)]
                                     + [nn.Linear(hid, 3, bias=False)])
        self.rigidity_network = nn.ModuleList([nn.Linear(3, rhid), nn.Linear(rhid, rhid), nn.Linear(rhid, 1)])
        with torch.no_grad():
            for layer in list(self.network[:-1]) + list(self.rigidity_network[:-1]):
                nn.init.kaiming_uniform_(layer.weight, a=0, mode="fan_in", nonlinearity="relu")
                nn.init.zeros_(layer.bias)
            self.network[-1].weight.zero_()          # start with straight rays
            self.rigidity_network[-1].weight.zero_()
            self.rigidity_network[-1].bias.zero_()

    def forward(self, input_pts, input_latents, details=None, special_loss_return=False):
        """Stand-alone bender evaluation.  The render path never calls this (the bender runs fused
        inside the field kernel); it exists for the divergence regulariser
        (run_nerf_helpers.py:42-49), which differentiates it twice, so it is plain autograd-able
        PyTorch over the SAME parameters (SURVEY.md section 8a row a11 / 7.3-1: out of kernel scope)."""
        if not special_loss_return:
            raise RuntimeError("nonrigid_nerf_b200: ray_bending.forward is only available with special_loss_return=True "
                               "(divergence regulariser); rendering uses the fused kernel")
        if details is None:
            details = {}
        xyz = input_pts[:, :3]
        h = torch.cat([xyz, input_latents], -1)
        for i, layer in enumerate(self.network):
            h = layer(h)
            if i != len(self.network) - 1:
                h = torch.relu(h)
        details["unmasked_offsets"] = h
        r = xyz
        for i, layer in enumerate(self.rigidity_network):
            r = layer(r)
            if i != len(self.rigidity_network) - 1:
                r = torch.relu(r)
        rigidity = (torch.tanh(r) + 1) / 2
        if self.rigidity_test_time_cutoff is not None:
            rigidity = torch.where(rigidity <= self.rigidity_test_time_cutoff, torch.zeros_like(rigidity), rigidity)
        masked = rigidity * h
        if self.test_time_scaling is not None:
            masked = masked * self.test_time_scaling
        details["rigidity_mask"] = rigidity
        details["masked_offsets"] = masked
        return details


class NeRF(nn.Module):
    """Canonical 8x256 radiance-field MLP (run_nerf_helpers.py:172-314), evaluated by the fused kernel."""

    def __init__(self, D=8, W=256, input_ch=3, input_ch_views=3, output_ch=4, skips=[4], use_viewdirs=False,
                 ray_bender=None, ray_bending_latent_size=0, embeddirs_fn=None, num_ray_samples=None,
                 approx_nonrigid_viewdirs=True, time_conditioned_baseline=False):
        super().__init__()
        if use_viewdirs:
            # the view-dependent head (run_nerf_helpers.py:233-236, 284-304), inference only; training raises at call time
            if input_ch_views != 27:
                raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True needs input_ch_views=27 (multires_views=4), "
                                   f"got {input_ch_views}")
            if time_conditioned_baseline:
                raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True together with time_conditioned_baseline is not implemented")
            if ray_bender is not None and not approx_nonrigid_viewdirs:
                raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True with approx_nonrigid_viewdirs=False (exact view "
                                   "directions through the ray bender) is not implemented")
            if ray_bender is not None and (num_ray_samples is None or num_ray_samples < 2):
                raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True with a ray bender needs num_ray_samples >= 2 "
                                   f"(finite-difference view directions), got {num_ray_samples}")
        if time_conditioned_baseline and ray_bending_latent_size != ops.LATENT:
            raise RuntimeError("nonrigid_nerf_b200: time_conditioned_baseline needs ray_bending_latent_size=32 "
                               f"(got {ray_bending_latent_size})")
        if D != 8 or W != 256 or list(skips) != [4] or input_ch != 63:
            raise RuntimeError("nonrigid_nerf_b200: only netdepth=8, netwidth=256, skips=[4], multires=10 is implemented")
        self.D, self.W = D, W
        self.input_ch, self.input_ch_views = input_ch, input_ch_views
        self.skips = skips
        self.use_viewdirs = use_viewdirs
        self.approx_nonrigid_viewdirs = approx_nonrigid_viewdirs
        self.embeddirs_fn = embeddirs_fn
        self.num_ray_samples = num_ray_samples
        self.test_time_nonrigid_object_removal_threshold = None
        self.time_conditioned_baseline = time_conditioned_baseline
        self.ray_bending_latent_size = ray_bending_latent_size
        self.ray_bender = (ray_bender,)  # 1-tuple: keeps the bender out of NeRF.parameters() (run_nerf_helpers.py:213-215)
        # naive NR-NeRF baseline (run_nerf_helpers.py:206-209): the per-frame latent joins the embedding at layer 0 and at the
        # skip layer, so those layers take 63 + 32 and 63 + 32 + 256 inputs.  The kernels fold the latent columns into a
        # per-ray bias of both layers (csrc/field_fwd.cu).
        lin_in = input_ch + (ray_bending_latent_size if time_conditioned_baseline else 0)
        self.pts_linears = nn.ModuleList([nn.Linear(lin_in, W)] + [nn.Linear(W, W) if i not in skips else nn.Linear(W + lin_in, W)
                                                                    for i in range(D - 1)])
        # use_viewdirs=False: views_linears is dead weight, kept for checkpoints
        self.views_linears = nn.ModuleList([nn.Linear(input_ch_views + W, W // 2)])
        if use_viewdirs:
            self.feature_linear = nn.Linear(W, W)
            self.alpha_linear = nn.Linear(W, 1)
            self.rgb_linear = nn.Linear(W // 2, 3)
        else:
            self.output_linear = nn.Linear(W, output_ch)

    def forward(self, x, detailed_output=False):
        """x: [P, input_ch + input_ch_views + latent] as built by run_network; only x[:, :3] (raw xyz)
        and the latent columns are read (the kernel re-derives the encoding)."""
        p = x.shape[0]
        pts = x[:, :3]
        lat = x[:, self.input_ch + self.input_ch_views:] if self.ray_bending_latent_size > 0 else None
        if self.use_viewdirs:
            # with a bender the rows form rays of num_ray_samples points (their bent points give the view directions,
            # run_nerf_helpers.py:316-356); without one the direction is the first three view columns (the raw d of the
            # embedded directions)
            vd = x[:, self.input_ch:self.input_ch + 3]
            raw, details = _ag.field_views(self, None, None, pts, lat, vd, detailed_output)
        else:
            raw, details = _ag.field_points(self, pts, lat, detailed_output)
        raw = raw.reshape(p, -1)
        if detailed_output:
            return raw, {k: v.reshape(p, -1) for k, v in details.items()}
        return raw


# ---- ray helpers (run_nerf_helpers.py:588-605) ------------------------------------------------------------
def get_rays(c2w, intrin):
    """rays_o, rays_d [H, W, 3] of the camera c2w [3(+), 4] with intrinsics intrin (dict: height, width, focal_x, focal_y,
    center_x, center_y) -- one kernel, bit-identical to the reference's float32 arithmetic."""
    return ops.get_rays(c2w, intrin)


# ---- hierarchical sampling (run_nerf_helpers.py:651-698) ------------------------------------------
def sample_pdf(bins, weights, N_samples, det=False, pytest=False):
    if pytest:
        raise RuntimeError("nonrigid_nerf_b200: the pytest= numpy-random hook is not supported; pass randomness explicitly")
    u = None if det else torch.rand(list(bins.shape[:-1]) + [N_samples], device=bins.device)
    lead = bins.shape[:-1]
    out = ops.sample_pdf_op(bins.reshape(-1, bins.shape[-1]), weights.reshape(-1, weights.shape[-1]), N_samples,
                            None if u is None else u.reshape(-1, N_samples))
    return out.reshape(*lead, N_samples)


# ---- disparity visualisation (run_nerf_helpers.py:701-793) ------------------------------------------------
def _disparity_image(depth_map, which: int):
    """One disparity map [H, W] through evaluation.disparity_images: a CUDA tensor gives a CUDA tensor [H, W, 3] (no
    host copy), anything else is read as a numpy array and gives a numpy array, like the reference."""
    from . import evaluation
    if isinstance(depth_map, torch.Tensor) and depth_map.is_cuda:
        return evaluation.disparity_images(depth_map[None], jet=which == 0, phong=which == 1)[which][0]
    d = torch.from_numpy(np.ascontiguousarray(depth_map, dtype=np.float32)).cuda()
    return evaluation.disparity_images(d[None], jet=which == 0, phong=which == 1)[which][0].cpu().numpy()


def visualize_disparity_with_jet_color_scheme(depth_map_in):
    """cm.jet colours [H, W, 3] of clip(depth_map_in, 0, 1) (fp32 values of the float64 table)."""
    return _disparity_image(depth_map_in, 0)


def visualize_disparity_with_blinn_phong(depth_map):
    """The reference's Blinn-Phong shading [H, W, 3] of the normals of the disparity map [H, W] (H, W >= 2), in fp32."""
    return _disparity_image(depth_map, 1)


# ---- divergence regulariser (run_nerf_helpers.py:22-116) --------------------------------------------
# Stays PyTorch autograd over the SAME bender parameters: it needs d(offset)/d(xyz) differentiated a
# second time w.r.t. the weights (double backward), which the first-order DGRAD/WGRAD kernels do not
# serve (SURVEY.md 7.3-1, section 8f row f2).  ~3 % of the step's FLOPs, coarse samples only.
def divergence_approx(input_points, offsets_of_inputs):
    """Hutchinson estimator e^T J e of the trace of the offset field's Jacobian (FFJORD)."""
    e = torch.randn_like(offsets_of_inputs)
    e_dydx = torch.autograd.grad(offsets_of_inputs, input_points, e, create_graph=True)[0]
    return (e_dydx * e).view(offsets_of_inputs.shape[0], -1).sum(dim=1)


def _get_minibatch_jacobian(y, x):
    """[N, D_y, D_x] Jacobian, one autograd pass per output dimension."""
    assert y.shape[0] == x.shape[0]
    y = y.view(y.shape[0], -1)
    rows = []
    for j in range(y.shape[1]):
        dy = torch.autograd.grad(y[:, j], x, torch.ones_like(y[:, j]), retain_graph=True, create_graph=True)[0]
        rows.append(dy.view(x.shape[0], 1, -1))
    return torch.cat(rows, 1)


def divergence_exact(input_points, offsets_of_inputs):
    jac = _get_minibatch_jacobian(offsets_of_inputs, input_points)
    return torch.diagonal(jac, dim1=1, dim2=2).sum(1)


def compute_divergence_loss(offsets_of_inputs, input_points, point_latents, ray_bender, exact, chunk, N_rays, weights=None,
                            backprop_into_weights=True):
    """Per-ray mean over samples of weights * divergence(offset field)^2."""
    divergence_fn = divergence_exact if exact else divergence_approx
    input_points = input_points.detach().requires_grad_(True)
    pieces = []
    for i in range(0, input_points.shape[0], chunk):
        sub = input_points[i:i + chunk, :]
        details = ray_bender(sub, point_latents[i:i + chunk, :], special_loss_return=True)
        offsets = details["masked_offsets"] if "masked_offsets" in details else details["unmasked_offsets"]
        pieces.append(divergence_fn(sub, offsets))
    div = torch.abs(torch.cat(pieces, dim=0)) ** 2
    if weights is not None:
        if not backprop_into_weights:
            weights = weights.detach()
        div = weights * div
    return torch.mean(div.view(N_rays, -1), dim=-1)
