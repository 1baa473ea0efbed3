"""CPU oracle for the NR-NeRF per-ray volumetric rendering hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in the shipped package (`nonrigid_nerf_b200/`) imports this
module; only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline legs may.  It is a
from-scratch restatement, in plain fp32 PyTorch-on-CPU tensor ops (the reference's own arithmetic
library), of the algorithm in the reference files cited per function (paths relative to
/root/reference).  It is written functionally -- explicit weight dictionaries, randomness passed in
as tensors -- so that the CUDA path and the oracle can be driven with byte-identical inputs.

Parity pinning: the reference ships no tests / golden vectors (SURVEY.md section 4), so the oracle
is pinned against outputs of the *executed, unmodified reference* (tests/golden/make_golden.py
imports /root/reference in the build container and stores its outputs; tests/test_oracle_golden.py
checks this file against them).

Conventions
-----------
nerf params  : dict  pts_w[i] [out,in], pts_b[i] [out] (i = 0..7), out_w [C,256], out_b [C]
bender params: dict  net_w[i], net_b[i] (i = 0..3), net_w[4] (no bias), rig_w[i], rig_b[i] (i = 0..2)
All tensors fp32.  `latents` is per-ray [N, Z].
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

Tensor = torch.Tensor

NERF_D = 8
NERF_W = 256
NERF_SKIP = 4  # after layer index 4 the embedding is concatenated in front of h
PE_L = 10      # multires
LATENT = 32


# --------------------------------------------------------------------------------------------
# deterministic weights / inputs (numpy RandomState => identical on every machine)
# --------------------------------------------------------------------------------------------
def make_nerf_params(seed: int, out_ch: int = 5, density_boost: float = 1.0, input_ch: int = 63) -> Dict[str, list]:
    """nn.Linear default init (U(-1/sqrt(fan_in), +1/sqrt(fan_in)) for weight and bias), as used by
    NeRF.__init__ (run_nerf_helpers.py:218-238).  `density_boost` multiplies the sigma row of the
    output layer so that test scenes are not almost transparent."""
    rs = np.random.RandomState(seed)
    p = {"pts_w": [], "pts_b": []}
    for i in range(NERF_D):
        fan_in = input_ch if i == 0 else (NERF_W + input_ch if i == NERF_SKIP + 1 else NERF_W)
        b = 1.0 / math.sqrt(fan_in)
        p["pts_w"].append(torch.from_numpy(rs.uniform(-b, b, size=(NERF_W, fan_in)).astype(np.float32)))
        p["pts_b"].append(torch.from_numpy(rs.uniform(-b, b, size=(NERF_W,)).astype(np.float32)))
    b = 1.0 / math.sqrt(NERF_W)
    ow = rs.uniform(-b, b, size=(out_ch, NERF_W)).astype(np.float32)
    ob = rs.uniform(-b, b, size=(out_ch,)).astype(np.float32)
    ow[3] *= density_boost
    ob[3] = ob[3] * density_boost + (0.5 * density_boost if density_boost != 1.0 else 0.0)
    p["out_w"] = torch.from_numpy(ow)
    p["out_b"] = torch.from_numpy(ob)
    return p


def make_view_params(seed: int, density_boost: float = 1.0) -> Dict[str, Tensor]:
    """The view-dependent branch of NeRF(use_viewdirs=True) (run_nerf_helpers.py:225-236): alpha_linear 256->1,
    feature_linear 256->256, views_linears[0] (256 + 27)->128, rgb_linear 128->3; nn.Linear default init."""
    rs = np.random.RandomState(seed)

    def lin(out_f, in_f):
        b = 1.0 / math.sqrt(in_f)
        return (torch.from_numpy(rs.uniform(-b, b, size=(out_f, in_f)).astype(np.float32)),
                torch.from_numpy(rs.uniform(-b, b, size=(out_f,)).astype(np.float32)))
    p = {}
    p["alpha_w"], p["alpha_b"] = lin(1, NERF_W)
    p["feature_w"], p["feature_b"] = lin(NERF_W, NERF_W)
    p["views_w"], p["views_b"] = lin(NERF_W // 2, NERF_W + 27)
    p["rgb_w"], p["rgb_b"] = lin(3, NERF_W // 2)
    if density_boost != 1.0:
        p["alpha_w"] = p["alpha_w"] * density_boost
        p["alpha_b"] = p["alpha_b"] * density_boost + 0.5 * density_boost
    return p


def make_bender_params(seed: int, latent: int = LATENT, offset_std: float = 0.01, rigid_std: float = 0.1) -> Dict[str, list]:
    """ray_bending init (run_nerf_helpers.py:433-505): kaiming-uniform(relu) hidden weights, zero
    hidden biases; the two zero-initialised output layers are re-drawn N(0, std) so that bending is
    not the identity (SURVEY.md section 8c)."""
    rs = np.random.RandomState(seed)
    p = {"net_w": [], "net_b": [], "rig_w": [], "rig_b": []}
    dims = [3 + latent, 64, 64, 64, 64]
    for i in range(4):
        bound = math.sqrt(6.0 / dims[i])
        p["net_w"].append(torch.from_numpy(rs.uniform(-bound, bound, size=(64, dims[i])).astype(np.float32)))
        p["net_b"].append(torch.zeros(64))
    p["net_w"].append(torch.from_numpy((rs.randn(3, 64) * offset_std).astype(np.float32)))
    rd = [3, 32]
    for i in range(2):
        bound = math.sqrt(6.0 / rd[i])
        p["rig_w"].append(torch.from_numpy(rs.uniform(-bound, bound, size=(32, rd[i])).astype(np.float32)))
        p["rig_b"].append(torch.zeros(32))
    p["rig_w"].append(torch.from_numpy((rs.randn(1, 32) * rigid_std).astype(np.float32)))
    p["rig_b"].append(torch.from_numpy((rs.randn(1) * rigid_std).astype(np.float32)))
    return p


def make_rays(seed: int, n: int, latent: int = LATENT) -> Dict[str, Tensor]:
    """Synthetic camera rays shaped like get_rays_np output (run_nerf_helpers.py:608-622) for the
    example sequence: common origin, un-normalised directions looking down -z, near/far from the
    example bounds (train.py:1419-1420), per-ray latents ~ N(0, 0.1^2)."""
    rs = np.random.RandomState(seed)
    H, W, focal = 384, 512, 256.61
    px = rs.randint(0, W, size=n).astype(np.float32)
    py = rs.randint(0, H, size=n).astype(np.float32)
    dirs = np.stack([(px - W * 0.5) / focal, -(py - H * 0.5) / focal, -np.ones_like(px)], -1)
    ang = 0.2
    rot = np.array([[math.cos(ang), 0, math.sin(ang)], [0, 1, 0], [-math.sin(ang), 0, math.cos(ang)]], dtype=np.float32)
    rays_d = (dirs @ rot.T).astype(np.float32)
    rays_o = np.broadcast_to(np.array([0.05, -0.02, 0.4], dtype=np.float32), rays_d.shape).copy()
    return {
        "rays_o": torch.from_numpy(rays_o),
        "rays_d": torch.from_numpy(rays_d),
        "near": 0.0022,
        "far": 1.0024,
        "latents": torch.from_numpy((rs.randn(n, latent) * 0.1).astype(np.float32)),
        "target": torch.from_numpy(rs.uniform(0, 1, size=(n, 3)).astype(np.float32)),
    }


def make_randomness(seed: int, n: int, s_c: int, n_imp: int) -> Dict[str, Tensor]:
    """The four random tensors render_rays draws, in the reference's order (train.py:861, 753,
    run_nerf_helpers.py:666, train.py:753 again)."""
    g = torch.Generator().manual_seed(seed)
    return {
        "t_rand": torch.rand(n, s_c, generator=g),
        "noise_c": torch.randn(n, s_c, generator=g),
        "u": torch.rand(n, n_imp, generator=g),
        "noise_f": torch.randn(n, s_c + n_imp, generator=g),
    }


# --------------------------------------------------------------------------------------------
# point-wise field evaluation
# --------------------------------------------------------------------------------------------
def positional_encoding(x: Tensor, n_freqs: int = PE_L) -> Tensor:
    """Embedder.embed with get_embedder's settings (run_nerf_helpers.py:120-168):
    [x, sin(2^0 x), cos(2^0 x), ..., sin(2^(L-1) x), cos(2^(L-1) x)]; frequencies are exact powers
    of two, no pi factor, raw input included first."""
    feats = [x]
    for k in range(n_freqs):
        f = float(2.0 ** k)
        feats.append(torch.sin(x * f))
        feats.append(torch.cos(x * f))
    return torch.cat(feats, -1)


def bender_forward(bp: Dict[str, list], xyz: Tensor, latents: Tensor,
                   rigidity_cutoff: Optional[float] = None, scaling: Optional[float] = None) -> Dict[str, Tensor]:
    """ray_bending.forward, mode simple_neural with rigidity network (run_nerf_helpers.py:507-584).
    xyz [P,3], latents [P,Z] -> unmasked_offsets [P,3], rigidity_mask [P,1], masked_offsets [P,3],
    bent [P,3]."""
    h = torch.cat([xyz, latents], -1)
    for i in range(5):
        h = F.linear(h, bp["net_w"][i], bp["net_b"][i] if i < 4 else None)
        if i != 4:
            h = F.relu(h)
    unmasked = h
    r = xyz
    for i in range(3):
        r = F.linear(r, bp["rig_w"][i], bp["rig_b"][i])
        if i != 2:
            r = F.relu(r)
    rigidity = (torch.tanh(r) + 1.0) / 2.0
    if rigidity_cutoff is not None:
        rigidity = torch.where(rigidity <= rigidity_cutoff, torch.zeros_like(rigidity), rigidity)
    masked = rigidity * unmasked
    if scaling is not None:
        masked = masked * scaling
    return {"unmasked_offsets": unmasked, "rigidity_mask": rigidity, "masked_offsets": masked, "bent": xyz + masked}


def nerf_mlp(npar: Dict[str, list], emb: Tensor) -> Tensor:
    """NeRF.forward without view directions (run_nerf_helpers.py:272-306): 8 x (Linear, ReLU) of
    width 256, with cat[embedding, h] after layer 4, then output_linear."""
    h = emb
    for i in range(NERF_D):
        h = F.relu(F.linear(h, npar["pts_w"][i], npar["pts_b"][i]))
        if i == NERF_SKIP:
            h = torch.cat([emb, h], -1)
    return F.linear(h, npar["out_w"], npar["out_b"])


def direction_encoding(d: Tensor) -> Tensor:
    """embeddirs_fn = get_embedder(multires_views = 4) (train.py:582-586): [d, sin(2^k d), cos(2^k d)], k = 0..3 -> 27."""
    return positional_encoding(d, 4)


def viewdirs_via_finite_differences(bent: Tensor) -> Tensor:
    """NeRF.viewdirs_via_finite_differences (run_nerf_helpers.py:316-356), difference_type = "backward": the direction of
    sample i is the normalised step from sample i-1 to sample i of the BENT ray (sample 0 copies sample 1's), eps = 1e-6
    added to the norm.  bent [N,S,3] -> [N*S, 27] (already encoded)."""
    eps = 0.000001
    diff = bent[:, 1:, :] - bent[:, :-1, :]
    back = diff / (torch.norm(diff, dim=-1, keepdim=True) + eps)
    dirs = torch.cat([back[:, 0, :].reshape(-1, 1, 3), back], dim=1)
    return direction_encoding(dirs.reshape(-1, 3))


def nerf_mlp_views(npar: Dict[str, list], vpar: Dict[str, Tensor], emb: Tensor, dirs_emb: Tensor) -> Tensor:
    """NeRF.forward with use_viewdirs=True (run_nerf_helpers.py:272-304): trunk as nerf_mlp without its output layer, then
    alpha = alpha_linear(h), feature = feature_linear(h), h = relu(views_linears[0](cat[feature, dirs])), rgb = rgb_linear(h);
    output = cat[rgb, alpha] (4 channels)."""
    h = emb
    for i in range(NERF_D):
        h = F.relu(F.linear(h, npar["pts_w"][i], npar["pts_b"][i]))
        if i == NERF_SKIP:
            h = torch.cat([emb, h], -1)
    alpha = F.linear(h, vpar["alpha_w"], vpar["alpha_b"])
    feature = F.linear(h, vpar["feature_w"], vpar["feature_b"])
    hv = F.relu(F.linear(torch.cat([feature, dirs_emb], -1), vpar["views_w"], vpar["views_b"]))
    rgb = F.linear(hv, vpar["rgb_w"], vpar["rgb_b"])
    return torch.cat([rgb, alpha], -1)


def query_field(npar, bp, pts: Tensor, latents: Tensor, rigidity_cutoff=None, scaling=None,
                removal_threshold=None, vpar=None, viewdirs: Optional[Tensor] = None) -> Tuple[Tensor, Dict[str, Tensor]]:
    """run_network + NeRF.forward for one pass (train.py:57-105, run_nerf_helpers.py:240-314).
    pts [N,S,3], latents [N,Z] -> raw [N,S,C], details (each [N,S,k]).
    vpar (make_view_params) switches to the view-dependent head; with a bender the view directions are the finite differences
    of the bent points (approx_nonrigid_viewdirs=True), without one the normalised ray directions `viewdirs` [N,3]."""
    n, s, _ = pts.shape
    flat = pts.reshape(-1, 3)
    details = {"initial_input_pts": flat.detach().clone()}
    if bp is not None:
        lat = latents[:, None, :].expand(n, s, latents.shape[-1]).reshape(n * s, -1)
        b = bender_forward(bp, flat, lat, rigidity_cutoff, scaling)
        bent = b.pop("bent")
        details.update(b)
    else:
        bent = flat
    details["input_pts"] = bent.detach().clone()
    if vpar is not None:
        if bp is not None:
            dirs_emb = viewdirs_via_finite_differences(bent.reshape(n, s, 3))
        else:
            dirs_emb = direction_encoding(viewdirs[:, None, :].expand(n, s, 3).reshape(-1, 3))
        raw = nerf_mlp_views(npar, vpar, positional_encoding(bent), dirs_emb)
    else:
        raw = nerf_mlp(npar, positional_encoding(bent))
    if removal_threshold is not None and bp is not None:
        kill = details["rigidity_mask"].flatten() >= removal_threshold
        raw = raw.clone()
        raw[kill, 3] = raw[kill, 3] * 0.0
    raw = raw.reshape(n, s, -1)
    details = {k: v.reshape(n, s, -1) for k, v in details.items()}
    return raw, details


# --------------------------------------------------------------------------------------------
# per-ray operations
# --------------------------------------------------------------------------------------------
def stratified_z(near: Tensor, far: Tensor, s: int, t_rand: Optional[Tensor], lindisp: bool = False) -> Tensor:
    """render_rays sampling part (train.py:847-869). near/far [N,1]."""
    t = torch.linspace(0.0, 1.0, steps=s, device=near.device)
    if not lindisp:
        z = near * (1.0 - t) + far * t
    else:
        z = 1.0 / (1.0 / near * (1.0 - t) + 1.0 / far * t)
    z = z.expand(near.shape[0], s)
    if t_rand is not None:
        mids = 0.5 * (z[:, 1:] + z[:, :-1])
        upper = torch.cat([mids, z[:, -1:]], -1)
        lower = torch.cat([z[:, :1], mids], -1)
        z = lower + (upper - lower) * t_rand
    return z


def raw2outputs(raw: Tensor, z: Tensor, rays_d: Tensor, noise: Optional[Tensor] = None,
                white_bkgd: bool = False):
    """train.py:724-789.  `noise` is the already-scaled additive sigma noise (randn * raw_noise_std).
    Returns rgb_map, disp_map, acc_map, alpha, weights, depth_map."""
    dists = z[:, 1:] - z[:, :-1]
    dists = torch.cat([dists, torch.full_like(dists[:, :1], 1e10)], -1)
    dists = dists * torch.norm(rays_d[:, None, :], dim=-1)
    rgb = torch.sigmoid(raw[..., :3])
    sigma = raw[..., 3] if noise is None else raw[..., 3] + noise
    alpha = 1.0 - torch.exp(-F.relu(sigma) * dists)
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    weights = alpha * trans
    rgb_map = torch.sum(weights[..., None] * rgb, -2)
    depth = torch.sum(weights * z, -1)
    acc = torch.sum(weights, -1)
    disp = 1.0 / torch.max(1e-10 * torch.ones_like(depth), depth / acc)
    if white_bkgd:
        rgb_map = rgb_map + (1.0 - acc[..., None])
    return rgb_map, disp, acc, alpha, weights, depth


def sample_pdf(bins: Tensor, weights: Tensor, u: Tensor) -> Tensor:
    """run_nerf_helpers.py:651-698 with `u` supplied ([N,n] random, or the deterministic linspace).
    bins [N,B], weights [N,B-1]."""
    w = weights + 1e-5
    pdf = w / torch.sum(w, -1, keepdim=True)
    cdf = torch.cat([torch.zeros_like(pdf[:, :1]), torch.cumsum(pdf, -1)], -1)
    u = u.contiguous()
    inds = torch.searchsorted(cdf.detach(), u, right=False)
    below = torch.clamp(inds - 1, min=0)
    above = torch.clamp(inds, max=cdf.shape[-1] - 1)
    cdf_b, cdf_a = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    bin_b, bin_a = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = cdf_a - cdf_b
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - cdf_b) / denom
    return bin_b + t * (bin_a - bin_b)


def det_u(n: int, n_imp: int, device=None) -> Tensor:
    return torch.linspace(0.0, 1.0, steps=n_imp, device=device).expand(n, n_imp).contiguous()


def render_rays(coarse, fine, bp, rays_o: Tensor, rays_d: Tensor, near, far, latents: Tensor,
                s_c: int = 64, n_imp: int = 64, perturb: bool = False, raw_noise_std: float = 0.0,
                rnd: Optional[Dict[str, Tensor]] = None, lindisp: bool = False, white_bkgd: bool = False,
                rigidity_cutoff=None, scaling=None, removal_threshold=None, detailed: bool = True,
                vpar_c=None, vpar_f=None) -> Dict[str, Tensor]:
    """render_rays (train.py:792-980) with the coarse / importance-sample / fine assembly; keys as
    in the reference's result dict.  vpar_c / vpar_f (make_view_params): view-dependent heads (use_viewdirs=True,
    train.py:364-381: viewdirs = rays_d / |rays_d|)."""
    viewdirs = rays_d / torch.norm(rays_d, dim=-1, keepdim=True) if vpar_c is not None else None
    n = rays_o.shape[0]
    # (device-agnostic: the training A/B of scripts/train_ab.py runs this restatement in fp32 on the GPU as the checker)
    near_t = torch.as_tensor(near, dtype=torch.float32, device=rays_o.device).expand(n).reshape(n, 1)
    far_t = torch.as_tensor(far, dtype=torch.float32, device=rays_o.device).expand(n).reshape(n, 1)
    z = stratified_z(near_t, far_t, s_c, rnd["t_rand"] if perturb else None, lindisp)
    pts = rays_o[:, None, :] + rays_d[:, None, :] * z[:, :, None]
    raw, det_c = query_field(coarse, bp, pts, latents, rigidity_cutoff, scaling, removal_threshold, vpar_c, viewdirs)
    noise_c = rnd["noise_c"] * raw_noise_std if raw_noise_std > 0 else None
    rgb, disp, acc, alpha, w, depth = raw2outputs(raw, z, rays_d, noise_c, white_bkgd)
    ret = {}
    if n_imp > 0:
        rgb0, disp0, acc0, alpha0, w0 = rgb, disp, acc, alpha, w
        z_mid = 0.5 * (z[:, 1:] + z[:, :-1])
        u = rnd["u"] if perturb else det_u(n, n_imp, rays_o.device)
        z_samples = sample_pdf(z_mid, w[:, 1:-1], u).detach()
        z_f, _ = torch.sort(torch.cat([z, z_samples], -1), -1)
        pts_f = rays_o[:, None, :] + rays_d[:, None, :] * z_f[:, :, None]
        raw, det_f = query_field(fine if fine is not None else coarse, bp, pts_f, latents, rigidity_cutoff, scaling,
                                 removal_threshold, vpar_f if fine is not None else vpar_c, viewdirs)
        noise_f = rnd["noise_f"] * raw_noise_std if raw_noise_std > 0 else None
        rgb, disp, acc, alpha, w, depth = raw2outputs(raw, z_f, rays_d, noise_f, white_bkgd)
        ret.update({"rgb0": rgb0, "disp0": disp0, "acc0": acc0,
                    "z_std": torch.std(z_samples, dim=-1, unbiased=False), "z_vals_fine": z_f})
        if detailed:
            ret["fine_visibility_weights"] = w
            ret["fine_opacity_alpha"] = alpha
            for k, v in det_f.items():
                ret["fine_" + k] = v
    else:
        alpha0, w0 = alpha, w
    ret.update({"rgb_map": rgb, "disp_map": disp, "acc_map": acc, "raw": raw, "z_vals_coarse": z})
    if detailed:
        ret["visibility_weights"] = w0
        ret["opacity_alpha"] = alpha0
        ret.update(det_c)
    return ret


# --------------------------------------------------------------------------------------------
# training loss (per-ray), train.py:152-287 minus the divergence term's randomness (passed in)
# --------------------------------------------------------------------------------------------
def training_loss(ret: Dict[str, Tensor], target: Tensor, offsets_w: float = 0.0, rigidity_w: float = 0.0,
                  sched: float = 1.0) -> Tensor:
    n = target.shape[0]
    loss = torch.mean(((ret["rgb_map"] - target) ** 2).view(n, -1), dim=1)
    if "rgb0" in ret:
        loss = loss + torch.mean(((ret["rgb0"] - target) ** 2).view(n, -1), dim=1)
    if offsets_w > 0.0:
        wts = ret["visibility_weights"].detach().reshape(-1)
        off = ret["unmasked_offsets"].reshape(-1, 3)
        rig = ret["rigidity_mask"].reshape(-1)
        ol = torch.mean((wts * torch.pow(torch.norm(off, dim=-1), 2.0 - rig)).view(n, -1), dim=-1)
        ol = ol + rigidity_w * torch.mean((wts * rig).view(n, -1), dim=-1)
        loss = loss + offsets_w * sched * ol
    return loss


def divergence_loss(bp, ret: Dict[str, Tensor], latents: Tensor, n_rays: int, s_c: int, e: Optional[Tensor] = None) -> Tensor:
    """Divergence regulariser of the offset field on the coarse samples (train.py:245-286 driving
    compute_divergence_loss / divergence_approx, run_nerf_helpers.py:22-116): Hutchinson estimate
    e^T J e with J = d(masked offsets)/d(xyz), squared, weighted by 1 - exp(-relu(alpha)) (detached),
    mean over the ray's samples.  `e` ~ N(0, 1) [P, 3] may be injected."""
    pts = ret["initial_input_pts"].reshape(-1, 3).detach().requires_grad_(True)
    lat = latents[:, None, :].expand(n_rays, s_c, latents.shape[-1]).reshape(-1, latents.shape[-1])
    w = (1.0 - torch.exp(-F.relu(ret["opacity_alpha"].reshape(-1)))).detach()
    off = bender_forward(bp, pts, lat)["masked_offsets"]
    if e is None:
        e = torch.randn_like(off)
    e_dydx = torch.autograd.grad(off, pts, e, create_graph=True)[0]
    div = (e_dydx * e).view(off.shape[0], -1).sum(dim=1)
    return torch.mean((w * torch.abs(div) ** 2).view(n_rays, -1), dim=-1)


def training_wrapper_loss(cp, fp, bp, rays: Dict[str, Tensor], latent_table: Tensor, imageid_to_timestepid, pixel_indices: Tensor,
                          rnd: Dict[str, Tensor], e: Tensor, global_step: int, n_iters: int, offsets_w: float,
                          divergence_w: float, rigidity_w: float, s_c: int = 64, n_imp: int = 64, vpar_c=None, vpar_f=None):
    """Per-ray loss [N] of training_wrapper_class.forward (train.py:152-287): latent lookup by the ray's image id
    (:173-189), training-mode render, data terms, offsets / rigidity regulariser and divergence regulariser, both
    scaled by the increasing schedule (1/100)^(1 - global_step / N_iters) (:229, :281).  vpar_c / vpar_f
    (make_view_params): the view-dependent heads (use_viewdirs=True), as in render_rays.  Returns (loss, ret)."""
    n = rays["rays_o"].shape[0]
    i2t = torch.as_tensor(imageid_to_timestepid, device=pixel_indices.device)
    lat = latent_table[i2t[pixel_indices[:, 0]], :]
    ret = render_rays(cp, fp, bp, rays["rays_o"], rays["rays_d"], rays["near"], rays["far"], lat, s_c, n_imp, perturb=True,
                      raw_noise_std=1.0, rnd=rnd, vpar_c=vpar_c, vpar_f=vpar_f)
    sched = (1.0 / 100.0) ** (1 - (global_step / n_iters))
    loss = training_loss(ret, rays["target"], offsets_w, rigidity_w, sched)
    if divergence_w > 0.0:
        loss = loss + divergence_w * sched * divergence_loss(bp, ret, lat, n, s_c, e)
    return loss, ret


def get_rays(c2w: Tensor, intrin) -> Tuple[Tensor, Tensor]:
    """get_rays / get_rays_np (run_nerf_helpers.py:588-622): rays_o, rays_d [H, W, 3] float32."""
    h, w = int(intrin["height"]), int(intrin["width"])
    i, j = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32), indexing="xy")
    dirs = np.stack([(i - np.float32(intrin["center_x"])) / np.float32(intrin["focal_x"]),
                     -(j - np.float32(intrin["center_y"])) / np.float32(intrin["focal_y"]), -np.ones_like(i)], -1)
    c = c2w.numpy().astype(np.float32)
    rays_d = np.sum(dirs[..., np.newaxis, :] * c[:3, :3], -1)
    rays_o = np.broadcast_to(c[:3, -1], np.shape(rays_d))
    return torch.from_numpy(np.ascontiguousarray(rays_o)), torch.from_numpy(rays_d.astype(np.float32))


def surface_selection(weights: Tensor, input_pts: Tensor, rigidity: Optional[Tensor]):
    """free_viewpoint_rendering.py:623-651: per ray the sample whose accumulated visibility is closest to 0.5, and the
    canonical point / rigidity at that sample.  weights [N,S], input_pts [N,S,3], rigidity [N,S(,1)]."""
    acc = torch.cumsum(weights, dim=-1)
    idx = torch.min(torch.abs(acc - 0.5), dim=-1)[1]
    rows = torch.arange(weights.shape[0])
    pts = input_pts[rows, idx, :]
    rig = rigidity.reshape(weights.shape[0], -1)[rows, idx] if rigidity is not None else None
    return idx, pts, rig


def clone_params(p, requires_grad=False):
    out = {}
    for k, v in p.items():
        if isinstance(v, list):
            out[k] = [t.clone().requires_grad_(requires_grad) for t in v]
        else:
            out[k] = v.clone().requires_grad_(requires_grad)
    return out


def flat_param_list(p):
    out = []
    for k in sorted(p.keys()):
        v = p[k]
        out.extend(v if isinstance(v, list) else [v])
    return out


FLOP_PER_POINT = 1_016_320  # SURVEY.md section 8(d): NeRF 984,576 + bender 31,744 (2 FLOP / MAC)
