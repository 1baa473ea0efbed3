"""Host-side mirror of the reference's train.py hot-path entry points.

render / batchify_rays / render_rays / run_network / batchify / raw2outputs keep the reference's
names, argument meaning, return structure and error behaviour (train.py:27-137, :326-416,
:724-980), but run on the fused sm_90a kernels.  torch.nn.DataParallel (train.py:290-323) is
replaced by ray sharding over torch.distributed/NCCL (parallel.py).

Randomness (t_rand, sigma noise coarse, u, sigma noise fine; train.py:861, :753, run_nerf_helpers.py:666) comes from the
global torch generator, but pooled: one torch.rand and one torch.randn per render_rays call, sliced into the four arrays --
the same distributions, NOT the same values a seeded reference run would draw with its four calls.  Exact reproduction of
a reference run goes through the `randomness=` keyword (the four tensors given explicitly).
"""
from __future__ import annotations

import numpy as np
import torch

from . import autograd as _ag
from . import ops
from .run_nerf_helpers import NeRF, img2mse, mse2psnr  # noqa: F401  (same star-import surface)

DEBUG = False  # reference: train.py:24 (NaN/Inf scan of every output when True)


# ---- run_network / batchify (train.py:27-105) ----------------------------------------------------
def batchify(fn, chunk, detailed_output=False):
    """Kept for API compatibility: the fused kernel needs no activation chunking, so `chunk` only
    bounds the size of one launch."""
    if chunk is None:
        return fn

    def ret(inputs):
        outs = [fn(inputs[i:i + chunk], detailed_output=detailed_output) for i in range(0, inputs.shape[0], chunk)]
        if detailed_output:
            outputs = torch.cat([o[0] for o in outs], 0)
            details = {k: torch.cat([o[1][k] for o in outs], 0) for k in outs[0][1]}
            return outputs, details
        return torch.cat(outs, 0)

    return ret


def run_network(inputs, viewdirs, additional_pixel_information, fn, embed_fn, embeddirs_fn, netchunk=1024 * 64,
                detailed_output=False):
    """Prepares inputs and applies network `fn` (train.py:57-105).  inputs: [N_rays, N_samples, 3]."""
    if viewdirs is not None:
        raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True is not implemented yet (SURVEY.md 8f row f1)")
    n, s = inputs.shape[0], inputs.shape[1]
    latents = additional_pixel_information["ray_bending_latents"]
    pts = inputs.reshape(-1, 3)
    lat = latents[:, None].expand(n, s, latents.shape[-1]).reshape(n * s, latents.shape[-1])
    raw, details = _ag.field_points(fn, pts, lat, detailed_output)
    outputs = raw.reshape(n, s, -1)
    if detailed_output:
        return outputs, {k: v.reshape(n, s, -1) for k, v in details.items()}
    return outputs


# ---- raw2outputs (train.py:724-789) ---------------------------------------------------------------
def raw2outputs(raw, z_vals, rays_d, raw_noise_std=0, white_bkgd=False, pytest=False):
    """Returns rgb_map, disp_map, acc_map, opacity_alpha, visibility_weights, depth_map."""
    if pytest:
        raise RuntimeError("nonrigid_nerf_b200: the pytest= numpy-random hook is not supported")
    noise = None
    if raw_noise_std > 0.0:
        noise = torch.randn(raw[..., 3].shape, device=raw.device) * raw_noise_std
    o = _ag.composite(raw, z_vals, rays_d, noise, white_bkgd)
    return o["rgb_map"], o["disp_map"], o["acc_map"], o["alpha"], o["weights"], o["depth_map"]


# ---- render_rays (train.py:792-980) ---------------------------------------------------------------
def render_rays(ray_batch, network_fn, network_query_fn, N_samples, retraw=False, lindisp=False, perturb=0.0,
                N_importance=0, network_fine=None, white_bkgd=False, raw_noise_std=0.0,
                additional_pixel_information=None, detailed_output=False, verbose=False, pytest=False, **dummy_kwargs):
    """Volumetric rendering of a ray batch [N, 8] = (o, d, near, far).  `network_query_fn` is accepted
    for signature compatibility; the field is evaluated by the fused kernel on `network_fn` /
    `network_fine` (which carry their ray bender as `.ray_bender[0]`).
    Extra keyword `randomness` (dict with t_rand, noise_c, u, noise_f; unit-variance noise) replaces
    the internal draws -- the supported way to reproduce a run exactly (the reference's `pytest` hook
    re-seeds numpy instead, train.py:863-867)."""
    if pytest:
        raise RuntimeError("nonrigid_nerf_b200: the pytest= numpy-random hook is not supported")
    if ray_batch.shape[-1] > 8:
        raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True is not implemented yet (SURVEY.md 8f row f1)")
    if not isinstance(network_fn, NeRF) or (network_fine is not None and not isinstance(network_fine, NeRF)):
        raise RuntimeError("nonrigid_nerf_b200: render_rays needs nonrigid_nerf_b200.run_nerf_helpers.NeRF modules")
    n = ray_batch.shape[0]
    dev = ray_batch.device
    rays = ray_batch if (ray_batch.dtype == torch.float32 and ray_batch.is_contiguous()) else ray_batch.float().contiguous()
    rays_d = rays[:, 3:6]
    latents = None
    if network_fn.ray_bender[0] is not None:
        latents = additional_pixel_information["ray_bending_latents"]

    rnd = dummy_kwargs.get("randomness", None)

    # The reference draws t_rand, the coarse noise, u and the fine noise with four generator calls
    # (train.py:861, 744, 915).  Here one torch.rand and one torch.randn fill a pool per call of render_rays and the
    # four arrays are contiguous slices of it: same distributions, two launches instead of four (+ two scalings).
    n_fine = N_samples + N_importance
    want = {"t_rand": (torch.rand, n * N_samples if perturb > 0.0 else 0),
            "u": (torch.rand, n * N_importance if (perturb > 0.0 and N_importance > 0) else 0),
            "noise_c": (torch.randn, n * N_samples if raw_noise_std > 0.0 else 0),
            "noise_f": (torch.randn, n * n_fine if (raw_noise_std > 0.0 and N_importance > 0) else 0)}
    pools = {}
    if rnd is None:
        for fn in (torch.rand, torch.randn):
            tot = sum(cnt for f, cnt in want.values() if f is fn)
            if tot:
                buf = fn(tot, device=dev)
                if fn is torch.randn and raw_noise_std != 1.0:
                    buf = buf * raw_noise_std
                o = 0
                for k, (f, cnt) in want.items():
                    if f is fn and cnt:
                        pools[k] = buf[o:o + cnt]
                        o += cnt

    def draw(key, fn, *shape):
        if rnd is not None:
            t = rnd[key].to(dev)
            return t * raw_noise_std if (fn is torch.randn and raw_noise_std != 1.0) else t
        return pools[key].view(*shape)

    # coarse depths (train.py:847-869); t_rand drawn first, like the reference
    t_rand = draw("t_rand", torch.rand, n, N_samples) if perturb > 0.0 else None
    z_vals = ops.sample_coarse(rays, N_samples, t_rand, lindisp)
    raw, details = _ag.field(network_fn, rays, z_vals, latents, detailed_output)
    noise = draw("noise_c", torch.randn, n, N_samples) if raw_noise_std > 0.0 else None   # already scaled by raw_noise_std

    if N_importance > 0:
        u = draw("u", torch.rand, n, N_importance) if perturb > 0.0 else None   # det=(perturb == 0), train.py:915
        c0 = _ag.composite(raw, z_vals, rays_d, noise, white_bkgd, N_importance, u)
        z_fine = c0["z_vals_out"]   # sorted union, detached (train.py:918-920)
        run_fn = network_fn if network_fine is None else network_fine
        raw, fine_details = _ag.field(run_fn, rays, z_fine, latents, detailed_output)
        noise_f = draw("noise_f", torch.randn, n, n_fine) if raw_noise_std > 0.0 else None
        c1 = _ag.composite(raw, z_fine, rays_d, noise_f, white_bkgd)
    else:
        c0 = None
        c1 = _ag.composite(raw, z_vals, rays_d, noise, white_bkgd)
        z_fine, run_fn = z_vals, network_fn

    ret = {"rgb_map": c1["rgb_map"], "disp_map": c1["disp_map"], "acc_map": c1["acc_map"]}
    if dummy_kwargs.get("surface_output", False):
        # Fused free-viewpoint post-processing (free_viewpoint_rendering.py:617-658): instead of shipping every sample's
        # bent point and rigidity to the host (11.5 KB per ray) and indexing there, pick the median-visibility sample on
        # the device and evaluate the bender for that ONE point per ray: 4 floats + an index per ray.
        with torch.no_grad():
            idx = ops.median_visibility_index(c1["weights"])
            z_s = torch.gather(z_fine, 1, idx[:, None])
            pts = rays[:, 0:3] + rays[:, 3:6] * z_s          # multiply, then add: the same rounding as the field kernel
            _, det = _ag.field_points(run_fn, pts, latents, True)
        ret["median_indices"] = idx
        ret["surface_pts"] = det["input_pts"].reshape(n, 3)
        if "rigidity_mask" in det:
            ret["surface_rigidity"] = det["rigidity_mask"].reshape(n)
    if retraw:
        ret["raw"] = raw
    if N_importance > 0:
        ret["rgb0"], ret["disp0"], ret["acc0"] = c0["rgb_map"], c0["disp_map"], c0["acc_map"]
        ret["z_std"] = c0["z_std"]
        if detailed_output:
            ret["fine_visibility_weights"] = c1["weights"]
            ret["fine_opacity_alpha"] = c1["alpha"]
            for key, val in fine_details.items():
                ret["fine_" + str(key)] = val
    if detailed_output:
        first = c0 if c0 is not None else c1   # (the reference raises UnboundLocalError here when N_importance == 0)
        ret["visibility_weights"] = first["weights"]
        ret["opacity_alpha"] = first["alpha"]
        for key, val in details.items():
            ret[key] = val
    if DEBUG:
        for k in ret:
            if torch.isnan(ret[k]).any() or torch.isinf(ret[k]).any():
                print(f"! [Numerical Error] {k} contains nan or inf.", flush=True)
    return ret


# ---- batchify_rays / render (train.py:108-137, :326-416) --------------------------------------------
def batchify_rays(rays_flat, additional_pixel_information, chunk=1024 * 32, detailed_output=False, **kwargs):
    """Render rays in chunks (`chunk` only bounds the per-launch working set; results do not depend on it)."""
    all_ret = {}
    for i in range(0, rays_flat.shape[0], chunk):
        info = {"ray_bending_latents": additional_pixel_information["ray_bending_latents"][i:i + chunk, :]}
        ret = render_rays(rays_flat[i:i + chunk], additional_pixel_information=info, detailed_output=detailed_output, **kwargs)
        for k in ret:
            all_ret.setdefault(k, []).append(ret[k])
    return {k: (v[0] if len(v) == 1 else torch.cat(v, 0)) for k, v in all_ret.items()}


def render(rays_o, rays_d, chunk=1024 * 32, ndc=True, near=0.0, far=1.0, use_viewdirs=False, c2w_staticcam=None,
           additional_pixel_information=None, detailed_output=False, **kwargs):
    """Render rays.  Returns [rgb_map, disp_map, acc_map, extras] (train.py:326-416)."""
    if use_viewdirs:
        raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True is not implemented yet (SURVEY.md 8f row f1)")
    sh = rays_d.shape
    if ndc:
        raise RuntimeError("not implemented. change H, W, focal to use ray_params instead")  # train.py:384-386
    if not rays_o.is_cuda:
        raise RuntimeError("nonrigid_nerf_b200: rays must be CUDA tensors (there is no CPU path)")
    rays_o = torch.reshape(rays_o, [-1, 3]).float()
    rays_d = torch.reshape(rays_d, [-1, 3]).float()
    if isinstance(near, torch.Tensor) or isinstance(far, torch.Tensor) or np.ndim(near) > 0 or np.ndim(far) > 0:
        near_t = torch.as_tensor(near, dtype=torch.float32, device=rays_d.device) * torch.ones_like(rays_d[..., :1])
        far_t = torch.as_tensor(far, dtype=torch.float32, device=rays_d.device) * torch.ones_like(rays_d[..., :1])
        rays = torch.cat([rays_o, rays_d, near_t, far_t], -1)
    else:
        rays = ops.pack_rays(rays_o, rays_d, float(near), float(far))     # scalar bounds (train.py:1463-1468): one launch
    all_ret = batchify_rays(rays, additional_pixel_information, chunk=chunk, detailed_output=detailed_output, **kwargs)
    for k in all_ret:
        all_ret[k] = torch.reshape(all_ret[k], list(sh[:-1]) + list(all_ret[k].shape[1:]))
    k_extract = ["rgb_map", "disp_map", "acc_map"]
    ret_list = [all_ret[k] for k in k_extract]
    ret_dict = {k: all_ret[k] for k in all_ret if k not in k_extract}
    return ret_list + [ret_dict]


# ---- batch sampling of the training loop (train.py:1498-1517, :1546-1564) on the device ------------------------------
class RayBatchSampler:
    """Keeps the images, poses and intrinsics resident on the GPU and produces a training batch -- random (image, x, y)
    pixels, their rays and target colours -- with one kernel, instead of gathering rows of a host-side table of every ray
    of every image (0.8 GB for the example sequence) and copying them to the device each iteration.

        sampler = RayBatchSampler(images, poses, intrinsics, dataset_extras["imageid_to_viewid"], device)
        batch_rays, target_s, batch_pixel_indices = sampler.sample(N_rand)        # [2, N, 3], [N, 3], [N, 3] (image, x, y)

    `generator` (a torch.Generator on the device) makes the draw reproducible and identical across ranks."""

    def __init__(self, images, poses, intrinsics, imageid_to_viewid=None, device="cuda"):
        dev = torch.device(device)
        self.images = torch.as_tensor(images, dtype=torch.float32).to(dev).contiguous()          # [n_img, H, W, 3]
        self.poses = torch.as_tensor(poses, dtype=torch.float32)[:, :3, :4].to(dev).contiguous()
        self.n_images, self.height, self.width = self.images.shape[0], self.images.shape[1], self.images.shape[2]
        if int(intrinsics[0]["height"]) != self.height or int(intrinsics[0]["width"]) != self.width:
            raise RuntimeError("nonrigid_nerf_b200: intrinsics do not match the image size")
        self.intrinsics = torch.tensor([ops.intrinsics_row(k) for k in intrinsics], dtype=torch.float32, device=dev)
        self.image_to_view = None if imageid_to_viewid is None else torch.as_tensor(list(imageid_to_viewid), dtype=torch.int32, device=dev)

    def sample(self, n_rand: int, generator=None):
        dev = self.images.device
        pix = torch.stack([torch.randint(self.n_images, (n_rand,), device=dev, generator=generator),
                           torch.randint(self.width, (n_rand,), device=dev, generator=generator),
                           torch.randint(self.height, (n_rand,), device=dev, generator=generator)], -1)    # (image, x, y)
        return self.rays_for(pix)

    def rays_for(self, pix: torch.Tensor):
        rays_o, rays_d, target = ops.ray_batch(pix, self.poses, self.intrinsics, self.image_to_view, self.images, self.height, self.width)
        return torch.stack([rays_o, rays_d], 0), target, pix
