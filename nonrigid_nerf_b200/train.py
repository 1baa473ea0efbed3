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
from . import geometry, ops
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
    views = getattr(fn, "use_viewdirs", False)
    if (viewdirs is not None) != views:
        raise RuntimeError("nonrigid_nerf_b200: " + ("a use_viewdirs=True model needs viewdirs" if views else
                                                     "viewdirs given to a model without the view-dependent head (use_viewdirs=False)"))
    n, s = inputs.shape[0], inputs.shape[1]
    latents = additional_pixel_information["ray_bending_latents"]
    pts = inputs.reshape(-1, 3)
    lat = latents[:, None].expand(n, s, latents.shape[-1]).reshape(n * s, latents.shape[-1])
    if views:   # the ray's direction for each of its samples (train.py:79-84); with a bender the kernels use the bent points'
        vd = viewdirs[:, None].expand(n, s, 3).reshape(n * s, 3)
        raw, details = _ag.field_views(fn, None, None, pts, lat, vd, detailed_output)
    else:
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
                additional_pixel_information=None, detailed_output=False, verbose=False, pytest=False, held_out=None, occupancy=None,
                early_termination=None, baked=None, **dummy_kwargs):
    """Volumetric rendering of a ray batch [N, 8] = (o, d, near, far).  `network_query_fn` is accepted
    for signature compatibility; the field is evaluated by the fused kernel on `network_fn` /
    `network_fine` (which carry their ray bender as `.ray_bender[0]`).
    Extra keyword `randomness` (dict with t_rand, noise_c, u, noise_f; unit-variance noise) replaces
    the internal draws -- the supported way to reproduce a run exactly (the reference's `pytest` hook
    re-seeds numpy instead, train.py:863-867).
    held_out [N] (bool or uint8, on the rays' device): rays of held-out frames.  With a ray bender their gradient reaches
    only their latent codes, not the coarse, fine or bender weights; without one they contribute no gradient at all.  So
    one backward of ((train + held_out) * loss).mean() gives the gradients of the reference's two backward passes
    (train.py:1595-1608).  None: the ordinary path.
    occupancy (geometry.OccupancyGrid, under torch.no_grad() only): each pass evaluates the NeRF trunk only on samples
    whose bent point lies in an occupied cell, outside the grid's box, or is not finite; the others get raw = 0.  None:
    every sample is evaluated.
    early_termination (a float t in [0, 1], under torch.no_grad() only; the reference has no such option): each pass
    evaluates its samples in segments of nrn_termination_segment() consecutive samples, in depth order, and stops
    evaluating a ray after the segment in which its transmittance T = prod (1 - alpha_i + 1e-10) (compositing's own
    alphas and noise, fp32, sample by sample) falls below t.  Samples not evaluated get raw = 0; with occupancy as well, a
    sample is evaluated only when both allow it.  extras["termination_index"] (int32 [N]) is the first sample the last
    pass skipped because of termination (S when the ray never died), and extras["termination_index0"] the coarse pass's
    when N_importance > 0.  Per ray |rgb - rgb_full| <= T and |acc - acc_full| <= T (2 T for rgb with white_bkgd) against
    the render without termination at the same depths, up to rounding, where T is the transmittance at which the ray
    died; the coarse weights of skipped samples are 0, so the fine depths follow a pdf within t of mass of the full one.
    t = 0 terminates nothing, nor does a NaN T.  None: every sample is evaluated (no termination_index keys).
    baked (geometry.BakedScene, under torch.no_grad() only; the reference has no such option): the coarse pass samples
    baked.coarse and the fine pass baked.fine (required when N_importance > 0) in place of the NeRF trunk for every sample
    whose bent point is finite and inside the grid's box: raw is the grid's trilinear lookup there (raw[..., 4] = 0, the
    object removal applied) and the trunk's raw elsewhere, so a box that holds no sample renders as without it.  With
    baked.deformation (geometry.FrameDeformation, a model with a ray bender) both passes take the bends of every ray whose
    samples all lie inside that grid's box from it (trilinear offset and rigidity, then the test-time knobs) instead of
    the bender; any other ray is bent by the bender exactly as without it.  Pass that frame's latent code as the rays'
    latents.  Not combined with occupancy or early_termination.  None: the trunk evaluates every sample.
    surface_normals=True (with surface_output=True) adds ret["surface_normals"] [N, 3]: the world-space unit normal
    geometry.normals_from_gradient(geometry.density_gradient(...)) of the pass's model, with the ray's latent code, at
    the frame-space point of the median-visibility sample (the point surface_pts and surface_rigidity are taken at).
    No other output changes.  Default False."""
    if pytest:
        raise RuntimeError("nonrigid_nerf_b200: the pytest= numpy-random hook is not supported")
    if not isinstance(network_fn, NeRF) or (network_fine is not None and not isinstance(network_fine, NeRF)):
        raise RuntimeError("nonrigid_nerf_b200: render_rays needs nonrigid_nerf_b200.run_nerf_helpers.NeRF modules")
    _check_views(ray_batch.shape[-1] > 8, network_fn, network_fine if N_importance > 0 else None, additional_pixel_information)
    n = ray_batch.shape[0]
    dev = ray_batch.device
    _ag.check_held_out(held_out, n, dev)
    rays = ray_batch if (ray_batch.dtype == torch.float32 and ray_batch.is_contiguous()) else ray_batch.float().contiguous()
    viewdirs = None
    if rays.shape[-1] > 8:   # (o, d, near, far, viewdirs): train.py:843
        viewdirs = rays[:, -3:]
        rays = rays[:, :8].contiguous()
    rays_d = rays[:, 3:6]
    latents = None
    if network_fn.ray_bender[0] is not None or getattr(network_fn, "time_conditioned_baseline", False):
        latents = additional_pixel_information["ray_bending_latents"]
    early_termination = _check_fast_paths(occupancy, early_termination, baked, network_fn, network_fine, N_importance, latents)
    term_index = {}

    def field(net, z, noise, key):
        if baked is not None:
            return _ag.field_baked(net, rays, z, latents, detailed_output, baked.coarse if key == "coarse" else baked.fine, baked.deformation)
        if early_termination is not None:
            raw, det, term_index[key] = _ag.field_terminate(net, rays, z, latents, detailed_output, early_termination, occupancy, noise)
            return raw, det
        if occupancy is None:
            return _ag.field(net, rays, z, latents, detailed_output, viewdirs, held_out)
        return _ag.field_occupancy(net, rays, z, latents, detailed_output, occupancy)

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
    # the noise is drawn before the field call: an early-terminating pass feeds it into its transmittance
    noise = draw("noise_c", torch.randn, n, N_samples) if raw_noise_std > 0.0 else None   # already scaled by raw_noise_std
    raw, details = field(network_fn, z_vals, noise, "coarse")

    if N_importance > 0:
        u = draw("u", torch.rand, n, N_importance) if perturb > 0.0 else None   # det=(perturb == 0), train.py:915
        c0 = _ag.composite(raw, z_vals, rays_d, noise, white_bkgd, N_importance, u)
        z_fine = c0["z_vals_out"]   # sorted union, detached (train.py:918-920)
        run_fn = network_fn if network_fine is None else network_fine
        noise_f = draw("noise_f", torch.randn, n, n_fine) if raw_noise_std > 0.0 else None
        raw, fine_details = field(run_fn, z_fine, noise_f, "fine")
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
            if not getattr(run_fn, "use_viewdirs", False):
                _, det = _ag.field_points(run_fn, pts, latents, True)
            elif run_fn.ray_bender[0] is not None:   # the surface point and rigidity do not depend on the head: bend pass alone
                _, det = _ag.field_views(run_fn, None, None, pts, latents, None, True, bend_only=True)
            else:                                     # no bender: the point itself
                det = {"input_pts": pts}
            if dummy_kwargs.get("surface_normals", False):
                # world-space unit normals of the frame's density at the median sample's frame-space point
                ret["surface_normals"] = geometry.normals_from_gradient(geometry.density_gradient(run_fn, pts, latents))
        ret["median_indices"] = idx
        ret["surface_pts"] = det["input_pts"].reshape(n, 3)
        if "rigidity_mask" in det:
            ret["surface_rigidity"] = det["rigidity_mask"].reshape(n)
    if retraw:
        ret["raw"] = raw
    if early_termination is not None:
        ret["termination_index"] = term_index["fine" if N_importance > 0 else "coarse"]
        if N_importance > 0:
            ret["termination_index0"] = term_index["coarse"]
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


def _check_views(batch_has_viewdirs, network_fn, network_fine, additional_pixel_information):
    """Before any launch: the ray batch carries view directions exactly when the models have the view-dependent head,
    and that head is only evaluated without autograd (_ag.views_check)."""
    for net in (network_fn, network_fine):
        if net is None:
            continue
        if getattr(net, "use_viewdirs", False) != batch_has_viewdirs:
            raise RuntimeError("nonrigid_nerf_b200: " + ("a use_viewdirs=True model needs ray batches with view directions "
                                                         "(render(use_viewdirs=True), 11 columns)" if not batch_has_viewdirs else
                                                         "ray batch with view directions (use_viewdirs=True) for a model "
                                                         "without the view-dependent head"))
        info = additional_pixel_information or {}
        _ag.views_check(net, info.get("ray_bending_latents"))


def _check_fast_paths(occupancy, early_termination, baked, network_fn, network_fine, n_importance, latents):
    """Before any launch: render(..., occupancy=, early_termination=, baked=) is refused for what they do not support
    (_check_baked, _ag.occupancy_check, _ag.termination_check); returns the early-termination threshold as a float, or
    None."""
    if baked is not None:
        _check_baked(baked, network_fn, network_fine, n_importance, latents, occupancy, early_termination)
    nets = [net for net in (network_fn, network_fine if n_importance > 0 else None) if net is not None]
    if occupancy is not None:
        for net in nets:
            _ag.occupancy_check(net, latents, occupancy)
    if early_termination is None:
        return None
    t = _ag.termination_threshold(early_termination)
    for net in nets:
        _ag.termination_check(net, latents, t)
    return t


def _check_baked(baked, network_fn, network_fine, n_importance, latents, occupancy, early_termination):
    """Before any launch: render(..., baked=scene) is refused for what it does not support (_ag.baked_check), with occupancy
    or early_termination, without a fine grid when N_importance > 0, and for a deformation that a pass's model cannot read
    (_ag.deformation_check)."""
    from .geometry import BakedScene
    if not isinstance(baked, BakedScene):
        raise RuntimeError(f"nonrigid_nerf_b200: baked must be a geometry.BakedScene, got {type(baked).__name__}")
    if occupancy is not None or early_termination is not None:
        raise RuntimeError("nonrigid_nerf_b200: rendering from a baked radiance grid is not combined with occupancy or "
                           "early_termination")
    _ag.baked_check(network_fn, latents, baked.coarse)
    if n_importance > 0:
        if baked.fine is None:
            raise RuntimeError("nonrigid_nerf_b200: N_importance > 0 needs a fine grid (BakedScene(coarse, fine))")
        _ag.baked_check(network_fn if network_fine is None else network_fine, latents, baked.fine)
    if baked.deformation is not None:
        _ag.deformation_check(network_fn, baked.deformation)
        if n_importance > 0:
            _ag.deformation_check(network_fn if network_fine is None else network_fine, baked.deformation)


# ---- batchify_rays / render (train.py:108-137, :326-416) --------------------------------------------
def batchify_rays(rays_flat, additional_pixel_information, chunk=1024 * 32, detailed_output=False, **kwargs):
    """Render rays in chunks (`chunk` only bounds the per-launch working set; results do not depend on it)."""
    all_ret = {}
    held_out = kwargs.pop("held_out", None)
    for i in range(0, rays_flat.shape[0], chunk):
        info = {"ray_bending_latents": additional_pixel_information["ray_bending_latents"][i:i + chunk, :]}
        held = None if held_out is None else held_out[i:i + chunk]
        ret = render_rays(rays_flat[i:i + chunk], additional_pixel_information=info, detailed_output=detailed_output,
                          held_out=held, **kwargs)
        for k in ret:
            all_ret.setdefault(k, []).append(ret[k])
    return {k: (v[0] if len(v) == 1 else torch.cat(v, 0)) for k, v in all_ret.items()}


def render(rays_o, rays_d, chunk=1024 * 32, ndc=True, near=0.0, far=1.0, use_viewdirs=False, c2w_staticcam=None,
           additional_pixel_information=None, detailed_output=False, **kwargs):
    """Render rays.  Returns [rgb_map, disp_map, acc_map, extras] (train.py:326-416).  Keyword held_out [N] (one entry
    per ray of the flattened batch), keyword occupancy (a geometry.OccupancyGrid), keyword early_termination (a float
    in [0, 1]) and keyword baked (a geometry.BakedScene): see render_rays."""
    if kwargs.get("network_fn") is not None:
        _check_fast_paths(kwargs.get("occupancy"), kwargs.get("early_termination"), kwargs.get("baked"), kwargs["network_fn"],
                          kwargs.get("network_fine"), kwargs.get("N_importance", 0), (additional_pixel_information or {}).get("ray_bending_latents"))
        _check_views(bool(use_viewdirs), kwargs["network_fn"], kwargs.get("network_fine") if kwargs.get("N_importance", 0) > 0 else None,
                     additional_pixel_information)
    elif kwargs.get("early_termination") is not None:
        _ag.termination_threshold(kwargs["early_termination"])
    viewdirs = None
    if use_viewdirs:   # provide ray directions as input (train.py:364-381)
        if c2w_staticcam is not None:
            raise RuntimeError("need to pull this call to get_rays out to render_path() for gpu parallelization to work")
        viewdirs = rays_d / torch.norm(rays_d, dim=-1, keepdim=True)
        viewdirs = torch.reshape(viewdirs, [-1, 3]).float()
    sh = rays_d.shape
    if ndc:
        raise RuntimeError("not implemented. change H, W, focal to use ray_params instead")  # train.py:384-386
    if not rays_o.is_cuda:
        raise RuntimeError("nonrigid_nerf_b200: rays must be CUDA tensors (there is no CPU path)")
    rays_o = torch.reshape(rays_o, [-1, 3]).float()
    rays_d = torch.reshape(rays_d, [-1, 3]).float()
    _ag.check_held_out(kwargs.get("held_out"), rays_d.shape[0], rays_d.device)
    if isinstance(near, torch.Tensor) or isinstance(far, torch.Tensor) or np.ndim(near) > 0 or np.ndim(far) > 0:
        near_t = torch.as_tensor(near, dtype=torch.float32, device=rays_d.device) * torch.ones_like(rays_d[..., :1])
        far_t = torch.as_tensor(far, dtype=torch.float32, device=rays_d.device) * torch.ones_like(rays_d[..., :1])
        rays = torch.cat([rays_o, rays_d, near_t, far_t], -1)
    else:
        rays = ops.pack_rays(rays_o, rays_d, float(near), float(far))     # scalar bounds (train.py:1463-1468): one launch
    if viewdirs is not None:
        rays = torch.cat([rays, viewdirs], -1)                               # train.py:398-399
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
