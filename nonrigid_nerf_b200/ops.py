"""Tensor-level wrappers over the C ABI (forward ops; autograd lives in autograd.py).

All tensors are fp32 CUDA tensors owned by PyTorch; kernels are enqueued on the current stream.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import torch

from . import _lib

LATENT = 32
FORCE_PACK = False   # set while capturing a CUDA graph: the repack kernels must be part of the graph


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(f"nonrigid_nerf_b200: {name} must be a CUDA tensor (there is no CPU path)")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def _ptr_array(tensors):
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


# ---------------------------------------------------------------------------------------------
# weight packing (cached per module, invalidated by the parameters' version counters)
# ---------------------------------------------------------------------------------------------
_PARAM_EPOCH = 0   # bumped by optimizers that update parameters behind autograd's back (optim.Adam)


def note_parameters_changed() -> None:
    """Invalidate every cached fp16 weight image: parameters were updated by a kernel that does not touch
    PyTorch's version counters."""
    global _PARAM_EPOCH
    _PARAM_EPOCH += 1


def _versions(params):
    return (_PARAM_EPOCH,) + tuple((p.data_ptr(), p._version) for p in params)


def nerf_param_list(net):
    ws = [net.pts_linears[i].weight for i in range(8)] + [net.output_linear.weight]
    bs = [net.pts_linears[i].bias for i in range(8)] + [net.output_linear.bias]
    return ws, bs


def bender_param_list(bender):
    net_w = [bender.network[i].weight for i in range(5)]
    net_b = [bender.network[i].bias for i in range(4)]
    rig_w = [bender.rigidity_network[i].weight for i in range(3)]
    rig_b = [bender.rigidity_network[i].bias for i in range(3)]
    return net_w, net_b, rig_w, rig_b


def pack_nerf(net) -> torch.Tensor:
    """fp16 wgmma operand image of a NeRF module's weights (see csrc/nrn_common.cuh)."""
    ws, bs = nerf_param_list(net)
    key = _versions(ws + bs)
    cache = getattr(net, "_nrn_pack", None)
    if cache is not None and cache[0] == key and not FORCE_PACK:
        return cache[1]
    lib = _lib.load()
    for t in ws + bs:
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise RuntimeError("nonrigid_nerf_b200: NeRF parameters must be contiguous fp32 CUDA tensors")
    if ws[0].shape != (256, 63) or ws[5].shape != (256, 319) or ws[8].shape[1] != 256:
        raise RuntimeError("nonrigid_nerf_b200: only D=8, W=256, skips=[4], multires=10, use_viewdirs=False is implemented "
                           f"(got layer shapes {[tuple(w.shape) for w in ws]})")
    buf = cache[1] if cache is not None else torch.empty(lib.nrn_packed_nerf_bytes(), dtype=torch.uint8, device=ws[0].device)
    out_ch = ws[8].shape[0]
    with torch.cuda.device(ws[0].device):
        _lib.check(lib.nrn_pack_nerf(_ptr_array([w.detach() for w in ws]), _ptr_array([b.detach() for b in bs]), 63, out_ch,
                                     _ptr(buf), _stream()), "pack_nerf")
    net._nrn_pack = (key, buf)
    return buf


def pack_bender(bender) -> torch.Tensor:
    net_w, net_b, rig_w, rig_b = bender_param_list(bender)
    allp = net_w + net_b + rig_w + rig_b
    key = _versions(allp)
    cache = getattr(bender, "_nrn_pack", None)
    if cache is not None and cache[0] == key and not FORCE_PACK:
        return cache[1]
    lib = _lib.load()
    for t in allp:
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise RuntimeError("nonrigid_nerf_b200: ray_bending parameters must be contiguous fp32 CUDA tensors")
    if net_w[0].shape != (64, 3 + LATENT):
        raise RuntimeError("nonrigid_nerf_b200: only ray_bending_latent_size=32, simple_neural is implemented")
    buf = cache[1] if cache is not None else torch.empty(lib.nrn_packed_bender_bytes(), dtype=torch.uint8, device=net_w[0].device)
    with torch.cuda.device(net_w[0].device):
        _lib.check(lib.nrn_pack_bender(_ptr_array([t.detach() for t in net_w]), _ptr_array([t.detach() for t in net_b]),
                                       _ptr_array([t.detach() for t in rig_w]), _ptr_array([t.detach() for t in rig_b]),
                                       LATENT, _ptr(buf), _stream()), "pack_bender")
    bender._nrn_pack = (key, buf)
    return buf


# ---------------------------------------------------------------------------------------------
# forward ops
# ---------------------------------------------------------------------------------------------
def sample_coarse(rays: torch.Tensor, n_samples: int, t_rand: Optional[torch.Tensor], lindisp: bool) -> torch.Tensor:
    """z_vals [N, S] (train.py:847-869)."""
    rays = _f32c(rays, "rays")
    n = rays.shape[0]
    z = torch.empty(n, n_samples, dtype=torch.float32, device=rays.device)
    if t_rand is not None:
        t_rand = _f32c(t_rand, "t_rand")
    with torch.cuda.device(rays.device):
        _lib.check(_lib.load().nrn_sample_coarse(_ptr(rays), _ptr(t_rand), n, n_samples, int(bool(lindisp)), _ptr(z), _stream()),
                   "sample_coarse")
    return z


def _field(rays, z_vals, points, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details, stash=None):
    a = _lib.NrnFieldArgs()
    keep = []
    if points is None:
        rays = _f32c(rays, "rays")
        z_vals = _f32c(z_vals, "z_vals")
        n, s = z_vals.shape
        dev = rays.device
        a.rays, a.z_vals = rays.data_ptr(), z_vals.data_ptr()
        keep += [rays, z_vals]
    else:
        if not points.is_cuda:
            raise RuntimeError("nonrigid_nerf_b200: points must be a CUDA tensor (there is no CPU path)")
        if points.dtype != torch.float32 or points.dim() != 2 or points.stride(1) != 1:
            points = points.reshape(points.shape[0], -1).float().contiguous()
        n, s = points.shape[0], 1
        dev = points.device
        a.points, a.points_stride = points.data_ptr(), points.stride(0)
        keep.append(points)
    a.n_rays, a.n_samples = n, s
    a.nerf_packed = nerf_pack.data_ptr()
    if bender_pack is not None:
        if latents is None:
            raise RuntimeError("nonrigid_nerf_b200: ray bending needs latents")
        if latents.dtype != torch.float32 or not latents.is_cuda:
            latents = latents.float().to(dev)
        # an expanded (stride-0) latent row is passed as a broadcast instead of being materialised;
        # a column slice of a wider row-major matrix (run_network's [P, 95] input) is read in place
        if not (latents.dim() == 2 and latents.shape[0] == n and latents.stride(1) == 1):
            latents = latents.reshape(n, -1).contiguous()
        if latents.shape[-1] != LATENT:
            raise RuntimeError(f"nonrigid_nerf_b200: latent size {latents.shape[-1]} unsupported (32)")
        a.latents, a.latent_stride = latents.data_ptr(), (latents.stride(0) if n > 1 else 0)
        a.bender_packed = bender_pack.data_ptr()
        keep.append(latents)
    a.out_ch = out_ch
    if cutoff is not None:
        a.use_cutoff, a.rigidity_cutoff = 1, float(cutoff)
    if scaling is not None:
        a.use_scaling, a.scaling = 1, float(scaling)
    if removal is not None:
        a.use_removal, a.removal_threshold = 1, float(removal)
    raw = torch.empty(n, s, out_ch, dtype=torch.float32, device=dev)
    a.raw = raw.data_ptr()
    details: Dict[str, torch.Tensor] = {}
    if want_details:
        details["initial_input_pts"] = torch.empty(n, s, 3, dtype=torch.float32, device=dev)
        details["input_pts"] = torch.empty(n, s, 3, dtype=torch.float32, device=dev)
        a.initial_input_pts, a.input_pts = details["initial_input_pts"].data_ptr(), details["input_pts"].data_ptr()
        if bender_pack is not None:
            details["unmasked_offsets"] = torch.empty(n, s, 3, dtype=torch.float32, device=dev)
            details["masked_offsets"] = torch.empty(n, s, 3, dtype=torch.float32, device=dev)
            details["rigidity_mask"] = torch.empty(n, s, 1, dtype=torch.float32, device=dev)
            a.unmasked_offsets = details["unmasked_offsets"].data_ptr()
            a.masked_offsets = details["masked_offsets"].data_ptr()
            a.rigidity_mask = details["rigidity_mask"].data_ptr()
    if stash is not None:
        a.stash = stash.data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nrn_field_forward(C.byref(a)), "field_forward")
    return raw, details


def field_forward(rays: torch.Tensor, z_vals: torch.Tensor, latents: Optional[torch.Tensor], nerf_pack: torch.Tensor,
                  bender_pack: Optional[torch.Tensor], out_ch: int, cutoff: Optional[float] = None,
                  scaling: Optional[float] = None, removal: Optional[float] = None,
                  want_details: bool = False, stash: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """One fused pass over rays x samples: raw [N, S, out_ch] (+ the reference's per-point `details`).
    `stash` (uint8, nrn_stash_bytes) switches the kernel to training mode (activations kept for backward)."""
    return _field(rays, z_vals, None, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details, stash)


def field_forward_points(points: torch.Tensor, latents: Optional[torch.Tensor], nerf_pack: torch.Tensor,
                         bender_pack: Optional[torch.Tensor], out_ch: int, cutoff=None, scaling=None, removal=None,
                         want_details: bool = False) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """Point mode (NeRF.forward(x)): one xyz (+ one latent) per row; returns raw [P, 1, out_ch]."""
    return _field(None, None, points, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details)


def composite(raw: torch.Tensor, z_vals: torch.Tensor, rays_d: torch.Tensor, noise: Optional[torch.Tensor] = None,
              white_bkgd: bool = False, n_importance: int = 0, u: Optional[torch.Tensor] = None,
              want_point_outputs: bool = True) -> Dict[str, torch.Tensor]:
    """raw2outputs (train.py:724-789), optionally fused with hierarchical resampling
    (run_nerf_helpers.py:651-698, train.py:910-923, :959)."""
    raw = _f32c(raw, "raw")
    z_vals = _f32c(z_vals, "z_vals")
    n, s, c = raw.shape
    dev = raw.device
    if rays_d.dtype != torch.float32 or rays_d.stride(-1) != 1 or rays_d.dim() != 2:
        rays_d = rays_d.reshape(n, -1).float().contiguous()
    a = _lib.NrnCompositeArgs()
    a.raw, a.z_vals, a.rays_d, a.rays_d_stride = raw.data_ptr(), z_vals.data_ptr(), rays_d.data_ptr(), rays_d.stride(0)
    if noise is not None:
        noise = _f32c(noise, "noise")
        a.noise = noise.data_ptr()
    a.n_rays, a.n_samples, a.channels, a.white_bkgd = n, s, c, int(bool(white_bkgd))
    out = {
        "rgb_map": torch.empty(n, 3, dtype=torch.float32, device=dev),
        "disp_map": torch.empty(n, dtype=torch.float32, device=dev),
        "acc_map": torch.empty(n, dtype=torch.float32, device=dev),
        "depth_map": torch.empty(n, dtype=torch.float32, device=dev),
    }
    a.rgb_map, a.disp_map, a.acc_map, a.depth_map = (out[k].data_ptr() for k in ("rgb_map", "disp_map", "acc_map", "depth_map"))
    if want_point_outputs:
        out["weights"] = torch.empty(n, s, dtype=torch.float32, device=dev)
        out["alpha"] = torch.empty(n, s, dtype=torch.float32, device=dev)
        a.weights, a.alpha = out["weights"].data_ptr(), out["alpha"].data_ptr()
    a.n_importance = n_importance
    if n_importance > 0:
        if u is not None:
            u = _f32c(u, "u")
            a.u = u.data_ptr()
        out["z_vals_out"] = torch.empty(n, s + n_importance, dtype=torch.float32, device=dev)
        out["z_std"] = torch.empty(n, dtype=torch.float32, device=dev)
        a.z_vals_out, a.z_std = out["z_vals_out"].data_ptr(), out["z_std"].data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nrn_composite(C.byref(a)), "composite")
    return out


def composite_backward(raw, z_vals, rays_d, noise, white_bkgd, d_rgb, d_acc=None) -> torch.Tensor:
    raw = _f32c(raw, "raw")
    z_vals = _f32c(z_vals, "z_vals")
    d_rgb = _f32c(d_rgb, "d_rgb")
    n, s, c = raw.shape
    if rays_d.dtype != torch.float32 or rays_d.stride(-1) != 1 or rays_d.dim() != 2:
        rays_d = rays_d.reshape(n, -1).float().contiguous()
    a = _lib.NrnCompositeBwdArgs()
    a.raw, a.z_vals, a.rays_d, a.rays_d_stride = raw.data_ptr(), z_vals.data_ptr(), rays_d.data_ptr(), rays_d.stride(0)
    if noise is not None:
        noise = _f32c(noise, "noise")
        a.noise = noise.data_ptr()
    a.n_rays, a.n_samples, a.channels, a.white_bkgd = n, s, c, int(bool(white_bkgd))
    a.d_rgb_map = d_rgb.data_ptr()
    if d_acc is not None:
        d_acc = _f32c(d_acc, "d_acc")
        a.d_acc_map = d_acc.data_ptr()
    d_raw = torch.empty_like(raw)
    a.d_raw = d_raw.data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    with torch.cuda.device(raw.device):
        _lib.check(_lib.load().nrn_composite_backward(C.byref(a)), "composite_backward")
    return d_raw


def sample_pdf_op(bins: torch.Tensor, weights: torch.Tensor, n_samples: int, u: Optional[torch.Tensor]) -> torch.Tensor:
    bins = _f32c(bins, "bins")
    weights = _f32c(weights, "weights")
    n, nb = bins.shape
    if weights.shape != (n, nb - 1):
        raise RuntimeError(f"sample_pdf: weights must be [N, len(bins)-1], got {tuple(weights.shape)} for bins {tuple(bins.shape)}")
    if u is not None:
        u = _f32c(u, "u")
    out = torch.empty(n, n_samples, dtype=torch.float32, device=bins.device)
    with torch.cuda.device(bins.device):
        _lib.check(_lib.load().nrn_sample_pdf(_ptr(bins), _ptr(weights), _ptr(u), n, nb, n_samples, _ptr(out), _stream()), "sample_pdf")
    return out


# ---------------------------------------------------------------------------------------------
# ray generation, batch sampling, free-viewpoint post-processing
# ---------------------------------------------------------------------------------------------
def intrinsics_row(intrin) -> list:
    return [float(intrin["focal_x"]), float(intrin["focal_y"]), float(intrin["center_x"]), float(intrin["center_y"])]


def pack_rays(rays_o: torch.Tensor, rays_d: torch.Tensor, near: float, far: float) -> torch.Tensor:
    """[N, 8] = (o, d, near, far) for scalar near / far in one launch (train.py:388-398)."""
    rays_o, rays_d = _f32c(rays_o, "rays_o"), _f32c(rays_d, "rays_d")
    n = rays_o.shape[0]
    rays = torch.empty(n, 8, dtype=torch.float32, device=rays_o.device)
    with torch.cuda.device(rays_o.device):
        _lib.check(_lib.load().nrn_pack_rays(_ptr(rays_o), _ptr(rays_d), float(near), float(far), n, _ptr(rays), _stream()), "pack_rays")
    return rays


def get_rays(c2w: torch.Tensor, intrin) -> Tuple[torch.Tensor, torch.Tensor]:
    """get_rays (run_nerf_helpers.py:588-605): rays_o, rays_d [H, W, 3] of one camera, computed on the device."""
    if not c2w.is_cuda:
        raise RuntimeError("nonrigid_nerf_b200: get_rays needs a CUDA pose (there is no CPU path)")
    h, w = int(intrin["height"]), int(intrin["width"])
    pose = c2w[:3, :4].float().contiguous()
    k = torch.tensor(intrinsics_row(intrin), dtype=torch.float32, device=c2w.device)
    rays_o = torch.empty(h, w, 3, dtype=torch.float32, device=c2w.device)
    rays_d = torch.empty(h, w, 3, dtype=torch.float32, device=c2w.device)
    with torch.cuda.device(c2w.device):
        _lib.check(_lib.load().nrn_get_rays(_ptr(pose), _ptr(k), h, w, _ptr(rays_o), _ptr(rays_d), _stream()), "get_rays")
    return rays_o, rays_d


def ray_batch(pix: torch.Tensor, poses: torch.Tensor, intrinsics: torch.Tensor, image_to_view: Optional[torch.Tensor],
              images: Optional[torch.Tensor], height: int, width: int):
    """Rays (and target colours) of the pixels pix [N, 3] = (image, x, y), computed from poses [n_img, 3, 4] and
    intrinsics [n_views, 4] instead of gathered from a table of every ray (train.py:1498-1517, :1546-1564)."""
    for t, nm in ((pix, "pix"), (poses, "poses"), (intrinsics, "intrinsics")):
        if not t.is_cuda:
            raise RuntimeError(f"nonrigid_nerf_b200: ray_batch needs CUDA tensors ({nm}); there is no CPU path")
    n = pix.shape[0]
    dev = pix.device
    pix = pix.long().contiguous()
    poses = poses[:, :3, :4].float().contiguous()
    intrinsics = intrinsics.float().contiguous()
    if image_to_view is not None:
        image_to_view = image_to_view.to(dev).int().contiguous()
    rays_o = torch.empty(n, 3, dtype=torch.float32, device=dev)
    rays_d = torch.empty(n, 3, dtype=torch.float32, device=dev)
    target = None
    if images is not None:
        if images.dtype != torch.float32 or not images.is_contiguous() or tuple(images.shape[1:]) != (height, width, 3):
            raise RuntimeError("nonrigid_nerf_b200: ray_batch images must be a contiguous fp32 [n_images, H, W, 3] CUDA tensor")
        target = torch.empty(n, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nrn_ray_batch(_ptr(pix), n, _ptr(poses), _ptr(intrinsics), _ptr(image_to_view), _ptr(images), height, width,
                                             _ptr(rays_o), _ptr(rays_d), _ptr(target), _stream()), "ray_batch")
    return rays_o, rays_d, target


def median_visibility_index(weights: torch.Tensor) -> torch.Tensor:
    """Index [N] (int64) of the sample whose accumulated visibility is closest to 0.5 (free_viewpoint_rendering.py:623-629)."""
    weights = _f32c(weights, "weights")
    n, s = weights.shape
    idx = torch.empty(n, dtype=torch.int64, device=weights.device)
    with torch.cuda.device(weights.device):
        _lib.check(_lib.load().nrn_median_visibility_index(_ptr(weights), n, s, _ptr(idx), _stream()), "median_visibility_index")
    return idx
