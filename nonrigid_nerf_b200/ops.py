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


def _views_trunk_params(net):
    """The trunk and alpha_linear of a NeRF(use_viewdirs=True)"""
    return ([net.pts_linears[i].weight for i in range(8)] + [net.alpha_linear.weight],
            [net.pts_linears[i].bias for i in range(8)] + [net.alpha_linear.bias])


def _cached_pack(owner, attr: str, params, kind: str, check_shapes, nbytes, pack) -> torch.Tensor:
    """The packed image of `params`, kept as owner.<attr> = (key, buffer) and rewritten in place when a parameter
    changed (or while FORCE_PACK is set).  `kind` names the parameters in the error; check_shapes() raises for a
    geometry the kernels do not implement; pack(lib, buf) writes the image."""
    key = _versions(params)
    cache = getattr(owner, attr, None)
    if cache is not None and cache[0] == key and not FORCE_PACK:
        return cache[1]
    for t in params:
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise RuntimeError(f"nonrigid_nerf_b200: {kind} parameters must be contiguous fp32 CUDA tensors")
    check_shapes()
    lib = _lib.load()
    dev = params[0].device
    buf = cache[1] if cache is not None else torch.empty(nbytes(lib), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        pack(lib, buf)
    setattr(owner, attr, (key, buf))
    return buf


def pack_nerf(net) -> torch.Tensor:
    """fp16 wgmma operand image of a NeRF module's weights (see csrc/nrn_common.cuh).  With use_viewdirs=True the head
    of the image is alpha_linear in row 3 under three zero rows, so the head step yields alpha in channel 3."""
    views = getattr(net, "use_viewdirs", False)
    ws, bs = _views_trunk_params(net) if views else nerf_param_list(net)
    in_ch = 63 + (LATENT if getattr(net, "time_conditioned_baseline", False) else 0)   # [embedding (| latent)]

    def check_shapes():
        if ws[0].shape != (256, in_ch) or ws[5].shape != (256, in_ch + 256) or ws[8].shape[1] != 256:
            raise RuntimeError("nonrigid_nerf_b200: only D=8, W=256, skips=[4], multires=10, use_viewdirs=False is implemented "
                               f"(got layer shapes {[tuple(w.shape) for w in ws]})")

    def pack(lib, buf):
        hw, hb = ws[8], bs[8]
        if views:   # [0, 0, 0, alpha]: the head rows of rgb + alpha
            hw, hb = torch.cat([hw.new_zeros(3, hw.shape[1]), hw], 0), torch.cat([hb.new_zeros(3), hb], 0)
        _lib.check(lib.nrn_pack_nerf(_ptr_array([w.detach() for w in ws[:8] + [hw]]), _ptr_array([b.detach() for b in bs[:8] + [hb]]),
                                     in_ch, hw.shape[0], _ptr(buf), _stream()), "pack_nerf")

    return _cached_pack(net, "_nrn_pack", ws + bs, "NeRF", check_shapes, lambda lib: lib.nrn_packed_nerf_bytes(), pack)


def views_param_list(net):
    ws = [net.feature_linear.weight, net.views_linears[0].weight, net.rgb_linear.weight]
    bs = [net.feature_linear.bias, net.views_linears[0].bias, net.rgb_linear.bias]
    return ws, bs


def _check_views_shapes(ws):
    if ws[0].shape != (256, 256) or ws[1].shape != (128, 256 + 27) or ws[2].shape != (3, 128):
        raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True needs W=256 and input_ch_views=27 "
                           f"(got view-head shapes {[tuple(w.shape) for w in ws]})")


def pack_views(net) -> torch.Tensor:
    """fp16 wgmma operand images of the view-dependent head (feature_linear, views_linears.0, rgb_linear)."""
    ws, bs = views_param_list(net)
    return _cached_pack(net, "_nrn_pack_views", ws + bs, "NeRF", lambda: _check_views_shapes(ws), lambda lib: lib.nrn_packed_views_bytes(),
                        lambda lib, buf: _lib.check(lib.nrn_pack_views(_ptr_array([w.detach() for w in ws]),
                                                                       _ptr_array([b.detach() for b in bs]), _ptr(buf), _stream()),
                                                    "pack_views"))


def pack_views_t(net) -> torch.Tensor:
    """fp16 transposed images of the view-dependent head for its backward (rgb_linear, views_linears.0's feature columns,
    feature_linear); cached like pack_views."""
    ws, _ = views_param_list(net)
    return _cached_pack(net, "_nrn_pack_views_t", ws, "NeRF", lambda: _check_views_shapes(ws), lambda lib: lib.nrn_packed_views_t_bytes(),
                        lambda lib, buf: _lib.check(lib.nrn_pack_views_t(_ptr_array([w.detach() for w in ws]), _ptr(buf), _stream()),
                                                    "pack_views_t"))


def pack_bender(bender) -> torch.Tensor:
    net_w, net_b, rig_w, rig_b = bender_param_list(bender)

    def check_shapes():
        if net_w[0].shape != (64, 3 + LATENT):
            raise RuntimeError("nonrigid_nerf_b200: only ray_bending_latent_size=32, simple_neural is implemented")

    def pack(lib, buf):
        _lib.check(lib.nrn_pack_bender(_ptr_array([t.detach() for t in net_w]), _ptr_array([t.detach() for t in net_b]),
                                       _ptr_array([t.detach() for t in rig_w]), _ptr_array([t.detach() for t in rig_b]),
                                       LATENT, _ptr(buf), _stream()), "pack_bender")

    return _cached_pack(bender, "_nrn_pack", net_w + net_b + rig_w + rig_b, "ray_bending", check_shapes,
                        lambda lib: lib.nrn_packed_bender_bytes(), pack)


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


def latent_rows(latents: torch.Tensor, n: int, dev) -> Tuple[torch.Tensor, int]:
    """The [n, 32] fp32 latents as the kernels read them, and their row stride in floats (0: one row for every ray).
    An expanded (stride-0) latent row is passed as a broadcast instead of being materialised; a column slice of a wider
    row-major matrix (run_network's [P, 95] input) is read in place."""
    if latents.dtype != torch.float32 or not latents.is_cuda:
        latents = latents.float().to(dev)
    if not (latents.dim() == 2 and latents.shape[0] == n and latents.stride(1) == 1):
        latents = latents.reshape(n, -1).contiguous()
    if latents.shape[-1] != LATENT:
        raise RuntimeError(f"nonrigid_nerf_b200: latent size {latents.shape[-1]} unsupported (32)")
    return latents, (latents.stride(0) if n > 1 else 0)


def tc_ray_bias(net, latents: torch.Tensor, stride: int) -> torch.Tensor:
    """Time-conditioned baseline: the per-ray biases of L0 and L5, rb[n][l] = b_l + W_l[:, 63:95] . z[n] (fp32, from the
    nn.Linear weights); one row when stride == 0."""
    w0, b0 = net.pts_linears[0].weight, net.pts_linears[0].bias
    w5, b5 = net.pts_linears[5].weight, net.pts_linears[5].bias
    for t in (w0, b0, w5, b5):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise RuntimeError("nonrigid_nerf_b200: NeRF parameters must be contiguous fp32 CUDA tensors")
    rows = 1 if stride == 0 else latents.shape[0]
    rb = torch.empty(rows, 2, 256, dtype=torch.float32, device=latents.device)
    with torch.cuda.device(latents.device):
        _lib.check(_lib.load().nrn_tc_latent_bias(_ptr(latents), stride, rows, _ptr(w0.detach()), _ptr(b0.detach()), _ptr(w5.detach()),
                                                  _ptr(b5.detach()), _ptr(rb), _stream()), "tc_latent_bias")
    return rb


def _rays8(rays: torch.Tensor) -> torch.Tensor:
    """rays [N, 8+] as the kernels read them: fp32 rows of 8 floats (o, d, near, far), 8 floats apart."""
    if not rays.is_cuda:
        raise RuntimeError("nonrigid_nerf_b200: rays must be a CUDA tensor (there is no CPU path)")
    if rays.dtype == torch.float32 and rays.stride(-1) == 1 and rays.stride(0) == 8:
        return rays
    return rays[:, :8].float().contiguous()


def _field_args(rays, z_vals, points, n_samples, latents, nerf_pack, bender_pack, out_ch, knobs, want_raw, want_details):
    """NrnFieldArgs of one field call.  Ray mode: rays [N, 8+] and z_vals [N, S]; point mode: points [N * n_samples, 3+],
    n_samples consecutive points forming one ray.  `latents` (None: not read) are those of each ray, or each point in
    point mode; knobs = (cutoff, scaling, removal).  raw [N, S, out_ch] (when want_raw) and the details are allocated here.
    Returns (args, raw, details, keep): keep holds the converted inputs the args point into (the latent rows last, when
    latents are given) and must live until the call is enqueued."""
    a = _lib.NrnFieldArgs()
    if points is None:
        rays, z_vals = _rays8(rays), _f32c(z_vals, "z_vals")
        n, s = z_vals.shape
        a.rays, a.z_vals = rays.data_ptr(), z_vals.data_ptr()
        keep = [rays, z_vals]
    else:
        if not points.is_cuda:
            raise RuntimeError("nonrigid_nerf_b200: points must be a CUDA tensor (there is no CPU path)")
        if points.dtype != torch.float32 or points.dim() != 2 or points.stride(1) != 1:
            points = points.reshape(points.shape[0], -1).float().contiguous()
        s = n_samples
        if points.shape[0] % s:
            raise RuntimeError(f"nonrigid_nerf_b200: use_viewdirs=True: {points.shape[0]} points do not form rays of num_ray_samples={s}")
        n = points.shape[0] // s
        a.points, a.points_stride = points.data_ptr(), points.stride(0)
        keep = [points]
    dev = keep[0].device
    a.n_rays, a.n_samples, a.out_ch = n, s, out_ch
    a.nerf_packed = nerf_pack.data_ptr()
    if bender_pack is not None:
        a.bender_packed = bender_pack.data_ptr()
    if latents is not None:
        latents, a.latent_stride = latent_rows(latents, n * s if points is not None else n, dev)
        a.latents = latents.data_ptr()
        keep.append(latents)
    cutoff, scaling, removal = knobs
    if cutoff is not None:
        a.use_cutoff, a.rigidity_cutoff = 1, float(cutoff)
    if scaling is not None:
        a.use_scaling, a.scaling = 1, float(scaling)
    if removal is not None:
        a.use_removal, a.removal_threshold = 1, float(removal)
    raw = None
    if want_raw:
        raw = torch.empty(n, s, out_ch, dtype=torch.float32, device=dev)
        a.raw = raw.data_ptr()
    details: Dict[str, torch.Tensor] = {}
    if want_details:
        names = ["initial_input_pts", "input_pts"] + (["unmasked_offsets", "masked_offsets", "rigidity_mask"] if bender_pack is not None else [])
        for k in names:
            details[k] = torch.empty(n, s, 1 if k == "rigidity_mask" else 3, dtype=torch.float32, device=dev)
            setattr(a, k, details[k].data_ptr())
    a.stream = torch.cuda.current_stream().cuda_stream
    return a, raw, details, keep


def _viewdirs(viewdirs: Optional[torch.Tensor], dev) -> Tuple[torch.Tensor, int]:
    """The view directions [N, 3+] as fp32 rows on `dev`, and their row stride in floats."""
    if viewdirs is None:
        raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True without a ray bender needs the view directions")
    if viewdirs.dtype != torch.float32 or viewdirs.dim() != 2 or viewdirs.stride(1) != 1 or not viewdirs.is_cuda:
        viewdirs = viewdirs.reshape(viewdirs.shape[0], -1).float().contiguous().to(dev)
    return viewdirs, viewdirs.stride(0) if viewdirs.shape[0] > 1 else 3


def _field(rays, z_vals, points, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details, stash=None, relu_mask=None,
           tc_net=None):
    tc = tc_net if bender_pack is None else None   # time-conditioned baseline: the latents enter as per-ray biases of L0 and L5
    if latents is None and (bender_pack is not None or tc is not None):
        raise RuntimeError("nonrigid_nerf_b200: " + ("ray bending" if tc is None else "time_conditioned_baseline") + " needs latents")
    a, raw, details, keep = _field_args(rays, z_vals, points, 1, latents if bender_pack is not None or tc is not None else None, nerf_pack,
                                        bender_pack, out_ch, (cutoff, scaling, removal), True, want_details)
    if stash is not None:
        a.stash = stash.data_ptr()
    if relu_mask is not None:
        a.relu_mask = relu_mask.data_ptr()
    with torch.cuda.device(keep[0].device):
        if tc is not None:
            ray_bias = tc_ray_bias(tc, keep[-1], a.latent_stride)
            _lib.check(_lib.load().nrn_field_forward_tc(C.byref(a), _ptr(ray_bias)), "field_forward_tc")
        else:
            _lib.check(_lib.load().nrn_field_forward(C.byref(a)), "field_forward")
    return raw, details


def field_forward(rays: torch.Tensor, z_vals: torch.Tensor, latents: Optional[torch.Tensor], nerf_pack: torch.Tensor,
                  bender_pack: Optional[torch.Tensor], out_ch: int, cutoff: Optional[float] = None,
                  scaling: Optional[float] = None, removal: Optional[float] = None,
                  want_details: bool = False, stash: Optional[torch.Tensor] = None,
                  relu_mask: Optional[torch.Tensor] = None, tc_net=None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """One fused pass over rays x samples: raw [N, S, out_ch] (+ the reference's per-point `details`).
    `stash` (uint8, nrn_stash_bytes) with `relu_mask` (uint8, nrn_relu_mask_bytes) switches the kernel to training mode
    (activations and ReLU masks kept for backward).  `tc_net`: the time-conditioned NeRF whose L0 / L5 weights turn
    `latents` into per-ray biases (no bender)."""
    return _field(rays, z_vals, None, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details, stash,
                  relu_mask, tc_net)


def field_forward_points(points: torch.Tensor, latents: Optional[torch.Tensor], nerf_pack: torch.Tensor,
                         bender_pack: Optional[torch.Tensor], out_ch: int, cutoff=None, scaling=None, removal=None,
                         want_details: bool = False, tc_net=None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """Point mode (NeRF.forward(x)): one xyz (+ one latent) per row; returns raw [P, 1, out_ch]."""
    return _field(None, None, points, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details,
                  tc_net=tc_net)


def _fast_pass(entry: str, sizer: str, size_flag: int, rays, z_vals, latents, nerf_pack, bender_pack, out_ch, knobs, want_details,
               structs, needs_latents: bool = False):
    """Run the render pass `entry` (nrn_field_forward_<entry>) with the workspace nrn_<sizer>_workspace_bytes(n, S, out_ch,
    size_flag) asks for: latents are passed with a bender, or always when needs_latents.  structs(a, dev): the C structs
    (or None) that follow NrnFieldArgs.  Returns (raw, details)."""
    if latents is None and (needs_latents or bender_pack is not None):
        raise RuntimeError("nonrigid_nerf_b200: ray bending needs latents")
    a, raw, details, keep = _field_args(rays, z_vals, None, 1, latents if needs_latents or bender_pack is not None else None, nerf_pack,
                                        bender_pack, out_ch, knobs, True, want_details)
    dev = keep[0].device
    args = [C.byref(x) if x is not None else None for x in structs(a, dev)]
    lib = _lib.load()
    nbytes = getattr(lib, f"nrn_{sizer}_workspace_bytes")(a.n_rays, a.n_samples, out_ch, size_flag)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(getattr(lib, f"nrn_field_forward_{entry}")(C.byref(a), *args, _ptr(ws), nbytes), f"field_forward_{entry}")
    return raw, details


def field_forward_occupancy(rays: torch.Tensor, z_vals: torch.Tensor, latents: Optional[torch.Tensor], nerf_pack: torch.Tensor,
                            bender_pack: Optional[torch.Tensor], out_ch: int, cutoff=None, scaling=None, removal=None,
                            want_details: bool = False, grid=None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """field_forward (inference) that runs the NeRF trunk only on samples the occupancy grid keeps (geometry.OccupancyGrid):
    raw [N, S, out_ch] equal to field_forward's where kept and 0 elsewhere; the details for every sample."""
    return _fast_pass("occupancy", "occupancy", int(bender_pack is not None), rays, z_vals, latents, nerf_pack, bender_pack,
                      out_ch, (cutoff, scaling, removal), want_details, lambda a, dev: [grid.c_struct(dev)])


def field_forward_baked(rays: torch.Tensor, z_vals: torch.Tensor, latents: Optional[torch.Tensor], nerf_pack: torch.Tensor,
                        bender_pack: Optional[torch.Tensor], out_ch: int, cutoff=None, scaling=None, removal=None,
                        want_details: bool = False, grid=None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """field_forward (inference) that samples the radiance grid (geometry.RadianceGrid) in place of the NeRF trunk for
    samples whose (bent) point lies inside its box: raw [N, S, out_ch] from the lookup there (raw[..., 4] = 0), equal to
    field_forward's elsewhere; the details for every sample."""
    return _fast_pass("baked", "baked", int(bender_pack is not None), rays, z_vals, latents, nerf_pack, bender_pack, out_ch,
                      (cutoff, scaling, removal), want_details, lambda a, dev: [grid.c_struct(dev)])


def field_forward_deformed(rays: torch.Tensor, z_vals: torch.Tensor, latents: torch.Tensor, nerf_pack: torch.Tensor, bender_pack: torch.Tensor,
                           out_ch: int, cutoff=None, scaling=None, removal=None, want_details: bool = False, grid=None,
                           deformation=None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """field_forward_baked whose bends come from one frame of a baked deformation grid (geometry.FrameDeformation) for every
    ray whose samples all lie inside its box; the other rays are bent by the bender with their latents and equal
    field_forward_baked's bit for bit.  raw [N, S, out_ch] and the details for every sample."""
    return _fast_pass("deformed", "deformed", int(want_details), rays, z_vals, latents, nerf_pack, bender_pack, out_ch,
                      (cutoff, scaling, removal), want_details, lambda a, dev: [grid.c_struct(dev), deformation.c_struct(dev)],
                      needs_latents=True)


def field_forward_terminate(rays: torch.Tensor, z_vals: torch.Tensor, latents: Optional[torch.Tensor], nerf_pack: torch.Tensor,
                            bender_pack: Optional[torch.Tensor], out_ch: int, cutoff=None, scaling=None, removal=None,
                            want_details: bool = False, threshold: float = 0.0, grid=None, noise: Optional[torch.Tensor] = None
                            ) -> Tuple[torch.Tensor, Dict[str, torch.Tensor], torch.Tensor]:
    """field_forward (inference) with early ray termination (nrn_field_forward_terminate): the samples run in segments of
    nrn_termination_segment(), and a ray stops being evaluated after the segment in which its transmittance falls below
    `threshold`; with `grid` (geometry.OccupancyGrid) a sample is also skipped where the grid would skip it.  noise [N, S]:
    the sigma noise compositing will add (already scaled), or None.  Returns raw [N, S, out_ch] (field_forward's where
    evaluated, 0 elsewhere), the details for every sample, and termination_index [N] int32."""
    term = noise_rows = None

    def structs(a, dev):
        nonlocal term, noise_rows
        g = grid.c_struct(dev) if grid is not None else None
        t = _lib.NrnTerminationArgs()
        t.threshold = float(threshold)
        if noise is not None:
            noise_rows = _f32c(noise, "noise")
            if tuple(noise_rows.shape) != (a.n_rays, a.n_samples):
                raise RuntimeError(f"nonrigid_nerf_b200: noise must be [{a.n_rays}, {a.n_samples}], got {list(noise_rows.shape)}")
            t.noise = noise_rows.data_ptr()
        term = torch.empty(a.n_rays, dtype=torch.int32, device=dev)
        t.termination_index = term.data_ptr()
        return [g, t]

    raw, details = _fast_pass("terminate", "termination", int(bender_pack is not None), rays, z_vals, latents, nerf_pack, bender_pack,
                              out_ch, (cutoff, scaling, removal), want_details, structs)
    return raw, details, term


def field_forward_views(rays: Optional[torch.Tensor], z_vals: Optional[torch.Tensor], points: Optional[torch.Tensor], n_samples: int,
                        latents: Optional[torch.Tensor], viewdirs: Optional[torch.Tensor], nerf_pack: torch.Tensor,
                        bender_pack: Optional[torch.Tensor], views_pack: Optional[torch.Tensor], cutoff=None, scaling=None,
                        removal=None, want_details: bool = False) -> Tuple[Optional[torch.Tensor], Dict[str, torch.Tensor]]:
    """The view-dependent head (inference): raw [N, S, 4] = [rgb, alpha].  Ray mode: rays [N, 8+] and z_vals [N, S].
    Point mode: points [P, 3+] with P = N * n_samples, n_samples consecutive points forming one ray (the finite
    differences of the bent points run inside each), latents per point.  With a bender the view directions are those
    differences; without one `viewdirs` (per ray, or per point in point mode) is used.  views_pack = None with a bender
    runs the bend pass alone (raw is None; the details are filled)."""
    if bender_pack is not None and latents is None:
        raise RuntimeError("nonrigid_nerf_b200: ray bending needs latents")
    a, raw, details, keep = _field_args(rays, z_vals, points, n_samples, latents if bender_pack is not None else None, nerf_pack,
                                        bender_pack, 4, (cutoff, scaling, removal), views_pack is not None, want_details)
    n, s, dev = a.n_rays, a.n_samples, keep[0].device
    lib = _lib.load()
    v = _lib.NrnViewArgs()
    if bender_pack is not None:
        ws = torch.empty(lib.nrn_views_workspace_bytes(n, s), dtype=torch.uint8, device=dev)
        v.workspace = ws.data_ptr()
    else:
        viewdirs, v.viewdirs_stride = _viewdirs(viewdirs, dev)
        v.viewdirs = viewdirs.data_ptr()
    if views_pack is not None:
        v.views_packed = views_pack.data_ptr()
    with torch.cuda.device(dev):
        _lib.check(lib.nrn_field_forward_views(C.byref(a), C.byref(v)), "field_forward_views")
    return raw, details


def bend_points(points: torch.Tensor, latent: torch.Tensor, bender_pack: torch.Tensor, nerf_pack: torch.Tensor, offsets: torch.Tensor,
                rigidity: torch.Tensor, workspace: torch.Tensor) -> None:
    """The ray bender alone, knobs off, at points [P, 3] (contiguous fp32) with one latent row [1, 32]: its unmasked offsets
    into offsets [P, 3] and its rigidity into rigidity [P] (both contiguous fp32, preallocated so that a caller looping over
    planes allocates nothing per call).  workspace: nrn_views_workspace_bytes(P, 1) bytes.  This is the bend pass of
    nrn_field_forward_views in point mode with raw NULL, so the view head does not run; the bend pass reads no NeRF
    weights, but the argument block names a packed NeRF, so nerf_pack is any 16-byte aligned buffer of
    nrn_packed_nerf_bytes() bytes."""
    n = points.shape[0]
    a = _lib.NrnFieldArgs()
    a.points, a.points_stride = points.data_ptr(), 3
    a.n_rays, a.n_samples, a.out_ch = n, 1, 4
    a.nerf_packed, a.bender_packed = nerf_pack.data_ptr(), bender_pack.data_ptr()
    a.latents, a.latent_stride = latent.data_ptr(), 0   # one row for every point
    a.unmasked_offsets, a.rigidity_mask = offsets.data_ptr(), rigidity.data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    v = _lib.NrnViewArgs()
    v.workspace = workspace.data_ptr()
    _lib.check(_lib.load().nrn_field_forward_views(C.byref(a), C.byref(v)), "bend_points")


def field_forward_views_train(rays: torch.Tensor, z_vals: torch.Tensor, viewdirs: torch.Tensor, nerf_pack: torch.Tensor,
                              views_pack: torch.Tensor, want_details: bool = False):
    """The view-dependent head without a bender, keeping what its backward needs: raw [N, S, 4], details, and the buffers
    (stash, relu_mask, views_stash, hv_mask)."""
    a, raw, details, keep = _field_args(rays, z_vals, None, 1, None, nerf_pack, None, 4, (None, None, None), True, want_details)
    n, s, dev = a.n_rays, a.n_samples, keep[0].device
    lib = _lib.load()
    bufs = {k: torch.empty(f(n, s), dtype=torch.uint8, device=dev) for k, f in (
        ("stash", lib.nrn_stash_bytes), ("relu_mask", lib.nrn_relu_mask_bytes), ("views_stash", lib.nrn_views_stash_bytes),
        ("hv_mask", lib.nrn_hv_mask_bytes))}
    a.stash, a.relu_mask = bufs["stash"].data_ptr(), bufs["relu_mask"].data_ptr()
    v, t = _lib.NrnViewArgs(), _lib.NrnViewTrainArgs()
    v.views_packed = views_pack.data_ptr()
    viewdirs, v.viewdirs_stride = _viewdirs(viewdirs, dev)
    v.viewdirs = viewdirs.data_ptr()
    t.views_stash, t.hv_mask = bufs["views_stash"].data_ptr(), bufs["hv_mask"].data_ptr()
    with torch.cuda.device(dev):
        _lib.check(lib.nrn_field_forward_views_train(C.byref(a), C.byref(v), C.byref(t)), "field_forward_views_train")
    return raw, details, bufs


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
