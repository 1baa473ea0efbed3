"""torch.autograd glue between the PyTorch-owned parameters and the fused kernels.

PyTorch owns every tensor (weights stay nn.Parameters with the reference's names); the extension
keeps a derived packed fp16 copy (ops.pack_*), rebuilt when a parameter's version counter changes.
Gradients come back from the DGRAD/WGRAD kernels as flat fp32 buffers laid out in the reference's
parameter shapes and are handed to autograd as views, so the reference's Adam, its two-pass
test-latent backward (train.py:1595-1608) and the PyTorch-side regularisers keep working unchanged.

Gradient flow implemented (SURVEY.md appendix C): rgb_map / acc_map -> raw -> both MLPs -> positional
encoding -> bent point -> bender weights and per-ray latents; plus upstream gradients on the coarse
`unmasked_offsets` / `rigidity_mask` details (offsets / rigidity regularisers, train.py:219-242).
z_vals, ray origins/directions and the importance samples carry no gradient (train.py:918).
"""
from __future__ import annotations

import ctypes as C
import numbers
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib, ops


def _knobs(net):
    bender = net.ray_bender[0]
    cutoff = getattr(bender, "rigidity_test_time_cutoff", None) if bender is not None else None
    scaling = getattr(bender, "test_time_scaling", None) if bender is not None else None
    removal = getattr(net, "test_time_nonrigid_object_removal_threshold", None)
    return cutoff, scaling, removal


def _packs(net):
    """(cutoff, scaling, removal, nerf_pack, bender_pack, out_ch) of an inference call on `net`; the view-dependent head
    (use_viewdirs=True, no output_linear) writes 4 channels."""
    bender = net.ray_bender[0]
    cutoff, scaling, removal = _knobs(net)
    nerf_pack = ops.pack_nerf(net)
    bender_pack = ops.pack_bender(bender) if bender is not None else None
    out_ch = 4 if getattr(net, "use_viewdirs", False) else net.output_linear.weight.shape[0]
    return cutoff, scaling, removal, nerf_pack, bender_pack, out_ch


def _tc_net(net):
    """The NeRF itself when it is a time-conditioned baseline (its latents enter L0 / L5 as per-ray biases), else None.
    Like train.py:574-576 the baseline runs without ray bending."""
    if not getattr(net, "time_conditioned_baseline", False):
        return None
    if net.ray_bender[0] is not None:
        raise RuntimeError("nonrigid_nerf_b200: the time_conditioned_baseline NeRF requires ray bending to be turned off "
                           "(ray_bender must be None)")
    return net


def _flat_params(net, bender):
    """Parameters in the flat order of the WGRAD output buffers (csrc/wgrad.cu); `net` may be None for the bender's
    alone."""
    nerf = []
    if net is not None:
        ws, bs = ops.nerf_param_list(net)
        for w, b in zip(ws, bs):
            nerf += [w, b]
    bend = []
    if bender is not None:
        net_w, net_b, rig_w, rig_b = ops.bender_param_list(bender)
        for i in range(4):
            bend += [net_w[i], net_b[i]]
        bend.append(net_w[4])
        for i in range(3):
            bend += [rig_w[i], rig_b[i]]
    return nerf, bend


def _split_flat(flat: torch.Tensor, like):
    out, o = [], 0
    for p in like:
        n = p.numel()
        out.append(flat[o:o + n].view_as(p))
        o += n
    assert o == flat.numel(), (o, flat.numel())
    return out


def check_held_out(held_out: Optional[torch.Tensor], n_rays: int, device) -> Optional[torch.Tensor]:
    """The per-ray held-out mask of render(..., held_out=) as the kernels read it (one byte per ray, nonzero = held out), or
    None.  Raises, before any launch, unless it is an [n_rays] bool or uint8 tensor on `device`.  Its contents are not read
    on the host, so a CUDA graph may replay a step with new ones."""
    if held_out is None:
        return None
    if not isinstance(held_out, torch.Tensor):
        raise RuntimeError("nonrigid_nerf_b200: held_out must be a tensor ([N] bool or uint8, one entry per ray)")
    if held_out.dtype not in (torch.bool, torch.uint8):
        raise RuntimeError(f"nonrigid_nerf_b200: held_out must be bool or uint8 (0/1 per ray), got {held_out.dtype}")
    if held_out.dim() != 1 or held_out.shape[0] != n_rays:
        raise RuntimeError(f"nonrigid_nerf_b200: held_out must have shape [{n_rays}] (one entry per ray), got {list(held_out.shape)}")
    if held_out.device != torch.device(device):
        raise RuntimeError(f"nonrigid_nerf_b200: held_out must be on the rays' device {device}, got {held_out.device}")
    return held_out.contiguous().view(torch.uint8)


def _zero_held_rows(d_raw: torch.Tensor, held: Optional[torch.Tensor]) -> torch.Tensor:
    """Without a bender a held-out ray contributes nothing (the reference's second backward pass only runs with a bender,
    train.py:1595-1597): its rows of the upstream gradient d_raw [N, S, C] are zeroed, which gives every parameter and latent
    the gradient of the loss weighted by the training rays alone."""
    if held is None:
        return d_raw
    return d_raw.masked_fill(held.view(-1, 1, 1).bool(), 0.0)


class _FieldTrainFn(torch.autograd.Function):
    """raw, unmasked_offsets, rigidity_mask (differentiable) + point details (not differentiable).
    params = the NeRF's parameters in WGRAD order, followed (with a bender) by the bender's parameters in WGRAD order.
    held: None, or the uint8 per-ray mask of check_held_out: with a bender a held-out ray's gradient reaches its latent
    only (the held-out DGRAD leaves it out of the weight gradients), without one it is dropped (_zero_held_rows).
    (No autograd object outlives an iteration: a cached graph fragment would pin AccumulateGrad nodes -- and the CUDA
    stream they were created on -- across iterations, which breaks CUDA-graph capture of the step.)"""

    @staticmethod
    def forward(ctx, net, rays, z_vals, latents, held, n_nerf, *params):
        bender = net.ray_bender[0]
        cutoff, scaling, removal = _knobs(net)
        if removal is not None:
            raise RuntimeError("nonrigid_nerf_b200: test_time_nonrigid_object_removal_threshold is a test-time knob; "
                               "it is not differentiable")
        nerf_pack = ops.pack_nerf(net)
        bender_pack = ops.pack_bender(bender) if bender is not None else None
        out_ch = net.output_linear.weight.shape[0]
        n, s = z_vals.shape
        lib = _lib.load()
        stash = torch.empty(lib.nrn_stash_bytes(n, s), dtype=torch.uint8, device=z_vals.device)
        relu_mask = torch.empty(lib.nrn_relu_mask_bytes(n, s), dtype=torch.uint8, device=z_vals.device)
        tc = _tc_net(net)
        ctx.tc_latents = None
        if tc is not None:   # the latents as the forward read them: the backward forms their gradient and dW0 / dW5's latent columns
            ctx.tc_latents = ops.latent_rows(latents.detach(), n, z_vals.device)
            latents = ctx.tc_latents[0]
        raw, det = ops.field_forward(rays, z_vals, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, None, True, stash,
                                     relu_mask, tc)
        ctx.net, ctx.n_nerf = net, n_nerf
        ctx.shape = (n, s, out_ch)
        ctx.knobs = (cutoff, scaling)
        ctx.packs = (nerf_pack, bender_pack)
        ctx.stash = stash
        ctx.relu_mask = relu_mask
        ctx.params = params
        ctx.held = held
        ctx.set_materialize_grads(False)
        if bender is not None:
            _register_relu_mask(det["unmasked_offsets"], relu_mask)
            ctx.save_for_backward(det["unmasked_offsets"], det["rigidity_mask"])
            outs = (raw, det["unmasked_offsets"], det["rigidity_mask"], det["initial_input_pts"], det["input_pts"],
                    det["masked_offsets"])
            ctx.mark_non_differentiable(*outs[3:])
        else:
            outs = (raw, det["initial_input_pts"], det["input_pts"])
            ctx.mark_non_differentiable(*outs[1:])
        return outs

    @staticmethod
    def backward(ctx, d_raw, *rest):
        net = ctx.net
        bender = net.ray_bender[0]
        n, s, out_ch = ctx.shape
        nerf_pack, bender_pack = ctx.packs
        cutoff, scaling = ctx.knobs
        dev = ctx.stash.device
        lib = _lib.load()
        d_un = d_rig = None
        if bender is not None:
            d_un, d_rig = rest[0], rest[1]
        if d_raw is None:
            d_raw = torch.zeros(n, s, out_ch, dtype=torch.float32, device=dev)
        held = ctx.held
        if bender is None:
            d_raw, held = _zero_held_rows(d_raw, held), None
        a = _lib.NrnFieldBwdArgs()
        a.n_rays, a.n_samples, a.out_ch = n, s, out_ch
        d_raw = d_raw.contiguous().float()
        a.d_raw = d_raw.data_ptr()
        a.stash, a.relu_mask = ctx.stash.data_ptr(), ctx.relu_mask.data_ptr()
        gstash = torch.empty(lib.nrn_grad_stash_bytes(n, s), dtype=torch.uint8, device=dev)
        scratch = torch.empty(lib.nrn_wgrad_scratch_bytes(), dtype=torch.uint8, device=dev)
        a.grad_stash, a.wgrad_scratch = gstash.data_ptr(), scratch.data_ptr()
        a.nerf_packed = nerf_pack.data_ptr()
        nerf_p = list(ctx.params[:ctx.n_nerf])   # the output_linear block (last two) goes to its own destination
        n_floats = lib.nrn_nerf_tc_grad_floats(out_ch) if ctx.tc_latents is not None else lib.nrn_nerf_grad_floats(out_ch)
        nerf_grad, a.nerf_grad, a.nerf_grad_head, a.accumulate_nerf = _grad_destination(nerf_p, len(nerf_p) - 2, n_floats, dev)
        bend_grad = d_lat = None
        keep = [d_raw]
        if bender is not None:
            un, rig = ctx.saved_tensors
            a.bender_packed = bender_pack.data_ptr()
            a.unmasked_offsets, a.rigidity_mask = un.data_ptr(), rig.data_ptr()
            if d_un is not None:
                d_un = d_un.contiguous().float()
                a.d_unmasked_offsets = d_un.data_ptr()
                keep.append(d_un)
            if d_rig is not None:
                d_rig = d_rig.contiguous().float()
                a.d_rigidity_mask = d_rig.data_ptr()
                keep.append(d_rig)
            if cutoff is not None:
                a.use_cutoff, a.rigidity_cutoff = 1, float(cutoff)
            if scaling is not None:
                a.use_scaling, a.scaling = 1, float(scaling)
            bend_p = list(ctx.params[ctx.n_nerf:])
            bend_grad, a.bender_grad, _, a.accumulate_bender = _grad_destination(bend_p, len(bend_p), lib.nrn_bender_grad_floats(), dev)
            d_lat = torch.empty(n, ops.LATENT, dtype=torch.float32, device=dev)
            a.d_latents = d_lat.data_ptr()
        a.stream = torch.cuda.current_stream().cuda_stream
        if ctx.tc_latents is not None:
            lat, stride = ctx.tc_latents
            t = _lib.NrnTcBwdArgs()
            t.latents, t.latent_stride = lat.data_ptr(), stride
            t.w0, t.w5 = net.pts_linears[0].weight.data_ptr(), net.pts_linears[5].weight.data_ptr()
            d_lat = torch.empty(n, ops.LATENT, dtype=torch.float32, device=dev)
            workspace = torch.empty(lib.nrn_tc_workspace_bytes(n), dtype=torch.uint8, device=dev)
            t.d_latents, t.workspace = d_lat.data_ptr(), workspace.data_ptr()
            with torch.cuda.device(dev):
                _lib.check(lib.nrn_field_backward_tc(C.byref(a), C.byref(t)), "field_backward_tc")
        elif bender is not None and torch.are_deterministic_algorithms_enabled():
            # the per-ray latent gradient in a fixed order (per-point rows, then one reduction) instead of fp32 atomics
            rows = torch.empty(lib.nrn_latent_rows_bytes(n, s) // 4, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                if held is not None:
                    _lib.check(lib.nrn_field_backward_det_held_out(C.byref(a), rows.data_ptr(), held.data_ptr()), "field_backward_det_held_out")
                else:
                    _lib.check(lib.nrn_field_backward_det(C.byref(a), rows.data_ptr()), "field_backward_det")
        elif held is not None:
            with torch.cuda.device(dev):
                _lib.check(lib.nrn_field_backward_held_out(C.byref(a), held.data_ptr()), "field_backward_held_out")
        else:
            with torch.cuda.device(dev):
                _lib.check(lib.nrn_field_backward(C.byref(a)), "field_backward")
        # the stash and the ReLU masks live as long as the autograd node: backward(retain_graph=True) followed by a second backward()
        # over the same graph (test-latent pass of the reference loop, train.py:1595-1606) reads it again
        grads = _param_grads(nerf_grad, nerf_p)
        if bender is not None:
            grads += _param_grads(bend_grad, bend_p)
        return (None, None, None, d_lat, None, None, *grads)


# ---------------------------------------------------------------------------------------------
# gradient arena look-ups (optim.Adam seats every .grad as a view of one flat buffer)
# ---------------------------------------------------------------------------------------------
def _arena_destination(params):
    from .optim import arena_destination
    return arena_destination(list(params))


def _grad_destination(params, split: int, n_floats: int, dev):
    """Where the WGRAD reduction puts the gradients of `params` (in its flat order; params[split:] is the block it writes
    to a head destination of its own, none when split == len(params)).  When every parameter requires a gradient and the
    .grad tensors of each block lie back to back in one buffer (optim.Adam's arena), it ADDS into them in place and
    autograd gets nothing to accumulate: (None, block address, head block address or None, 1).  Otherwise a fresh flat
    buffer of n_floats, handed to autograd as per-parameter views by _param_grads (torch.optim.Adam, or after the caller
    re-bound gradients -- the reference sets weights.grad = None between its two backward passes, train.py:1598-1604):
    (buffer, its address, None, 0)."""
    if all(p.requires_grad for p in params):
        dst = _arena_destination(params[:split])
        head = _arena_destination(params[split:]) if dst is not None and split < len(params) else None
        if dst is not None and (head is not None or split == len(params)):
            return None, dst, head, 1
    flat = torch.empty(n_floats, dtype=torch.float32, device=dev)
    return flat, flat.data_ptr(), None, 0


def _param_grads(flat: Optional[torch.Tensor], params):
    """What backward returns for `params` after _grad_destination: nothing where WGRAD added into the arena, else views of
    the flat buffer (None for a parameter that needs no gradient)."""
    if flat is None:
        return [None] * len(params)
    return [g if p.requires_grad else None for g, p in zip(_split_flat(flat, params), params)]


class _LatentGatherFn(torch.autograd.Function):
    """latents[timestep[i]] for every ray i (train.py:173-189: stack the per-frame latents, index by the ray's time step).
    The per-frame latents are views of the optimizer's flat buffer, so the table is read in place; the backward adds the
    per-ray gradients [N, Z] into the latents' .grad arena with one index_add_ (fallback: per-latent gradient views).
    Under torch.use_deterministic_algorithms(True) PyTorch's CUDA index_add_ sums in a fixed order by itself (and can be
    captured in a CUDA graph), so deterministic mode needs nothing of its own here."""

    @staticmethod
    def forward(ctx, timestep, *latents):
        z = latents[0].numel()
        base, contiguous = latents[0].data_ptr(), True
        for i, l in enumerate(latents):
            if l.data_ptr() != base + 4 * z * i or l.dtype != torch.float32 or not l.is_contiguous():
                contiguous = False
                break
        if contiguous and latents[0].untyped_storage().nbytes() >= latents[0].storage_offset() * 4 + 4 * z * len(latents):
            table = latents[0].detach().as_strided((len(latents), z), (z, 1))
        else:
            table = torch.stack([l.detach() for l in latents], 0)
        ctx.save_for_backward(timestep)
        ctx.latents = latents
        ctx.z = z
        return torch.index_select(table, 0, timestep)

    @staticmethod
    def backward(ctx, d_sel):
        (timestep,) = ctx.saved_tensors
        latents, z = ctx.latents, ctx.z
        t = len(latents)
        dst = _arena_destination(latents) if all(l.requires_grad for l in latents) else None
        if dst is not None:
            g0 = latents[0].grad
            g0.as_strided((t, z), (z, 1)).index_add_(0, timestep, d_sel.contiguous().float())
            return (None,) * (t + 1)
        g = torch.zeros(t, z, dtype=torch.float32, device=d_sel.device).index_add_(0, timestep, d_sel.float())
        return (None, *[g[i] if l.requires_grad else None for i, l in enumerate(latents)])


def gather_latents(latents, timestep: torch.Tensor) -> torch.Tensor:
    """[N, Z] per-ray latents from the list of per-frame leaf tensors and the rays' time-step ids."""
    return _LatentGatherFn.apply(timestep, *latents)


# ---------------------------------------------------------------------------------------------
# divergence regulariser (fused; SURVEY.md section 8f row f2)
# ---------------------------------------------------------------------------------------------
_MASK_BY_PTR = {}   # data_ptr of a coarse pass's unmasked_offsets -> weakref to that pass's ReLU masks


def _register_relu_mask(unmasked: torch.Tensor, relu_mask: torch.Tensor) -> None:
    import weakref
    for k in [k for k, v in _MASK_BY_PTR.items() if v() is None]:
        del _MASK_BY_PTR[k]
    _MASK_BY_PTR[unmasked.data_ptr()] = weakref.ref(relu_mask)


def lookup_relu_mask(unmasked: torch.Tensor) -> Optional[torch.Tensor]:
    """The ReLU masks of the coarse pass that produced `unmasked`: found by walking the tensor's autograd history
    (through the reshapes of render()) to the _FieldTrainFn node, which owns them; the address table is only the
    fallback for detached tensors."""
    fn = unmasked.grad_fn
    for _ in range(8):
        if fn is None:
            break
        relu_mask = getattr(fn, "relu_mask", None)
        if isinstance(relu_mask, torch.Tensor):
            return relu_mask
        nxt = [f for f, _ in fn.next_functions if f is not None]
        fn = nxt[0] if len(nxt) == 1 else None
    ref = _MASK_BY_PTR.get(unmasked.data_ptr())
    return ref() if ref is not None else None


def _div_args(ctx):
    """The NrnDivArgs fields the divergence forward and backward share, from the tensors the forward keeps in ctx."""
    un, rg, w, e, relu_mask, bender_pack, tan, scal = ctx.keep
    a = _lib.NrnDivArgs()
    a.n_rays, a.n_samples = ctx.shape
    a.relu_mask, a.e, a.unmasked_offsets, a.rigidity_mask, a.weights = relu_mask.data_ptr(), e.data_ptr(), un.data_ptr(), rg.data_ptr(), w.data_ptr()
    a.weights_are_opacity_alpha = 1 if ctx.w_is_alpha else 0
    a.bender_packed = bender_pack.data_ptr()
    a.tangent_stash = tan.data_ptr()
    a.d, a.alpha, a.beta, a.tau_c = (scal[i].data_ptr() for i in range(4))
    a.stream = torch.cuda.current_stream().cuda_stream
    return a


class _DivergenceFn(torch.autograd.Function):
    """per-ray mean_s(w * (e^T J e)^2) of the offset field, closed-form forward and backward (csrc/div.cu).  held: None or
    the uint8 per-ray mask of check_held_out: a held-out ray's term then reaches the bender's weights not at all, its
    latent through the gradients w.r.t. unmasked / rigidity."""

    @staticmethod
    def forward(ctx, unmasked, rigidity, weights, e, relu_mask, bender, w_is_alpha, held, *bend_p):
        n, s = unmasked.shape[0], unmasked.shape[1]
        dev = unmasked.device
        lib = _lib.load()
        un = unmasked.detach().contiguous().float()
        rg = rigidity.detach().contiguous().float()
        w = weights.detach().contiguous().float()
        e = e.contiguous().float()
        bender_pack = ops.pack_bender(bender)   # the cached fp16 images the coarse pass ran with
        tan = torch.empty(lib.nrn_div_stash_bytes(n, s), dtype=torch.uint8, device=dev)
        scal = torch.empty(4, n * s, dtype=torch.float32, device=dev)
        loss = torch.empty(n, dtype=torch.float32, device=dev)
        ctx.keep = (un, rg, w, e, relu_mask, bender_pack, tan, scal)
        ctx.w_is_alpha = bool(w_is_alpha)
        ctx.shape = (n, s)
        a = _div_args(ctx)
        a.loss = loss.data_ptr()
        if torch.are_deterministic_algorithms_enabled():   # the per-ray loss in a fixed order instead of fp32 atomics
            rows = torch.empty(lib.nrn_div_loss_rows_bytes(n, s) // 4, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _lib.check(lib.nrn_divergence_forward_det(C.byref(a), rows.data_ptr()), "divergence_forward_det")
        else:
            with torch.cuda.device(dev):
                _lib.check(lib.nrn_divergence_forward(C.byref(a)), "divergence_forward")
        ctx.bend_p = bend_p
        ctx.held = held
        ctx.in_shapes = (unmasked.shape, rigidity.shape)
        return loss

    @staticmethod
    def backward(ctx, g):
        n, s = ctx.shape
        dev = ctx.keep[0].device
        lib = _lib.load()
        # G = dL/dd per point = g_ray * 2 * w * d / S, computed (with its max, the loss-scale source) by the library
        g = g.reshape(n).contiguous().float()
        G = torch.empty(n * s, dtype=torch.float32, device=dev)
        a = _div_args(ctx)
        a.g_ray, a.G_workspace = g.data_ptr(), G.data_ptr()
        adj = torch.empty(lib.nrn_div_grad_stash_bytes(n, s), dtype=torch.uint8, device=dev)
        scratch = torch.empty(lib.nrn_wgrad_scratch_bytes(), dtype=torch.uint8, device=dev)
        d_un = torch.empty(n * s, 3, dtype=torch.float32, device=dev)
        d_rg = torch.empty(n * s, dtype=torch.float32, device=dev)
        bend_p = list(ctx.bend_p)
        bend_grad, a.bender_grad, _, a.accumulate_bender = _grad_destination(bend_p, len(bend_p), lib.nrn_bender_grad_floats(), dev)
        a.adjoint_stash, a.wgrad_scratch = adj.data_ptr(), scratch.data_ptr()
        a.d_unmasked_offsets, a.d_rigidity_mask = d_un.data_ptr(), d_rg.data_ptr()
        with torch.cuda.device(dev):
            if ctx.held is not None:
                _lib.check(lib.nrn_divergence_backward_held_out(C.byref(a), ctx.held.data_ptr()), "divergence_backward_held_out")
            else:
                _lib.check(lib.nrn_divergence_backward(C.byref(a)), "divergence_backward")
        return (d_un.view(ctx.in_shapes[0]), d_rg.view(ctx.in_shapes[1]), None, None, None, None, None, None,
                *_param_grads(bend_grad, bend_p))


def divergence_loss(unmasked: torch.Tensor, rigidity: torch.Tensor, weights: Optional[torch.Tensor], bender,
                    e: Optional[torch.Tensor] = None, opacity_alpha: Optional[torch.Tensor] = None,
                    held_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Fused divergence regulariser on the coarse samples of the LAST differentiable coarse pass.
    unmasked [N,S,3], rigidity [N,S,1] must be that pass's outputs (they locate its ReLU masks and
    carry the gradient w.r.t. the primal bender evaluation); weights [N,S] are used detached; `e` [N*S,3]
    are the Hutchinson probes (drawn with torch.randn like run_nerf_helpers.py:110 when None).
    Instead of `weights`, `opacity_alpha` [N,S] may be given: the kernels then apply the reference's
    1 - exp(-relu(opacity_alpha)) (train.py:267) themselves.  held_out [N] (bool or uint8): rays whose term reaches their
    latent only, not the bender's weights (render(..., held_out=))."""
    held = check_held_out(held_out, unmasked.shape[0], unmasked.device)
    relu_mask = lookup_relu_mask(unmasked)
    if relu_mask is None:
        raise RuntimeError("nonrigid_nerf_b200: no ReLU masks for these offsets -- the fused divergence term needs the "
                           "un-chunked coarse pass of the current differentiable render() call (N_rand <= chunk)")
    n, s = unmasked.shape[0], unmasked.shape[1]
    if e is None:
        e = torch.randn(n * s, 3, device=unmasked.device)
    _, bend_p = _flat_params(None, bender)
    if opacity_alpha is not None:
        return _DivergenceFn.apply(unmasked, rigidity, opacity_alpha, e, relu_mask, bender, True, held, *bend_p)
    return _DivergenceFn.apply(unmasked, rigidity, weights, e, relu_mask, bender, False, held, *bend_p)


class _RayLossFn(torch.autograd.Function):
    """Per-ray loss of training_wrapper_class.forward (train.py:208-287) in one kernel (csrc/loss.cu): data terms, offsets /
    rigidity regulariser, and the (already reduced) divergence regulariser with its weight and the regularisers' schedule."""

    @staticmethod
    def forward(ctx, rgb, rgb0, target, weights, unmasked, rigidity, lam_o, lam_r, sched_step, sched_n_iters, div, lam_div):
        n = rgb.shape[0]
        dev = rgb.device
        lib = _lib.load()
        a = _lib.NrnRayLossArgs()
        keep = [rgb.detach().contiguous().float(), target.contiguous().float()]
        a.rgb, a.target = keep[0].data_ptr(), keep[1].data_ptr()
        u_rgb = torch.empty(n, 3, dtype=torch.float32, device=dev)
        a.u_rgb = u_rgb.data_ptr()
        u_rgb0 = u_off = u_rig = u_div = None
        if rgb0 is not None:
            keep.append(rgb0.detach().contiguous().float())
            a.rgb0 = keep[-1].data_ptr()
            u_rgb0 = torch.empty(n, 3, dtype=torch.float32, device=dev)
            a.u_rgb0 = u_rgb0.data_ptr()
        s = 1
        if unmasked is not None:
            s = unmasked.shape[1]
            keep += [weights.detach().contiguous().float(), unmasked.detach().contiguous().float(), rigidity.detach().contiguous().float()]
            a.weights, a.unmasked_offsets, a.rigidity_mask = (t.data_ptr() for t in keep[-3:])
            u_off = torch.empty(n, s, 3, dtype=torch.float32, device=dev)
            u_rig = torch.empty(rigidity.shape, dtype=torch.float32, device=dev)
            a.u_unmasked_offsets, a.u_rigidity_mask = u_off.data_ptr(), u_rig.data_ptr()
        a.n_rays, a.n_samples = n, s
        a.lam_offsets, a.lam_rigidity = float(lam_o), float(lam_r)
        if sched_step is not None:
            keep.append(sched_step.detach().float().contiguous())
            a.sched_step, a.sched_n_iters = keep[-1].data_ptr(), float(sched_n_iters)
        if div is not None:
            keep.append(div.detach().contiguous().float())
            u_div = torch.empty(n, dtype=torch.float32, device=dev)
            a.divergence, a.lam_divergence, a.u_divergence = keep[-1].data_ptr(), float(lam_div), u_div.data_ptr()
        loss = torch.empty(n, dtype=torch.float32, device=dev)
        a.loss = loss.data_ptr()
        a.stream = torch.cuda.current_stream().cuda_stream
        with torch.cuda.device(dev):
            _lib.check(lib.nrn_ray_loss(C.byref(a)), "ray_loss")
        ctx.units = (u_rgb, u_rgb0, u_off, u_rig, u_div)
        ctx.ns = (n, s)
        return loss

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        g = g.contiguous().float()
        a = _lib.NrnRayLossBwdArgs()
        a.n_rays, a.n_samples = ctx.ns
        a.g = g.data_ptr()
        outs = [None if u is None else torch.empty_like(u) for u in ctx.units]
        names = ("rgb", "rgb0", "unmasked_offsets", "rigidity_mask", "divergence")
        for nm, u, o in zip(names, ctx.units, outs):
            if u is not None:
                setattr(a, "u_" + nm, u.data_ptr())
                setattr(a, "d_" + nm, o.data_ptr())
        a.stream = torch.cuda.current_stream().cuda_stream
        with torch.cuda.device(g.device):
            _lib.check(lib.nrn_ray_loss_backward(C.byref(a)), "ray_loss_backward")
        d_rgb, d_rgb0, d_off, d_rig, d_div = outs
        return d_rgb, d_rgb0, None, None, d_off, d_rig, None, None, None, None, d_div, None


def ray_loss(rgb, rgb0, target, weights=None, unmasked=None, rigidity=None, lam_offsets=0.0, lam_rigidity=0.0,
             sched_step: Optional[torch.Tensor] = None, sched_n_iters: float = 1.0, divergence: Optional[torch.Tensor] = None,
             lam_divergence: float = 0.0):
    """loss[N] = img2mse(rgb) + img2mse(rgb0) + sched * lam_offsets * (offsets + lam_rigidity * rigidity regulariser)
                 + sched * lam_divergence * divergence,   sched = (1/100)^(1 - sched_step / sched_n_iters) evaluated on the device
    from the 0-dim CUDA tensor `sched_step` (CUDA-graph-safe), or 1 when sched_step is None (the caller folds the schedule
    into the weights)."""
    return _RayLossFn.apply(rgb, rgb0, target, weights, unmasked, rigidity, lam_offsets, lam_rigidity, sched_step, sched_n_iters,
                            divergence, lam_divergence)


class _CompositeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, raw, z_vals, rays_d, noise, white_bkgd, n_importance, u):
        o = ops.composite(raw, z_vals, rays_d, noise, white_bkgd, n_importance, u, True)
        ctx.save_for_backward(raw, z_vals, rays_d, noise if noise is not None else raw.new_empty(0))
        ctx.has_noise = noise is not None
        ctx.white = bool(white_bkgd)
        ctx.set_materialize_grads(False)
        outs = [o["rgb_map"], o["acc_map"], o["disp_map"], o["depth_map"], o["weights"], o["alpha"]]
        if n_importance > 0:
            outs += [o["z_vals_out"], o["z_std"]]
        ctx.mark_non_differentiable(*outs[2:])
        return tuple(outs)

    @staticmethod
    def backward(ctx, d_rgb, d_acc, *unsupported):
        raw, z_vals, rays_d, noise = ctx.saved_tensors
        if d_rgb is None and d_acc is None:
            return None, None, None, None, None, None, None
        if d_rgb is None:
            d_rgb = torch.zeros(raw.shape[0], 3, dtype=torch.float32, device=raw.device)
        d_raw = ops.composite_backward(raw, z_vals, rays_d, noise if ctx.has_noise else None, ctx.white, d_rgb, d_acc)
        return d_raw, None, None, None, None, None, None


# ---------------------------------------------------------------------------------------------
# entry points used by train.py / run_nerf_helpers.py
# ---------------------------------------------------------------------------------------------
def _needs_grad(net, latents) -> bool:
    if not torch.is_grad_enabled():
        return False
    bender = net.ray_bender[0]
    if latents is not None and latents.requires_grad:
        return True
    if any(p.requires_grad for p in net.parameters()):
        return True
    return bender is not None and any(p.requires_grad for p in bender.parameters())


_SEATED = object()


def views_check(net, latents=None, bender=_SEATED) -> None:
    """Raise for what the view-dependent head (use_viewdirs=True) does not support: with a bender (the seated one, or
    `bender`, which the caller is about to seat), exact view directions, rays of fewer than two samples and any
    differentiable call (training with a bender is not implemented; without one the head trains)."""
    if not getattr(net, "use_viewdirs", False):
        return
    if bender is _SEATED:
        bender = net.ray_bender[0]
    if bender is None:
        return
    if not net.approx_nonrigid_viewdirs:
        raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True with approx_nonrigid_viewdirs=False (exact view directions "
                           "through the ray bender) is not implemented")
    if net.num_ray_samples is None or net.num_ray_samples < 2:
        raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True with a ray bender needs num_ray_samples >= 2 (the view "
                           f"directions are finite differences along each ray; got {net.num_ray_samples})")
    if _needs_grad(net, latents) or (torch.is_grad_enabled() and any(p.requires_grad for p in bender.parameters())):
        raise RuntimeError("nonrigid_nerf_b200: use_viewdirs=True: training with the view-dependent head is not implemented yet; "
                           "rendering works under torch.no_grad()")


def _views_flat_params(net):
    """A use_viewdirs=True NeRF's parameters in the flat order of nrn_field_backward_views: the trunk's (W0 b0 .. W7 b7),
    then the head block in module order."""
    ws, bs = ops._views_trunk_params(net)
    trunk = []
    for w, b in zip(ws[:8], bs[:8]):
        trunk += [w, b]
    head = [net.views_linears[0].weight, net.views_linears[0].bias, net.feature_linear.weight, net.feature_linear.bias,
            net.alpha_linear.weight, net.alpha_linear.bias, net.rgb_linear.weight, net.rgb_linear.bias]
    return trunk, head


class _ViewsTrainFn(torch.autograd.Function):
    """The view-dependent head without a bender: raw (differentiable) + point details (not).  params = the trunk's
    parameters, then the head block's (_views_flat_params).  The view direction is the ray's own, so like the reference no
    gradient leaves the field but the parameters': the latents get none."""

    @staticmethod
    def forward(ctx, net, rays, z_vals, viewdirs, held, n_trunk, *params):
        if getattr(net, "test_time_nonrigid_object_removal_threshold", None) is not None:
            raise RuntimeError("nonrigid_nerf_b200: test_time_nonrigid_object_removal_threshold is a test-time knob; "
                               "it is not differentiable")
        nerf_pack, views_pack = ops.pack_nerf(net), ops.pack_views(net)
        views_t = ops.pack_views_t(net)   # the weights this forward ran with, for the backward
        raw, det, bufs = ops.field_forward_views_train(rays, z_vals, viewdirs, nerf_pack, views_pack, True)
        ctx.n_trunk, ctx.params = n_trunk, params
        ctx.shape = z_vals.shape
        ctx.packs = (nerf_pack, views_t)
        # the stashes live as long as the autograd node (a second backward over a retained graph reads them again)
        ctx.bufs = bufs
        ctx.held = held
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(det["initial_input_pts"], det["input_pts"])
        return raw, det["initial_input_pts"], det["input_pts"]

    @staticmethod
    def backward(ctx, d_raw, *rest):
        n, s = ctx.shape
        nerf_pack, views_t = ctx.packs
        bufs = ctx.bufs
        dev = nerf_pack.device
        lib = _lib.load()
        if d_raw is None:
            d_raw = torch.zeros(n, s, 4, dtype=torch.float32, device=dev)
        d_raw = _zero_held_rows(d_raw, ctx.held).contiguous().float()
        a = _lib.NrnFieldBwdArgs()
        a.n_rays, a.n_samples, a.out_ch = n, s, 4
        a.d_raw = d_raw.data_ptr()
        a.stash, a.relu_mask = bufs["stash"].data_ptr(), bufs["relu_mask"].data_ptr()
        gstash = torch.empty(lib.nrn_grad_stash_bytes(n, s), dtype=torch.uint8, device=dev)
        vgstash = torch.empty(lib.nrn_views_grad_stash_bytes(n, s), dtype=torch.uint8, device=dev)
        scratch = torch.empty(lib.nrn_wgrad_scratch_bytes(), dtype=torch.uint8, device=dev)
        a.grad_stash, a.wgrad_scratch = gstash.data_ptr(), scratch.data_ptr()
        a.nerf_packed = nerf_pack.data_ptr()
        params = list(ctx.params)   # the trunk's, then the head block's
        flat, a.nerf_grad, a.nerf_grad_head, a.accumulate_nerf = _grad_destination(params, ctx.n_trunk, lib.nrn_nerf_views_grad_floats(), dev)
        a.stream = torch.cuda.current_stream().cuda_stream
        v = _lib.NrnViewBwdArgs()
        v.views_t_packed, v.views_stash, v.views_grad_stash, v.hv_mask = (
            views_t.data_ptr(), bufs["views_stash"].data_ptr(), vgstash.data_ptr(), bufs["hv_mask"].data_ptr())
        with torch.cuda.device(dev):
            _lib.check(lib.nrn_field_backward_views(C.byref(a), C.byref(v)), "field_backward_views")
        return (None, None, None, None, None, None, *_param_grads(flat, params))


def field_views(net, rays, z_vals, points, latents, viewdirs, want_details, bend_only=False):
    """The view-dependent head (inference): ray mode (rays, z_vals) or point mode (points grouped into rays of
    net.num_ray_samples).  bend_only: the bend pass alone (details only, raw is None).  Differentiable ray-mode calls
    without a bender go through field()."""
    views_check(net, latents)
    if _needs_grad(net, latents):
        raise RuntimeError("nonrigid_nerf_b200: the point-wise NeRF.forward / run_network entry is inference-only; "
                           "differentiable rendering goes through render() / render_rays()")
    cutoff, scaling, removal, nerf_pack, bender_pack, _ = _packs(net)
    views_pack = None if bend_only else ops.pack_views(net)
    s = net.num_ray_samples if (points is not None and bender_pack is not None and not bend_only) else 1
    return ops.field_forward_views(rays, z_vals, points, s, latents, viewdirs, nerf_pack, bender_pack, views_pack, cutoff,
                                   scaling, removal, want_details)


def field(net, rays: torch.Tensor, z_vals: torch.Tensor, latents: Optional[torch.Tensor],
          want_details: bool, viewdirs: Optional[torch.Tensor] = None,
          held_out: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """Fused field evaluation for rays x samples; differentiable when autograd is recording.  viewdirs [N, 3]: the
    normalised ray directions a use_viewdirs=True model takes.  held_out [N] (bool or uint8): rays whose gradient reaches
    their latent only with a bender, and nothing without one (check_held_out)."""
    held = check_held_out(held_out, rays.shape[0], rays.device)
    bender = net.ray_bender[0]
    if getattr(net, "use_viewdirs", False):
        if viewdirs is None:
            raise RuntimeError("nonrigid_nerf_b200: a use_viewdirs=True model needs ray batches with view directions (11 columns)")
        views_check(net, latents)   # with a bender: raises for a differentiable call
        if bender is None and _needs_grad(net, latents):
            trunk, head = _views_flat_params(net)
            raw, init, bent = _ViewsTrainFn.apply(net, rays, z_vals, viewdirs, held, len(trunk), *trunk, *head)
            return raw, ({"initial_input_pts": init, "input_pts": bent} if want_details else {})
        return field_views(net, rays, z_vals, None, latents, viewdirs, want_details)
    _tc_net(net)
    if not _needs_grad(net, latents):
        return field_rays(net, rays, z_vals, latents, want_details)
    nerf_p, bend_p = _flat_params(net, bender)
    outs = _FieldTrainFn.apply(net, rays, z_vals, latents, held, len(nerf_p), *nerf_p, *bend_p)
    if bender is not None:
        raw, un, rig, init, bent, masked = outs
        details = {"initial_input_pts": init, "unmasked_offsets": un, "rigidity_mask": rig, "masked_offsets": masked,
                   "input_pts": bent}
    else:
        raw, init, bent = outs
        details = {"initial_input_pts": init, "input_pts": bent}
    return raw, (details if want_details else {})


def _skip_check(net, latents, what: str, why: str) -> None:
    """Raise for what a render pass that skips samples (`what`: "with an occupancy grid", ...) does not support: the
    view-dependent head, the time-conditioned baseline and differentiable calls (`why` the skipped samples get no gradient)."""
    if getattr(net, "use_viewdirs", False):
        raise RuntimeError(f"nonrigid_nerf_b200: rendering {what} is not implemented for use_viewdirs=True")
    if getattr(net, "time_conditioned_baseline", False):
        raise RuntimeError(f"nonrigid_nerf_b200: rendering {what} is not implemented for time_conditioned_baseline=True")
    if _needs_grad(net, latents):
        raise RuntimeError(f"nonrigid_nerf_b200: rendering {what} is inference only; call render() under torch.no_grad() ({why})")


def occupancy_check(net, latents, grid) -> None:
    """Raise, before any launch, for what render(..., occupancy=grid) does not support: the view-dependent head, the
    time-conditioned baseline and differentiable calls."""
    from .geometry import OccupancyGrid
    if not isinstance(grid, OccupancyGrid):
        raise RuntimeError(f"nonrigid_nerf_b200: occupancy must be a geometry.OccupancyGrid, got {type(grid).__name__}")
    _skip_check(net, latents, "with an occupancy grid", "skipped samples would get no gradient")


def field_occupancy(net, rays, z_vals, latents, want_details, grid):
    """field_rays that evaluates the NeRF trunk only on the samples the occupancy grid keeps; raw is 0 for the others."""
    occupancy_check(net, latents, grid)
    cutoff, scaling, removal, nerf_pack, bender_pack, out_ch = _packs(net)
    return ops.field_forward_occupancy(rays, z_vals, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details,
                                       grid)


def baked_check(net, latents, grid) -> None:
    """Raise, before any launch, for what render(..., baked=) does not support: a pass without a geometry.RadianceGrid,
    the view-dependent head, the time-conditioned baseline and differentiable calls."""
    from .geometry import RadianceGrid, bake_check
    if not isinstance(grid, RadianceGrid):
        raise RuntimeError(f"nonrigid_nerf_b200: a baked render pass needs a geometry.RadianceGrid, got {type(grid).__name__}")
    bake_check(net)
    if _needs_grad(net, latents):
        raise RuntimeError("nonrigid_nerf_b200: rendering from a baked radiance grid is inference only; call render() under "
                           "torch.no_grad() (the grid carries no gradient)")


def deformation_check(net, deformation) -> None:
    """Raise, before any launch, unless `deformation` is a geometry.FrameDeformation that a pass of `net` can read: the model
    has a ray bender, and the grid is well formed and on the model's device."""
    from .geometry import FrameDeformation
    if not isinstance(deformation, FrameDeformation):
        raise RuntimeError(f"nonrigid_nerf_b200: a baked deformation must be a geometry.FrameDeformation (DeformationGrid.frame(i)), got "
                           f"{type(deformation).__name__}")
    if net.ray_bender[0] is None:
        raise RuntimeError("nonrigid_nerf_b200: a baked deformation needs a model with a ray bender (its rays that leave the grid are "
                           "bent by it)")
    deformation.c_struct(net.output_linear.weight.device)


def field_baked(net, rays, z_vals, latents, want_details, grid, deformation=None):
    """field_rays that samples the radiance grid in place of the NeRF trunk for samples inside its box; with `deformation`
    (geometry.FrameDeformation) the bends of the rays inside its box come from that grid in place of the ray bender."""
    baked_check(net, latents, grid)
    cutoff, scaling, removal, nerf_pack, bender_pack, out_ch = _packs(net)
    if deformation is not None:
        deformation_check(net, deformation)
        return ops.field_forward_deformed(rays, z_vals, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details,
                                          grid, deformation)
    return ops.field_forward_baked(rays, z_vals, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details, grid)


def termination_threshold(threshold) -> float:
    """The early-termination threshold as a float; raises unless it is a finite real number in [0, 1] (not a bool or a
    tensor)."""
    if isinstance(threshold, (bool, np.bool_, torch.Tensor)) or not isinstance(threshold, numbers.Real):
        raise RuntimeError(f"nonrigid_nerf_b200: early_termination must be a real number in [0, 1], got {type(threshold).__name__}")
    t = float(threshold)
    if not (0.0 <= t <= 1.0):
        raise RuntimeError(f"nonrigid_nerf_b200: early_termination must be a finite real number in [0, 1], got {t!r}")
    return t


def termination_check(net, latents, threshold) -> float:
    """Raise, before any launch, for what render(..., early_termination=t) does not support: a threshold that is not a
    finite real in [0, 1], the view-dependent head, the time-conditioned baseline and differentiable calls.  Returns t."""
    t = termination_threshold(threshold)
    _skip_check(net, latents, "with early_termination", "samples that are not evaluated would get no gradient")
    return t


def field_terminate(net, rays, z_vals, latents, want_details, threshold, grid=None, noise=None):
    """field_rays with early ray termination (and, with `grid`, the occupancy grid's skipping): raw is 0 for samples not
    evaluated.  Returns (raw, details, termination_index)."""
    t = termination_check(net, latents, threshold)
    if grid is not None:
        occupancy_check(net, latents, grid)
    cutoff, scaling, removal, nerf_pack, bender_pack, out_ch = _packs(net)
    return ops.field_forward_terminate(rays, z_vals, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details, t,
                                       grid, noise)


def field_rays(net, rays, z_vals, latents, want_details):
    """Inference path (no stash)."""
    cutoff, scaling, removal, nerf_pack, bender_pack, out_ch = _packs(net)
    return ops.field_forward(rays, z_vals, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details,
                             tc_net=_tc_net(net))


def field_points(net, pts, latents, want_details):
    """NeRF.forward(x) semantics: one xyz (+ latent) per row.  Inference only."""
    if getattr(net, "use_viewdirs", False):
        raise RuntimeError("nonrigid_nerf_b200: a use_viewdirs=True model is evaluated point-wise by field_views")
    _tc_net(net)
    if _needs_grad(net, latents):
        raise RuntimeError("nonrigid_nerf_b200: the point-wise NeRF.forward / run_network entry is inference-only; "
                           "differentiable rendering goes through render() / render_rays()")
    cutoff, scaling, removal, nerf_pack, bender_pack, out_ch = _packs(net)
    return ops.field_forward_points(pts, latents, nerf_pack, bender_pack, out_ch, cutoff, scaling, removal, want_details,
                                    tc_net=_tc_net(net))


def composite(raw, z_vals, rays_d, noise=None, white_bkgd=False, n_importance=0, u=None) -> Dict[str, torch.Tensor]:
    """raw2outputs (+ hierarchical resampling); differentiable w.r.t. raw through rgb_map / acc_map."""
    if torch.is_grad_enabled() and raw.requires_grad:
        outs = _CompositeFn.apply(raw, z_vals, rays_d, noise, white_bkgd, n_importance, u)
        keys = ["rgb_map", "acc_map", "disp_map", "depth_map", "weights", "alpha"] + (["z_vals_out", "z_std"] if n_importance > 0 else [])
        return dict(zip(keys, outs))
    return ops.composite(raw, z_vals, rays_d, noise, white_bkgd, n_importance, u, True)
