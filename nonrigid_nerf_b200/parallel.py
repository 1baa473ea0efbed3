"""Ray-sharded multi-GPU execution: the replacement of torch.nn.DataParallel in the reference
(train.py:290-297, :320-323; call sites train.py:1566-1577 and :473-480).

One process per GPU (torchrun), `torch.distributed` with the NCCL backend.  The callables returned by
get_parallelized_{training,render}_function keep DataParallel's calling convention (SURVEY.md
appendix D): every tensor argument whose leading dimension is the ray count is split along dim 0
(tensors nested in dicts / lists / tuples too), everything else is passed by reference, and the
outputs are concatenated along dim 0 -- here with an all-gather, so that EVERY rank holds the full
result and can keep executing the unmodified training loop in lock-step.

Collectives on the path (SURVEY.md section 8e):
  * inputs: one broadcast of the step's ray batch from rank 0 (ranks sample with unseeded numpy in
    the reference, train.py:1546-1564; <= 3 MB), then each rank takes rows [r*ceil(N/G), (r+1)*ceil(N/G))
  * outputs: all-gather of the per-ray losses [N] (training) or of the rendered maps (inference)
  * gradients: ONE flat fp32 all-reduce (SUM) per optimizer step, issued from an optimizer
    pre-step hook, i.e. after every backward pass of the iteration (the reference runs two when test
    latents are optimised, train.py:1595-1608) has accumulated into .grad.
Weights stay replicated; Adam runs identically on every rank.
With world_size == 1 (or torch.distributed not initialised) the wrappers call straight through.
"""
from __future__ import annotations

import weakref
from typing import Any, Callable, List, Optional

import torch
import torch.distributed as dist

from . import autograd as _ag
from . import train as T


# ---------------------------------------------------------------------------------------------
# distributed plumbing
# ---------------------------------------------------------------------------------------------
def _world() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _rank() -> int:
    return dist.get_rank() if _world() > 1 else 0


def shard_bounds(n: int, world: int, rank: int):
    """DataParallel-style chunking: ceil(n / world) rows per rank, trailing ranks may get fewer/none."""
    per = (n + world - 1) // world
    lo = min(rank * per, n)
    return lo, min(lo + per, n)


def _map_tensors(obj: Any, fn: Callable[[torch.Tensor], Any]) -> Any:
    """Apply fn to every tensor nested in dicts / lists / tuples.  Containers without tensors are returned
    as the SAME object (DataParallel passes non-tensor arguments by reference)."""
    if isinstance(obj, torch.Tensor):
        return fn(obj)
    if isinstance(obj, dict):
        new = {k: _map_tensors(v, fn) for k, v in obj.items()}
        return obj if all(new[k] is obj[k] for k in obj) else new
    if isinstance(obj, (tuple, list)):
        new = [_map_tensors(v, fn) for v in obj]
        if all(a is b for a, b in zip(new, obj)):
            return obj
        return tuple(new) if isinstance(obj, tuple) else new
    return obj


def _first_tensor(obj: Any) -> Optional[torch.Tensor]:
    if isinstance(obj, torch.Tensor):
        return obj
    if isinstance(obj, dict):
        obj = list(obj.values())
    if isinstance(obj, (list, tuple)):
        for v in obj:
            t = _first_tensor(v)
            if t is not None:
                return t
    return None


class _AllGatherRows(torch.autograd.Function):
    """Concatenate per-rank row blocks (uneven allowed).  Backward: this rank's slice of the incoming
    gradient -- every rank evaluates the same scalar loss on the gathered tensor, so no communication
    is needed there; parameter gradients are summed later by the optimizer pre-step hook."""

    @staticmethod
    def forward(ctx, local: torch.Tensor, n_total: int):
        world, rank = _world(), _rank()
        per = (n_total + world - 1) // world
        lo, hi = shard_bounds(n_total, world, rank)
        ctx.bounds = (lo, hi)
        pad = local.new_zeros((per,) + tuple(local.shape[1:]))
        pad[: hi - lo] = local
        out = local.new_empty((world * per,) + tuple(local.shape[1:]))
        dist.all_gather_into_tensor(out, pad.contiguous()) if hasattr(dist, "all_gather_into_tensor") and local.is_cuda else \
            _all_gather_list(out, pad, world)
        return out[:n_total]

    @staticmethod
    def backward(ctx, grad):
        lo, hi = ctx.bounds
        return grad[lo:hi].contiguous(), None


def _all_gather_list(out, pad, world):
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad.contiguous())
    out.copy_(torch.cat(parts, 0))


def all_reduce_gradients(params: List[torch.Tensor]) -> None:
    """One flat SUM all-reduce over the gradients of `params` (None gradients travel as zeros; a
    per-parameter presence flag rides in the same buffer so that a gradient that is None on every
    rank -- e.g. the dead views_linears, SURVEY.md 7.3-6 -- stays None)."""
    if _world() == 1:
        return
    params = [p for p in params if p.requires_grad]
    if not params:
        return
    dev = params[0].device
    if UNIFORM_GRADS or (dev.type == "cuda" and torch.cuda.is_current_stream_capturing()):
        # inside a CUDA-graph capture no host read-back is possible: gradients that are None must be None on
        # every rank (true for this path: the same graph runs everywhere), so only the present ones travel
        live = [p for p in params if p.grad is not None]
        flat = torch.cat([p.grad.reshape(-1) for p in live])          # one gather kernel
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)                    # ONE collective over every gradient
        views, o = [], 0
        for p in live:
            n = p.numel()
            views.append(flat[o:o + n].view_as(p))
            o += n
        torch._foreach_copy_([p.grad for p in live], views)            # one multi-tensor scatter back
        return
    chunks = [(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1).float() for p in params]
    flags = torch.tensor([0.0 if p.grad is None else 1.0 for p in params], dtype=torch.float32, device=dev)
    flat = torch.cat(chunks + [flags])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    o = 0
    flags = flat[-len(params):]
    present = (flags > 0).tolist()
    for p, here in zip(params, present):
        n = p.numel()
        if here:
            g = flat[o:o + n].view_as(p).to(p.dtype)
            if p.grad is None:
                p.grad = g.clone()
            else:
                p.grad.copy_(g)
        o += n


_HOOK_INSTALLED = False
_SHARDED_PARAMS: dict = {}   # id(tensor) -> weak reference, for every tensor a ray-sharded training function differentiates
                             # (the reference is checked: a recycled id() of a freed model can never enrol an unrelated optimizer)
UNIFORM_GRADS = False   # True: a gradient that is None on one rank is None on all (skips the presence flags + host sync)


def _register_sharded_params(params) -> None:
    for k in [k for k, r in _SHARDED_PARAMS.items() if r() is None]:
        del _SHARDED_PARAMS[k]
    for p in params:
        _SHARDED_PARAMS[id(p)] = weakref.ref(p)


def _owns_sharded_params(optimizer) -> bool:
    """Only an optimizer that steps parameters of a ray-sharded training function takes part in the gradient
    all-reduce.  Any other optimizer in the process (a CPU baseline, a user's second model) is left alone."""
    for g in optimizer.param_groups:
        for p in g["params"]:
            ref = _SHARDED_PARAMS.get(id(p))
            if ref is not None and ref() is p:
                return True
    return False


class NcclArenaReducer:
    """In-place SUM all-reduce over an optim.Adam gradient arena: ONE collective over ONE persistent buffer whose views
    are the parameters' .grad tensors (no gather before, no scatter after)."""

    fused_adam = False

    def step(self, optimizer, adam_args) -> bool:
        if _world() > 1:
            dist.all_reduce(optimizer.gradient_arena(), op=dist.ReduceOp.SUM)
        return False        # the optimizer launches its Adam kernel on the reduced arena


def attach_optimizer(optimizer, reducer=None) -> None:
    """Tell an nonrigid_nerf_b200.optim.Adam that its parameters are trained ray-sharded: its step() then reduces the
    gradient arena across ranks itself.  Called automatically (with the NCCL reducer) from the optimizer hook the first
    time such an optimizer steps; call it explicitly to install another reducer (peer.PeerArenaReducer)."""
    if hasattr(optimizer, "gradient_arena"):
        optimizer._reducer = reducer if reducer is not None else NcclArenaReducer()


def _install_optimizer_hook() -> None:
    """Optimizer pre-step hook (the reference builds its optimizer before it builds the parallel wrappers and never
    hands it over, train.py:656-658 vs :1455-1461, so the hook cannot be attached to one instance): all-reduce the
    gradients of an optimizer that owns the sharded parameters; every other optimizer passes through untouched."""
    global _HOOK_INSTALLED
    if _HOOK_INSTALLED:
        return
    from torch.optim.optimizer import register_optimizer_step_pre_hook

    def hook(optimizer, args, kwargs):
        if _world() == 1 or not _owns_sharded_params(optimizer):
            return
        if hasattr(optimizer, "gradient_arena") and getattr(optimizer, "_reducer", None) is None:
            attach_optimizer(optimizer)
        if not getattr(optimizer, "reduces_gradients_itself", False):
            all_reduce_gradients([p for g in optimizer.param_groups for p in g["params"]])

    register_optimizer_step_pre_hook(hook)
    _HOOK_INSTALLED = True


class RayShardedFunction:
    """Callable with nn.DataParallel's scatter / gather convention over torch.distributed ranks."""

    def __init__(self, module: Callable, broadcast_inputs: bool = True):
        self.module = module
        self.broadcast_inputs = broadcast_inputs

    def __call__(self, *args, **kwargs):
        world, rank = _world(), _rank()
        if world == 1:
            return self.module(*args, **kwargs)
        lead = _first_tensor(args)
        if lead is None:
            lead = _first_tensor(kwargs)
        if lead is None:
            raise RuntimeError("RayShardedFunction: no tensor argument to shard")
        n = lead.shape[0]
        lo, hi = shard_bounds(n, world, rank)

        def shard(t: torch.Tensor):
            if t.dim() == 0 or t.shape[0] != n:
                return t
            # host tensors cannot travel over an NCCL-only group: they are taken as identical on every rank
            if self.broadcast_inputs and not t.requires_grad and (t.is_cuda or dist.get_backend() != "nccl"):
                t = t.contiguous()
                dist.broadcast(t, src=0)
            return t[lo:hi]

        out = self.module(*_map_tensors(args, shard), **_map_tensors(kwargs, shard))
        return _map_tensors(out, lambda t: _AllGatherRows.apply(t, n))


# ---------------------------------------------------------------------------------------------
# the modules DataParallel used to wrap (train.py:140-287, :300-317)
# ---------------------------------------------------------------------------------------------
class training_wrapper_class(torch.nn.Module):
    """Per-rank training step: latent lookup, render, data term and regularisers -> per-ray loss [N].
    Mirrors training_wrapper_class.forward (train.py:152-287) argument for argument."""

    def __init__(self, coarse_model, latents, fine_model=None, ray_bender=None):
        super().__init__()
        self.coarse_model = coarse_model
        self.latents = latents            # python list of leaf tensors [Z] (train.py:1448-1453)
        self.fine_model = fine_model
        self.ray_bender = ray_bender

    def forward(self, args, rays_o, rays_d, i, render_kwargs_train, target_s, global_step, start, dataset_extras,
                batch_pixel_indices, held_out=None):
        """held_out [N] (bool or uint8, on the rays' device): rays of held-out frames (test_block_size, train.py:1376-1395),
        whose loss reaches only their latent codes with a ray bender and nothing without one, so that one
        ((train + test) * loss).mean().backward() with held_out=test gives the gradients of the reference's two backward
        passes (train.py:1595-1608)."""
        # the view-dependent head cannot be trained with a bender yet: raise before any launch, for the bender seated below
        for net in (self.coarse_model, self.fine_model):
            if net is not None:
                _ag.views_check(net, bender=self.ray_bender)
        if held_out is not None:
            _ag.check_held_out(held_out, rays_o.shape[0], target_s.device)
        self.coarse_model.ray_bender = (self.ray_bender,)
        render_kwargs_train["network_fn"] = self.coarse_model
        render_kwargs_train["ray_bender"] = self.ray_bender
        if self.fine_model is not None:
            self.fine_model.ray_bender = (self.ray_bender,)
            render_kwargs_train["network_fine"] = self.fine_model
        dev = target_s.device
        key = tuple(dataset_extras["imageid_to_timestepid"])
        if getattr(self, "_i2t", (None, None))[0] != (key, dev):   # one H2D copy, not one per step (train.py:178-180)
            self._i2t = ((key, dev), torch.as_tensor(dataset_extras["imageid_to_timestepid"], device=dev))
        imageid_to_timestepid = self._i2t[1]
        timestep = imageid_to_timestepid[batch_pixel_indices[:, 0].to(dev).long()]
        # [N, Z] per-ray latents (train.py:173-189).  The per-frame latents are read in place (they are views of the
        # optimizer's flat buffer) and their gradient is one index_add_ into the .grad arena.
        info = {"ray_bending_latents": _ag.gather_latents(self.latents, timestep)}
        detailed = args.offsets_loss_weight > 0.0 or args.divergence_loss_weight > 0.0
        rgb, disp, acc, extras = T.render(rays_o, rays_d, chunk=args.chunk, verbose=i < 10, retraw=True,
                                          additional_pixel_information=info, detailed_output=detailed, held_out=held_out,
                                          **render_kwargs_train)
        # increasing schedule of the regularisers, (1/100)^(1 - global_step / N_iters) (train.py:229, :281).  `global_step` may be
        # a 0-dim CUDA tensor: the schedule is then evaluated inside the loss kernel, so a step captured in a CUDA graph
        # follows it when replayed.
        if isinstance(global_step, torch.Tensor):
            sched, sched_step = 1.0, global_step
        else:
            sched, sched_step = (1.0 / 100.0) ** (1 - (global_step / args.N_iters)), None
        use_offsets = self.ray_bender is not None and args.offsets_loss_weight > 0.0
        div = None
        if self.ray_bender is not None and args.divergence_loss_weight > 0.0:
            # exact_divergence = False, backprop_into_weights = False (train.py:246-247); fused closed-form kernels; the weights
            # 1 - exp(-relu(opacity_alpha)) (train.py:267) are formed inside them.  Hutchinson probes: torch.randn like
            # run_nerf_helpers.py:110, or injected with the other random draws (render_kwargs_train["randomness"]["e"],
            # [N, N_samples, 3] or [N * N_samples, 3]) for exact reproduction
            rnd = render_kwargs_train.get("randomness")
            probes = rnd.get("e") if isinstance(rnd, dict) else None
            div = _ag.divergence_loss(extras["unmasked_offsets"], extras["rigidity_mask"], None, self.ray_bender,
                                      e=None if probes is None else probes.to(dev).reshape(-1, 3), opacity_alpha=extras["opacity_alpha"],
                                      held_out=held_out)
        # data term (fine + coarse), offsets / rigidity regulariser (train.py:208-242) and the weighted divergence term
        # (train.py:278-286) in one fused kernel
        loss = _ag.ray_loss(rgb, extras.get("rgb0"), target_s,
                            extras["visibility_weights"] if use_offsets else None,
                            extras["unmasked_offsets"] if use_offsets else None,
                            extras["rigidity_mask"] if use_offsets else None,
                            args.offsets_loss_weight * sched if use_offsets else 0.0, args.rigidity_loss_weight,
                            sched_step, float(args.N_iters), div, args.divergence_loss_weight * sched)
        return loss


class render_wrapper_class(torch.nn.Module):
    """train.render with the wrapped models; every keyword (held_out, occupancy, early_termination, baked, ...) is passed
    on.  An occupancy grid, an early-termination threshold and a baked scene reach every rank whole: none is a tensor or a
    tuple, so RayShardedFunction does not shard them."""

    def __init__(self, coarse_model, fine_model=None, ray_bender=None):
        super().__init__()
        self.coarse_model, self.fine_model, self.ray_bender = coarse_model, fine_model, ray_bender

    def forward(self, *args, **kwargs):
        self.coarse_model.ray_bender = (self.ray_bender,)
        kwargs["network_fn"] = self.coarse_model
        kwargs["ray_bender"] = self.ray_bender
        if self.fine_model is not None:
            self.fine_model.ray_bender = (self.ray_bender,)
            kwargs["network_fine"] = self.fine_model
        return T.render(*args, **kwargs)


def get_parallelized_training_function(coarse_model, latents, fine_model=None, ray_bender=None):
    _register_sharded_params(list(latents) + list(coarse_model.parameters())
                             + (list(fine_model.parameters()) if fine_model is not None else [])
                             + (list(ray_bender.parameters()) if ray_bender is not None else []))
    _install_optimizer_hook()
    return RayShardedFunction(training_wrapper_class(coarse_model, latents, fine_model=fine_model, ray_bender=ray_bender))


def get_parallelized_render_function(coarse_model, fine_model=None, ray_bender=None):
    return RayShardedFunction(render_wrapper_class(coarse_model, fine_model=fine_model, ray_bender=ray_bender))
