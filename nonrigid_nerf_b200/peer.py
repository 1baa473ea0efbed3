"""Peer-memory gradient reduction (csrc/peer.cu): the H100-native replacement of DataParallel's gradient reduce + Adam.

One process per GPU on one NVSwitch node.  Every rank's gradient arena lives in a CUDA-IPC window the other ranks map;
`optimizer.step()` becomes ONE fused sequence of plain kernels that reads the peers' arenas over NVLink while summing them
and applies Adam -- no NCCL call, no staging copy, capturable in a CUDA graph together with the rest of the iteration.
torch.distributed is used only for the plumbing (exchanging the 64-byte IPC handles, barriers at set-up / tear-down).

    opt = optim.Adam(grad_vars, lr=5e-4)
    train_fn = parallel.get_parallelized_training_function(coarse, latents, fine, bender)
    parallel.attach_optimizer(opt, peer.PeerArenaReducer(opt))      # instead of the default NCCL all-reduce
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch
import torch.distributed as dist

from . import _lib


class _DeviceBuffer:
    """CUDA array interface over a raw device pointer (memory owned by the library, not by PyTorch)."""

    def __init__(self, ptr: int, n_floats: int):
        self.__cuda_array_interface__ = {"shape": (n_floats,), "typestr": "<f4", "data": (ptr, False), "version": 3, "strides": None}


class PeerArenaReducer:
    fused_adam = True

    def __init__(self, optimizer, slot_floats: int = 1 << 16):
        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("nonrigid_nerf_b200.peer: torch.distributed must be initialised (one process per GPU)")
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        if self.world > 8:
            raise RuntimeError("nonrigid_nerf_b200.peer: at most 8 ranks (one NVSwitch node)")
        lib = _lib.load()
        self._lib = lib
        dev = optimizer._dev
        self._dev = dev
        total = optimizer._total
        self.slot_floats = int(slot_floats)
        nbytes = lib.nrn_peer_window_bytes(total, self.slot_floats)
        own = C.c_void_p()
        handle = C.create_string_buffer(64)
        # every phase that can fail is followed by an exchange of the outcome, so that either ALL ranks get a reducer or ALL
        # ranks raise (a rank that failed alone would leave the others waiting in a collective)
        err = None
        try:
            with torch.cuda.device(dev):
                _lib.check(lib.nrn_peer_alloc(nbytes, C.byref(own), handle), "peer_alloc")
        except RuntimeError as exc:
            err = str(exc)
        self._own = own.value
        infos = [None] * self.world
        dist.all_gather_object(infos, (err, bytes(handle.raw)))
        if any(e is not None for e, _ in infos):
            raise RuntimeError("nonrigid_nerf_b200.peer: window allocation failed: " + "; ".join(f"rank {r}: {e}" for r, (e, _) in enumerate(infos) if e))
        handles = [h for _, h in infos]
        self._mapped = [None] * self.world
        ctx = _lib.NrnPeerCtx()
        err = None
        for r in range(self.world):
            if r == self.rank:
                ctx.window[r] = self._own
                continue
            p = C.c_void_p()
            try:
                with torch.cuda.device(dev):
                    _lib.check(lib.nrn_peer_open(handles[r], C.byref(p)), f"peer_open(rank {r})")
            except RuntimeError as exc:
                err = str(exc)
                break
            self._mapped[r] = p.value
            ctx.window[r] = p.value
        errs = [None] * self.world
        dist.all_gather_object(errs, err)
        if any(e is not None for e in errs):
            raise RuntimeError("nonrigid_nerf_b200.peer: mapping the peers' windows failed: " + "; ".join(f"rank {r}: {e}" for r, e in enumerate(errs) if e))
        ctx.world, ctx.rank, ctx.arena_floats, ctx.slot_floats = self.world, self.rank, total, self.slot_floats
        self._state = torch.zeros(4, dtype=torch.int32, device=dev)
        self._reduced = torch.empty(max(total, 1), dtype=torch.float32, device=dev)
        ctx.state, ctx.reduced = self._state.data_ptr(), self._reduced.data_ptr()
        self._ctx = ctx
        slot_bytes = (self.slot_floats * 4 + 255) // 256 * 256
        arena_ptr = self._own + 1024 + 2 * slot_bytes
        self._arena_holder = _DeviceBuffer(arena_ptr, total)
        arena = torch.as_tensor(self._arena_holder, device=dev)
        optimizer.rebind_arena(arena)
        torch.cuda.synchronize(dev)
        dist.barrier()          # every window is mapped everywhere before the first flag is written
        self._closed = False

    # -- optimizer hook: the whole step (reduce + Adam) in the fused kernels -------------------------------------
    def step(self, optimizer, adam_args) -> bool:
        with torch.cuda.device(self._dev):
            _lib.check(self._lib.nrn_peer_reduce_adam(C.byref(self._ctx), C.byref(adam_args)), "peer_reduce_adam")
        return True

    def gather_rows(self, local: torch.Tensor) -> torch.Tensor:
        """All-gather of a small fp32 tensor with the same number of elements on every rank -> [world * n] (rank order)."""
        local = local.detach().contiguous().float()
        n = local.numel()
        out = torch.empty(self.world * n, dtype=torch.float32, device=local.device)
        with torch.cuda.device(self._dev):
            _lib.check(self._lib.nrn_peer_gather_rows(C.byref(self._ctx), C.c_void_p(local.data_ptr()), n, C.c_void_p(out.data_ptr()),
                                                      C.c_void_p(torch.cuda.current_stream().cuda_stream)), "peer_gather_rows")
        return out

    def close(self) -> None:
        if self._closed:
            return
        self._closed = True
        torch.cuda.synchronize(self._dev)
        if dist.is_initialized():
            dist.barrier()      # nobody unmaps while a peer may still read
        for p in self._mapped:
            if p is not None:
                self._lib.nrn_peer_close(C.c_void_p(p))
        if dist.is_initialized():
            dist.barrier()
        # the arena tensor handed to the optimizer aliases the window: it is deliberately leaked rather than freed under
        # live .grad views when the process is about to exit anyway


def reducer_for(optimizer) -> Optional[PeerArenaReducer]:
    r = getattr(optimizer, "_reducer", None)
    return r if isinstance(r, PeerArenaReducer) else None
