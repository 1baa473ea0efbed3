"""CUDA-graph capture of a whole training iteration.

At N_rand = 1024 the fused kernels need ~2 ms per step, but an iteration also launches several hundred
tiny PyTorch kernels (loss arithmetic, the double-backward divergence regulariser, per-latent gradient
accumulation, Adam): launch-bound.  Capturing forward + backward + optimizer step once and replaying the
graph removes the host from the loop ("CUDA streams and graphs instead of a tracing compiler").
Everything the eager step does is still executed by every replay, including the weight re-packing kernels.
"""
from __future__ import annotations

from typing import Callable, Sequence

import torch

from . import ops


class GraphedStep:
    """`fn(*tensors) -> tensor(s)` captured once; call with new input tensors of the same shapes.
    Requirements on `fn`: no host synchronisation, optimizers constructed with capturable=True, and
    `optimizer.zero_grad(set_to_none=True)` before `backward()` inside `fn` (PyTorch's whole-network
    capture recipe).  Python scalars used inside `fn` are frozen at capture time."""

    def __init__(self, fn: Callable, example_inputs: Sequence[torch.Tensor], warmup: int = 3):
        self.static_inputs = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                fn(*self.static_inputs)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        ops.FORCE_PACK = True
        try:
            with torch.cuda.graph(self.graph):
                self.static_out = fn(*self.static_inputs)
        finally:
            ops.FORCE_PACK = False

    def __call__(self, *inputs: torch.Tensor):
        """Replay with new inputs (device tensors, or pinned host tensors: those are copied straight into the graph's input
        buffers, one H2D copy each and no intermediate device tensor)."""
        for s, t in zip(self.static_inputs, inputs):
            if s.data_ptr() != t.data_ptr():
                s.copy_(t, non_blocking=True)
        self.graph.replay()
        return self.static_out
