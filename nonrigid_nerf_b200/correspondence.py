"""Pixel correspondences between rendered frames through the canonical volume, on the GPU.

render(..., surface_output=True) gives every pixel of a frame its canonical surface point (train.py:159-176), and
free_viewpoint_rendering.py:615-645 paints those points as a checkerboard in which equal colours mean the same scene
point.  match_frames() turns them into correspondences: for each pixel of a query frame, the pixel of a target frame whose
canonical point is nearest, the pixel flow to it, and optionally whether matching back lands where it started (the usual
occlusion test).  The answer is the brute-force one, bit for bit (csrc/match.cu describes the search).

Like evaluation.py, it takes CUDA tensors, enqueues its kernels on the current stream, allocates outputs and workspace
through PyTorch's allocator and never synchronises, so it can be captured in a CUDA graph.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple, Optional

import torch

from . import _lib
from .ops import _stream

MAX_SIDE = 1 << 24          # frame height and width at most (pixel coordinates exact in fp32)
MAX_POINTS = 2 ** 31 - 1    # pixels of one frame at most (point indices are int32)
MAX_FRAMES = 65535


class Correspondences(NamedTuple):
    index: torch.Tensor                   # [F, Hq, Wq] int32: y * Wt + x of the matched target pixel, or -1
    distance: torch.Tensor                # [F, Hq, Wq] fp32: canonical distance to the match, +inf where index == -1
    flow: torch.Tensor                    # [F, Hq, Wq, 2] fp32: (x_t - x_q, y_t - y_q) in pixels, NaN where index == -1
    consistent: Optional[torch.Tensor]    # [F, Hq, Wq] bool (round_trip=True): the match matches back within tolerance


def _points(t: torch.Tensor, name: str, size) -> tuple:
    if not isinstance(t, torch.Tensor):
        raise RuntimeError(f"nonrigid_nerf_b200: {name} must be a CUDA tensor (there is no CPU path)")
    if t.dim() == 4 and t.shape[-1] == 3:
        f, h, w = t.shape[:3]
        if size is not None and tuple(size) != (h, w):
            raise RuntimeError(f"nonrigid_nerf_b200: {name} is {tuple(t.shape)}, not frames of {tuple(size)}")
    elif t.dim() == 3 and t.shape[-1] == 3:
        if size is None:
            raise RuntimeError(f"nonrigid_nerf_b200: {name} of shape [F, H*W, 3] needs its frame size (H, W)")
        h, w = (int(v) for v in size)
        f = t.shape[0]
        if h * w != t.shape[1]:
            raise RuntimeError(f"nonrigid_nerf_b200: {name} holds {t.shape[1]} points per frame, not {h} x {w}")
    else:
        raise RuntimeError(f"nonrigid_nerf_b200: {name} must be [F, H, W, 3] or [F, H*W, 3], got {tuple(t.shape)}")
    if h < 1 or w < 1 or h > MAX_SIDE or w > MAX_SIDE or h * w > MAX_POINTS:
        raise RuntimeError(f"nonrigid_nerf_b200: {name} frames of {h} x {w} pixels: height and width must be 1 to {MAX_SIDE} "
                           f"and a frame at most {MAX_POINTS} pixels")
    if f > MAX_FRAMES:
        raise RuntimeError(f"nonrigid_nerf_b200: {name} has {f} frames, at most {MAX_FRAMES} are supported")
    return t, f, h, w


def _mask(m, name: str, f: int, h: int, w: int, dev):
    if m is None:
        return None
    if not isinstance(m, torch.Tensor) or tuple(m.shape) not in ((f, h, w), (f, h * w)) or m.device != dev:
        got = tuple(m.shape) if isinstance(m, torch.Tensor) else type(m)
        raise RuntimeError(f"nonrigid_nerf_b200: {name} must be [{f}, {h}, {w}] or [{f}, {h * w}] on {dev}, got {got}")
    return (m != 0).to(torch.uint8).contiguous()


def workspace_bytes(fq: int, hq: int, wq: int, ft: int, ht: int, wt: int, round_trip: bool) -> int:
    """Bytes of device workspace match_frames uses for these frame stacks (nrn_match_workspace_bytes); 0 when out of range."""
    return int(_lib.load().nrn_match_workspace_bytes(fq, hq, wq, ft, ht, wt, 1 if round_trip else 0))


def match_frames(query: torch.Tensor, target: torch.Tensor, query_mask: Optional[torch.Tensor] = None,
                 target_mask: Optional[torch.Tensor] = None, max_distance: float = math.inf, round_trip: bool = False,
                 round_trip_pixels: float = 1.0, *, size=None, target_size=None) -> Correspondences:
    """Match every pixel of the query frames to the target pixel with the nearest canonical surface point.

    query [Fq, Hq, Wq, 3] and target [Ft, Ht, Wt, 3] are canonical surface points (surface_pts of
    render(..., surface_output=True)), or [F, H*W, 3] as surface_pts stacks, with size=(Hq, Wq) (and target_size=(Ht, Wt)
    when the target frames differ).  Frame k is matched against frame k (Fq == Ft), one query frame against every target
    frame (Fq == 1) or every query frame against one target frame (Ft == 1).  query_mask / target_mask [F, H, W] (or
    [F, H*W]) mark the pixels that have a surface (False: none; e.g. acc_map > 0.5); a point with a non-finite coordinate
    counts as masked.  A pixel is matched when its nearest valid target point lies within max_distance (canonical units);
    the nearest is the smallest d2 = (dx*dx + dy*dy) + dz*dz in fp32, ties going to the smaller target index.
    round_trip=True also matches each matched target pixel back against its query frame: `consistent` is True where that
    lands within round_trip_pixels (Euclidean) of the query pixel, False where it does not or there is no match."""
    query, fq, hq, wq = _points(query, "query", size)
    target, ft, ht, wt = _points(target, "target", size if target_size is None else target_size)
    dev = query.device
    if target.device != dev:
        raise RuntimeError(f"nonrigid_nerf_b200: query is on {dev}, target on {target.device}")
    if not (fq == ft or fq == 1 or ft == 1):
        raise RuntimeError(f"nonrigid_nerf_b200: {fq} query frames do not pair with {ft} target frames "
                           "(equal counts, or one frame on either side)")
    max_distance = float(max_distance)
    if not max_distance >= 0.0:
        raise RuntimeError(f"nonrigid_nerf_b200: max_distance must be >= 0, got {max_distance}")
    round_trip_pixels = float(round_trip_pixels)
    if round_trip and not round_trip_pixels >= 0.0:
        raise RuntimeError(f"nonrigid_nerf_b200: round_trip_pixels must be >= 0, got {round_trip_pixels}")
    qm = _mask(query_mask, "query_mask", fq, hq, wq, dev)
    tm = _mask(target_mask, "target_mask", ft, ht, wt, dev)
    if not query.is_cuda:
        raise RuntimeError("nonrigid_nerf_b200: match_frames takes CUDA tensors (there is no CPU path)")
    query, target = query.float().contiguous(), target.float().contiguous()
    f = fq if (fq == ft or ft == 1) else ft
    index = torch.empty((f, hq, wq), dtype=torch.int32, device=dev)
    distance = torch.empty((f, hq, wq), dtype=torch.float32, device=dev)
    flow = torch.empty((f, hq, wq, 2), dtype=torch.float32, device=dev)
    consistent = torch.empty((f, hq, wq), dtype=torch.bool, device=dev) if round_trip else None
    if f == 0:
        return Correspondences(index, distance, flow, consistent)
    lib = _lib.load()
    ws_bytes = workspace_bytes(fq, hq, wq, ft, ht, wt, round_trip)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    a = _lib.NrnMatchArgs()
    a.query, a.target = query.data_ptr(), target.data_ptr()
    a.query_mask, a.target_mask = (None if m is None else m.data_ptr() for m in (qm, tm))
    a.n_query_frames, a.query_height, a.query_width = fq, hq, wq
    a.n_target_frames, a.target_height, a.target_width = ft, ht, wt
    a.max_distance, a.round_trip, a.round_trip_pixels = max_distance, 1 if round_trip else 0, round_trip_pixels
    a.index, a.distance, a.flow = index.data_ptr(), distance.data_ptr(), flow.data_ptr()
    a.consistent = None if consistent is None else consistent.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws_bytes
    with torch.cuda.device(dev):
        a.stream = _stream().value
        _lib.check(lib.nrn_match(C.byref(a)), "match_frames")
    return Correspondences(index, distance, flow, consistent)
