"""Scores and images of rendered frames on the GPU: what free_viewpoint_rendering.py computes on the host with numpy,
scikit-image and matplotlib once the frames are rendered (PSNR, SSIM and the error images of :786-876, the jet and
Blinn-Phong disparity images of :725-745 / run_nerf_helpers.py:701-793, the background-stability map of :770-785, and
the uint8 images and videos it saves, :615-766).

Every function takes CUDA tensors, enqueues its kernels on the current stream, allocates its outputs and workspace
through PyTorch's allocator and never synchronises, so it can be captured in a CUDA graph.  Colours index matplotlib's
256-entry cm.jet table (`jet_colormap()`) as the reference does.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import _lib
from .ops import _ptr, _stream


class ImageScores(NamedTuple):
    psnr: torch.Tensor                    # [F] fp32
    ssim: torch.Tensor                    # [F] fp32
    ssim_map: Optional[torch.Tensor]      # [F, H, W, 3] fp32, the SSIM map S (ssim_map=True)
    error_rgb: Optional[torch.Tensor]     # [F, H, W, 3] uint8 (error_maps=True)
    error_ssim: Optional[torch.Tensor]    # [F, H, W, 3] uint8 (error_maps=True)


class FrameImages(NamedTuple):
    """The uint8 images free_viewpoint_rendering.py saves (:660-766); None where the input is missing."""
    rgb: Optional[torch.Tensor]               # [F, H, W, 3] to8b(rgb)
    disp: Optional[torch.Tensor]              # [F, H, W]    each frame divided by its maximum
    disp_video: Optional[torch.Tensor]        # [F, H, W]    divided by the maximum over all frames (video_disp.mp4)
    disp_jet: Optional[torch.Tensor]          # [F, H, W, 3]
    disp_phong: Optional[torch.Tensor]        # [F, H, W, 3] (None for frames with fewer than 2 rows or columns)
    correspondences: Optional[torch.Tensor]   # [F, H, W, 3] the 100-voxel checkerboard of the canonical point
    rigidity: Optional[torch.Tensor]          # [F, H, W]
    rigidity_jet: Optional[torch.Tensor]      # [F, H, W, 3]


def _frames(t: torch.Tensor, name: str, ndim: int) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"nonrigid_nerf_b200: {name} must be a CUDA tensor (there is no CPU path)")
    if t.dim() != ndim or (ndim == 4 and t.shape[-1] != 3):
        shape = "[F, H, W, 3]" if ndim == 4 else "[F, H, W]"
        raise RuntimeError(f"nonrigid_nerf_b200: {name} must be {shape}, got {tuple(t.shape)}")
    return t.float().contiguous()


def jet_colormap() -> np.ndarray:
    """matplotlib's cm.jet table as the kernels use it: [256, 3] float64, cm.jet(i)[:3]."""
    rgb = np.empty((256, 3), dtype=np.float64)
    _lib.check(_lib.load().nrn_jet_colormap(rgb.ctypes.data_as(C.c_void_p), None), "jet_colormap")
    return rgb


def image_scores(gt: torch.Tensor, generated: torch.Tensor, mask: Optional[torch.Tensor] = None, error_maps: bool = False,
                 ssim_map: bool = False) -> ImageScores:
    """PSNR and SSIM of every frame of generated [F, H, W, 3] against gt, as free_viewpoint_rendering.py:818-862 scores
    them.  mask [H, W] (nonzero = pixel zeroed in both images) defaults to the pixels of gt[0] whose channels sum to 0,
    the mask the reference builds from the first frame it scores.  error_maps=True adds the two uint8 error images
    (scaled RGB error and 1 - SSIM, on jet); ssim_map=True adds the SSIM map S."""
    gt = _frames(gt, "gt", 4)
    generated = _frames(generated, "generated", 4)
    if gt.shape != generated.shape or gt.device != generated.device:
        raise RuntimeError(f"nonrigid_nerf_b200: gt {tuple(gt.shape)} and generated {tuple(generated.shape)} differ")
    f, h, w, _ = gt.shape
    dev = gt.device
    if mask is not None:
        if tuple(mask.shape) != (h, w) or mask.device != dev:
            raise RuntimeError(f"nonrigid_nerf_b200: mask must be [{h}, {w}] on {dev}, got {tuple(mask.shape)}")
        mask = (mask != 0).to(torch.uint8).contiguous()
    lib = _lib.load()
    ws = torch.empty(max(int(lib.nrn_image_scores_bytes(f, h, w)), 16), dtype=torch.uint8, device=dev)
    psnr = torch.empty(f, dtype=torch.float32, device=dev)
    ssim = torch.empty(f, dtype=torch.float32, device=dev)
    smap = torch.empty_like(gt) if ssim_map else None
    err_rgb = torch.empty(gt.shape, dtype=torch.uint8, device=dev) if error_maps else None
    err_ssim = torch.empty(gt.shape, dtype=torch.uint8, device=dev) if error_maps else None
    a = _lib.NrnImageScoreArgs()
    a.gt, a.generated, a.mask = gt.data_ptr(), generated.data_ptr(), None if mask is None else mask.data_ptr()
    a.n_frames, a.height, a.width = f, h, w
    a.psnr, a.ssim = psnr.data_ptr(), ssim.data_ptr()
    a.ssim_map = None if smap is None else smap.data_ptr()
    a.error_rgb = None if err_rgb is None else err_rgb.data_ptr()
    a.error_ssim = None if err_ssim is None else err_ssim.data_ptr()
    a.workspace = ws.data_ptr()
    with torch.cuda.device(dev):
        a.stream = _stream().value
        _lib.check(lib.nrn_image_scores(C.byref(a)), "image_scores")
    return ImageScores(psnr, ssim, smap, err_rgb, err_ssim)


def disparity_images(disps: torch.Tensor, jet: bool = True, phong: bool = True):
    """(jet, phong) images [F, H, W, 3] fp32 of disparity frames [F, H, W], as visualize_disparity_with_jet_color_scheme
    and visualize_disparity_with_blinn_phong (run_nerf_helpers.py:701-793) make them; an image not asked for is None.
    The Phong image needs H, W >= 2."""
    disps = _frames(disps, "disps", 3)
    out_jet = torch.empty(disps.shape + (3,), dtype=torch.float32, device=disps.device) if jet else None
    out_phong = torch.empty(disps.shape + (3,), dtype=torch.float32, device=disps.device) if phong else None
    f, h, w = disps.shape
    with torch.cuda.device(disps.device):
        _lib.check(_lib.load().nrn_disparity_images(_ptr(disps), f, h, w, _ptr(out_jet), _ptr(out_phong), _stream()),
                   "disparity_images")
    return out_jet, out_phong


def background_stability(rgbs: torch.Tensor):
    """(image, std) of a fixed-camera sequence rgbs [F, H, W, 3] (free_viewpoint_rendering.py:770-785): std [H, W, 3] =
    np.std(rgbs, axis=0), image [H, W, 3] fp32 = the jet colour of 10 * the mean of std over the channels."""
    rgbs = _frames(rgbs, "rgbs", 4)
    f, h, w, _ = rgbs.shape
    if f == 0:
        raise RuntimeError("nonrigid_nerf_b200: background_stability needs at least one frame")
    image = torch.empty((h, w, 3), dtype=torch.float32, device=rgbs.device)
    std = torch.empty((h, w, 3), dtype=torch.float32, device=rgbs.device)
    with torch.cuda.device(rgbs.device):
        _lib.check(_lib.load().nrn_frame_std_image(_ptr(rgbs), f, h, w, _ptr(std), _ptr(image), _stream()), "background_stability")
    return image, std


def _volume_point(p, name: str) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray(p, dtype=np.float64).reshape(-1))
    if a.shape != (3,):
        raise RuntimeError(f"nonrigid_nerf_b200: {name} must hold 3 values, got {a.size}")
    return a


def frame_images(rgbs: Optional[torch.Tensor] = None, disps: Optional[torch.Tensor] = None,
                 surface_pts: Optional[torch.Tensor] = None, surface_rigidity: Optional[torch.Tensor] = None,
                 min_point=None, max_point=None) -> FrameImages:
    """The uint8 images free_viewpoint_rendering.py saves for a stack of rendered frames (:615-766), in one call:
    rgbs [F, H, W, 3] and disps [F, H, W] as render() returns them per frame (at least one of them: they give the frame
    size), surface_pts [F, H*W, 3] and surface_rigidity [F, H*W] as render(..., surface_output=True) returns them (or
    [F, H, W, 3] / [F, H, W]), and the volume extent min_point / max_point (3 values each, the checkpoint's
    scripts_dict["min_nerf_volume_point"] / ["max_nerf_volume_point"]) that the correspondence image needs.  Each image
    is computed when its input is given (rigidity images need surface_rigidity, which a model without a bender does not
    have).  The values equal the reference's numpy code bit for bit, except that disp_phong is to8b of
    disparity_images' fp32 Phong value and can be one level below the reference's float64 one.  The Phong image needs
    H, W >= 2 (np.gradient); smaller frames get disp_phong = None."""
    if any(t is not None and not isinstance(t, torch.Tensor) for t in (rgbs, disps, surface_pts, surface_rigidity)):
        raise RuntimeError("nonrigid_nerf_b200: frame_images inputs must be CUDA tensors (there is no CPU path)")
    if rgbs is not None and (rgbs.dim() != 4 or rgbs.shape[-1] != 3):
        raise RuntimeError(f"nonrigid_nerf_b200: rgbs must be [F, H, W, 3], got {tuple(rgbs.shape)}")
    if disps is not None and disps.dim() != 3:
        raise RuntimeError(f"nonrigid_nerf_b200: disps must be [F, H, W], got {tuple(disps.shape)}")
    if rgbs is None and disps is None:
        raise RuntimeError("nonrigid_nerf_b200: frame_images needs rgbs or disps (they give the frame size)")
    f, h, w = (rgbs if rgbs is not None else disps).shape[:3]
    if disps is not None and tuple(disps.shape) != (f, h, w):
        raise RuntimeError(f"nonrigid_nerf_b200: disps {tuple(disps.shape)} and rgbs {tuple(rgbs.shape)} differ")
    for t, name, tail in ((surface_pts, "surface_pts", (3,)), (surface_rigidity, "surface_rigidity", ())):
        if t is not None and tuple(t.shape) not in ((f, h * w) + tail, (f, h, w) + tail):
            raise RuntimeError(f"nonrigid_nerf_b200: {name} must be {[f, h * w] + list(tail)} or {[f, h, w] + list(tail)} "
                               f"for these frames, got {tuple(t.shape)}")
    if surface_pts is not None:
        if min_point is None or max_point is None:
            raise RuntimeError("nonrigid_nerf_b200: the correspondence image needs min_point and max_point")
        lo, hi = _volume_point(min_point, "min_point"), _volume_point(max_point, "max_point")
        if not np.all(hi > lo):
            raise RuntimeError(f"nonrigid_nerf_b200: max_point {hi.tolist()} must exceed min_point {lo.tolist()} on every axis")
    given = [t for t in (rgbs, disps, surface_pts, surface_rigidity) if t is not None]
    dev = given[0].device
    if any(not t.is_cuda or t.device != dev for t in given):
        raise RuntimeError("nonrigid_nerf_b200: frame_images inputs must be CUDA tensors on one device (there is no CPU path)")
    rgbs, disps, surface_pts, surface_rigidity = (None if t is None else t.float().contiguous()
                                                  for t in (rgbs, disps, surface_pts, surface_rigidity))

    def img(cond, channels):
        return torch.empty((f, h, w) + ((3,) if channels == 3 else ()), dtype=torch.uint8, device=dev) if cond else None

    out = FrameImages(rgb=img(rgbs is not None, 3), disp=img(disps is not None, 1), disp_video=img(disps is not None, 1),
                      disp_jet=img(disps is not None, 3), disp_phong=img(disps is not None and h >= 2 and w >= 2, 3),
                      correspondences=img(surface_pts is not None, 3), rigidity=img(surface_rigidity is not None, 1),
                      rigidity_jet=img(surface_rigidity is not None, 3))
    disp_max = torch.empty(f, dtype=torch.float32, device=dev) if disps is not None else None
    a = _lib.NrnFrameImageArgs()
    a.rgb, a.disp, a.surface_pts, a.surface_rigidity = (None if t is None else t.data_ptr()
                                                        for t in (rgbs, disps, surface_pts, surface_rigidity))
    if surface_pts is not None:
        a.min_point, a.max_point = lo.ctypes.data, hi.ctypes.data
    a.n_frames, a.height, a.width = f, h, w
    a.disp_max = None if disp_max is None else disp_max.data_ptr()
    for name, t in zip(FrameImages._fields, out):
        setattr(a, "out_" + name, None if t is None else t.data_ptr())
    with torch.cuda.device(dev):
        a.stream = _stream().value
        _lib.check(_lib.load().nrn_frame_images(C.byref(a)), "frame_images")
    return out
