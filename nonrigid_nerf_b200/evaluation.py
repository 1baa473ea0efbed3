"""Scores and images of rendered frames on the GPU: what free_viewpoint_rendering.py computes on the host with numpy,
scikit-image and matplotlib once the frames are rendered (PSNR, SSIM and the error images of :786-876, the jet and
Blinn-Phong disparity images of :725-745 / run_nerf_helpers.py:701-793, the background-stability map of :770-785).

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
