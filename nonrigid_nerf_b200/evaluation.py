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


# ---- LPIPS (free_viewpoint_rendering.py:788-849, :868) ------------------------------------------------------------------
# lpips.LPIPS(net='alex') state-dict keys: the AlexNet convolutions ([out, in, k, k] weight, [out] bias), the tap weights
# lin{k}.model.1.weight [1, C_k, 1, 1] and the scaling layer's shift / scale [1, 3, 1, 1] (defaults when absent)
LPIPS_CONVS = (("net.slice1.0", 64, 3, 11), ("net.slice2.3", 192, 64, 5), ("net.slice3.6", 384, 192, 3),
               ("net.slice4.8", 256, 384, 3), ("net.slice5.10", 256, 256, 3))
LPIPS_SHIFT = (-0.030, -0.088, -0.188)
LPIPS_SCALE = (0.458, 0.448, 0.450)
LPIPS_MIN_SIDE = 31   # the smallest frame height and width for which every tap has a pixel


def lpips_state(source) -> list:
    """The 17 fp32 tensors nrn_lpips_pack takes, in its order (conv weight and bias of the five layers, the five tap
    weights flattened to [C_k], shift [3], scale [3]), from an lpips.LPIPS(net='alex') module or its state dict.
    Raises before anything reaches the device when the source is not that network: another backbone (VGG, SqueezeNet),
    missing keys, wrong shapes, or a module configured for a different score (version 0.0, spatial maps)."""
    if isinstance(source, torch.nn.Module):
        if str(getattr(source, "version", "0.1")) != "0.1":
            raise RuntimeError(f"nonrigid_nerf_b200: LPIPS version {source.version} is not supported (0.1 only)")
        if getattr(source, "spatial", False):
            raise RuntimeError("nonrigid_nerf_b200: spatial LPIPS maps are not supported (one score per frame)")
        if getattr(source, "pnet_type", "alex") != "alex":
            raise RuntimeError(f"nonrigid_nerf_b200: the {source.pnet_type} backbone is not supported (net='alex' only)")
        source = source.state_dict()
    if not isinstance(source, dict):
        raise RuntimeError(f"nonrigid_nerf_b200: lpips weights come from an lpips.LPIPS module or its state dict, got {type(source)}")
    if any(k in source for k in ("lin5.model.1.weight", "lin6.model.1.weight")):
        raise RuntimeError("nonrigid_nerf_b200: this LPIPS state dict has more than five taps (SqueezeNet); net='alex' only")

    def get(key, shape):
        if key not in source:
            raise RuntimeError(f"nonrigid_nerf_b200: LPIPS state dict lacks {key} (net='alex' only)")
        t = source[key]
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != shape:
            got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t)
            raise RuntimeError(f"nonrigid_nerf_b200: LPIPS {key} must be {list(shape)}, got {got} "
                               "(net='alex' only; VGG and SqueezeNet backbones are not supported)")
        t = t.detach().float()
        if not bool(torch.isfinite(t).all()):
            raise RuntimeError(f"nonrigid_nerf_b200: LPIPS {key} holds non-finite values")
        return t

    out = []
    for key, cout, cin, k in LPIPS_CONVS:
        out += [get(key + ".weight", (cout, cin, k, k)), get(key + ".bias", (cout,))]
    out += [get(f"lin{k}.model.1.weight", (1, c[1], 1, 1)).reshape(-1) for k, c in enumerate(LPIPS_CONVS)]
    for key, default in (("scaling_layer.shift", LPIPS_SHIFT), ("scaling_layer.scale", LPIPS_SCALE)):
        out.append(get(key, (1, 3, 1, 1)).reshape(-1) if key in source else torch.tensor(default, dtype=torch.float32))
    return out


class LpipsWeights:
    """An LPIPS weight set packed for the kernels (nrn_lpips_pack): fp16 convolution images, fp32 biases, tap weights and
    scaling.  Made once by lpips_weights(); `packed` lives on `device`."""

    def __init__(self, packed: torch.Tensor, sources: list):
        self.packed = packed
        self.device = packed.device
        self._sources = sources   # the pack reads them on the stream; kept alive with the packed block


def lpips_weights(source, device=None) -> LpipsWeights:
    """Validate an lpips.LPIPS(net='alex') module or its state dict (lpips_state) and pack it once on `device` (default:
    the current CUDA device), on the current stream."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("nonrigid_nerf_b200: LPIPS weights are packed on a CUDA device (there is no CPU path)")
    state = lpips_state(source)
    lib = _lib.load()
    with torch.cuda.device(dev):
        src = [t.to(dev).contiguous() for t in state]
        packed = torch.empty(int(lib.nrn_lpips_packed_bytes()), dtype=torch.uint8, device=dev)
        ptrs = (C.c_void_p * len(src))(*[t.data_ptr() for t in src])
        _lib.check(lib.nrn_lpips_pack(ptrs, packed.data_ptr(), _stream()), "lpips_weights")
    return LpipsWeights(packed, src)


def lpips(gt: torch.Tensor, generated: torch.Tensor, weights: LpipsWeights, mask: Optional[torch.Tensor] = None,
          per_layer: bool = False, *, chunk_frames: Optional[int] = None):
    """LPIPS (v0.1, AlexNet) of every frame of generated [F, H, W, 3] against gt in [0, 1], as
    free_viewpoint_rendering.py:836-849 scores them: [F] fp32, or ([F], [F, 5] tap scores) with per_layer=True.  mask
    [H, W] (nonzero = pixel zeroed in both images) defaults to the pixels of gt[0] whose channels sum to 0, as in
    image_scores.  H and W must be at least 31.  Frames go through the network in chunks of chunk_frames (default: as
    many as fit 256 MiB of activations); a frame's score does not depend on the chunk or batch it is in.
    Activations are stored in fp16.  A convolution output above 65504 (the largest fp16 value) would be clamped and
    give a finite but wrong score, so a frame with such an output in either image scores NaN instead, and so do its tap
    scores from that convolution's tap on; the earlier taps stay finite.  There is no higher-precision path."""
    if not isinstance(weights, LpipsWeights):
        raise RuntimeError("nonrigid_nerf_b200: weights must come from evaluation.lpips_weights()")
    gt = _frames(gt, "gt", 4)
    generated = _frames(generated, "generated", 4)
    if gt.shape != generated.shape or gt.device != generated.device:
        raise RuntimeError(f"nonrigid_nerf_b200: gt {tuple(gt.shape)} and generated {tuple(generated.shape)} differ")
    f, h, w, _ = gt.shape
    dev = gt.device
    if weights.device != dev:
        raise RuntimeError(f"nonrigid_nerf_b200: LPIPS weights are on {weights.device}, the frames on {dev}")
    if h < LPIPS_MIN_SIDE or w < LPIPS_MIN_SIDE:
        raise RuntimeError(f"nonrigid_nerf_b200: LPIPS needs frames of at least {LPIPS_MIN_SIDE} x {LPIPS_MIN_SIDE} pixels "
                           f"(every AlexNet tap needs a pixel), got {h} x {w}")
    if mask is not None:
        if tuple(mask.shape) != (h, w) or mask.device != dev:
            raise RuntimeError(f"nonrigid_nerf_b200: mask must be [{h}, {w}] on {dev}, got {tuple(mask.shape)}")
        mask = (mask != 0).to(torch.uint8).contiguous()
    lib = _lib.load()
    if chunk_frames is None:
        ws_bytes = int(lib.nrn_lpips_workspace_bytes(f, h, w))
    else:
        if int(chunk_frames) < 1:
            raise RuntimeError(f"nonrigid_nerf_b200: chunk_frames must be at least 1, got {chunk_frames}")
        base = int(lib.nrn_lpips_workspace_bytes(0, h, w))
        ws_bytes = base + min(int(chunk_frames), f) * (int(lib.nrn_lpips_workspace_bytes(1, h, w)) - base)
    if ws_bytes == 0:
        raise RuntimeError(f"nonrigid_nerf_b200: LPIPS frames of {h} x {w} pixels are out of range")
    out = torch.empty(f, dtype=torch.float32, device=dev)
    layers = torch.empty((f, 5), dtype=torch.float32, device=dev) if per_layer else None
    if f > 0:
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        a = _lib.NrnLpipsArgs()
        a.gt, a.generated, a.mask = gt.data_ptr(), generated.data_ptr(), None if mask is None else mask.data_ptr()
        a.n_frames, a.height, a.width = f, h, w
        a.packed, a.lpips, a.per_layer = weights.packed.data_ptr(), out.data_ptr(), None if layers is None else layers.data_ptr()
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws_bytes
        with torch.cuda.device(dev):
            a.stream = _stream().value
            _lib.check(lib.nrn_lpips(C.byref(a)), "lpips")
    return (out, layers) if per_layer else out


def normal_images(normals: torch.Tensor, c2w: torch.Tensor) -> torch.Tensor:
    """uint8 [F, H, W, 3] images of world-space unit normals [F, H, W, 3] (render(..., surface_normals=True)) seen from the
    cameras c2w [F, 3, 4+] (camera-to-world, get_rays convention: x right, y up, z toward the viewer).  Per pixel, in
    fp32 with every operation rounded on its own: c_k = (R[0][k] n_0 + R[1][k] n_1) + R[2][k] n_2 (R = c2w[:, :3, :3], so
    c = R^T n), v = (c + 1) * 0.5, out = to8b(v) = uint8(trunc(255 * clip(v, 0, 1))); a zero normal (no surface) gives 0."""
    normals = _frames(normals, "normals", 4)
    if normals.shape[-1] != 3:
        raise RuntimeError(f"nonrigid_nerf_b200: normals must be [F, H, W, 3], got {tuple(normals.shape)}")
    if not isinstance(c2w, torch.Tensor) or c2w.dim() != 3 or c2w.shape[0] != normals.shape[0] or c2w.shape[1] < 3 or c2w.shape[2] < 3:
        raise RuntimeError(f"nonrigid_nerf_b200: c2w must be [F, 3, 4] for {normals.shape[0]} frames")
    r = c2w[:, :3, :3].to(device=normals.device, dtype=torch.float32)[:, None, None]   # [F, 1, 1, 3, 3]
    n = normals
    c = [(r[..., 0, k] * n[..., 0] + r[..., 1, k] * n[..., 1]) + r[..., 2, k] * n[..., 2] for k in range(3)]
    v = (torch.stack(c, -1) + 1.0) * 0.5
    out = (255.0 * v.clamp(0.0, 1.0)).to(torch.uint8)
    zero = (n == 0).all(-1, keepdim=True)
    return torch.where(zero, torch.zeros_like(out), out)
