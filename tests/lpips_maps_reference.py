"""Spatial LPIPS maps (lpips.LPIPS(net='alex', spatial=True), retPerLayer=True for the per-tap maps) restated for the
tests of evaluation.lpips_maps, on top of tests/lpips_reference.py:

- distances(): the per-pixel distance d_l [F, h_l, w_l] of every tap in fp64, the quantity lpips_reference.lpips
  averages;
- maps64(): per tap F.interpolate(d_l, size=(H, W), mode="bilinear", align_corners=False) in fp64 and their sum in tap
  order (val += res[l]);
- upsample32() / maps32(): the kernel's fp32 rule with every operation rounded on its own (numpy float32 rounds each
  operation and never contracts), for bit-for-bit checks of the upsampling of the kernel's own tap maps, with the NaN rule
  of frames whose convolution clamped an output;
- upsample_loop(): PyTorch's index rule as a plain loop in fp64, which pins F.interpolate's reading of it;
- error_image(): to8b(jet(clip(map, 0, 1))) with the library's jet table and its NaN rule (index 0);
- the workspace of nrn_lpips_maps: tests/lpips_layout.py's chunk, then the five tap maps [fc][h_l][w_l] fp32, each tap a
  256-byte aligned buffer.
"""
import numpy as np
import torch
import torch.nn.functional as F

from tests import lpips_layout as L
from tests import lpips_reference as R


# ---- fp64 restatement --------------------------------------------------------------------------------------------------
def distances(gt, gen, sd: dict, mask=None, device="cpu") -> list:
    """[d_0 .. d_4], d_l [F, h_l, w_l] fp64 (on `device`): per pixel sum_c w_c (g_c / (|g| + 1e-10) - r_c / (|r| + 1e-10))^2
    of tap l, for frames gt, gen [F, H, W, 3] (numpy or tensors) with the mask rule of lpips_reference.lpips"""
    gt = torch.as_tensor(np.asarray(gt) if not isinstance(gt, torch.Tensor) else gt).to(device, torch.float64).clone()
    gen = torch.as_tensor(np.asarray(gen) if not isinstance(gen, torch.Tensor) else gen).to(device, torch.float64).clone()
    m = R.mask_from(gt[0].cpu().numpy()) if mask is None else np.asarray(mask) != 0
    m = torch.as_tensor(m, device=device)
    gt[:, m] = 0
    gen[:, m] = 0
    sdd = {k: v.to(device) for k, v in sd.items()}
    out = [[] for _ in range(L.TAPS)]
    for i in range(gt.shape[0]):   # frame by frame, as the scores
        fa, fb = R.taps(_scaled(gt[i:i + 1], sdd), sdd), R.taps(_scaled(gen[i:i + 1], sdd), sdd)
        for k, (a, b) in enumerate(zip(fa, fb)):
            na = a / (torch.sqrt((a * a).sum(dim=1, keepdim=True)) + R.EPS)
            nb = b / (torch.sqrt((b * b).sum(dim=1, keepdim=True)) + R.EPS)
            w = sdd[f"lin{k}.model.1.weight"].double().reshape(1, -1, 1, 1)
            out[k].append((w * (na - nb) ** 2).sum(dim=1)[0])
    return [torch.stack(d) for d in out]


def _scaled(img, sd):
    shift = sd.get("scaling_layer.shift", torch.tensor(R.SHIFT)).double().reshape(1, 3, 1, 1).to(img.device)
    scale = sd.get("scaling_layer.scale", torch.tensor(R.SCALE)).double().reshape(1, 3, 1, 1).to(img.device)
    return (2 * img.permute(0, 3, 1, 2) - 1 - shift) / scale


def upsample64(d: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """[F, h_l, w_l] -> [F, H, W]: F.interpolate(bilinear, align_corners=False) in fp64"""
    return F.interpolate(d.double()[:, None], size=(h, w), mode="bilinear", align_corners=False)[:, 0]


def maps64(gt, gen, sd: dict, mask=None, device="cpu"):
    """(map [F, H, W], layer_maps [F, 5, H, W]) in fp64: lpips.LPIPS(net='alex', spatial=True) of the frames"""
    h, w = np.shape(gt)[1:3]
    ups = [upsample64(d, h, w) for d in distances(gt, gen, sd, mask, device)]
    total = ups[0].clone()
    for u in ups[1:]:
        total += u
    return total, torch.stack(ups, dim=1)


def upsample_loop(d: np.ndarray, h: int, w: int) -> np.ndarray:
    """[h_l, w_l] -> [H, W] in fp64 by PyTorch's rule for align_corners=False and an explicit size, written out:
    scale = in / out, src = max(scale (dst + 0.5) - 0.5, 0), i0 = floor, i1 = i0 + (i0 < in - 1), l1 = src - i0"""
    hi, wi = d.shape
    out = np.empty((h, w))
    for y in range(h):
        sy = max((hi / h) * (y + 0.5) - 0.5, 0.0)
        y0 = int(sy)
        y1 = y0 + (1 if y0 < hi - 1 else 0)
        ly1 = sy - y0
        for x in range(w):
            sx = max((wi / w) * (x + 0.5) - 0.5, 0.0)
            x0 = int(sx)
            x1 = x0 + (1 if x0 < wi - 1 else 0)
            lx1 = sx - x0
            out[y, x] = (1 - ly1) * ((1 - lx1) * d[y0, x0] + lx1 * d[y0, x1]) + ly1 * ((1 - lx1) * d[y1, x0] + lx1 * d[y1, x1])
    return out


def fp32_bound(d_max, h_l, w_l):
    """|fp32 rule - fp64 interpolate| <= d_max 2^-24 (6 (h_l + w_l + 2) + 8): the source coordinates src = scale (y + 0.5)
    - 0.5 carry about 3 (|src| + 1) 2^-24 of fp32 rounding into l1 along each axis, each of which multiplies a difference of
    two non-negative neighbours (at most d_max), and the six products and sums round once each"""
    return d_max * 2.0 ** -24 * (6 * (h_l + w_l + 2) + 8)


# ---- the kernel's fp32 rule --------------------------------------------------------------------------------------------
def _axis32(n_out: int, n_in: int):
    f32 = np.float32
    scale = f32(n_in) / f32(n_out)
    src = scale * (np.arange(n_out).astype(f32) + f32(0.5)) - f32(0.5)
    src = np.where(src < f32(0), f32(0), src).astype(f32)
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < n_in - 1)
    l1 = (src - i0.astype(f32)).astype(f32)
    return i0, i1, (f32(1) - l1).astype(f32), l1


def upsample32(d: np.ndarray, h: int, w: int) -> np.ndarray:
    """[F, h_l, w_l] fp32 -> [F, H, W] fp32: v = hl0 (wl0 x00 + wl1 x01) + hl1 (wl0 x10 + wl1 x11), each operation rounded
    to fp32 on its own"""
    d = np.asarray(d, dtype=np.float32)
    y0, y1, hl0, hl1 = _axis32(h, d.shape[1])
    x0, x1, wl0, wl1 = _axis32(w, d.shape[2])
    r0, r1 = d[:, y0], d[:, y1]                            # [F, H, w_l]
    top = wl0 * r0[:, :, x0] + wl1 * r0[:, :, x1]          # [F, H, W]
    bot = wl0 * r1[:, :, x0] + wl1 * r1[:, :, x1]
    return (hl0[None, :, None] * top + hl1[None, :, None] * bot).astype(np.float32)


def maps32(taps, h: int, w: int, first=None):
    """(map [F, H, W], layer_maps [F, 5, H, W]) fp32 from the tap maps [d_0 .. d_4] (each [F, h_l, w_l] fp32); first [F]:
    each frame's first tap whose convolution clamped an output (5 or None: none), NaN from it on"""
    ups = np.stack([upsample32(d, h, w) for d in taps], axis=1)
    if first is not None:
        for f, k in enumerate(first):
            ups[f, k:] = np.nan
    total = ups[:, 0].copy()
    for k in range(1, L.TAPS):
        total = (total + ups[:, k]).astype(np.float32)
    return total, ups


def lut_index(v: np.ndarray) -> np.ndarray:
    """the jet index of eval.cuh's lut_index: int(fp32(255 * clip(v, 0, 1))), NaN -> 0"""
    v = np.asarray(v, dtype=np.float32)
    k = (np.float32(255) * np.clip(np.nan_to_num(v, nan=0.0), np.float32(0), np.float32(1))).astype(np.float32)
    return np.where(np.isnan(v), 0, k.astype(np.int64))


def jet8() -> np.ndarray:
    """[256, 3] uint8 to8b(cm.jet(i)[:3]), the library's table"""
    import ctypes as C
    from nonrigid_nerf_b200 import _lib
    t = np.empty((256, 3), dtype=np.uint8)
    _lib.check(_lib.load().nrn_jet_colormap(None, t.ctypes.data_as(C.c_void_p)), "jet_colormap")
    return t


def error_image(map32: np.ndarray) -> np.ndarray:
    """[F, H, W] fp32 -> [F, H, W, 3] uint8 to8b(jet(clip(map, 0, 1)))"""
    return jet8()[lut_index(map32)]


# ---- workspace of nrn_lpips_maps ---------------------------------------------------------------------------------------
def tap_map_bytes(h, w, tap):
    return L.px(h, w, L.TAP_STAGES[tap]) * 4


def map_frame_bytes(h, w):
    return L.frame_bytes(h, w) + sum(L.a256(tap_map_bytes(h, w, k)) for k in range(L.TAPS))


def workspace_bytes(f, h, w):
    """nrn_lpips_maps_workspace_bytes(f, h, w): 0 out of range"""
    if f < 0 or not (L.MIN_SIDE <= h <= L.MAX_SIDE and L.MIN_SIDE <= w <= L.MAX_SIDE):
        return 0
    fb = map_frame_bytes(h, w)
    return L.mask_bytes(h, w) + min(max(1, min(L.CHUNK_BUDGET // fb, L.MAX_CHUNK)), f) * fb


def tap_map_offset(fc, h, w, tap):
    o = L.mask_bytes(h, w) + fc * L.frame_bytes(h, w)
    return o + sum(L.a256(fc * tap_map_bytes(h, w, k)) for k in range(tap))


def tap_map(ws, fc, h, w, tap):
    """Tap `tap`'s map of a chunk of fc frames from the workspace bytes ws (uint8 tensor) -> [fc, h_l, w_l] fp32"""
    hh, ww = L.dims(h, w)[L.TAP_STAGES[tap]]
    off = tap_map_offset(fc, h, w, tap)
    return ws[off:off + fc * tap_map_bytes(h, w, tap)].view(torch.float32).view(fc, hh, ww)
