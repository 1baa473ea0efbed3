"""numpy / scipy restatements of the reference's evaluation and visualisation (free_viewpoint_rendering.py:725-876,
run_nerf_helpers.py:701-793), the checkers of nonrigid_nerf_b200.evaluation.  scikit-image and matplotlib, which the
reference calls, are optional: where they can be imported the tests compare against them as well.

- jet: matplotlib's cm.jet rebuilt from its published segment data the way LinearSegmentedColormap builds its table;
- SSIM: skimage.metrics.structural_similarity(data_range=1, gaussian_weights=True, sigma=1.5,
  use_sample_covariance=False, multichannel=True, full=True) written out with scipy.ndimage.gaussian_filter, in fp64;
- Blinn-Phong: the shading of run_nerf_helpers.py:718-793 with np.gradient normals, in fp64.
"""
from __future__ import annotations

import numpy as np
from scipy.ndimage import gaussian_filter

# matplotlib/_cm.py: _jet_data, (x, y0, y1) per breakpoint
JET_DATA = {
    "red": ((0.00, 0, 0), (0.35, 0, 0), (0.66, 1, 1), (0.89, 1, 1), (1.00, 0.5, 0.5)),
    "green": ((0.000, 0, 0), (0.125, 0, 0), (0.375, 1, 1), (0.640, 1, 1), (0.910, 0, 0), (1.000, 0, 0)),
    "blue": ((0.00, 0.5, 0.5), (0.11, 1, 1), (0.34, 1, 1), (0.65, 0, 0), (1, 0, 0)),
}


def _segment_table(data, n=256):
    a = np.asarray(data, dtype=np.float64)
    x, y0, y1 = a[:, 0] * (n - 1), a[:, 1], a[:, 2]
    xind = (n - 1) * np.linspace(0, 1, n) ** 1.0
    ind = np.searchsorted(x, xind)[1:-1]
    distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
    return np.clip(lut, 0.0, 1.0)


def jet_lut() -> np.ndarray:
    """[256, 3] float64 = cm.jet(i)[:3]."""
    return np.stack([_segment_table(JET_DATA[c]) for c in ("red", "green", "blue")], axis=-1)


def to8b(x):
    return (255 * np.clip(x, 0, 1)).astype(np.uint8)


def lut_index(v):
    """uint8(255 * clip(v, 0, 1)) as .astype("uint8") truncates it, in v's precision; NaN -> 0."""
    return (255.0 * np.clip(np.nan_to_num(np.asarray(v), nan=0.0), 0, 1)).astype(np.uint8)


def near_bin_edge(v, eps=1e-6):
    """Where v lies within eps of a LUT bin edge k / 255 (the fp32 / fp64 truncation may fall either way there)."""
    s = 255.0 * np.asarray(v, dtype=np.float64)
    return np.abs(s - np.round(s)) < 255.0 * eps


def mask_from(gt0):
    return np.sum(gt0, axis=-1) == 0.0


def apply_mask(gt, gen, mask):
    gt, gen = gt.copy(), gen.copy()
    gt[..., mask, :] = 0.0
    gen[..., mask, :] = 0.0
    return gt, gen


def psnr(gt, gen):
    mse = np.mean((gt.astype(np.float64) - gen.astype(np.float64)) ** 2)
    with np.errstate(divide="ignore"):
        return -10.0 * np.log10(mse)


def ssim(gt, gen):
    """(score, S [H, W, 3]) in fp64 for one frame [H, W, 3]."""
    filt = lambda a: gaussian_filter(a, sigma=1.5, truncate=3.5, mode="reflect")  # noqa: E731
    S = np.empty(gt.shape, dtype=np.float64)
    for c in range(3):
        x, y = gt[..., c].astype(np.float64), gen[..., c].astype(np.float64)
        ux, uy, uxx, uyy, uxy = filt(x), filt(y), filt(x * x), filt(y * y), filt(x * y)
        vx, vy, vxy = uxx - ux * ux, uyy - uy * uy, uxy - ux * uy
        C1, C2 = 0.01 ** 2, 0.03 ** 2
        S[..., c] = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux * ux + uy * uy + C1) * (vx + vy + C2))
    with np.errstate(invalid="ignore"):
        crop = S[5:-5, 5:-5] if min(gt.shape[:2]) > 10 else S[:0]
        score = np.float64(np.nan) if crop.size == 0 else crop.mean(dtype=np.float64)
    return score, S


def error_rgb_value(gt, gen):
    """10 |gt - gen|_2 / sqrt(3) on the float32 frames, as free_viewpoint_rendering.py:847-849 computes it."""
    return np.linalg.norm(gt - gen, axis=-1) / np.sqrt(1 + 1 + 1) * 10.0


def error_ssim_value(S):
    return 1.0 - np.mean(S.astype(np.float64), axis=-1)


def std_image(rgbs):
    """(image [H, W, 3] fp64 colours, std [H, W, 3] fp32) of free_viewpoint_rendering.py:771-780."""
    std = np.std(rgbs, axis=0)
    v = 10 * np.mean(std, axis=-1)
    return jet_lut()[lut_index(v)], std, v


def phong(d):
    """Blinn-Phong image [H, W, 3] (fp64) of a disparity map [H, W]; also the Lambertian term [H, W] before clipping."""
    d = np.asarray(d)
    h, w = d.shape
    zy, zx = np.gradient(d, 2.0 / (h - 1))
    n = np.stack([-zx, zy, np.ones_like(d)], axis=-1).astype(np.float64)
    n = n / np.linalg.norm(n, axis=-1, keepdims=True)
    cols, rows = np.meshgrid(np.arange(w, dtype=np.float32) / w, np.arange(h, dtype=np.float32) / w, indexing="xy")
    pos = np.stack([cols, rows, d], axis=-1).astype(np.float64)
    to_light = 1.0 - pos
    dist = np.linalg.norm(to_light, axis=-1, keepdims=True)
    to_light = to_light / dist
    att = (dist + 1.0) ** 2
    lam_raw = np.sum(to_light * n, axis=-1)
    lam = np.clip(lam_raw, 0.0, None)[..., None]
    view = -pos / np.linalg.norm(pos, axis=-1, keepdims=True)
    half = to_light + view
    half = half / np.linalg.norm(half, axis=-1, keepdims=True)
    spec = np.clip(np.sum(half * -n, axis=-1), 0.0, None)[..., None] ** 2.0
    spec[lam <= 0.0] = 0.0
    diffuse, ambient = np.array([0.5, 0.0, 0.0]), np.array([0.1, 0.0, 0.0])
    return lam * diffuse * 2.0 / att + spec * 2.0 / att + ambient, lam_raw


def frames(kind, f, h, w, seed):
    """Test frames [F, H, W, 3] fp32 in [0, 1]: (gt, generated) pairs of several structures."""
    rng = np.random.default_rng(seed)
    if kind == "random":
        gt = rng.random((f, h, w, 3), dtype=np.float32)
        gen = np.clip(gt + rng.normal(0, 0.1, gt.shape), 0, 1).astype(np.float32)
    elif kind == "smooth":
        yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
        base = np.stack([xx, yy, 0.5 * (xx + yy)], axis=-1)
        gt = np.stack([np.clip(base * (0.5 + 0.5 * rng.random()), 0, 1) for _ in range(f)]).astype(np.float32)
        gen = np.clip(gt + 0.02 * np.sin(7 * base + rng.random()), 0, 1).astype(np.float32)
    elif kind == "edges":
        yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        gt = np.stack([np.stack([((xx // 4 + yy // 3 + i) % 2).astype(np.float32)] * 3, -1) * np.float32(0.8) for i in range(f)])
        gen = np.roll(gt, 1, axis=2) * np.float32(0.9)
    elif kind == "masked":   # black borders in every ground-truth frame, as undistortion leaves them
        gt = rng.random((f, h, w, 3), dtype=np.float32) * np.float32(0.9) + np.float32(0.05)
        b = max(1, min(h, w) // 8)
        gt[:, :b], gt[:, :, :b] = 0.0, 0.0
        gen = np.clip(gt + rng.normal(0, 0.05, gt.shape), 0, 1).astype(np.float32)
    else:
        raise ValueError(kind)
    return gt.astype(np.float32), gen.astype(np.float32)
