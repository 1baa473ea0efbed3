"""numpy restatement of the images free_viewpoint_rendering.py saves for rendered frames: the canonical-correspondence
image (:640-644), the per-frame images (:660-704) and the video stacks (:706-766), with the convert_*_to_saveable /
_jet / _phong helpers of :346-378.  It takes the per-pixel results of render(..., surface_output=True) (the canonical
point and rigidity of each pixel's median-visibility sample) in place of the reference's detailed output, and is the
checker of nonrigid_nerf_b200.evaluation.frame_images.  to8b, the cm.jet table, the LUT index and the Blinn-Phong
shading are tests/eval_reference.py's.
"""
from __future__ import annotations

import numpy as np

from tests.eval_reference import jet_lut, lut_index, phong, to8b

VOXELS = 100   # the reference's number_of_small_rgb_voxels


def normalized(disp, normalize=True):
    """disp / np.max(disp) in disp's precision (float32 for a rendered map), or disp itself."""
    return disp / np.max(disp) if normalize else disp.copy()


def disparity_saveable(disp, normalize=True):
    return to8b(normalized(disp, normalize))


def disparity_jet(disp, normalize=True):
    """to8b of the jet colours: the reference indexes cm.jet with uint8(255 * clip(d, 0, 1)) in d's precision."""
    return to8b(jet_lut()[lut_index(normalized(disp, normalize))])


def disparity_phong(disp, normalize=True):
    """to8b of the float64 Blinn-Phong restatement of the normalised map (H, W >= 2)."""
    return to8b(phong(normalized(disp, normalize))[0])


def correspondence_rgb(surface_pixels, min_point, max_point):
    """float64 fraction image of float32 canonical points [..., 3] in a float64 extent: the checkerboard of VOXELS
    voxels per axis, c - c.astype(int) (truncation toward zero, so points below min give negative values)."""
    lo = np.asarray(min_point, dtype=np.float64).reshape(-1)
    hi = np.asarray(max_point, dtype=np.float64).reshape(-1)
    c = (np.asarray(surface_pixels, dtype=np.float32) - lo) / (hi - lo)
    c *= VOXELS
    with np.errstate(invalid="ignore"):
        return c - c.astype(np.int64)


def frame_images(rgbs=None, disps=None, surface_pts=None, surface_rigidity=None, min_point=None, max_point=None):
    """{name: uint8 stack} of every image the inputs allow, named as evaluation.FrameImages.  rgbs [F, H, W, 3] and / or
    disps [F, H, W] (they give the frame size), surface_pts [F, H*W, 3], surface_rigidity [F, H*W]."""
    f, h, w = (rgbs if rgbs is not None else disps).shape[:3]
    out = {}
    if rgbs is not None:
        out["rgb"] = to8b(rgbs)
    if disps is not None:
        out["disp"] = np.stack([disparity_saveable(d) for d in disps])
        out["disp_video"] = disparity_saveable(disps)   # one maximum over the whole stack, as the video is written
        out["disp_jet"] = np.stack([disparity_jet(d) for d in disps])
        if h >= 2 and w >= 2:
            out["disp_phong"] = np.stack([disparity_phong(d) for d in disps])
    if surface_pts is not None:
        pts = np.asarray(surface_pts).reshape(f, h, w, 3)
        out["correspondences"] = to8b(correspondence_rgb(pts, min_point, max_point))
    if surface_rigidity is not None:
        rig = np.asarray(surface_rigidity).reshape(f, h, w)
        out["rigidity"] = np.stack([disparity_saveable(r, normalize=False) for r in rig])
        out["rigidity_jet"] = np.stack([disparity_jet(r, normalize=False) for r in rig])
    return out


def seeded_inputs(f, h, w, seed):
    """Test inputs (rgbs, disps, surface_pts [F, H*W, 3], surface_rigidity [F, H*W], min_point, max_point): colours
    and rigidity in and outside [0, 1] with exact 0 and 1, disparity frames of different maxima (the first with its
    maximum in a corner), canonical points inside and outside the extent, on voxel boundaries and on its faces."""
    rng = np.random.default_rng(seed)
    lo, hi = np.array([-1.5, -0.75, -2.0]), np.array([1.25, 0.5, -0.125])
    n = h * w
    rgbs = rng.uniform(-0.1, 1.1, (f, h, w, 3)).astype(np.float32)
    flat = rgbs.reshape(-1)
    flat[: min(6, flat.size)] = np.array([0.0, 1.0, -0.0, np.nextafter(np.float32(1), np.float32(2)),
                                          np.nextafter(np.float32(0), np.float32(-1)), 0.5], dtype=np.float32)[: min(6, flat.size)]
    disps = (rng.uniform(0.0, 1.0, (f, h, w)) * (1.0 + np.arange(f)[:, None, None])).astype(np.float32)
    disps[0, h - 1, w - 1] = np.float32(1.5) * (1.0 + disps[0].max())
    pts = (lo + (hi - lo) * rng.uniform(-0.1, 1.1, (f, n, 3))).astype(np.float32)
    k = max(1, n // 4)
    grid = rng.integers(-3, VOXELS + 4, (f, k, 3))   # voxel boundaries, some outside the extent
    on = (lo + (hi - lo) * grid / VOXELS).astype(np.float32)
    pts[:, :k] = on
    pts[0, 0], pts[-1, -1] = lo.astype(np.float32), hi.astype(np.float32)
    rig = rng.uniform(-0.2, 1.2, (f, n)).astype(np.float32)
    rig.reshape(-1)[: min(4, rig.size)] = np.array([0.0, 1.0, -1e-8, 1.0 + 1e-7], dtype=np.float32)[: min(4, rig.size)]
    return rgbs, disps, pts, rig, lo, hi
