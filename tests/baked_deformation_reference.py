"""numpy restatement of baked deformation grids (csrc/baked.cuh, nrnerf_b200.h): the fp16 store of the bender's offset and
rigidity, the per-ray rule that decides which rays take their bends from the grid, and the lookup followed by the
test-time knobs, in the same fp32 operations (tests/baked_reference.py restates the trilinear lookup itself)."""
import numpy as np

from tests import baked_reference as R


def to_f16(offsets: np.ndarray, rigidity: np.ndarray) -> np.ndarray:
    """[..., 4] fp16 of offsets [..., 3] and rigidity [...] or [..., 1]: the radiance store's rounding."""
    o = np.asarray(offsets, np.float32)
    r = np.asarray(rigidity, np.float32).reshape(o.shape[:-1] + (1,))
    return R.to_f16(np.concatenate([o, r], -1))


def sample_points(rays: np.ndarray, z: np.ndarray) -> np.ndarray:
    """[N, S, 3] fp32 x = o + d z of rays [N, 8+] and depths [N, S], multiply then add."""
    rays, z = np.asarray(rays, np.float32), np.asarray(z, np.float32)
    return rays[:, None, 0:3] + rays[:, None, 3:6] * z[..., None]


def deformed_rays(x: np.ndarray, lo, hi) -> np.ndarray:
    """[N] bool: every sample of the ray finite and inside [lo, hi] (the others fall back to the bender)."""
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    with np.errstate(invalid="ignore"):
        return np.all((x >= lo) & (x <= hi), axis=(1, 2))


def bend(x: np.ndarray, values: np.ndarray, lo, hi, cutoff=None, scaling=None):
    """The bend of points x [P, 3] inside the box from one frame's grid values [nz, ny, nx, 4] fp16: dict of
    unmasked_offsets o [P, 3], rigidity_mask r~ [P], masked_offsets m [P, 3] and input_pts c [P, 3], each operation an fp32
    one rounded on its own: r~ = (r <= cutoff) ? 0 : r, m = r~ o, m = m s, c = x + m."""
    x = np.asarray(x, np.float32).reshape(-1, 3)
    inside, v = R.lookup(x, values, lo, hi)
    assert inside.all()
    return knobs(x, v, cutoff, scaling)


def knobs(x: np.ndarray, v: np.ndarray, cutoff=None, scaling=None):
    """bend's algebra on looked-up values v [P, 4] = (o, r) at points x [P, 3]."""
    x = np.asarray(x, np.float32).reshape(-1, 3)
    o, r = v[:, :3].astype(np.float32), v[:, 3].astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        rt = np.where(r <= np.float32(cutoff), np.float32(0), r) if cutoff is not None else r
        m = rt[:, None] * o
        if scaling is not None:
            m = m * np.float32(scaling)
        c = x + m
    return {"unmasked_offsets": o, "rigidity_mask": rt.astype(np.float32), "masked_offsets": m.astype(np.float32),
            "input_pts": c.astype(np.float32), "initial_input_pts": x}
