"""numpy restatement of the baked radiance grid (csrc/baked.cuh): the vertex positions, the fp16 store and the fp32 lookup,
in the same fp32 operations."""
import numpy as np

from tests import mesh_reference as M


def vertex_points(min_point, max_point, res) -> np.ndarray:
    """[nz, ny, nx, 3] fp32 vertex positions: the mesh grid's points (mesh_reference.grid_points_plane, one formula for
    both); res = (nx, ny, nz)."""
    return np.stack([M.grid_points_plane(min_point, max_point, res, k) for k in range(res[2])])


def to_f16(raw: np.ndarray) -> np.ndarray:
    """[..., 4] fp16 of raw [..., >= 4] channels 0..3: round to nearest even, finite values saturated to +-65504, inf and
    NaN kept."""
    r = np.asarray(raw, np.float32)[..., :4]
    fin = np.isfinite(r)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.where(fin, np.clip(r, np.float32(-65504), np.float32(65504)), r).astype(np.float16)


def scale(lo, hi, res) -> np.ndarray:
    """fl((n - 1) / fl(hi - lo)) per axis; res = (nx, ny, nz)."""
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    return (np.asarray(res, np.float32) - np.float32(1)) / (hi - lo)


def cells(points: np.ndarray, res, lo, hi):
    """(inside [P] bool, lower corner [P, 3] int64 (i, j, k), fractions [P, 3] fp32) of each point; the corner and fractions
    of a point outside are 0."""
    x = np.asarray(points, np.float32).reshape(-1, 3)
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    n = np.asarray(res, np.int64)
    with np.errstate(invalid="ignore"):
        inside = np.all((x >= lo) & (x <= hi), axis=1)
        u = (np.where(inside[:, None], x, lo) - lo) * scale(lo, hi, res)
    c = np.minimum(np.floor(u).astype(np.int64), n - 2)
    f = u - c.astype(np.float32)
    return inside, c, f.astype(np.float32)


def lerp(a, b, t):
    return a + t * (b - a)


def interpolate(corners: np.ndarray, f: np.ndarray) -> np.ndarray:
    """raw [P, 4] fp32 from corners [P, 8, 4] (corner q = dx + 2 dy + 4 dz, fp16 or fp32) and fractions f [P, 3]: along x,
    then y, then z."""
    v = np.asarray(corners).astype(np.float32)
    fx, fy, fz = (f[:, a:a + 1].astype(np.float32) for a in range(3))
    with np.errstate(invalid="ignore", over="ignore"):
        x = [lerp(v[:, q], v[:, q + 1], fx) for q in (0, 2, 4, 6)]   # (dy, dz) = (0, 0), (1, 0), (0, 1), (1, 1)
        y = [lerp(x[0], x[1], fy), lerp(x[2], x[3], fy)]
        return lerp(y[0], y[1], fz)


def corner_index(c: np.ndarray, res) -> np.ndarray:
    """[P, 8] flat vertex indices (k * ny + j) * nx + i of the 8 corners of cells c [P, 3]."""
    nx, ny, _ = res
    q = np.arange(8)
    d = np.stack([q & 1, (q >> 1) & 1, (q >> 2) & 1], 1)   # [8, 3]
    v = c[:, None, :] + d[None]
    return (v[..., 2] * ny + v[..., 1]) * nx + v[..., 0]


def lookup(points: np.ndarray, values: np.ndarray, lo, hi):
    """(inside [P] bool, raw [P, 4] fp32, NaN where not inside) of points in the grid values [nz, ny, nx, 4] fp16."""
    nz, ny, nx, _ = values.shape
    res = (nx, ny, nz)
    inside, c, f = cells(points, res, lo, hi)
    corners = values.reshape(-1, 4)[corner_index(c, res)]
    raw = interpolate(corners, f)
    return inside, np.where(inside[:, None], raw, np.float32(np.nan))
