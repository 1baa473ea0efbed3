"""numpy restatement of the occupancy grid (csrc/occupancy.cu): the build from corner densities, the bit layout, the point
lookup and the compaction, in the same fp32 operations."""
import numpy as np


def build(sigma: np.ndarray, threshold: float, dilation: int) -> np.ndarray:
    """occupied [nz, ny, nx] bool from sigma [nz + 1, ny + 1, nx + 1]: any corner > threshold or NaN, then dilated by
    `dilation` cells in the Chebyshev sense."""
    s = np.asarray(sigma, np.float32)
    t = np.float32(threshold)
    v = ~(s <= t)
    occ = np.zeros((s.shape[0] - 1, s.shape[1] - 1, s.shape[2] - 1), bool)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                occ |= v[dz:dz + occ.shape[0], dy:dy + occ.shape[1], dx:dx + occ.shape[2]]
    for axis in range(3):
        out = occ.copy()
        n = occ.shape[axis]
        for sft in range(1, min(dilation, n - 1) + 1):
            lo = [slice(None)] * 3
            hi = [slice(None)] * 3
            lo[axis], hi[axis] = slice(0, n - sft), slice(sft, n)
            out[tuple(lo)] |= occ[tuple(hi)]
            out[tuple(hi)] |= occ[tuple(lo)]
        occ = out
    return occ


def pack(occ: np.ndarray) -> np.ndarray:
    """int32 words: cell c = (k * ny + j) * nx + i at bit c % 32 of word c // 32."""
    flat = np.asarray(occ, bool).reshape(-1)
    words = (flat.size + 31) // 32
    padded = np.zeros(words * 32, bool)
    padded[:flat.size] = flat
    return np.packbits(padded, bitorder="little").view("<i4").copy()


def unpack(bits: np.ndarray, shape) -> np.ndarray:
    n = int(np.prod(shape))
    return np.unpackbits(np.asarray(bits, "<i4").view(np.uint8), bitorder="little")[:n].astype(bool).reshape(shape)


def scale(lo, hi, res) -> np.ndarray:
    """fl(n / fl(hi - lo)) per axis; res = (nx, ny, nz)."""
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    return (np.asarray(res, np.float32) / (hi - lo)).astype(np.float32)


def cells(points: np.ndarray, res, lo, hi) -> np.ndarray:
    """[P] int64 flat cell index (k * ny + j) * nx + i of each point, -1 outside the box or non-finite; res = (nx, ny, nz)."""
    x = np.asarray(points, np.float32).reshape(-1, 3)
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    res = np.asarray(res)
    with np.errstate(invalid="ignore"):
        inside = np.all((x >= lo) & (x <= hi), axis=1)
        c = np.floor((x - lo) * scale(lo, hi, res))
    c = np.minimum(np.where(inside[:, None], c, 0).astype(np.int64), res - 1)
    return np.where(inside, (c[:, 2] * res[1] + c[:, 1]) * res[0] + c[:, 0], -1)


def keep(points: np.ndarray, occ: np.ndarray, lo, hi) -> np.ndarray:
    """[P] bool: outside the box or non-finite, or in an occupied cell of occ [nz, ny, nx]."""
    nz, ny, nx = occ.shape
    c = cells(points, (nx, ny, nz), lo, hi)
    return (c < 0) | occ.reshape(-1)[np.maximum(c, 0)]


def compact(points: np.ndarray, occ: np.ndarray, lo, hi):
    """(kept xyz [K, 3], kept indices [K] ascending)."""
    x = np.asarray(points, np.float32).reshape(-1, 3)
    idx = np.nonzero(keep(x, occ, lo, hi))[0].astype(np.int32)
    return x[idx], idx
