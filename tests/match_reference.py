"""numpy restatement of nonrigid_nerf_b200.correspondence.match_frames: brute force over every valid target point in fp32,
d2 = (dx*dx + dy*dy) + dz*dz with each operation rounded on its own (numpy float32 arithmetic does not contract), the
smallest (d2, index) pair, kept when d2 <= fl(max_distance^2).  The round trip matches the matched target point back
against the query frame by the same rule."""
import numpy as np


def _valid(pts, mask):
    ok = np.all(np.isfinite(pts), axis=-1)
    return ok if mask is None else ok & (np.asarray(mask).reshape(ok.shape) != 0)


def nearest(q, pts, valid, max_d2):
    """(index, d2) of the nearest valid point of pts [N, 3] to each q [M, 3] (fp32), -1 / inf where none qualifies."""
    q = np.asarray(q, dtype=np.float32).reshape(-1, 3)
    cand = np.nonzero(valid)[0]
    idx = np.full(len(q), -1, dtype=np.int64)
    d2 = np.full(len(q), np.inf, dtype=np.float32)
    if len(cand) == 0 or len(q) == 0:
        return idx, d2
    p = pts[cand].astype(np.float32)
    step = max(1, (1 << 22) // len(cand))
    with np.errstate(over="ignore", invalid="ignore"):
        for s in range(0, len(q), step):
            qq = q[s:s + step]
            dx = p[None, :, 0] - qq[:, None, 0]
            dy = p[None, :, 1] - qq[:, None, 1]
            dz = p[None, :, 2] - qq[:, None, 2]
            dd = (dx * dx + dy * dy) + dz * dz
            k = np.argmin(dd, axis=1)                # the first minimum: the smallest index among ties
            best = dd[np.arange(len(qq)), k]
            ok = best <= max_d2
            idx[s:s + step] = np.where(ok, cand[k], -1)
            d2[s:s + step] = np.where(ok, best, np.float32(np.inf))
    return idx, d2


def match(query, target, query_mask=None, target_mask=None, max_distance=np.inf, round_trip=False, round_trip_pixels=1.0):
    """query [Fq, Hq, Wq, 3], target [Ft, Ht, Wt, 3] (numpy) -> (index, distance, flow, consistent) as match_frames."""
    query = np.asarray(query, dtype=np.float32)
    target = np.asarray(target, dtype=np.float32)
    fq, hq, wq, _ = query.shape
    ft, ht, wt, _ = target.shape
    assert fq == ft or fq == 1 or ft == 1
    f = fq if (fq == ft or ft == 1) else ft
    max_d2 = np.float32(max_distance) * np.float32(max_distance)
    tol2 = np.float32(round_trip_pixels) * np.float32(round_trip_pixels)
    index = np.full((f, hq * wq), -1, dtype=np.int32)
    distance = np.full((f, hq * wq), np.inf, dtype=np.float32)
    flow = np.full((f, hq * wq, 2), np.nan, dtype=np.float32)
    consistent = np.zeros((f, hq * wq), dtype=bool)
    xq = (np.arange(hq * wq) % wq).astype(np.float32)
    yq = (np.arange(hq * wq) // wq).astype(np.float32)
    for k in range(f):
        qf, tf = (0 if fq == 1 else k), (0 if ft == 1 else k)
        qp, tp = query[qf].reshape(-1, 3), target[tf].reshape(-1, 3)
        qv = _valid(qp, None if query_mask is None else query_mask[qf])
        tv = _valid(tp, None if target_mask is None else target_mask[tf])
        rows = np.nonzero(qv)[0]
        j, d2 = nearest(qp[rows], tp, tv, max_d2)
        hit = rows[j >= 0]
        j, d2 = j[j >= 0], d2[j >= 0]
        index[k, hit] = j
        distance[k, hit] = np.sqrt(d2)
        flow[k, hit, 0] = (j % wt).astype(np.float32) - xq[hit]
        flow[k, hit, 1] = (j // wt).astype(np.float32) - yq[hit]
        if round_trip and len(hit):
            back, _ = nearest(tp[j], qp, qv, max_d2)
            dx = (back % wq).astype(np.float32) - xq[hit]
            dy = (back // wq).astype(np.float32) - yq[hit]
            consistent[k, hit] = (back >= 0) & ((dx * dx + dy * dy) <= tol2)
    shape = (f, hq, wq)
    return index.reshape(shape), distance.reshape(shape), flow.reshape(shape + (2,)), consistent.reshape(shape) if round_trip else None
