"""numpy restatement of geometry.marching_cubes (csrc/mesh.cu), written from the specification alone, with its own cube table.

Numbering.  Corner c of a cell sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) in (x, y, z); the case index is the sum of
occupied(c) << c.  Edge e = 4 * axis + r runs along `axis` from its lower corner, whose offsets on the two other axes (in
increasing axis order) are r & 1 and r >> 1.  A grid edge belongs to its lower grid point, so its key is (k, j, i, axis).

Table.  On each of the six faces the crossed edges (one occupied end) are joined by segments: two crossed edges give one
segment; four (an ambiguous face, occupied corners on one diagonal) give two, each cutting off one occupied corner.  Each
segment P -> Q is oriented so that an occupied corner C it separates lies to its right seen from outside the cell:
((Q - P) x (C - P)) . n_out < 0, with P, Q the edge midpoints.  The segments then chain into closed loops (every crossed
edge starts exactly one segment), whose triangles' normals point out of the occupied region.  Loops are taken in order of
their lowest-numbered edge, each started there and fanned: (l0, l1, l2), (l0, l2, l3), ...
"""
import numpy as np

CORNERS = [(c & 1, (c >> 1) & 1, (c >> 2) & 1) for c in range(8)]


def _edge(e):
    axis, r = divmod(e, 4)
    o = [0, 0, 0]
    a1, a2 = [a for a in range(3) if a != axis]
    o[a1], o[a2] = r & 1, r >> 1
    return axis, o[0] | (o[1] << 1) | (o[2] << 2)


EDGES = [_edge(e) for e in range(12)]                      # (axis, lower corner)
EDGE_OFFSETS = [CORNERS[lo] for _, lo in EDGES]            # (dx, dy, dz) of each edge's lower corner


def _ends(e):
    axis, lo = EDGES[e]
    return lo, lo | (1 << axis)


def _mid2(e):
    """Twice the edge midpoint (integers)."""
    axis, lo = EDGES[e]
    return np.array(CORNERS[lo]) * 2 + np.eye(3, dtype=int)[axis]


def _case_triangles(case):
    occ = [(case >> c) & 1 for c in range(8)]
    nxt = {}
    for axis in range(3):
        for side in range(2):
            n_out = np.zeros(3, dtype=int)
            n_out[axis] = 2 * side - 1
            f_edges = [e for e in range(12) if EDGES[e][0] != axis and CORNERS[EDGES[e][1]][axis] == side]
            crossed = [e for e in f_edges if occ[_ends(e)[0]] != occ[_ends(e)[1]]]
            if len(crossed) == 2:
                occupied = [c for c in range(8) if CORNERS[c][axis] == side and occ[c]]
                segs = [(crossed[0], crossed[1], occupied[0])]
            elif len(crossed) == 4:
                segs = []
                for c in range(8):
                    if CORNERS[c][axis] == side and occ[c]:
                        p, q = [e for e in crossed if c in _ends(e)]
                        segs.append((p, q, c))
            else:
                assert not crossed
                segs = []
            for p, q, c in segs:
                mp, mq, mc = _mid2(p), _mid2(q), np.array(CORNERS[c]) * 2
                if np.dot(np.cross(mq - mp, mc - mp), n_out) > 0:
                    p, q = q, p
                assert p not in nxt, (case, p)
                nxt[p] = q
    assert sorted(nxt) == sorted(nxt.values())
    tris, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start
        tris += [(loop[0], loop[i], loop[i + 1]) for i in range(1, len(loop) - 1)]
    return tris


def build_table():
    """(tri_count [256] int, tri_edges [256, max_tris, 3] int (-1 padded))."""
    per_case = [_case_triangles(c) for c in range(256)]
    mx = max(len(t) for t in per_case)
    edges = -np.ones((256, mx, 3), dtype=np.int64)
    for c, t in enumerate(per_case):
        if t:
            edges[c, :len(t)] = t
    return np.array([len(t) for t in per_case], dtype=np.int64), edges


TRI_COUNT, TRI_EDGES = build_table()


def grid_axis(lo, hi, n):
    """x_i = lo + (hi - lo) * (i / (n - 1)) in fp32 (lo, hi rounded to fp32 first; each operation rounded), and x_{n-1} = hi."""
    lo, hi = np.float32(lo), np.float32(hi)
    t = np.arange(n, dtype=np.float32) / np.float32(n - 1)
    x = lo + (hi - lo) * t
    x[-1] = hi
    return x


def grid_points_plane(min_point, max_point, shape_xyz, k):
    """[ny, nx, 3] fp32 points of z-plane k."""
    nx, ny, nz = shape_xyz
    xs, ys, zs = (grid_axis(min_point[a], max_point[a], n) for a, n in enumerate((nx, ny, nz)))
    p = np.empty((ny, nx, 3), dtype=np.float32)
    p[..., 0] = xs[None, :]
    p[..., 1] = ys[:, None]
    p[..., 2] = zs[k]
    return p


def _axes(min_point, max_point, nx, ny, nz):
    return [grid_axis(min_point[a], max_point[a], n) for a, n in enumerate((nx, ny, nz))]


def plane_edges(s0, s1, t):
    """flags [ny, nx, 3] of the edges owned by plane s0's points (+z only when s1, the next plane, is given)."""
    o0 = s0 > t
    f = np.zeros(s0.shape + (3,), dtype=bool)
    f[:, :-1, 0] = o0[:, :-1] != o0[:, 1:]
    f[:-1, :, 1] = o0[:-1, :] != o0[1:, :]
    if s1 is not None:
        f[:, :, 2] = o0 != (s1 > t)
    return f


def plane_vertices(s0, s1, k, axes, t):
    """Vertices [n, 3] of the edges owned by z-plane k (s0 = plane k, s1 = plane k + 1 or None), in (j, i, axis) order."""
    xs, ys, zs = axes
    f = plane_edges(s0, s1, t)
    jj, ii, aa = np.nonzero(f)
    v0 = np.where(np.isnan(s0), np.float32(0), s0)
    v1 = None if s1 is None else np.where(np.isnan(s1), np.float32(0), s1)
    pa = np.stack([xs[ii], ys[jj], np.full(ii.shape, zs[k], dtype=np.float32)], -1)
    ib, jb = ii + (aa == 0), jj + (aa == 1)
    pb = np.stack([xs[np.minimum(ib, len(xs) - 1)], ys[np.minimum(jb, len(ys) - 1)],
                   np.where(aa == 2, zs[min(k + 1, len(zs) - 1)], zs[k]).astype(np.float32)], -1)
    sa = v0[jj, ii]
    sb = np.where(aa == 2, (v1 if v1 is not None else v0)[jj, ii], v0[np.minimum(jb, v0.shape[0] - 1), np.minimum(ib, v0.shape[1] - 1)])
    w = (t - sa) / (sb - sa)
    return (pa + w[:, None] * (pb - pa)).astype(np.float32), f


def _ids(f, base):
    ids = -np.ones(f.shape, dtype=np.int64)
    ids[f] = base + np.arange(int(f.sum()))
    return ids


def layer_faces(s0, s1, ids0, ids1, t):
    """Faces [m, 3] of cell layer between planes s0 and s1, with ids0 / ids1 the vertex ids of both planes' edges."""
    o0, o1 = s0 > t, s1 > t
    case = np.zeros((s0.shape[0] - 1, s0.shape[1] - 1), dtype=np.int64)
    for c, (dx, dy, dz) in enumerate(CORNERS):
        o = o1 if dz else o0
        case |= o[dy:dy + case.shape[0], dx:dx + case.shape[1]].astype(np.int64) << c
    cnt = TRI_COUNT[case]
    jj, ii = np.nonzero(cnt)
    n = cnt[jj, ii]
    cj, ci = np.repeat(jj, n), np.repeat(ii, n)
    m = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
    edges = TRI_EDGES[case[cj, ci], m]                        # [T, 3]
    ax = np.array([a for a, _ in EDGES])[edges]
    off = np.array(EDGE_OFFSETS)[edges]                       # [T, 3, 3]
    both = np.stack([ids0, ids1])                             # [2, ny, nx, 3]
    return both[off[..., 2], cj[:, None] + off[..., 1], ci[:, None] + off[..., 0], ax]


def slab(planes, k, axes, t, vbase):
    """Plane k's vertices and cell layer k's faces, from sigma planes k, k + 1, k + 2 (as many as exist) and the global id of
    plane k's first vertex: (vertices, faces, number of vertices of plane k)."""
    s0 = planes[0]
    s1 = planes[1] if len(planes) > 1 else None
    verts, f0 = plane_vertices(s0, s1, k, axes, t)
    if s1 is None:
        return verts, np.zeros((0, 3), dtype=np.int64), len(verts)
    f1 = plane_edges(s1, planes[2] if len(planes) > 2 else None, t)
    ids0, ids1 = _ids(f0, vbase), _ids(f1, vbase + len(verts))
    return verts, layer_faces(s0, s1, ids0, ids1, t), len(verts)


def marching_cubes(sigma, min_point, max_point, threshold):
    """(vertices [V, 3] fp32, faces [T, 3] int64, vertex offset of each plane [nz + 1], face offset of each layer [nz])."""
    sigma = np.asarray(sigma, dtype=np.float32)
    nz, ny, nx = sigma.shape
    t = np.float32(threshold)
    axes = _axes(min_point, max_point, nx, ny, nz)
    vs, fs, voff, foff = [], [], [0], []
    for k in range(nz):
        v, f, n = slab(sigma[k:k + 3], k, axes, t, voff[-1])
        foff.append(sum(len(x) for x in fs))
        vs.append(v)
        fs.append(f)
        voff.append(voff[-1] + n)
    return (np.concatenate(vs).reshape(-1, 3), np.concatenate(fs).reshape(-1, 3), np.array(voff, dtype=np.int64),
            np.array(foff, dtype=np.int64))
