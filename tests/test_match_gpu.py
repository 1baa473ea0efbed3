"""GPU tests of frame correspondences (correspondence.match_frames): bit for bit against the brute-force restatement
tests/match_reference.py on edge cases and random frames in every pairing mode, against a chunked brute force in torch at
504 x 378 and 1008 x 756 and over 86 frame pairs, reruns and CUDA-graph replay, a synthetic occluder for the round trip,
and the flow of two rendered frames against reprojection."""
import math

import numpy as np
import pytest
import torch

from tests import match_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _match(*args, **kw):
    from nonrigid_nerf_b200 import correspondence as M
    return M.match_frames(*args, **kw)


def _same(ours, ref):
    index, distance, flow, consistent = ref
    assert np.array_equal(ours.index.cpu().numpy(), index)
    assert np.array_equal(ours.distance.cpu().numpy(), distance)
    assert np.array_equal(ours.flow.cpu().numpy(), flow, equal_nan=True)
    if consistent is not None:
        assert np.array_equal(ours.consistent.cpu().numpy(), consistent)


def check(query, target, query_mask=None, target_mask=None, **kw):
    """match_frames on the GPU equals the restatement bit for bit; returns the GPU result."""
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    out = _match(t(query), t(target), t(query_mask), t(target_mask), **kw)
    _same(out, R.match(query, target, query_mask, target_mask, **kw))
    return out


def surface(rs, f, h, w, shift=0.0, noise=1e-3):
    """Frames of a wavy height field seen from above, shifted by `shift` per frame: [f, h, w, 3] fp32."""
    u, v = np.meshgrid(np.linspace(-1, 1, w), np.linspace(-0.75, 0.75, h))
    out = []
    for k in range(f):
        uu = u + shift * k
        z = 0.2 * np.sin(3 * uu) * np.cos(2 * v)
        out.append(np.stack([uu, v, z], -1) + noise * rs.randn(h, w, 3))
    return np.stack(out).astype(np.float32)


def test_tiny_frames():
    check(np.zeros((1, 1, 1, 3), np.float32), np.ones((1, 1, 1, 3), np.float32), round_trip=True)
    rs = np.random.RandomState(0)
    q, t = rs.randn(1, 5, 4, 3).astype(np.float32), rs.randn(1, 3, 7, 3).astype(np.float32)
    mask = np.zeros((1, 3, 7), bool)
    mask[0, 2, 5] = True                                   # a single valid target point: every query matches it
    out = check(q, t, target_mask=mask, round_trip=True)
    assert (out.index == 2 * 7 + 5).all()
    out = check(q, t, target_mask=np.zeros((1, 3, 7), bool), round_trip=True)   # all targets masked
    assert (out.index == -1).all() and torch.isinf(out.distance).all() and torch.isnan(out.flow).all()
    assert not out.consistent.any()


def test_one_cell_and_duplicates():
    rs = np.random.RandomState(1)
    same = np.broadcast_to(np.float32([0.5, -2.0, 3.0]), (1, 20, 30, 3)).copy()   # a flat box on every axis: one cell
    check(rs.randn(1, 9, 11, 3).astype(np.float32), same, round_trip=True)
    dup = (np.round(rs.randn(2, 40, 50, 3) * 2) / 4).astype(np.float32)           # many exact duplicates: ties
    out = check(dup, dup[::-1].copy(), round_trip=True)
    assert out.index.min() >= 0
    check(dup, dup, round_trip=True, round_trip_pixels=0.0)


def test_max_distance_boundary():
    t = np.zeros((1, 1, 4, 3), np.float32)
    t[0, 0, :, 0] = [1.0, -1.0, np.nextafter(np.float32(2), np.float32(3)), 3.0]
    q = np.zeros((1, 2, 2, 3), np.float32)
    q[0, 0, 1, 0] = 4.0
    q[0, 1, 0] = [4.0, 2.0, 0.0]
    for md in (1.0, np.nextafter(np.float32(1), np.float32(0)), 2.0, float(np.nextafter(np.float32(2), np.float32(3))), 0.0, math.inf):
        check(q, t, max_distance=float(md), round_trip=True)
    out = _match(torch.from_numpy(q).to(DEV), torch.from_numpy(t).to(DEV), max_distance=1.0)
    assert out.index[0, 0, 0] == 0 and out.index[0, 0, 1] == 3 and out.index[0, 1, 0] == -1


def test_non_finite_points():
    rs = np.random.RandomState(2)
    q = rs.randn(2, 13, 17, 3).astype(np.float32)
    t = rs.randn(2, 15, 11, 3).astype(np.float32)
    for a in (q, t):
        flat = a.reshape(-1, 3)
        pick = rs.choice(len(flat), 60, replace=False)
        flat[pick[:20], 0] = np.nan
        flat[pick[20:40], 1] = np.inf
        flat[pick[40:], 2] = -np.inf
    check(q, t, round_trip=True)
    check(q, t, rs.rand(2, 13, 17) > 0.3, rs.rand(2, 15, 11) > 0.3, round_trip=True, max_distance=0.5)


def test_cluster_with_far_outliers():
    rs = np.random.RandomState(3)
    t = (rs.randn(1, 30, 40, 3) * 1e-3).astype(np.float32)
    flat = t.reshape(-1, 3)
    flat[:5] = [[1e6, 0, 0], [-1e6, 3, 0], [0, 0, 1e5], [2e4, -3e4, 7e3], [0, 1e7, -1e7]]
    q = (rs.randn(1, 20, 20, 3) * 1e-3).astype(np.float32)
    qf = q.reshape(-1, 3)
    qf[:8] = [[5e5, 0, 0], [-3e6, 0, 0], [0, 0, -1e6], [1e4, 1e4, 1e4], [0, 2e7, -2e7], [1e30, 0, 0], [-1e38, 1e38, 0], [0.5, 0.5, 0.5]]
    check(q, t, round_trip=True)
    check(q, t, round_trip=True, max_distance=1e4)


@pytest.mark.parametrize("fq,ft", [(3, 3), (1, 4), (4, 1)])
def test_random_frames_each_pairing(fq, ft):
    rs = np.random.RandomState(10 + fq + ft)
    q = surface(rs, fq, 23, 31, shift=0.02)
    t = surface(rs, ft, 29, 19, shift=0.03)
    out = check(q, t, round_trip=True, round_trip_pixels=1.5)
    assert tuple(out.index.shape) == (max(fq, ft), 23, 31) and tuple(out.flow.shape) == (max(fq, ft), 23, 31, 2)
    check(q, t, rs.rand(fq, 23, 31) > 0.2, rs.rand(ft, 29, 19) > 0.2, max_distance=0.05, round_trip=True)
    # [F, H*W, 3] as surface_pts stacks, with the frame sizes given
    flat = _match(torch.from_numpy(q.reshape(fq, -1, 3)).to(DEV), torch.from_numpy(t.reshape(ft, -1, 3)).to(DEV),
                  round_trip=True, round_trip_pixels=1.5, size=(23, 31), target_size=(29, 19))
    for a, b in zip(flat, out):
        assert torch.equal(a, b)


def brute_force_torch(q, t, tvalid, qrows, chunk):
    """Nearest valid target (index, d2) of the query points q[qrows] by a chunked brute force in torch: each elementwise
    operation is its own kernel, rounded as the _rn intrinsics round; argmin takes the first minimum."""
    cand = torch.nonzero(tvalid).reshape(-1)
    p = t[cand]
    idx, d2 = [], []
    for s in range(0, len(qrows), chunk):
        qq = q[qrows[s:s + chunk]]
        dx = p[None, :, 0] - qq[:, None, 0]
        dy = p[None, :, 1] - qq[:, None, 1]
        dz = p[None, :, 2] - qq[:, None, 2]
        dd = (dx * dx + dy * dy) + dz * dz
        k = torch.argmin(dd, dim=1)
        idx.append(cand[k])
        d2.append(torch.gather(dd, 1, k[:, None])[:, 0])
    return torch.cat(idx).int(), torch.cat(d2)


def _against_torch(q, t, tmask, out, f, qf, tf, rows, chunk):
    qp, tp = q[qf].reshape(-1, 3), t[tf].reshape(-1, 3)
    tv = torch.isfinite(tp).all(-1) & tmask[tf].reshape(-1)
    j, d2 = brute_force_torch(qp, tp, tv, rows, chunk)
    assert torch.equal(out.index[f].reshape(-1)[rows], j)
    assert torch.equal(out.distance[f].reshape(-1)[rows], torch.sqrt(d2))


def test_full_frames_504x378():
    rs = np.random.RandomState(4)
    q = torch.from_numpy(surface(rs, 1, 378, 504)).to(DEV)
    t = torch.from_numpy(surface(rs, 1, 378, 504, shift=0.01)[0:1] + np.float32(0.004)).to(DEV)
    tmask = torch.from_numpy(rs.rand(1, 378, 504) > 0.1).to(DEV)
    out = _match(q, t, target_mask=tmask)
    _against_torch(q, t, tmask, out, 0, 0, 0, torch.arange(378 * 504, device=DEV), 256)


def test_sampled_queries_1008x756():
    rs = np.random.RandomState(5)
    q = torch.from_numpy(surface(rs, 1, 756, 1008)).to(DEV)
    t = torch.from_numpy(surface(rs, 1, 756, 1008, shift=0.01) + np.float32(0.002)).to(DEV)
    tmask = torch.ones(1, 756, 1008, dtype=torch.bool, device=DEV)
    out = _match(q, t, round_trip=True)
    rows = torch.from_numpy(rs.choice(756 * 1008, 8192, replace=False)).to(DEV)
    _against_torch(q, t, tmask, out, 0, 0, 0, rows, 64)


def test_86_frame_pairs_in_one_call():
    rs = np.random.RandomState(6)
    q = torch.from_numpy(surface(rs, 86, 48, 64, shift=0.01)).to(DEV)
    t = torch.from_numpy(surface(rs, 87, 48, 64, shift=0.01)[1:].copy()).to(DEV)   # frame i against frame i + 1
    tmask = torch.from_numpy(rs.rand(86, 48, 64) > 0.05).to(DEV)
    out = _match(q, t, target_mask=tmask, round_trip=True)
    for f in range(86):
        _against_torch(q, t, tmask, out, f, f, f, torch.arange(48 * 64, device=DEV), 3072)
    # tracking frame 0 through the sequence, and every frame against frame 0
    for fq, ft in ((1, 86), (86, 1)):
        qq, tt = q[:fq], t[:ft]
        o = _match(qq, tt, target_mask=tmask[:ft])
        for f in (0, 41, 85):
            _against_torch(qq, tt, tmask[:ft], o, f, 0 if fq == 1 else f, 0 if ft == 1 else f, torch.arange(48 * 64, device=DEV), 3072)


def test_reruns_and_graph_replay_are_bit_identical():
    rs = np.random.RandomState(7)
    q = torch.from_numpy(surface(rs, 4, 60, 80, shift=0.02)).to(DEV)
    t = torch.from_numpy(surface(rs, 4, 60, 80, shift=0.02) + np.float32(0.003)).to(DEV)
    kw = dict(round_trip=True, max_distance=0.1)
    first = _match(q, t, **kw)
    for _ in range(3):
        for a, b in zip(_match(q, t, **kw), first):
            assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _match(q, t, **kw)                                  # warm the allocator outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = _match(q, t, **kw)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(captured, first):
        assert torch.equal(a, b)


def test_round_trip_fails_behind_an_occluder():
    """Frame A sees a plane z = 0; frame B sees the same plane except where a square far in front of it hides it.  Pixels of A
    behind the square match plane points at the square's rim in B, which match back to the rim in A: the round trip fails
    there and holds everywhere else."""
    h, w = 40, 50
    u, v = np.meshgrid(np.arange(w, dtype=np.float32) * np.float32(0.01), np.arange(h, dtype=np.float32) * np.float32(0.01))
    a = np.stack([u, v, np.zeros_like(u)], -1)[None]
    b = a.copy()
    inside = np.zeros((h, w), bool)
    inside[10:30, 15:35] = True
    b[0, inside, 2] = 5.0
    out = check(a, b, round_trip=True, round_trip_pixels=1.0)
    cons = out.consistent[0].cpu().numpy()
    assert cons[~inside].all()
    assert not cons[12:28, 17:33].any()


def test_rendered_flow_agrees_with_reprojection():
    """Two frames of a model with a fresh bender (identity deformation) from cameras 0.01 apart: for pixels with
    acc_map > 0.5 the matched flow is compared with the projection of the query pixel's surface point into the target
    camera (get_rays intrinsics)."""
    import oracle.nrnerf_oracle as O
    from tests import helpers
    from nonrigid_nerf_b200 import run_nerf_helpers as H, train as T

    embed_fn, input_ch = H.get_embedder(10, 0)
    torch.manual_seed(0)
    bender = H.ray_bending(input_ch, 32, "simple_neural", embed_fn).to(DEV)   # fresh: its last layer is zero, rays stay straight
    nets = dict(D=8, W=256, input_ch=input_ch, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False,
                ray_bender=bender, ray_bending_latent_size=32)
    coarse = helpers.load_nerf_module(H.NeRF(num_ray_samples=64, **nets), O.make_nerf_params(31, 5, 30.0)).to(DEV)
    fine = helpers.load_nerf_module(H.NeRF(num_ray_samples=128, **nets), O.make_nerf_params(32, 5, 30.0)).to(DEV)
    h, w = 96, 128
    intrin = {"height": h, "width": w, "focal_x": 64.0, "focal_y": 64.0, "center_x": 64.0, "center_y": 48.0}
    r = O.make_rays(0, 1)
    poses = []
    for dx in (0.0, 0.01):
        c2w = torch.eye(4)[:3].clone()
        c2w[:, 3] = torch.tensor([0.05 + dx, -0.02, 0.4])
        poses.append(c2w.to(DEV))
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=64, network_fine=fine, N_samples=64, network_fn=coarse,
              ray_bender=bender, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False,
              near=r["near"], far=r["far"])
    pts, accs = [], []
    with torch.no_grad():
        for c2w in poses:
            ro, rd = H.get_rays(c2w, intrin)
            lat = torch.zeros(1, 32, device=DEV).expand(h * w, 32)
            _, _, acc, ex = T.render(ro.reshape(-1, 3), rd.reshape(-1, 3), chunk=4096,
                                     additional_pixel_information={"ray_bending_latents": lat}, surface_output=True, **kw)
            pts.append(ex["surface_pts"].reshape(h, w, 3))
            accs.append(acc.reshape(h, w))
    q, t = torch.stack(pts[:1]), torch.stack(pts[1:])
    out = _match(q, t, accs[0][None] > 0.5, accs[1][None] > 0.5, round_trip=True, round_trip_pixels=1.5)

    def project(p, c2w):
        loc = (p - c2w[:, 3]) @ c2w[:, :3]
        return (intrin["center_x"] + intrin["focal_x"] * loc[..., 0] / -loc[..., 2],
                intrin["center_y"] + intrin["focal_y"] * loc[..., 1] / loc[..., 2])

    jj, ii = torch.meshgrid(torch.arange(h, device=DEV), torch.arange(w, device=DEV), indexing="ij")
    x0, y0 = project(pts[0], poses[0])                      # the projection convention: its own camera gives the pixel back
    sel = accs[0] > 0.5
    assert sel.float().mean() > 0.2
    assert float((x0 - ii)[sel].abs().max()) < 1e-2 and float((y0 - jj)[sel].abs().max()) < 1e-2
    x1, y1 = project(pts[0], poses[1])
    ok = sel & (out.index[0] >= 0)
    err = torch.hypot(out.flow[0, ..., 0] - (x1 - ii), out.flow[0, ..., 1] - (y1 - jj))[ok]
    cons = out.consistent[0][ok]
    q50, q90 = float(err.quantile(0.5)), float(err.quantile(0.9))
    print(f"rendered flow vs reprojection over {int(ok.sum())} pixels: median {q50:.3f} px, 90th percentile {q90:.3f} px, "
          f"max {float(err.max()):.3f} px; round trip holds for {float(cons.float().mean()):.3f}; "
          f"median error where it holds {float(err[cons].quantile(0.5)) if cons.any() else float('nan'):.3f} px")
    assert q50 <= FLOW_MEDIAN_BOUND and q90 <= FLOW_P90_BOUND
    assert float(cons.float().mean()) >= 0.3 and float(err[cons].quantile(0.5)) <= FLOW_CONSISTENT_MEDIAN_BOUND


# Bounds on the flow error in pixels, from this test's own printout on one H100 80GB HBM3 (700 W): over the 12288 pixels
# with acc_map > 0.5 in the query frame and a match, median 1.49 px, 90th percentile 7.99 px (max 25.8 px); the round trip
# held for 47 % of them, with a median error of 0.44 px there.  The seeded model's density is random, so its median-
# visibility "surface" is view dependent and noisy; the bounds leave about a third of headroom over what was measured.
FLOW_MEDIAN_BOUND = 2.0
FLOW_P90_BOUND = 10.5
FLOW_CONSISTENT_MEDIAN_BOUND = 0.6
