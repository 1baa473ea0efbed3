"""The density gradient on the GPU (geometry.density_gradient, csrc/field_grad.cu) against its fp64 restatement
(tests/normals_reference.py) on the kernels' fp16-rounded weights, its identities, mesh vertex normals, render's
surface_normals and the normal images."""
import copy

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from nonrigid_nerf_b200 import _lib, evaluation, geometry, ops, train as T
from nonrigid_nerf_b200 import autograd as _ag
from nonrigid_nerf_b200 import run_nerf_helpers as H
from tests import helpers, normals_reference as R, stash_layout as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# Against an fp64 evaluation with its own ReLU masks (free-running), a point within rounding of a kink may take the other
# one-sided derivative; that comparison is reported and its median bounded.  The per-point bound is taken on the kernels'
# own path instead (test_against_fp64_on_the_kernels_masks).
MEDIAN = 1e-2


def _views_model(with_bender):
    torch.manual_seed(11)
    embed_fn, input_ch = H.get_embedder(10, 0)
    bender = None
    if with_bender:
        bender = helpers.load_bender_module(H.ray_bending(input_ch, 32, "simple_neural", embed_fn), O.make_bender_params(13)).to(DEV)
    net = H.NeRF(D=8, W=256, input_ch=input_ch, output_ch=4, skips=[4], input_ch_views=27, use_viewdirs=True, ray_bender=bender,
                 ray_bending_latent_size=32, num_ray_samples=64).to(DEV)
    with torch.no_grad():
        net.alpha_linear.weight.mul_(30.0)
    return net


def _model(kind):
    if kind == "tc":
        return helpers.tc_models(5, DEV)[0]
    if kind.startswith("views"):
        return _views_model(kind == "views_bender")
    coarse, _, _, _ = helpers.build_models(O, 7, DEV, with_bender=kind != "canonical")
    b = coarse.ray_bender[0]
    if kind == "bender_cutoff":
        b.rigidity_test_time_cutoff = 0.5
    elif kind == "bender_scaling":
        b.test_time_scaling = 2.5
    elif kind == "bender_removal":
        coarse.test_time_nonrigid_object_removal_threshold = 0.5
    return coarse


def _knobs(net):
    b = net.ray_bender[0]
    return dict(cutoff=getattr(b, "rigidity_test_time_cutoff", None) if b is not None else None,
                scaling=getattr(b, "test_time_scaling", None) if b is not None else None,
                removal=getattr(net, "test_time_nonrigid_object_removal_threshold", None))


def _points(n, seed=3):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, 3, generator=g) * 2.4 - 1.2).to(DEV)


def _check(net, x, z, kind, report):
    g = geometry.density_gradient(net, x, z)
    _lib.device_error_check()
    npar, bp = R.params(net, fp16=True, device=DEV)
    zz = None if z is None else torch.as_tensor(z, device=DEV)
    ref = R.density_gradient(npar, bp if zz is not None and bp is not None else None, x, zz, tc=kind == "tc", **_knobs(net))
    err = (g.double() - ref).norm(dim=1)
    rel = err / ref.norm(dim=1).clamp_min(1e-6)
    ok = (rel <= 2e-2) | (err <= 1e-6)
    n64, n32 = R.normals(ref), geometry.normals_from_gradient(g).double()
    ang = torch.rad2deg(torch.acos((n64 * n32).sum(1).clamp(-1, 1)))[ref.norm(dim=1) > 1e-6]
    report.append(f"{kind} P={x.shape[0]}: median rel {float(rel.median()):.2e}, within bound {float(ok.double().mean()):.5f}, "
                  f"angle median {float(ang.median()):.3e} deg, p99 {float(ang.quantile(0.99)) if ang.numel() else 0:.3e} deg")
    assert float(rel.median()) <= MEDIAN, report[-1]
    return g


def _tiles(n):
    return ((n + S.TILE_M - 1) // S.TILE_M + 1) // 2 * 2


def _readback(ws, n, layout=None):
    """The last chunk's n points in the workspace of a call of `layout` = min(P, chunk) points (include/nrnerf_b200.h):
    mask bits, E, unmasked offsets, rigidity."""
    layout = n if layout is None else layout
    t = _tiles(layout)
    up = lambda b: (b + 255) // 256 * 256   # noqa: E731
    e_off = up(t * S.MASK_TILE)
    u_off = e_off + up(t * S.E_BYTES)
    r_off = u_off + up(layout * 12)
    masks = {f"H{l + 1}": S.relu_bits(ws, S.MK_H[l][0], 256, t)[:n] for l in range(8)}
    for name, (off, cols) in (("Hb1", S.MK_HB1), ("Hb2", S.MK_HB2), ("Hb3", S.MK_HB3), ("Hb4", S.MK_HB4)):
        masks[name] = S.relu_bits(ws, off, cols, t)[:n]
    E = S.image(ws[e_off:], S.E_BYTES, 0, 8, t)[:n].double()
    un = ws[u_off:u_off + n * 12].view(torch.float32).view(n, 3)
    rig = ws[r_off:r_off + n * 4].view(torch.float32)
    return masks, E, un, rig, (e_off, u_off, r_off)


# Per point, the kernels and R.fixed_mask_chain take the same path (the masks, E, offsets and rigidity read back) with the
# same fp16 weights.  They differ by the fp16 roundings of the chain's gradient operands (8 in the trunk, 6 more with a
# bender) and the fp32 sums: R.rounding_bound carries each through the chain's own linear map to g, to first order.
# SLACK = 2 covers the second-order terms, the fp32 positional-encoding backward and the fp32 bend; ATOL fp16 underflow of
# gradients below 2^-24 / 2^9 in true units.  A saturated fp16 operand (|y| 2^9 > 65504) would break the bound.
SLACK, ATOL = 2.0, 1e-6


def _fixed_mask_check(net, x, z, kind, ws, report):
    n = x.shape[0]
    g = geometry._density_gradient(net, x, z, ws)
    _lib.device_error_check()
    masks, E, un, rig, _ = _readback(ws, n)
    npar, bp = R.params(net, fp16=True, device=DEV)
    bent = bp is not None and z is not None
    kn = _knobs(net) if bent else {}
    ref, bound, sigma = R.rounding_bound(npar, bp if bent else None, masks, E, un, rig, **kn)
    bound = SLACK * bound + ATOL
    err = (g.double() - ref).abs()
    ratio = float((err / bound).max())
    zs = float((err / (sigma + ATOL)).median())
    nz = ref.norm(dim=1) > 1e-6
    ang = torch.rad2deg(torch.acos((R.normals(ref) * geometry.normals_from_gradient(g).double()).sum(1).clamp(-1, 1)))[nz]
    rel = ((g.double() - ref).norm(dim=1) / ref.norm(dim=1).clamp_min(1e-12))[nz]
    report.append(f"{kind} P={n} (kernel masks): max err / bound {ratio:.3f}, median err / sigma {zs:.2f}, median rel {float(rel.median()):.2e}, max rel "
                  f"{float(rel.max()):.2e}, angle max {float(ang.max()):.3e} deg, median {float(ang.median()):.3e} deg")
    assert bool((err <= bound).all()), report[-1]
    # the typical error is that of independent roundings: the median component error is a few sigma at most
    assert zs <= 3.0, report[-1]
    if bent:
        # sigma resolves the bender's part of g: d raw / d bent alone (the bend backward dropped) is many sigma off
        dx = R.fixed_mask_chain(npar, None, masks, E)
        moved = ~(rig.double() >= kn["removal"]) if kn.get("removal") is not None else torch.ones(n, dtype=torch.bool, device=DEV)
        off = ((dx - ref).abs() / (sigma + ATOL)).amax(1)[moved]
        report[-1] += f"; bend backward dropped: median {float(off.median()):.1f} sigma"
        assert float(off.median()) >= 10.0, report[-1]
    return g


KINDS = ["canonical", "bender", "bender_cutoff", "bender_scaling", "bender_removal", "tc", "views", "views_bender"]


def _latent(kind):
    return None if kind in ("canonical", "views") else torch.randn(32, generator=torch.Generator().manual_seed(4)).to(DEV) * 0.3


@pytest.mark.parametrize("kind", KINDS)
def test_against_fp64_on_the_kernels_masks(kind):
    net = _model(kind)
    n = 1000
    ws = torch.empty(_lib.load().nrn_density_gradient_workspace_bytes(n, 0), dtype=torch.uint8, device=DEV)
    report = []
    _fixed_mask_check(net, _points(n), _latent(kind), kind, ws, report)
    print(report[-1])


@pytest.mark.parametrize("kind", KINDS)
def test_forward_matches_the_training_forward(kind):
    """field_fwd_grad_kernel's mask bits, encoding E, offsets and rigidity equal the training forward's (field_fwd.cu)
    for the same points, bit for bit: the encoding and mask epilogues field_grad.cu shares stay those of field_fwd.cu."""
    net = _model(kind)
    n = 1000
    x, z = _points(n), _latent(kind)
    lib = _lib.load()
    ws = torch.empty(lib.nrn_density_gradient_workspace_bytes(n, 0), dtype=torch.uint8, device=DEV)
    geometry._density_gradient(net, x, z, ws)
    _, _, un, rig, (e_off, _, _) = _readback(ws, n)
    tc = _ag._tc_net(net)
    bent = net.ray_bender[0] is not None and z is not None
    rays = torch.cat([x, torch.zeros(n, 3, device=DEV), torch.full((n, 1), 0.5, device=DEV), torch.full((n, 1), 2.0, device=DEV)], 1)
    zv = torch.ones(n, 1, device=DEV)   # o + 0 * z = o: the same points
    stash = torch.empty(lib.nrn_stash_bytes(n, 1), dtype=torch.uint8, device=DEV)
    mask = torch.empty(lib.nrn_relu_mask_bytes(n, 1), dtype=torch.uint8, device=DEV)
    kn = _knobs(net) if bent else dict(cutoff=None, scaling=None, removal=None)
    out_ch = 4 if getattr(net, "use_viewdirs", False) else net.output_linear.weight.shape[0]
    _, det = ops.field_forward(rays, zv, z.expand(n, 32) if z is not None else None, ops.pack_nerf(net),
                               ops.pack_bender(net.ray_bender[0]) if bent else None, out_ch, kn["cutoff"], kn["scaling"], kn["removal"],
                               want_details=True, stash=stash, relu_mask=mask, tc_net=tc)
    torch.cuda.synchronize()
    t = _tiles(n)
    mk_ws, mk_tr = ws[:t * S.MASK_TILE].view(t, S.MASK_TILE), mask[:t * S.MASK_TILE].view(t, S.MASK_TILE)
    used = S.MASK_TILE if bent else S.MK_HB1[0]   # without a bender the Hb images are written by neither kernel
    assert torch.equal(mk_ws[:, :used], mk_tr[:, :used])
    e_ws = S.image(ws[e_off:], S.E_BYTES, 0, 8, t).view(torch.int16)
    e_tr = S.image(stash, S.STASH_TILE, S.ST_E[0], 8, t).view(torch.int16)
    assert torch.equal(e_ws, e_tr)
    if bent:
        assert torch.equal(un, det["unmasked_offsets"].reshape(n, 3))
        assert torch.equal(rig, det["rigidity_mask"].reshape(n))


@pytest.mark.parametrize("kind", KINDS)
def test_against_fp64(kind):
    net = _model(kind)
    latent = None if kind in ("canonical", "views") else torch.randn(32, generator=torch.Generator().manual_seed(4)).to(DEV) * 0.3
    report = []
    x = _points(1000)
    g = _check(net, x, latent, kind, report)
    print(report[-1])
    # each point's gradient depends on that point only: 1, 127, 128, 129 and a ragged 1000 - 129 points give the same bits
    for a, b in ((0, 1), (0, 127), (0, 128), (0, 129), (129, 1000)):
        assert torch.equal(geometry.density_gradient(net, x[a:b].clone(), latent), g[a:b]), (a, b)


def test_past_one_chunk_with_per_point_latents():
    net = _model("bender")
    n = _lib.load().nrn_density_gradient_chunk() + 300
    x = _points(n)
    lat = (torch.randn(n, 32, generator=torch.Generator().manual_seed(5)) * 0.3).to(DEV)
    ws = torch.empty(_lib.load().nrn_density_gradient_workspace_bytes(n, 0), dtype=torch.uint8, device=DEV)
    report = []
    g = _check(net, x, lat, "bender", report)
    print(report[-1])
    # the last chunk (300 points) against fp64 on the kernels' own masks: the workspace holds that chunk
    gw = geometry._density_gradient(net, x, lat, ws)
    assert torch.equal(gw, g)
    chunk = _lib.load().nrn_density_gradient_chunk()
    masks, E, un, rig, _ = _readback(ws, n - chunk, chunk)
    npar, bp = R.params(net, fp16=True, device=DEV)
    ref, bound, _ = R.rounding_bound(npar, bp, masks, E, un, rig)
    assert bool(((g[chunk:].double() - ref).abs() <= SLACK * bound + ATOL).all())
    # each point's gradient depends on that point only: the tail of the second chunk alone gives the same bits
    tail = geometry.density_gradient(net, x[-300:].clone(), lat[-300:].clone())
    assert torch.equal(g[-300:], tail)


def test_tc_per_point_latents():
    net = _model("tc")
    x = _points(700)
    lat = (torch.randn(700, 32, generator=torch.Generator().manual_seed(6)) * 0.3).to(DEV)
    report = []
    _check(net, x, lat, "tc", report)
    print(report[-1])
    one = geometry.density_gradient(net, x[:5], lat[3])
    assert torch.equal(one[3], geometry.density_gradient(net, x[3:4], lat[3:4])[0])


def test_non_finite_points():
    net = _model("bender")
    z = torch.randn(32, generator=torch.Generator().manual_seed(4)).to(DEV) * 0.3
    x = _points(300)
    g0 = geometry.density_gradient(net, x, z)
    y = x.clone()
    y[7, 0], y[100, 1], y[200, 2] = float("nan"), float("inf"), float("-inf")
    g = geometry.density_gradient(net, y, z)
    bad = torch.zeros(300, dtype=torch.bool, device=DEV)
    bad[[7, 100, 200]] = True
    assert not torch.isfinite(g[bad]).all(1).any()
    assert torch.equal(g[~bad], g0[~bad])
    n = geometry.normals_from_gradient(g)
    assert torch.equal(n[bad], torch.zeros_like(n[bad]))


def test_zero_offsets_give_the_canonical_gradient_and_reruns_and_graphs_are_bit_identical():
    net = _model("bender")
    x = _points(5000)
    z = torch.randn(32, generator=torch.Generator().manual_seed(4)).to(DEV) * 0.3
    flat = copy.deepcopy(net)
    with torch.no_grad():
        flat.ray_bender[0].network[4].weight.zero_()
    assert torch.equal(geometry.density_gradient(flat, x, z), geometry.density_gradient(net, x))   # latent None: canonical
    a = geometry.density_gradient(net, x, z)
    assert torch.equal(a, geometry.density_gradient(net, x, z))
    # CUDA-graph replay (packs cached by the first calls)
    out = torch.empty_like(a)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        geometry.density_gradient(net, x, z)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            out.copy_(geometry.density_gradient(net, x, z))
    torch.cuda.synchronize()
    out.zero_()
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)


def test_timing_kinds():
    kinds = (_lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + _lib.DET_KERNEL_KINDS
             + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + _lib.MESH_KERNEL_KINDS
             + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS + _lib.OCCUPANCY_KERNEL_KINDS + _lib.TERMINATION_KERNEL_KINDS
             + _lib.DEFORM_KERNEL_KINDS)
    assert len(kinds) == 42
    net = _model("bender")
    _lib.timing_enable(True)
    geometry.density_gradient(net, _points(1000), torch.zeros(32, device=DEV))
    t = _lib.timing_read(kinds + _lib.NORMAL_KERNEL_KINDS)
    _lib.timing_enable(False)
    assert t["density_grad_fwd"][1] == 1 and t["density_grad_dgrad"][1] == 1


@pytest.mark.parametrize("frame", [False, True])
def test_mesh_vertex_normals(frame, tmp_path):
    # a smooth field (the embedding's octaves above 2^1 cut from L0 and L5), so that a 48^3 mesh resolves its surface
    net = _model("bender")
    with torch.no_grad():
        net.pts_linears[0].weight[:, 15:63] = 0.0
        net.pts_linears[5].weight[:, 15:63] = 0.0
    lo, hi = [-1.2] * 3, [1.2] * 3
    sigma = geometry.density_grid(net, lo, hi, 48)
    thr = float(sigma.quantile(0.7))
    mesh = geometry.extract_mesh(net, lo, hi, 48, thr)
    latent = None
    if frame:
        latent = torch.randn(32, generator=torch.Generator().manual_seed(9)).to(DEV) * 0.3
        mesh = geometry.deform_mesh(net.ray_bender[0], mesh, latent).mesh
    assert mesh.vertices.shape[0] > 1000
    n = geometry.vertex_normals(net, mesh, latent)
    assert torch.equal(n, geometry.normals_from_gradient(geometry.density_gradient(net, mesh.vertices, latent)))
    v, f = mesh.vertices.double(), mesh.faces.long()
    fn = torch.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]], dim=1)   # area-weighted, out of the occupied region
    acc = torch.zeros_like(v).index_add_(0, f[:, 0], fn).index_add_(0, f[:, 1], fn).index_add_(0, f[:, 2], fn)
    agree = float(((acc * n.double()).sum(1) > 0).double().mean())
    print(f"frame={frame}: V={v.shape[0]}, sign agreement {agree:.4f}")
    assert agree >= 0.9
    geometry.write_ply(tmp_path / "m.ply", mesh, normals=n)
    geometry.write_obj(tmp_path / "m.obj", mesh, normals=n)
    lines = (tmp_path / "m.obj").read_text().splitlines()
    vn = np.array([[float(t) for t in l.split()[1:]] for l in lines if l.startswith("vn ")], dtype=np.float32)
    assert np.array_equal(vn, n.cpu().numpy())


def test_render_surface_normals_and_images():
    coarse, fine, bender, _ = helpers.build_models(O, 21, DEV)
    r = O.make_rays(21, 2 * 600)
    lat = torch.cat([torch.randn(1, 32).expand(600, 32), torch.randn(1, 32).expand(600, 32)], 0).to(DEV) * 0.1
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=32, network_fine=fine, N_samples=32, network_fn=coarse,
              ray_bender=bender, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    args = (r["rays_o"].to(DEV), r["rays_d"].to(DEV))
    info = {"ray_bending_latents": lat}
    with torch.no_grad():
        base = T.render(*args, chunk=500, near=r["near"], far=r["far"], additional_pixel_information=info, surface_output=True, **kw)
        out = T.render(*args, chunk=500, near=r["near"], far=r["far"], additional_pixel_information=info, surface_output=True,
                       surface_normals=True, **kw)
    for a, b in zip(base[:3], out[:3]):
        assert torch.equal(a, b)
    assert set(out[3]) == set(base[3]) | {"surface_normals"}
    for k in base[3]:
        assert torch.equal(base[3][k], out[3][k]), k
    idx = out[3]["median_indices"]
    # the frame-space point of the median sample: o + d z as render_rays forms it
    with torch.no_grad():
        _, _, _, ex = T.render(*args, chunk=500, near=r["near"], far=r["far"], additional_pixel_information=info, detailed_output=True,
                               **kw)
    rays_o, rays_d = args
    z = ex["fine_initial_input_pts"] if "fine_initial_input_pts" in ex else None
    pts = z[torch.arange(1200, device=DEV), idx] if z is not None else None
    want = geometry.normals_from_gradient(geometry.density_gradient(fine, pts, lat))
    assert torch.equal(out[3]["surface_normals"], want)
    # the ray-sharded render wrapper at world size 1
    from nonrigid_nerf_b200 import parallel
    fn = parallel.get_parallelized_render_function(coarse, fine, bender)
    with torch.no_grad():
        sh = fn(*args, chunk=500, near=r["near"], far=r["far"], additional_pixel_information=info, surface_output=True,
                surface_normals=True, **{k: v for k, v in kw.items() if k not in ("network_fn", "network_fine", "ray_bender")})
    assert torch.equal(sh[3]["surface_normals"], out[3]["surface_normals"])
    # normal images against their numpy restatement, bit for bit
    nrm = out[3]["surface_normals"].reshape(2, 20, 30, 3).contiguous()
    nrm[0, 0, 0] = 0.0
    c2w = torch.stack([torch.eye(4)[:3], torch.tensor(
        [[0.0, -1.0, 0.0, 0.1], [1.0, 0.0, 0.0, 0.2], [0.0, 0.0, 1.0, 0.3]])]).to(DEV)
    img = evaluation.normal_images(nrm, c2w).cpu().numpy()
    n_np, r_np = nrm.cpu().numpy(), c2w[:, :3, :3].cpu().numpy().astype(np.float32)
    want = np.empty(img.shape, np.uint8)
    for f_ in range(2):
        R3 = r_np[f_]
        c = np.stack([(R3[0, k] * n_np[f_, ..., 0] + R3[1, k] * n_np[f_, ..., 1]) + R3[2, k] * n_np[f_, ..., 2] for k in range(3)], -1)
        v = (c + np.float32(1.0)) * np.float32(0.5)
        o = (np.float32(255.0) * np.clip(v, np.float32(0), np.float32(1))).astype(np.uint8)
        o[(n_np[f_] == 0).all(-1)] = 0
        want[f_] = o
    assert np.array_equal(img, want)
    assert img[0, 0, 0].tolist() == [0, 0, 0]
