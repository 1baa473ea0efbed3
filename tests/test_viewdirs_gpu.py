"""The view-dependent head (NeRF(use_viewdirs=True), inference): golden case K, the head against its fp64 reference from
the kernel's own h8 and bent points (tests/viewdirs_reference.py), rays that cross tiles, bit-for-bit consistency of the
entry points, the test-time knobs, and the refusal to run under autograd.

Bounds: rendered maps as tests/test_render_gpu.py (RGB / acc L-inf <= 5e-4 against the executed reference)."""
import os

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import stash_layout as SL
from tests.parity import DEV
from tests.viewdirs_reference import build_view_models, directions_fp32, head_reference

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _render(coarse, fine, r, n_samples=64, n_imp=64, chunk=32768, detailed=False, use_viewdirs=True, lat=None, **extra):
    from nonrigid_nerf_b200 import train as T
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=n_imp, network_fine=fine if n_imp > 0 else None,
              N_samples=n_samples, network_fn=coarse, white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    kw.update(extra)
    lat = r["latents"].to(DEV) if lat is None else lat
    return T.render(r["rays_o"].to(DEV), r["rays_d"].to(DEV), chunk=chunk, near=r["near"], far=r["far"], use_viewdirs=use_viewdirs,
                    additional_pixel_information={"ray_bending_latents": lat}, detailed_output=detailed, retraw=True, **kw)


def test_golden_caseK_forward_with_and_without_bender():
    from nonrigid_nerf_b200 import _lib
    g = np.load(os.path.join(GOLD, "caseK_viewdirs.npz"))
    seed, n = int(g["seed"]), int(g["n"])
    r = O.make_rays(seed, n)
    for with_b, pre in ((True, ""), (False, "static_")):
        coarse, fine, bender, (cp, fp, bp, vc, vf) = build_view_models(O, seed, DEV, with_bender=with_b)
        with torch.no_grad():
            rgb, disp, acc, ex = _render(coarse, fine, r, detailed=True)
        _lib.device_error_check()
        assert ex["raw"].shape == (n, 128, 4)
        for name, ours in (("rgb_map", rgb), ("rgb0", ex["rgb0"])) + ((("acc_map", acc),) if with_b else ()):
            d = np.abs(ours.cpu().numpy() - g[pre + name]).max()
            print(f"{pre}{name}: L-inf {d:.3e}")
            assert d <= 5e-4, (pre + name, d)
        ref = g[pre + "raw"]
        got = ex["raw"][:8].cpu().numpy()
        rel = np.abs(got - ref) / (1.0 + np.abs(ref))
        print(f"{pre}raw[:8] vs the reference: max |d| / (1 + |ref|) rgb {rel[..., :3].max():.3e}, alpha {rel[..., 3].max():.3e}")
        assert rel[..., 3].max() <= 5e-3, rel[..., 3].max()   # alpha does not depend on the direction
        # rgb: with a bender the direction is (p_i - p_{i-1}) / |p_i - p_{i-1}|, which magnifies the fp16 bender's error in
        # the bent points by 1 / |p_i - p_{i-1}| (closely spaced fine samples): the kernel's rgb is checked against the
        # oracle evaluated on the kernel's own bent points, where that conditioning no longer enters
        bent = ex["fine_input_pts"][:8].reshape(-1, 3).cpu()
        dirs = directions_fp32(bent, 128) if with_b else (r["rays_d"][:8] / torch.norm(r["rays_d"][:8], dim=-1, keepdim=True))[:, None].expand(8, 128, 3).reshape(-1, 3)
        o = O.nerf_mlp_views(fp, vf, O.positional_encoding(bent), O.direction_encoding(dirs)).reshape(8, 128, 4).numpy()
        rel_o = np.abs(got - o) / (1.0 + np.abs(o))
        print(f"{pre}raw[:8] vs the oracle on the kernel's bent points: max |d| / (1 + |ref|) {rel_o.max():.3e}")
        assert rel_o.max() <= 5e-3, rel_o.max()
        if not with_b:
            assert rel.max() <= 5e-3, rel.max()


def _rays_z(seed, n, s):
    r = O.make_rays(seed, n)
    g = torch.Generator().manual_seed(seed)
    t = torch.sort(torch.rand(n, s, generator=g), -1).values
    z = r["near"] * (1.0 - t) + r["far"] * t
    return r, helpers.rays8(r, DEV), z.float().to(DEV)


def _views_and_h8(net, rays, z, lat, removal=None):
    """raw and details of the view-head path on (rays, z), and h8 of the training kernel on the same points"""
    from nonrigid_nerf_b200 import _lib, ops, autograd as ag
    bender = net.ray_bender[0]
    n, s = z.shape
    vd = torch.nn.functional.normalize(rays[:, 3:6], dim=-1)
    with torch.no_grad():
        raw, det = ag.field_views(net, rays, z, None, lat, vd, True)
        lib = _lib.load()
        stash = torch.empty(lib.nrn_stash_bytes(n, s), dtype=torch.uint8, device=DEV)
        mask = torch.empty(lib.nrn_relu_mask_bytes(n, s), dtype=torch.uint8, device=DEV)
        _, det_t = ops.field_forward(rays, z, lat, ops.pack_nerf(net), ops.pack_bender(bender) if bender is not None else None, 4,
                                     want_details=True, stash=stash, relu_mask=mask)
    _lib.device_error_check()
    P = n * s
    T = (P + 127) // 128
    h8 = SL.image(stash, SL.STASH_TILE, *SL.ST_H[7], T)[:P]
    assert torch.equal(det_t["input_pts"], det["input_pts"]), "training kernel and bend pass bend differently"
    return raw, det, h8, vd


def _check_head(net, raw, det, h8, vd, s, tag):
    bent = det["input_pts"].reshape(-1, 3).cpu()
    n = bent.shape[0] // s
    if net.ray_bender[0] is not None:
        dirs = directions_fp32(bent, s)
    else:
        dirs = vd.cpu()[:, None].expand(n, s, 3).reshape(-1, 3)
    exact, bound = head_reference(net, h8.cpu(), dirs)
    got = raw.reshape(-1, 4).cpu().double()
    assert bool(torch.isfinite(got).all()), tag
    err = (got - exact).abs()
    ratio = (err / bound).max(0).values
    print(f"  [{tag}] rgb / alpha: max |kernel - exact| / bound per channel {[f'{float(x):.3f}' for x in ratio]}")
    assert bool((err <= bound).all()), (tag, int((err > bound).sum()), float(ratio.max()))


@pytest.mark.parametrize("n,s,with_b", [(96, 64, True), (96, 128, True), (50, 192, True), (40, 100, True), (300, 2, True),
                                        (1023, 64, True), (96, 64, False), (45, 100, False)])
def test_view_head_matches_fp64_reference_from_its_own_inputs(n, s, with_b):
    """Every sample of every ray, tiles crossed mid-ray (S = 192, 100), S = 2, a ragged last tile (1023 x 64)."""
    coarse, _, _, _ = build_view_models(O, 3100 + s, DEV, with_bender=with_b, s_coarse=s)
    r, rays, z = _rays_z(3100 + s, n, s)
    raw, det, h8, vd = _views_and_h8(coarse, rays, z, r["latents"].to(DEV))
    _check_head(coarse, raw, det, h8, vd, s, f"n={n} S={s} bender={with_b}")


def test_bend_pass_matches_todays_kernel_and_details_do_not_change_raw():
    from nonrigid_nerf_b200 import ops, autograd as ag
    coarse, _, bender, _ = build_view_models(O, 77, DEV)
    r, rays, z = _rays_z(77, 333, 64)
    lat = r["latents"].to(DEV)
    vd = torch.nn.functional.normalize(rays[:, 3:6], dim=-1)
    with torch.no_grad():
        raw_d, det = ag.field_views(coarse, rays, z, None, lat, vd, True)
        raw_n, _ = ag.field_views(coarse, rays, z, None, lat, vd, False)
        _, det_today = ops.field_forward(rays, z, lat, ops.pack_nerf(coarse), ops.pack_bender(bender), 4, want_details=True)
    for k in ("input_pts", "initial_input_pts", "unmasked_offsets", "masked_offsets", "rigidity_mask"):
        assert torch.equal(det[k], det_today[k]), k
    assert torch.equal(raw_d, raw_n)
    # broadcast latent (stride 0) vs the same row repeated
    one = lat[:1]
    with torch.no_grad():
        raw_b, _ = ag.field_views(coarse, rays, z, None, one.expand(333, 32), vd, False)
        raw_r, _ = ag.field_views(coarse, rays, z, None, one.repeat(333, 1).contiguous(), vd, False)
    assert torch.equal(raw_b, raw_r)


@pytest.mark.parametrize("with_b", [True, False])
def test_entry_points_agree_bit_for_bit(with_b):
    """render chunked vs unchunked; run_network and NeRF.forward(x) vs render_rays' raw; surface_output vs the gather
    from detailed_output."""
    from nonrigid_nerf_b200 import train as T
    seed, n = 515, 150
    coarse, fine, bender, _ = build_view_models(O, seed, DEV, with_bender=with_b)
    r = O.make_rays(seed, n)
    with torch.no_grad():
        rgb, _, _, ex = _render(coarse, fine, r, detailed=True)
        rgb_c, _, _, ex_c = _render(coarse, fine, r, chunk=100, detailed=True)
        _, _, _, ex_s = _render(coarse, fine, r, surface_output=True)
    assert torch.equal(rgb, rgb_c) and torch.equal(ex["raw"], ex_c["raw"]) and torch.equal(ex["rgb0"], ex_c["rgb0"])
    # the fine pass again, point-wise: run_network(inputs [N, S, 3], viewdirs) and NeRF.forward on [P, 63 + 27 + 32]
    pts = ex["fine_initial_input_pts"]
    rd = r["rays_d"].to(DEV)
    vd = rd / torch.norm(rd, dim=-1, keepdim=True)
    lat = r["latents"].to(DEV)
    with torch.no_grad():
        raw_rn = T.run_network(pts, vd, {"ray_bending_latents": lat}, fine, None, None)
        x = torch.zeros(n * 128, 63 + 27 + 32, device=DEV)
        x[:, :3] = pts.reshape(-1, 3)
        x[:, 63:66] = vd[:, None].expand(n, 128, 3).reshape(-1, 3)
        x[:, 90:] = lat[:, None].expand(n, 128, 32).reshape(-1, 32)
        raw_fw = fine(x)
    assert torch.equal(raw_rn, ex["raw"]), float((raw_rn - ex["raw"]).abs().max())
    assert torch.equal(raw_fw.reshape(n, 128, 4), ex["raw"])
    from nonrigid_nerf_b200 import ops
    idx = ex_s["median_indices"]
    assert torch.equal(idx, ops.median_visibility_index(ex["fine_visibility_weights"]))
    surf = torch.gather(ex["fine_input_pts"], 1, idx[:, None, None].expand(n, 1, 3))[:, 0]
    assert torch.equal(ex_s["surface_pts"], surf)
    if with_b:
        rig = torch.gather(ex["fine_rigidity_mask"][..., 0], 1, idx[:, None])[:, 0]
        assert torch.equal(ex_s["surface_rigidity"], rig)


def test_test_time_knobs():
    """Object removal zeroes channel 3 only, at its >= edge; cut-off and scaling against the oracle."""
    from nonrigid_nerf_b200 import autograd as ag
    seed = 808
    coarse, _, bender, (cp, _, bp, vc, _) = build_view_models(O, seed, DEV)
    r, rays, z = _rays_z(seed, 64, 64)
    lat = r["latents"].to(DEV)
    vd = torch.nn.functional.normalize(rays[:, 3:6], dim=-1)
    with torch.no_grad():
        raw0, det = ag.field_views(coarse, rays, z, None, lat, vd, True)
        rig = det["rigidity_mask"].flatten()
        thr = float(rig.sort().values[rig.numel() // 2])   # a value some points have exactly: the >= edge is exercised
        coarse.test_time_nonrigid_object_removal_threshold = thr
        raw1, _ = ag.field_views(coarse, rays, z, None, lat, vd, False)
        coarse.test_time_nonrigid_object_removal_threshold = None
    kill = (rig >= thr).reshape(raw0.shape[:2])
    assert bool(kill.any()) and bool((~kill).any())
    assert torch.equal(raw1[..., :3], raw0[..., :3])
    assert bool((raw1[..., 3][kill] == 0).all()) and torch.equal(raw1[..., 3][~kill], raw0[..., 3][~kill])
    # cut-off and scaling: the bent points (and so the directions) against the oracle's bender
    bender.rigidity_test_time_cutoff, bender.test_time_scaling = 0.45, 1.7
    with torch.no_grad():
        raw2, det2 = ag.field_views(coarse, rays, z, None, lat, vd, True)
    bender.rigidity_test_time_cutoff = bender.test_time_scaling = None
    pts = rays[:, None, :3].cpu() + rays[:, None, 3:6].cpu() * z[..., None].cpu()
    lat_p = r["latents"][:, None].expand(64, 64, 32).reshape(-1, 32)
    ref = O.bender_forward(bp, pts.reshape(-1, 3), lat_p, 0.45, 1.7)
    rm = det2["rigidity_mask"].reshape(-1).cpu()
    keep = (ref["rigidity_mask"].reshape(-1) - 0.45).abs() > 1e-3   # the cut-off decision is only defined up to precision
    assert bool(keep.float().mean() > 0.9)
    np.testing.assert_allclose(rm[keep].numpy(), ref["rigidity_mask"].reshape(-1)[keep].numpy(), atol=3e-4)
    np.testing.assert_allclose(det2["input_pts"].reshape(-1, 3).cpu()[keep].numpy(), ref["bent"][keep].numpy(), atol=2e-4)
    assert bool(torch.isfinite(raw2).all())


def test_no_backward_raises_before_any_launch():
    from nonrigid_nerf_b200 import _lib
    seed, n = 4242, 16
    coarse, fine, bender, _ = build_view_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    _lib.device_error_check()
    lat = r["latents"].to(DEV).requires_grad_(True)
    kinds = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS
    _lib.timing_enable(True)
    try:
        with pytest.raises(RuntimeError, match="use_viewdirs"):
            _render(coarse, fine, r, lat=lat)
        with pytest.raises(RuntimeError, match="use_viewdirs"):   # parameters that require grad alone
            _render(coarse, fine, r)
        with torch.no_grad():   # the same render without autograd does run (and is counted)
            _render(coarse, fine, r)
    finally:
        _lib.timing_enable(False)
    counts = {k: c for k, (_, c) in _lib.timing_read(kinds).items()}
    _lib.device_error_check()
    assert counts["views_bend"] == 2 and counts["views_field"] == 2 and counts["field_fwd"] == 0, counts
