"""GPU tests of evaluation.frame_images (nrn_frame_images) against the numpy restatement in
tests/frame_images_reference.py and golden case O: every uint8 image bit for bit (disp_phong within one level), values
at and just outside [0, 1], canonical points on voxel boundaries and outside the volume, the per-frame and per-stack
disparity maxima, untouched NULL outputs, reruns and CUDA-graph replay, the empty stack, and frames rendered by
render(..., surface_output=True)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import frame_images_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "caseO_frame_images.npz")
IMAGES = ("rgb", "disp", "disp_video", "disp_jet", "disp_phong", "correspondences", "rigidity", "rigidity_jet")


def _ev():
    from nonrigid_nerf_b200 import evaluation
    return evaluation


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _compare(out, ref, label):
    """Every image bit for bit, disp_phong within one level (to8b of the fp32 Phong value against the float64 one);
    returns the number of Phong values one level off."""
    phong_off = 0
    for k in IMAGES:
        got = getattr(out, k)
        if k not in ref:
            assert got is None, (label, k)
            continue
        got = got.cpu().numpy()
        assert got.dtype == np.uint8 and got.shape == ref[k].shape, (label, k, got.shape, ref[k].shape)
        if k == "disp_phong":
            d = np.abs(got.astype(np.int16) - ref[k].astype(np.int16))
            assert d.max() <= 1, (label, int(d.max()))
            phong_off = int((d != 0).sum())
        else:
            bad = got != ref[k]
            assert not bad.any(), (label, k, int(bad.sum()), np.argwhere(bad)[:3].tolist())
    print(f"{label}: disp_phong one level off at {phong_off} values")
    return phong_off


@pytest.mark.parametrize("f,h,w", [(1, 1, 1), (1, 7, 5), (3, 24, 32), (37, 756, 1008)])
def test_every_image_equals_the_restatement(f, h, w):
    rgbs, disps, pts, rig, lo, hi = R.seeded_inputs(f, h, w, seed=f * 7919 + h * 31 + w)
    out = _ev().frame_images(_cuda(rgbs), _cuda(disps), _cuda(pts), _cuda(rig), lo.tolist(), hi.tolist())
    ref = R.frame_images(rgbs, disps, pts, rig, lo, hi)
    _compare(out, ref, f"{f}x{h}x{w}")


def test_case_o_golden():
    g = np.load(GOLD)
    out = _ev().frame_images(_cuda(g["rgbs"]), _cuda(g["disps"]), _cuda(g["surface_pts"]), _cuda(g["surface_rigidity"]),
                             g["min_point"], g["max_point"])
    _compare(out, {k: g[k] for k in IMAGES}, "case O")


def test_values_at_the_edges():
    """0, 1, one ulp outside, NaN and +-inf in the colours and the rigidity; canonical points exactly on voxel
    boundaries (extents of 100 * 2^-k, so that every boundary is a float32 number), one ulp either side, below min
    (negative fractions), above max, and non-finite."""
    one, zero = np.float32(1), np.float32(0)
    vals = np.array([0.0, 1.0, -0.0, np.nextafter(one, 2 * one), np.nextafter(zero, -one), np.nextafter(one, zero),
                     np.nextafter(zero, one), 0.5, 1 / 255, 254.5 / 255, np.nan, np.inf, -np.inf, 2.0, -1.0], dtype=np.float32)
    n = len(vals)
    rgbs = np.stack([vals, vals[::-1], np.roll(vals, 3)], axis=-1).reshape(1, 3, 5, 3)
    rig = np.roll(vals, 5).reshape(1, n)
    lo, hi = np.array([-3.125, 0.0, 0.5]), np.array([3.125, 6.25, 3.625])   # extents 6.25, 6.25, 3.125
    j = np.arange(-2, n - 2, dtype=np.float64)[:, None] * 7
    b = lo + (hi - lo) * j / 100                                            # on boundaries (below min for j < 0)
    assert np.array_equal(b.astype(np.float32).astype(np.float64), b)
    b = b.astype(np.float32)
    pts = b.copy()
    pts[1::3] = np.nextafter(b[1::3], np.float32(-np.inf))
    pts[2::3] = np.nextafter(b[2::3], np.float32(np.inf))
    pts[-1] = [np.nan, np.inf, -np.inf]
    pts[-2] = hi.astype(np.float32) * 3
    pts = pts.reshape(1, n, 3)
    disps = np.abs(np.nan_to_num(vals, nan=0.25, posinf=3.0, neginf=0.0)).reshape(1, 3, 5)
    with np.errstate(invalid="ignore", over="ignore"):
        ref = R.frame_images(rgbs, disps, pts, rig, lo, hi)
    out = _ev().frame_images(_cuda(rgbs), _cuda(disps), _cuda(pts), _cuda(rig), lo, hi)
    _compare(out, ref, "edges")
    c = R.correspondence_rgb(pts, lo, hi)
    assert (c < 0).any() and (c == 0).any()
    # a NaN disparity makes its frame's maximum NaN (np.max), so every normalised value is NaN, to8b 0
    dn = disps.copy()
    dn[0, 1, 2] = np.nan
    out = _ev().frame_images(disps=_cuda(dn))
    assert int(out.disp.max()) == 0 and int(out.disp_video.max()) == 0
    assert out.rgb is None and out.correspondences is None and out.rigidity is None


def test_video_uses_the_stack_maximum_and_images_the_frame_maximum():
    d = np.stack([np.full((4, 6), 0.5 * 2.0 ** k, dtype=np.float32) for k in range(3)])   # maxima 0.5, 1, 2
    d[:, 0, 0] = [1.0, 2.0, 4.0]
    out = _ev().frame_images(disps=_cuda(d))
    assert np.all(out.disp[:, 1:].cpu().numpy() == 127)          # 0.5 of each frame's maximum
    video = out.disp_video.cpu().numpy()
    assert np.all(video[0, 1:] == 31) and np.all(video[1, 1:] == 63) and np.all(video[2, 1:] == 127)   # of 4
    assert np.array_equal(out.disp_video.cpu().numpy(), R.disparity_saveable(d))


def test_null_outputs_are_left_untouched():
    from nonrigid_nerf_b200 import _lib
    f, h, w = 2, 9, 11
    rgbs, disps, pts, rig, lo, hi = R.seeded_inputs(f, h, w, seed=5)
    ref = R.frame_images(rgbs, disps, pts, rig, lo, hi)
    ins = {k: _cuda(v) for k, v in (("rgb", rgbs), ("disp", disps), ("surface_pts", pts), ("surface_rigidity", rig))}
    disp_max = torch.full((f,), -7.0, device=DEV)
    lib = _lib.load()
    for keep in (("rgb",), ("disp_video", "correspondences"), ("disp_phong", "rigidity_jet"), ("disp", "rigidity")):
        bufs = {k: torch.full(ref[k].shape, 0xA5, dtype=torch.uint8, device=DEV) for k in IMAGES}
        a = _lib.NrnFrameImageArgs()
        for k, t in ins.items():
            setattr(a, k, t.data_ptr())
        a.min_point, a.max_point = lo.ctypes.data, hi.ctypes.data
        a.n_frames, a.height, a.width = f, h, w
        a.disp_max = disp_max.data_ptr()
        for k in keep:
            setattr(a, "out_" + k, bufs[k].data_ptr())
        a.stream = torch.cuda.current_stream().cuda_stream
        assert lib.nrn_frame_images(C.byref(a)) == 0, lib.nrn_last_error()
        torch.cuda.synchronize()
        for k in IMAGES:
            got = bufs[k].cpu().numpy()
            if k in keep:
                assert np.abs(got.astype(np.int16) - ref[k].astype(np.int16)).max() <= (1 if k == "disp_phong" else 0), (keep, k)
            else:
                assert np.all(got == 0xA5), (keep, k)
    assert np.array_equal(disp_max.cpu().numpy(), disps.reshape(f, -1).max(axis=1))


def test_rerun_and_graph_replay_are_bit_identical():
    ev = _ev()
    rgbs, disps, pts, rig, lo, hi = (_cuda(x) if isinstance(x, np.ndarray) and x.dtype == np.float32 else x
                                     for x in R.seeded_inputs(5, 120, 160, seed=9))
    a = ev.frame_images(rgbs, disps, pts, rig, lo, hi)
    b = ev.frame_images(rgbs, disps, pts, rig, lo, hi)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up on the capture stream
        ev.frame_images(rgbs, disps, pts, rig, lo, hi)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = ev.frame_images(rgbs, disps, pts, rig, lo, hi)
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(a, c):
        assert torch.equal(x, y)
    disps.mul_(0.5)   # a replay reads the inputs anew: the normalised images do not change, the video neither
    rgbs.mul_(0.5)
    g.replay()
    torch.cuda.synchronize()
    d = ev.frame_images(rgbs, disps, pts, rig, lo, hi)
    for x, y in zip(c, d):
        assert torch.equal(x, y)


def test_empty_stack_launches_nothing():
    from nonrigid_nerf_b200 import _lib as L
    ev = _ev()
    kinds = L.KERNEL_KINDS + L.TC_KERNEL_KINDS + L.VIEW_KERNEL_KINDS + L.VIEW_TRAIN_KERNEL_KINDS + L.DET_KERNEL_KINDS + \
        L.HELD_OUT_KERNEL_KINDS + L.EVAL_KERNEL_KINDS + L.FRAME_IMAGE_KERNEL_KINDS
    lo, hi = [0.0] * 3, [1.0] * 3
    torch.cuda.synchronize()
    L.timing_enable(True)
    try:
        out = ev.frame_images(torch.zeros(0, 4, 5, 3, device=DEV), torch.zeros(0, 4, 5, device=DEV),
                              torch.zeros(0, 20, 3, device=DEV), torch.zeros(0, 20, device=DEV), lo, hi)
        ev.frame_images(torch.zeros(2, 0, 5, 3, device=DEV), surface_rigidity=torch.zeros(2, 0, device=DEV))
        empty = L.timing_read(kinds)["frame_images"][1]
        ev.frame_images(torch.zeros(1, 4, 5, 3, device=DEV), torch.ones(1, 4, 5, device=DEV))
        ev.frame_images(torch.zeros(1, 4, 5, 3, device=DEV))
        counts = L.timing_read(kinds)
    finally:
        L.timing_enable(False)
    assert empty == 0
    assert counts["frame_images"][1] == 3   # the disparity maxima and the images, then the images alone
    assert all(c == 0 for k, (_, c) in counts.items() if k != "frame_images")
    assert all(t is not None and t.numel() == 0 for t in out)


def test_rendered_frames_end_to_end():
    """Two 24 x 32 frames rendered by a small bending model with render(..., surface_output=True): the images equal
    the host restatement of free_viewpoint_rendering.py:640-704 on the same tensors copied to the host."""
    import oracle.nrnerf_oracle as O
    from nonrigid_nerf_b200 import _lib, train as T
    from tests import helpers
    seed, h, w = 4321, 24, 32
    coarse, fine, bender, _ = helpers.build_models(O, seed, DEV)
    kw = dict(network_query_fn=None, perturb=0.0, N_importance=64, network_fine=fine, N_samples=64, network_fn=coarse,
              ray_bender=bender, use_viewdirs=False, white_bkgd=False, raw_noise_std=0.0, ndc=False, lindisp=False)
    frames = []
    for k in range(2):
        r = O.make_rays(seed + k, h * w)
        lat = r["latents"][:1].to(DEV).expand(h * w, 32)   # one latent per frame
        with torch.no_grad():
            rgb, disp, _, ex = T.render(r["rays_o"].reshape(h, w, 3).to(DEV), r["rays_d"].reshape(h, w, 3).to(DEV),
                                        chunk=1024, near=r["near"], far=r["far"],
                                        additional_pixel_information={"ray_bending_latents": lat}, surface_output=True, **kw)
        frames.append((rgb, disp, ex["surface_pts"].reshape(h * w, 3), ex["surface_rigidity"].reshape(h * w)))
    _lib.device_error_check()
    rgbs, disps, pts, rig = (torch.stack([fr[i] for fr in frames]) for i in range(4))
    # the volume extent as a checkpoint stores it: Python floats
    p = pts.cpu().numpy().reshape(-1, 3).astype(np.float64)
    lo, hi = (p.min(axis=0) - 0.01).tolist(), (p.max(axis=0) + 0.01).tolist()
    out = _ev().frame_images(rgbs, disps, pts, rig, lo, hi)
    ref = R.frame_images(rgbs.cpu().numpy(), disps.cpu().numpy(), pts.cpu().numpy(), rig.cpu().numpy(), lo, hi)
    _compare(out, ref, "rendered")
    assert len(np.unique(ref["correspondences"])) > 20 and ref["rigidity"].std() > 0
