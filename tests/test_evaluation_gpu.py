"""GPU tests of nonrigid_nerf_b200.evaluation against the fp64 numpy / scipy restatements in tests/eval_reference.py:
PSNR, SSIM and the SSIM map, the error images, the disparity images, the background-stability map; reproducibility,
CUDA-graph replay and NaN inputs."""
import numpy as np
import pytest
import torch

from tests import eval_reference as R

pytestmark = pytest.mark.gpu

# the kernel filters the moments in fp64 and writes S in fp32; the score is its fp64 sum
S_ATOL = 1e-6
SSIM_ATOL = 1e-6
PSNR_RTOL = 1e-6

# Phong in fp32 against fp64, relative to the frame's largest value: the half vector normalises the sum of the light and
# view directions, which nearly cancel where a vertex lies between the origin and the light
PHONG_RTOL = 1e-3

SHAPES = [(1, 1, 1), (1, 7, 13), (1, 11, 11), (1, 378, 504), (1, 756, 1008), (37, 378, 504)]


def _ev():
    from nonrigid_nerf_b200 import evaluation
    return evaluation


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _check_colours(out, idx_ref, value, table):
    """out [..., 3] equals table[idx_ref], except for a +-1 index where value lies within 1e-6 of a bin edge."""
    ok = np.all(out == table[idx_ref], axis=-1)
    near = R.near_bin_edge(value)
    for dk in (-1, 1):
        alt = np.clip(idx_ref.astype(np.int64) + dk, 0, 255)
        ok |= near & np.all(out == table[alt], axis=-1)
    assert ok.all(), f"{(~ok).sum()} pixels off the LUT colour, first at {np.argwhere(~ok)[:3].tolist()}"


def _phong_error(out, ref, lam):
    """max |out - ref| / max |ref| away from pixels whose Lambertian term is ~0 (where fp32 and fp64 may disagree on
    the reference's invalid_mask)."""
    keep = np.abs(lam) > 1e-4
    return float(np.abs(out - ref)[keep].max() / np.abs(ref).max()) if keep.any() else 0.0


@pytest.mark.parametrize("f,h,w", SHAPES)
@pytest.mark.parametrize("kind", ["random", "smooth", "edges", "masked"])
def test_scores_and_ssim_map_against_fp64(kind, f, h, w):
    if f * h * w > 378 * 504 and kind != "random" and kind != "masked":
        pytest.skip("the large sizes run the random and masked frames")
    gt, gen = R.frames(kind, f, h, w, seed=f * 1000 + h + w)
    out = _ev().image_scores(_cuda(gt), _cuda(gen), error_maps=True, ssim_map=True)
    psnr, ssim, smap = out.psnr.cpu().numpy(), out.ssim.cpu().numpy(), out.ssim_map.cpu().numpy()
    err_rgb, err_ssim = out.error_rgb.cpu().numpy(), out.error_ssim.cpu().numpy()
    mask = R.mask_from(gt[0])
    lut8 = R.to8b(R.jet_lut())
    worst = 0.0
    for i in range(f):
        g, r = R.apply_mask(gt[i], gen[i], mask)
        ref_psnr = R.psnr(g, r)
        score, S = R.ssim(g, r)
        if np.isinf(ref_psnr):
            assert np.isinf(psnr[i]) and psnr[i] > 0
        else:
            assert psnr[i] == pytest.approx(ref_psnr, rel=PSNR_RTOL, abs=1e-5)
        if np.isnan(score):
            assert np.isnan(ssim[i])
        else:
            assert ssim[i] == pytest.approx(score, abs=SSIM_ATOL)
        worst = max(worst, float(np.abs(smap[i] - S).max()))
        assert np.abs(smap[i] - S).max() <= S_ATOL, (i, np.abs(smap[i] - S).max())
        v = R.error_rgb_value(g, r)
        _check_colours(err_rgb[i], R.lut_index(v), v, lut8)
        v = R.error_ssim_value(smap[i])   # the colouring of the kernel's own S
        _check_colours(err_ssim[i], R.lut_index(v), v, lut8)
    print(f"{kind} {f}x{h}x{w}: max |S - S_fp64| = {worst:.3e}")


def test_given_mask_and_skimage():
    gt, gen = R.frames("random", 3, 40, 50, seed=7)
    mask = np.zeros((40, 50), dtype=bool)
    mask[5:9, 10:30] = True
    out = _ev().image_scores(_cuda(gt), _cuda(gen), mask=_cuda(mask), ssim_map=True)
    for i in range(3):
        g, r = R.apply_mask(gt[i], gen[i], mask)
        assert out.psnr[i].item() == pytest.approx(R.psnr(g, r), rel=PSNR_RTOL)
        assert out.ssim[i].item() == pytest.approx(R.ssim(g, r)[0], abs=SSIM_ATOL)
    try:
        from skimage.metrics import structural_similarity
    except ImportError as e:
        print(f"scikit-image not importable ({e}): compared against the fp64 restatement only")
        return
    g, r = R.apply_mask(gt[0], gen[0], mask)
    ref, ref_S = structural_similarity(g, r, data_range=1.0, channel_axis=-1, gaussian_weights=True, sigma=1.5,
                                       use_sample_covariance=False, full=True)
    assert out.ssim[0].item() == pytest.approx(ref, abs=SSIM_ATOL)
    assert np.abs(out.ssim_map[0].cpu().numpy() - ref_S).max() <= S_ATOL


def test_identical_frames_give_psnr_inf_and_ssim_one():
    gt, _ = R.frames("random", 2, 30, 40, seed=1)
    out = _ev().image_scores(_cuda(gt), _cuda(gt))
    assert torch.isinf(out.psnr).all() and (out.psnr > 0).all()
    assert torch.allclose(out.ssim, torch.ones_like(out.ssim), atol=1e-5)


def test_two_runs_bit_identical_and_graph_replay_equals_eager():
    ev = _ev()
    gt, gen = R.frames("random", 37, 378, 504, seed=11)
    gt, gen = _cuda(gt), _cuda(gen)
    d = _cuda(np.random.default_rng(2).random((4, 60, 80), dtype=np.float32))
    a = ev.image_scores(gt, gen, error_maps=True, ssim_map=True)
    b = ev.image_scores(gt, gen, error_maps=True, ssim_map=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up on the capture stream
        ev.image_scores(gt, gen, error_maps=True, ssim_map=True)
        ev.disparity_images(d)
        ev.background_stability(gen)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = ev.image_scores(gt, gen, error_maps=True, ssim_map=True)
        dj, dp = ev.disparity_images(d)
        bi, bs = ev.background_stability(gen)
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(a, c):
        assert torch.equal(x, y)
    ej, ep = ev.disparity_images(d)
    ei, es = ev.background_stability(gen)
    assert torch.equal(dj, ej) and torch.equal(dp, ep) and torch.equal(bi, ei) and torch.equal(bs, es)


@pytest.mark.parametrize("f,h,w", [(1, 2, 2), (1, 7, 13), (3, 378, 504)])
def test_disparity_images(f, h, w):
    rng = np.random.default_rng(h * w)
    yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
    d = np.stack([np.clip(0.2 + 0.6 * xx * yy + 0.05 * rng.random((h, w)), 0, 1) for _ in range(f)]).astype(np.float32)
    d[0, 0, 0] = 1.5   # clipped by the jet image
    jet, phong = _ev().disparity_images(_cuda(d))
    jet, phong = jet.cpu().numpy(), phong.cpu().numpy()
    lut = R.jet_lut()
    lutf = lut.astype(np.float32)
    worst = 0.0
    for i in range(f):
        _check_colours(jet[i], R.lut_index(d[i]), d[i], lutf)
        ref, lam = R.phong(d[i])
        err = _phong_error(phong[i], ref, lam)
        worst = max(worst, err)
        assert err <= PHONG_RTOL, err
    print(f"phong {f}x{h}x{w}: max |phong - phong_fp64| / max |phong_fp64| = {worst:.3e}")
    try:
        from matplotlib import cm  # noqa: F401
    except ImportError as e:
        print(f"matplotlib not importable ({e}): jet checked against the segment-data table")


def test_drop_in_names_numpy_and_cuda():
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    d = np.random.default_rng(0).random((20, 30), dtype=np.float32)
    j = H.visualize_disparity_with_jet_color_scheme(d)
    p = H.visualize_disparity_with_blinn_phong(d)
    assert isinstance(j, np.ndarray) and j.shape == (20, 30, 3) and isinstance(p, np.ndarray) and p.shape == (20, 30, 3)
    assert np.array_equal(j, R.jet_lut().astype(np.float32)[R.lut_index(d)])
    ref, lam = R.phong(d)
    assert _phong_error(p, ref, lam) <= PHONG_RTOL
    dc = _cuda(d)
    jc = H.visualize_disparity_with_jet_color_scheme(dc)
    pc = H.visualize_disparity_with_blinn_phong(dc)
    assert jc.is_cuda and pc.is_cuda and np.array_equal(jc.cpu().numpy(), j) and np.array_equal(pc.cpu().numpy(), p)


@pytest.mark.parametrize("f,h,w", [(1, 3, 4), (37, 378, 504)])
def test_background_stability_against_np_std(f, h, w):
    rgbs = np.random.default_rng(f + h).random((f, h, w, 3), dtype=np.float32)
    rgbs[:, : h // 2] *= np.float32(0.02)   # a steady half, whose colours stay low on the jet scale
    image, std = _ev().background_stability(_cuda(rgbs))
    ref_img, ref_std, v = R.std_image(rgbs)
    std = std.cpu().numpy()
    assert np.allclose(std, ref_std, rtol=2e-6, atol=1e-7), np.abs(std - ref_std).max()
    print(f"std {f}x{h}x{w}: {np.mean(std == ref_std):.6f} of the values bit-equal to np.std")
    _check_colours(image.cpu().numpy(), R.lut_index(v), v, R.jet_lut().astype(np.float32))


def test_nan_inputs_follow_the_reference():
    gt, gen = R.frames("random", 2, 40, 50, seed=5)
    gen[0, 20, 25, 1] = np.nan
    gen[1, 0, 0, 0] = np.nan
    out = _ev().image_scores(_cuda(gt), _cuda(gen), error_maps=True, ssim_map=True)
    smap = out.ssim_map.cpu().numpy()
    for i in range(2):
        score, S = R.ssim(gt[i], gen[i])
        assert np.array_equal(np.isnan(smap[i]), np.isnan(S)), i
        assert np.isnan(out.psnr[i].item())
        assert np.isnan(score) == np.isnan(out.ssim[i].item())
    d = np.random.default_rng(1).random((1, 12, 16), dtype=np.float32)
    d[0, 5, 7] = np.nan
    jet, phong = _ev().disparity_images(_cuda(d))
    ref, _ = R.phong(d[0])
    assert np.array_equal(np.isnan(phong[0].cpu().numpy()), np.isnan(ref))
    assert np.array_equal(jet[0, 5, 7].cpu().numpy(), R.jet_lut()[0].astype(np.float32))
    from nonrigid_nerf_b200 import _lib
    _lib.device_error_check()
