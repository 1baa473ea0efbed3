"""CPU tests of the frame evaluation: the numpy / scipy restatements on hand-computed cases, the library's cm.jet table
against matplotlib's segment data, and the C entry points' size queries and argument checks (no kernel is launched)."""
import ctypes as C

import numpy as np
import pytest

from tests import eval_reference as R


def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


def test_constant_image_has_ssim_one_and_identical_images_psnr_inf():
    img = np.full((16, 17, 3), 0.3, dtype=np.float32)
    score, S = R.ssim(img, img)
    assert score == pytest.approx(1.0, abs=1e-12) and np.allclose(S, 1.0, atol=1e-12)
    assert R.psnr(img, img) == np.inf   # the reference's -10 log10(0)
    other = img.copy()
    other[3, 4, 1] += 0.1
    assert R.psnr(img, other) == pytest.approx(-10 * np.log10(0.01 / (16 * 17 * 3)), rel=1e-6)
    assert np.isnan(R.ssim(img[:10], img[:10])[0])   # a 5-pixel crop of 10 rows leaves nothing to average


def test_ssim_restatement_against_skimage():
    try:
        from skimage.metrics import structural_similarity
    except ImportError as e:
        pytest.skip(f"scikit-image not importable ({e}); the fp64 restatement stands alone")
    gt, gen = R.frames("random", 1, 23, 31, 3)
    score, S = R.ssim(gt[0], gen[0])
    ref, ref_S = structural_similarity(gt[0], gen[0], data_range=1.0, channel_axis=-1, gaussian_weights=True, sigma=1.5,
                                       use_sample_covariance=False, full=True)
    assert score == pytest.approx(ref, abs=1e-12) and np.allclose(S, ref_S, atol=1e-12)


def test_jet_table_endpoints_and_breakpoints():
    lut = R.jet_lut()
    assert np.array_equal(lut[0], [0.0, 0.0, 0.5]) and np.array_equal(lut[255], [0.5, 0.0, 0.0])
    # red rises from 0 at x = 0.35 to 1 at 0.66, green from 0 at 0.125 to 1 at 0.375, blue from 1 at 0.34 to 0 at 0.65
    x = np.arange(256) / 255.0
    assert np.all(lut[x <= 0.35, 0] == 0) and np.all(lut[(x >= 0.66) & (x <= 0.89), 0] == 1)
    assert np.all(lut[x <= 0.125, 1] == 0) and np.all(lut[(x >= 0.375) & (x <= 0.64), 1] == 1) and np.all(lut[x >= 0.91, 1] == 0)
    assert np.all(lut[(x >= 0.11) & (x <= 0.34), 2] == 1) and np.all(lut[x >= 0.65, 2] == 0)
    assert lut[1, 2] == pytest.approx(0.5 + 0.5 * (1.0 / (0.11 * 255)), rel=1e-12)


def test_library_jet_table_is_the_segment_data_table():
    from nonrigid_nerf_b200 import evaluation
    L, lib = _lib()
    assert np.array_equal(evaluation.jet_colormap(), R.jet_lut())
    rgb8 = np.zeros((256, 3), dtype=np.uint8)
    assert lib.nrn_jet_colormap(None, rgb8.ctypes.data_as(C.c_void_p)) == 0
    assert np.array_equal(rgb8, R.to8b(R.jet_lut()))
    assert lib.nrn_jet_colormap(None, None) == -1


def test_jet_table_against_matplotlib():
    try:
        from matplotlib import cm
    except ImportError as e:
        pytest.skip(f"matplotlib not importable ({e}); the table is checked against its segment data instead")
    assert np.array_equal(R.jet_lut(), np.array([cm.jet(i)[:3] for i in range(256)]))


def test_image_scores_workspace_size():
    _, lib = _lib()
    tiles = ((504 + 31) // 32) * ((378 + 7) // 8)
    assert lib.nrn_image_scores_bytes(37, 378, 504) == 37 * tiles * 16 + (378 * 504 + 15) // 16 * 16
    assert lib.nrn_image_scores_bytes(1, 1, 1) == 16 + 16
    assert lib.nrn_image_scores_bytes(0, 7, 13) == 96   # the mask alone
    assert lib.nrn_image_scores_bytes(-1, 7, 13) == 0 and lib.nrn_image_scores_bytes(1, 0, 13) == 0


def _fake(n=64):
    buf = C.create_string_buffer(n + 16)
    return C.c_void_p((C.addressof(buf) + 15) & ~15), buf   # 16-byte aligned, never dereferenced


def _score_args(p, f=2, h=7, w=13):
    L, _ = _lib()
    a = L.NrnImageScoreArgs()
    a.gt = a.generated = a.psnr = a.ssim = a.workspace = p
    a.n_frames, a.height, a.width = f, h, w
    return a


def test_image_scores_rejects_bad_arguments_before_any_cuda_call():
    L, lib = _lib()
    p, keep = _fake()
    assert lib.nrn_image_scores(None) == -1
    for field, value, msg in (("n_frames", -1, b"bad sizes"), ("height", 0, b"bad sizes"), ("width", -3, b"bad sizes"),
                              ("gt", None, b"null"), ("generated", None, b"null"), ("psnr", None, b"null"),
                              ("ssim", None, b"null"), ("workspace", None, b"null"),
                              ("workspace", p.value + 8, b"16-byte aligned"), ("gt", p.value + 2, b"4-byte aligned"),
                              ("ssim_map", p.value + 1, b"4-byte aligned")):
        a = _score_args(p)
        setattr(a, field, value)
        assert lib.nrn_image_scores(C.byref(a)) == -1, field
        assert msg in lib.nrn_last_error(), (field, lib.nrn_last_error())
    a = _score_args(p, f=100000, h=4096, w=4096)   # 3.3e9 tiles
    assert lib.nrn_image_scores(C.byref(a)) == -1 and b"too many" in lib.nrn_last_error()
    # an empty batch is valid and launches nothing, even with every pointer NULL
    a = L.NrnImageScoreArgs()
    a.n_frames, a.height, a.width = 0, 7, 13
    assert lib.nrn_image_scores(C.byref(a)) == 0


def test_disparity_and_std_entry_points_reject_bad_arguments_before_any_cuda_call():
    _, lib = _lib()
    p, keep = _fake()
    assert lib.nrn_disparity_images(p, 1, 0, 5, p, None, None) == -1
    assert lib.nrn_disparity_images(p, -1, 4, 5, p, None, None) == -1
    assert lib.nrn_disparity_images(None, 1, 4, 5, p, p, None) == -1 and b"null" in lib.nrn_last_error()
    assert lib.nrn_disparity_images(p, 1, 4, 5, None, None, None) == -1
    assert lib.nrn_disparity_images(p, 1, 1, 5, None, p, None) == -1 and b"np.gradient" in lib.nrn_last_error()
    assert lib.nrn_disparity_images(p, 1, 4, 1, None, p, None) == -1
    assert lib.nrn_disparity_images(C.c_void_p(p.value + 2), 1, 4, 5, p, None, None) == -1 and b"aligned" in lib.nrn_last_error()
    assert lib.nrn_disparity_images(None, 0, 1, 5, None, None, None) == 0   # empty batch; H = 1 is fine without Phong
    assert lib.nrn_frame_std_image(p, 3, 0, 5, p, p, None) == -1
    assert lib.nrn_frame_std_image(p, -1, 4, 5, p, p, None) == -1
    assert lib.nrn_frame_std_image(None, 3, 4, 5, p, p, None) == -1 and b"null" in lib.nrn_last_error()
    assert lib.nrn_frame_std_image(p, 3, 4, 5, None, None, None) == -1
    assert lib.nrn_frame_std_image(p, 3, 4, 5, C.c_void_p(p.value + 1), None, None) == -1 and b"aligned" in lib.nrn_last_error()
    assert lib.nrn_frame_std_image(None, 0, 4, 5, None, None, None) == 0


def test_timing_kinds_and_drop_in_names():
    from nonrigid_nerf_b200 import _lib as L, run_nerf_helpers as H
    assert L.EVAL_KERNEL_KINDS == ("image_scores", "disparity_images", "frame_std_image")
    kinds = L.KERNEL_KINDS + L.TC_KERNEL_KINDS + L.VIEW_KERNEL_KINDS + L.VIEW_TRAIN_KERNEL_KINDS + L.DET_KERNEL_KINDS + \
        L.HELD_OUT_KERNEL_KINDS
    assert len(kinds) == 17   # the evaluation kinds are 17 to 19
    assert callable(H.visualize_disparity_with_jet_color_scheme) and callable(H.visualize_disparity_with_blinn_phong)
