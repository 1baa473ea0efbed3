"""CPU tests of the saved frame images (evaluation.frame_images): the numpy restatement against golden case O, the C
entry point's argument checks (each rejected before any CUDA call, on pointers that are never dereferenced) and the
Python wrapper's shape and device refusals."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import frame_images_reference as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "caseO_frame_images.npz")
IMAGES = ("rgb", "disp", "disp_video", "disp_jet", "disp_phong", "correspondences", "rigidity", "rigidity_jet")


def test_restatement_equals_case_o_bit_for_bit():
    g = np.load(GOLD)
    out = R.frame_images(g["rgbs"], g["disps"], g["surface_pts"], g["surface_rigidity"], g["min_point"], g["max_point"])
    assert sorted(out) == sorted(IMAGES)
    for k in IMAGES:
        assert out[k].dtype == np.uint8 and out[k].shape == g[k].shape, k
        assert np.array_equal(out[k], g[k]), (k, int((out[k] != g[k]).sum()))
    # the inputs reach what the fixture is for: negative fractions, both ends of to8b, frames of different maxima
    c = R.correspondence_rgb(g["surface_pts"], g["min_point"], g["max_point"])
    assert (c < 0).any() and (c == 0).any() and (g["correspondences"] == 254).any()
    assert len(np.unique(g["disps"].reshape(3, -1).max(axis=1))) == 3
    assert (g["rigidity"] == 0).any() and (g["rigidity"] == 255).any() and (g["rgb"] == 0).any() and (g["rgb"] == 255).any()


def test_correspondence_truncates_toward_zero():
    lo, hi = np.zeros(3), np.ones(3)
    p = np.array([[[-0.0125, 0.0, 0.5]], [[0.0125, 1.0, 1.0125]]], dtype=np.float32)   # c = -1.25, 0, 50 / 1.25, 100, 101.25
    c = R.correspondence_rgb(p, lo, hi)
    assert c[0, 0, 0] == pytest.approx(-0.25, abs=1e-5) and c[0, 0, 1] == 0 and c[0, 0, 2] == 0
    assert c[1, 0, 0] == pytest.approx(0.25, abs=1e-5) and c[1, 0, 1] == 0 and c[1, 0, 2] == pytest.approx(0.25, abs=1e-4)
    img = np.asarray(R.to8b(c))
    assert img[0, 0, 0] == 0 and img[1, 0, 0] == 63   # a negative fraction clips to 0; c - floor(c) would give 191


def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


def _fake(n=64):
    buf = C.create_string_buffer(n + 16)
    return C.c_void_p((C.addressof(buf) + 15) & ~15), buf   # 16-byte aligned, never dereferenced


def _args(p, lo, hi, f=2, h=7, w=5):
    L, _ = _lib()
    a = L.NrnFrameImageArgs()
    a.rgb = a.disp = a.surface_pts = a.surface_rigidity = a.disp_max = p
    a.min_point, a.max_point = lo.ctypes.data, hi.ctypes.data
    a.n_frames, a.height, a.width = f, h, w
    for k in IMAGES:
        setattr(a, "out_" + k, p)
    return a


def test_entry_point_rejects_bad_arguments_before_any_cuda_call():
    L, lib = _lib()
    p, keep = _fake()
    lo, hi = np.zeros(3), np.ones(3)
    assert lib.nrn_frame_images(None) == -1 and b"null args" in lib.nrn_last_error()
    flat_lo = np.array([0.0, 1.0, 0.0])
    cases = [("n_frames", -1, b"bad sizes"), ("height", -2, b"bad sizes"), ("width", -1, b"bad sizes"),
             ("rgb", None, b"without its input"), ("disp", None, b"without its input"), ("disp_max", None, b"without its input"),
             ("surface_pts", None, b"without its input"), ("min_point", None, b"without its input"),
             ("max_point", None, b"without its input"), ("surface_rigidity", None, b"without its input"),
             ("min_point", flat_lo.ctypes.data, b"must exceed"), ("max_point", lo.ctypes.data, b"must exceed"),
             ("rgb", p.value + 2, b"4-byte aligned"), ("disp", p.value + 1, b"4-byte aligned"),
             ("surface_pts", p.value + 3, b"4-byte aligned"), ("surface_rigidity", p.value + 2, b"4-byte aligned"),
             ("disp_max", p.value + 2, b"4-byte aligned"), ("height", 1, b"np.gradient"), ("width", 1, b"np.gradient")]
    for field, value, msg in cases:
        a = _args(p, lo, hi)
        setattr(a, field, value)
        assert lib.nrn_frame_images(C.byref(a)) == -1, field
        assert msg in lib.nrn_last_error(), (field, lib.nrn_last_error())
    nan = np.array([0.0, np.nan, 0.0])
    a = _args(p, nan, hi)
    assert lib.nrn_frame_images(C.byref(a)) == -1 and b"must exceed" in lib.nrn_last_error()
    a = _args(p, lo, hi, f=1 << 30, h=1 << 20, w=1 << 20)
    assert lib.nrn_frame_images(C.byref(a)) == -1 and b"too many" in lib.nrn_last_error()
    a = _args(p, lo, hi)
    for k in IMAGES:
        setattr(a, "out_" + k, None)
    assert lib.nrn_frame_images(C.byref(a)) == -1 and b"no output" in lib.nrn_last_error()
    # an empty stack (F = 0 or H * W = 0) is valid and launches nothing, even with every pointer NULL
    for f, h, w in ((0, 7, 5), (3, 0, 5), (3, 7, 0)):
        e = L.NrnFrameImageArgs()
        e.n_frames, e.height, e.width = f, h, w
        assert lib.nrn_frame_images(C.byref(e)) == 0, (f, h, w)


def test_wrapper_refusals():
    from nonrigid_nerf_b200 import evaluation as ev
    rgbs, disps = torch.zeros(2, 4, 5, 3), torch.zeros(2, 4, 5)
    pts, rig = torch.zeros(2, 20, 3), torch.zeros(2, 20)
    lo, hi = [0.0, 0.0, 0.0], [1.0, 1.0, 1.0]
    for kw, msg in (
            (dict(), "needs rgbs or disps"),
            (dict(surface_pts=pts, min_point=lo, max_point=hi), "needs rgbs or disps"),
            (dict(rgbs=torch.zeros(2, 4, 5)), "rgbs must be"),
            (dict(disps=torch.zeros(2, 20)), "disps must be"),
            (dict(rgbs=rgbs, disps=torch.zeros(2, 5, 4)), "differ"),
            (dict(rgbs=rgbs, surface_pts=torch.zeros(2, 21, 3), min_point=lo, max_point=hi), "surface_pts must be"),
            (dict(rgbs=rgbs, surface_pts=torch.zeros(3, 20, 3), min_point=lo, max_point=hi), "surface_pts must be"),
            (dict(disps=disps, surface_rigidity=torch.zeros(2, 20, 1)), "surface_rigidity must be"),
            (dict(rgbs=rgbs, surface_pts=pts), "needs min_point and max_point"),
            (dict(rgbs=rgbs, surface_pts=pts, min_point=lo), "needs min_point and max_point"),
            (dict(rgbs=rgbs, surface_pts=pts, min_point=[0.0, 0.0], max_point=hi), "3 values"),
            (dict(rgbs=rgbs, surface_pts=pts, min_point=lo, max_point=[1.0, 0.0, 1.0]), "must exceed"),
            (dict(rgbs=rgbs, disps=disps, surface_pts=pts, surface_rigidity=rig, min_point=lo, max_point=hi), "CUDA tensors"),
            (dict(rgbs=rgbs.numpy()), "CUDA tensors")):
        with pytest.raises(RuntimeError, match=msg):
            ev.frame_images(**kw)


def test_timing_kind():
    from nonrigid_nerf_b200 import _lib as L
    kinds = L.KERNEL_KINDS + L.TC_KERNEL_KINDS + L.VIEW_KERNEL_KINDS + L.VIEW_TRAIN_KERNEL_KINDS + L.DET_KERNEL_KINDS + \
        L.HELD_OUT_KERNEL_KINDS + L.EVAL_KERNEL_KINDS
    assert len(kinds) == 20 and L.FRAME_IMAGE_KERNEL_KINDS == ("frame_images",)   # kind 20
