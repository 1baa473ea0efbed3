"""Training the view-dependent head without a bender, on the CPU: the C entry points' sizes and argument checks (each
rejected before any CUDA call), and the refusals that stay (a bender, seated or about to be seated by the wrapper)."""
import ctypes

import pytest
import torch

from tests.test_viewdirs_cpu import _bender, _fake, _net


def test_sizes():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    assert lib.nrn_packed_views_t_bytes() == 200704
    assert lib.nrn_nerf_views_grad_floats() == 595844
    tiles = ((1023 * 64 + 127) // 128 + 1) & ~1   # rounded up to even: 512
    assert lib.nrn_views_stash_bytes(1023, 64) == tiles * 106496
    assert lib.nrn_views_grad_stash_bytes(1023, 64) == tiles * 98304
    assert lib.nrn_hv_mask_bytes(1023, 64) == tiles * 2048
    assert lib.nrn_views_stash_bytes(-1, 64) == 0 and lib.nrn_hv_mask_bytes(4, 0) == 0
    # the view model's parameter count equals the flat layout's
    net = _net()
    assert sum(p.numel() for p in net.parameters()) == lib.nrn_nerf_views_grad_floats()


def test_entry_points_validate_their_arguments():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()
    arr = (ctypes.c_void_p * 3)(p.value, p.value, p.value)
    assert lib.nrn_pack_views_t(None, p, None) == -1 and b"null" in lib.nrn_last_error()
    assert lib.nrn_pack_views_t(arr, ctypes.c_void_p(p.value + 4), None) == -1 and b"aligned" in lib.nrn_last_error()

    def fwd_args():
        a, v, t = _lib.NrnFieldArgs(), _lib.NrnViewArgs(), _lib.NrnViewTrainArgs()
        a.n_rays, a.n_samples, a.out_ch = 4, 64, 4
        a.rays = a.z_vals = a.nerf_packed = a.raw = a.stash = a.relu_mask = p
        v.views_packed, v.viewdirs, v.viewdirs_stride = p, p, 3
        t.views_stash = t.hv_mask = p
        return a, v, t

    def fwd(a, v, t, msg):
        assert lib.nrn_field_forward_views_train(ctypes.byref(a), ctypes.byref(v), ctypes.byref(t)) == -1
        assert msg in lib.nrn_last_error(), lib.nrn_last_error()

    a, v, t = fwd_args(); a.bender_packed = a.latents = p
    fwd(a, v, t, b"not implemented with a ray bender")
    a, v, t = fwd_args(); a.points, a.points_stride = p, 3
    fwd(a, v, t, b"ray mode")
    a, v, t = fwd_args(); a.out_ch = 5
    fwd(a, v, t, b"out_ch=5")
    a, v, t = fwd_args(); a.use_removal = 1
    fwd(a, v, t, b"test-time knob")
    a, v, t = fwd_args(); v.viewdirs = None
    fwd(a, v, t, b"viewdirs")
    a, v, t = fwd_args(); t.hv_mask = None
    fwd(a, v, t, b"hv_mask")
    a, v, t = fwd_args(); a.stash = ctypes.c_void_p(p.value + 8)
    fwd(a, v, t, b"aligned")
    a, v, t = fwd_args(); a.n_samples = 0
    fwd(a, v, t, b"bad sizes")
    assert lib.nrn_field_forward_views_train(None, None, None) == -1

    def bwd_args():
        a, v = _lib.NrnFieldBwdArgs(), _lib.NrnViewBwdArgs()
        a.n_rays, a.n_samples, a.out_ch = 4, 64, 4
        a.d_raw = a.stash = a.grad_stash = a.wgrad_scratch = a.nerf_packed = a.nerf_grad = a.relu_mask = p
        v.views_t_packed = v.views_stash = v.views_grad_stash = v.hv_mask = p
        return a, v

    def bwd(a, v, msg):
        assert lib.nrn_field_backward_views(ctypes.byref(a), ctypes.byref(v)) == -1
        assert msg in lib.nrn_last_error(), lib.nrn_last_error()

    a, v = bwd_args(); a.bender_packed = p
    bwd(a, v, b"not implemented with a ray bender")
    a, v = bwd_args(); a.out_ch = 5
    bwd(a, v, b"out_ch=5")
    a, v = bwd_args(); a.nerf_grad = None
    bwd(a, v, b"nerf_grad")
    a, v = bwd_args(); v.views_grad_stash = None
    bwd(a, v, b"views_grad_stash")
    a, v = bwd_args(); a.relu_mask = None
    bwd(a, v, b"null argument")
    a, v = bwd_args(); v.views_stash = ctypes.c_void_p(p.value + 4)
    bwd(a, v, b"aligned")
    assert lib.nrn_field_backward_views(None, None) == -1


def test_bender_seated_by_the_wrapper_is_refused_before_any_launch():
    """CPU tensors: a launch would fail with a different message, so the error proves nothing ran first."""
    from nonrigid_nerf_b200 import parallel
    views = _net()   # built without a bender
    assert views.ray_bender[0] is None
    lat = [torch.zeros(32, requires_grad=True)]
    wrapper = parallel.training_wrapper_class(views, lat, ray_bender=_bender())
    with pytest.raises(RuntimeError, match="training with the view-dependent head is not implemented"):
        wrapper.forward(None, None, None, 0, {}, torch.zeros(4, 3), 0, 0, {"imageid_to_timestepid": [0]}, torch.zeros(4, 3))
