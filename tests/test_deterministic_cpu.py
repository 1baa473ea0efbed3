"""Deterministic mode on the CPU: the workspace size queries of the fixed-order entry points and every argument check,
each rejected before any CUDA call.  No kernel is launched here."""
import ctypes

from tests.test_div_abi_cpu import _fake, _full_args


def test_sizes():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    assert lib.nrn_latent_rows_bytes(1024, 128) == 1024 * 128 * 32 * 4
    assert lib.nrn_latent_rows_bytes(3, 100) == 3 * 100 * 128
    assert lib.nrn_div_loss_rows_bytes(1024, 64) == 1024 * 64 * 4
    assert lib.nrn_div_loss_rows_bytes(8192, 64) == 8192 * 64 * 4
    # past 2^31 bytes: sizes are computed in size_t
    assert lib.nrn_latent_rows_bytes(65536, 512) == 65536 * 512 * 128
    for f in (lib.nrn_latent_rows_bytes, lib.nrn_div_loss_rows_bytes):
        assert f(0, 64) == 0 and f(-1, 64) == 0 and f(4, 0) == 0


def test_det_kinds_follow_the_view_training_kinds():
    from nonrigid_nerf_b200 import _lib
    kinds = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS
    assert len(kinds) == 13 and _lib.DET_KERNEL_KINDS == ("latent_reduce", "div_loss_reduce")


def _bwd_args(p):
    """Every pointer of a bender backward call set (to a dummy 16-byte aligned address), 4 rays x 64 samples."""
    from nonrigid_nerf_b200 import _lib
    a = _lib.NrnFieldBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = 4, 64, 4
    for name, typ in _lib.NrnFieldBwdArgs._fields_:
        if typ is ctypes.c_void_p and name not in ("stream", "nerf_grad_head", "d_unmasked_offsets", "d_rigidity_mask"):
            setattr(a, name, p)
    return a


def test_field_backward_det_validates_its_arguments():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()

    def bad(a, rows, msg):
        assert lib.nrn_field_backward_det(ctypes.byref(a) if a is not None else None, rows) == -1
        assert msg in lib.nrn_last_error(), lib.nrn_last_error()

    bad(None, p, b"null args")
    a = _bwd_args(p); a.n_samples = 0
    bad(a, p, b"bad sizes")
    a = _bwd_args(p); a.n_rays = -1
    bad(a, p, b"bad sizes")
    a = _bwd_args(p); a.bender_packed = None
    bad(a, p, b"needs a bender")
    a = _bwd_args(p); a.d_latents = None
    bad(a, p, b"d_latents")
    a = _bwd_args(p)
    bad(a, None, b"latent_rows")
    bad(a, ctypes.c_void_p(p.value + 4), b"latent_rows")
    for name in ("d_raw", "stash", "grad_stash", "wgrad_scratch", "nerf_packed", "nerf_grad", "unmasked_offsets",
                 "rigidity_mask", "bender_grad"):
        a = _bwd_args(p); setattr(a, name, None)
        bad(a, p, b"null")
    a = _bwd_args(p); a.relu_mask = None
    bad(a, p, b"relu_mask")
    a = _bwd_args(p); a.out_ch = 6
    bad(a, p, b"out_ch=6")
    for name in ("nerf_packed", "stash", "grad_stash", "relu_mask"):
        a = _bwd_args(p); setattr(a, name, p.value + 4)
        bad(a, p, b"16-byte aligned")
    a = _bwd_args(p); a.n_rays = a.n_samples = 0x7fffffff
    bad(a, p, b"nrn_field_backward_det: too many points")


def test_divergence_forward_det_validates_its_arguments():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()

    def bad(a, rows, msg):
        assert lib.nrn_divergence_forward_det(ctypes.byref(a) if a is not None else None, rows) == -1
        assert msg in lib.nrn_last_error(), lib.nrn_last_error()

    bad(None, p, b"null args")
    a = _full_args(p); a.n_samples = 0
    bad(a, p, b"bad sizes")
    a = _full_args(p); a.relu_mask = None
    bad(a, p, b"relu_mask")
    a = _full_args(p); a.bender_packed = None
    bad(a, p, b"bender_packed")
    a = _full_args(p); a.bender_packed = ctypes.c_void_p(p.value + 4)
    bad(a, p, b"aligned")
    for name in ("e", "unmasked_offsets", "rigidity_mask", "weights", "tangent_stash", "d", "alpha", "beta", "tau_c"):
        a = _full_args(p); setattr(a, name, None)
        bad(a, p, b"null argument")
    a = _full_args(p); a.loss = None
    bad(a, p, b"null loss")
    bad(_full_args(p), None, b"loss_rows")


def test_empty_divergence_batch_returns_before_any_cuda_call():
    """n_rays = 0: OK, and nothing is launched (on a machine without a GPU any CUDA call would fail)."""
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()
    a = _full_args(p); a.n_rays = 0
    assert lib.nrn_divergence_forward_det(ctypes.byref(a), None) == 0
