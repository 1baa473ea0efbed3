"""CPU-only tests of the ReLU mask buffer that the training forward writes for DGRAD: its size and the argument checks
that keep a training call from running without it.  No kernel is launched here."""
import ctypes


def test_relu_mask_bytes_follow_the_stash_tiles():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    assert lib.nrn_relu_mask_bytes(1024, 64) == 512 * 40_960       # 8 x 4 KB (H1..H8) + 4 x 2 KB (Hb1..Hb4) per tile
    assert lib.nrn_relu_mask_bytes(1, 7) == 2 * 40_960              # one ragged tile, rounded up to a tile pair like the stash
    assert lib.nrn_relu_mask_bytes(0, 64) == 0


def _fake(n=16):
    buf = ctypes.create_string_buffer(n + 16)
    return ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15), buf   # 16-byte aligned, never dereferenced


def test_training_forward_without_relu_mask_is_rejected():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()
    a = _lib.NrnFieldArgs()
    a.rays = a.z_vals = a.nerf_packed = a.raw = a.stash = p
    a.n_rays, a.n_samples, a.out_ch = 4, 64, 4
    assert lib.nrn_field_forward(ctypes.byref(a)) == -1
    assert b"relu_mask" in lib.nrn_last_error()
    a.stash, a.relu_mask = None, p                                   # masks without a stash: not a training call either
    assert lib.nrn_field_forward(ctypes.byref(a)) == -1
    assert b"relu_mask" in lib.nrn_last_error()


def test_backward_without_relu_mask_is_rejected():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()
    a = _lib.NrnFieldBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = 4, 64, 4
    a.nerf_packed = a.nerf_grad = a.d_raw = a.stash = a.grad_stash = a.wgrad_scratch = p
    assert lib.nrn_field_backward(ctypes.byref(a)) == -1
    assert b"relu_mask" in lib.nrn_last_error()


def test_misaligned_buffers_and_too_many_tiles_are_rejected():
    """The kernels move the stashes with bulk copies (16-byte aligned addresses) and count tiles in int: a misaligned
    buffer or more than INT32_MAX tiles comes back as NRN_E_INVALID, naming the entry point called, before any CUDA call."""
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()
    off = p.value + 4

    def bad(rc, who, msg):
        assert rc == -1, (who, lib.nrn_last_error())
        assert lib.nrn_last_error().startswith(who + b": ") and msg in lib.nrn_last_error(), lib.nrn_last_error()

    def fwd_args():
        a = _lib.NrnFieldArgs()
        a.rays = a.z_vals = a.nerf_packed = a.raw = a.stash = a.relu_mask = p
        a.n_rays, a.n_samples, a.out_ch = 4, 64, 4
        return a

    fwd = {b"nrn_field_forward": lambda a: lib.nrn_field_forward(ctypes.byref(a)),
           b"nrn_field_forward_tc": lambda a: lib.nrn_field_forward_tc(ctypes.byref(a), p)}
    for who, call in fwd.items():
        for name in ("stash", "relu_mask"):
            a = fwd_args(); setattr(a, name, off)
            bad(call(a), who, b"16-byte aligned")
        a = fwd_args(); a.n_rays = a.n_samples = 0x7fffffff
        bad(call(a), who, b"too many points")

    def bwd_args():
        a = _lib.NrnFieldBwdArgs()
        a.n_rays, a.n_samples, a.out_ch = 4, 64, 4
        a.nerf_packed = a.nerf_grad = a.d_raw = a.stash = a.grad_stash = a.wgrad_scratch = a.relu_mask = p
        return a

    t = _lib.NrnTcBwdArgs()
    t.latents = t.w0 = t.w5 = t.d_latents = t.workspace = p
    t.latent_stride = 32
    bwd = {b"nrn_field_backward": lambda a: lib.nrn_field_backward(ctypes.byref(a)),
           b"nrn_field_backward_tc": lambda a: lib.nrn_field_backward_tc(ctypes.byref(a), ctypes.byref(t))}
    for who, call in bwd.items():
        for name in ("nerf_packed", "stash", "grad_stash", "relu_mask"):
            a = bwd_args(); setattr(a, name, off)
            bad(call(a), who, b"16-byte aligned")
        a = bwd_args(); a.n_rays = a.n_samples = 0x7fffffff
        bad(call(a), who, b"too many points")
