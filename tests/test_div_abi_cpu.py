"""CPU-only tests of the divergence entry points' arguments (ABI version 4): they take the coarse pass's ReLU mask bits
and packed bender, and refuse to run without them.  No kernel is launched here."""
import ctypes


def test_div_args_carry_relu_mask_and_packed_bender():
    from nonrigid_nerf_b200 import _lib
    names = [f[0] for f in _lib.NrnDivArgs._fields_]
    assert _lib.ABI_VERSION == 4 and _lib.load().nrn_abi_version() == 4
    assert "relu_mask" in names and "bender_packed" in names
    assert not {"stash", "net_w", "rig_w"} & set(names)


def _fake(n=16):
    buf = ctypes.create_string_buffer(n + 16)
    return ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15), buf   # 16-byte aligned, never dereferenced


def _full_args(p):
    """Every pointer of a forward and a backward call set (to a dummy address), sizes of 4 rays x 64 samples."""
    from nonrigid_nerf_b200 import _lib
    a = _lib.NrnDivArgs()
    a.n_rays, a.n_samples = 4, 64
    for name, typ in _lib.NrnDivArgs._fields_:
        if typ is ctypes.c_void_p and name != "stream":
            setattr(a, name, p)
    return a


def test_divergence_calls_without_relu_mask_or_bender_are_rejected():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    p, keep = _fake()
    for call in (lib.nrn_divergence_forward, lib.nrn_divergence_backward):
        a = _full_args(p)
        a.relu_mask = None
        assert call(ctypes.byref(a)) == -1
        assert b"relu_mask" in lib.nrn_last_error()
        a = _full_args(p)
        a.bender_packed = None
        assert call(ctypes.byref(a)) == -1
        assert b"bender_packed" in lib.nrn_last_error()
        a = _full_args(p)
        a.bender_packed = ctypes.c_void_p(p.value + 4)                  # the weight images are read by bulk TMA
        assert call(ctypes.byref(a)) == -1
        assert b"aligned" in lib.nrn_last_error()
