"""ctypes binding of libnrnerf_b200.so (C ABI declared in include/nrnerf_b200.h).

There is no fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
Build it with `python -c "import __graft_entry__ as g; g.build()"` or `make -C nonrigid_nerf_b200/csrc`.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnrnerf_b200.so")
ABI_VERSION = 2

_f32p = C.POINTER(C.c_float)
_vp = C.c_void_p


class NrnFieldArgs(C.Structure):
    _fields_ = [
        ("rays", _vp), ("z_vals", _vp), ("points", _vp), ("points_stride", C.c_int64),
        ("latents", _vp), ("latent_stride", C.c_int64),
        ("n_rays", C.c_int32), ("n_samples", C.c_int32),
        ("nerf_packed", _vp), ("bender_packed", _vp),
        ("out_ch", C.c_int32),
        ("use_cutoff", C.c_int32), ("rigidity_cutoff", C.c_float),
        ("use_scaling", C.c_int32), ("scaling", C.c_float),
        ("use_removal", C.c_int32), ("removal_threshold", C.c_float),
        ("raw", _vp), ("initial_input_pts", _vp), ("input_pts", _vp), ("unmasked_offsets", _vp),
        ("masked_offsets", _vp), ("rigidity_mask", _vp),
        ("stash", _vp),
        ("stream", _vp),
    ]


class NrnFieldBwdArgs(C.Structure):
    _fields_ = [
        ("n_rays", C.c_int32), ("n_samples", C.c_int32), ("out_ch", C.c_int32),
        ("d_raw", _vp), ("stash", _vp), ("grad_stash", _vp), ("wgrad_scratch", _vp),
        ("nerf_packed", _vp), ("bender_packed", _vp),
        ("unmasked_offsets", _vp), ("rigidity_mask", _vp), ("d_unmasked_offsets", _vp), ("d_rigidity_mask", _vp),
        ("use_cutoff", C.c_int32), ("rigidity_cutoff", C.c_float),
        ("use_scaling", C.c_int32), ("scaling", C.c_float),
        ("nerf_grad", _vp), ("bender_grad", _vp), ("d_latents", _vp),
        ("stream", _vp),
        ("nerf_grad_head", _vp), ("accumulate_nerf", C.c_int32), ("accumulate_bender", C.c_int32),
    ]


class NrnDivArgs(C.Structure):
    _fields_ = [
        ("n_rays", C.c_int32), ("n_samples", C.c_int32),
        ("stash", _vp), ("e", _vp), ("unmasked_offsets", _vp), ("rigidity_mask", _vp), ("weights", _vp),
        ("weights_are_opacity_alpha", C.c_int32),
        ("net_w", C.POINTER(_vp)), ("rig_w", C.POINTER(_vp)),
        ("tangent_stash", _vp), ("d", _vp), ("alpha", _vp), ("beta", _vp), ("tau_c", _vp), ("loss", _vp),
        ("G", _vp), ("g_ray", _vp), ("G_workspace", _vp), ("adjoint_stash", _vp), ("wgrad_scratch", _vp), ("d_unmasked_offsets", _vp),
        ("d_rigidity_mask", _vp), ("bender_grad", _vp),
        ("stream", _vp),
        ("accumulate_bender", C.c_int32),
    ]


class NrnRayLossArgs(C.Structure):
    _fields_ = [
        ("n_rays", C.c_int32), ("n_samples", C.c_int32),
        ("rgb", _vp), ("rgb0", _vp), ("target", _vp), ("weights", _vp), ("unmasked_offsets", _vp), ("rigidity_mask", _vp),
        ("lam_offsets", C.c_float), ("lam_rigidity", C.c_float),
        ("loss", _vp), ("u_rgb", _vp), ("u_rgb0", _vp), ("u_unmasked_offsets", _vp), ("u_rigidity_mask", _vp),
        ("stream", _vp),
        ("sched_step", _vp), ("sched_n_iters", C.c_float), ("divergence", _vp), ("lam_divergence", C.c_float), ("u_divergence", _vp),
    ]


class NrnRayLossBwdArgs(C.Structure):
    _fields_ = [
        ("n_rays", C.c_int32), ("n_samples", C.c_int32), ("g", _vp),
        ("u_rgb", _vp), ("u_rgb0", _vp), ("u_unmasked_offsets", _vp), ("u_rigidity_mask", _vp), ("u_divergence", _vp),
        ("d_rgb", _vp), ("d_rgb0", _vp), ("d_unmasked_offsets", _vp), ("d_rigidity_mask", _vp), ("d_divergence", _vp),
        ("stream", _vp),
    ]


class NrnAdamArgs(C.Structure):
    _fields_ = [
        ("params", _vp), ("exp_avg", _vp), ("exp_avg_sq", _vp), ("grad_ptrs", _vp), ("blocks", _vp), ("n_tensors", C.c_int32), ("n_blocks", C.c_int32),
        ("lr", _vp), ("step", _vp), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("stream", _vp),
    ]


class NrnPeerCtx(C.Structure):
    _fields_ = [
        ("window", _vp * 8), ("world", C.c_int32), ("rank", C.c_int32), ("arena_floats", C.c_int64), ("slot_floats", C.c_int64),
        ("state", _vp), ("reduced", _vp),
    ]


class NrnCompositeArgs(C.Structure):
    _fields_ = [
        ("raw", _vp), ("z_vals", _vp), ("rays_d", _vp), ("rays_d_stride", C.c_int32), ("noise", _vp),
        ("n_rays", C.c_int32), ("n_samples", C.c_int32), ("channels", C.c_int32), ("white_bkgd", C.c_int32),
        ("rgb_map", _vp), ("disp_map", _vp), ("acc_map", _vp), ("depth_map", _vp), ("weights", _vp), ("alpha", _vp),
        ("n_importance", C.c_int32), ("u", _vp), ("z_vals_out", _vp), ("z_std", _vp),
        ("stream", _vp),
    ]


class NrnCompositeBwdArgs(C.Structure):
    _fields_ = [
        ("raw", _vp), ("z_vals", _vp), ("rays_d", _vp), ("rays_d_stride", C.c_int32), ("noise", _vp),
        ("n_rays", C.c_int32), ("n_samples", C.c_int32), ("channels", C.c_int32), ("white_bkgd", C.c_int32),
        ("d_rgb_map", _vp), ("d_acc_map", _vp), ("d_raw", _vp),
        ("stream", _vp),
    ]


# every symbol include/nrnerf_b200.h declares: (restype, argtypes)
SYMBOLS = {
    "nrn_abi_version": (C.c_int, []),
    "nrn_last_error": (C.c_char_p, []),
    "nrn_device_error": (C.c_int, [C.POINTER(C.c_int)]),
    "nrn_packed_nerf_bytes": (C.c_size_t, []),
    "nrn_packed_bender_bytes": (C.c_size_t, []),
    "nrn_pack_nerf": (C.c_int, [C.POINTER(_vp), C.POINTER(_vp), C.c_int, C.c_int, _vp, _vp]),
    "nrn_pack_bender": (C.c_int, [C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.c_int, _vp, _vp]),
    "nrn_sample_coarse": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, _vp, _vp]),
    "nrn_get_rays": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp]),
    "nrn_pack_rays": (C.c_int, [_vp, _vp, C.c_float, C.c_float, C.c_int, _vp, _vp]),
    "nrn_ray_batch": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp]),
    "nrn_median_visibility_index": (C.c_int, [_vp, C.c_int, C.c_int, _vp, _vp]),
    "nrn_field_forward": (C.c_int, [C.POINTER(NrnFieldArgs)]),
    "nrn_composite": (C.c_int, [C.POINTER(NrnCompositeArgs)]),
    "nrn_sample_pdf": (C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, C.c_int, _vp, _vp]),
    "nrn_composite_backward": (C.c_int, [C.POINTER(NrnCompositeBwdArgs)]),
    "nrn_stash_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_grad_stash_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_wgrad_scratch_bytes": (C.c_size_t, []),
    "nrn_nerf_grad_floats": (C.c_int, [C.c_int]),
    "nrn_bender_grad_floats": (C.c_int, []),
    "nrn_field_backward": (C.c_int, [C.POINTER(NrnFieldBwdArgs)]),
    "nrn_div_stash_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_div_grad_stash_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_divergence_forward": (C.c_int, [C.POINTER(NrnDivArgs)]),
    "nrn_divergence_backward": (C.c_int, [C.POINTER(NrnDivArgs)]),
    "nrn_ray_loss": (C.c_int, [C.POINTER(NrnRayLossArgs)]),
    "nrn_scale_rows": (C.c_int, [_vp, _vp, _vp, C.c_int64, C.c_int, _vp]),
    "nrn_ray_loss_backward": (C.c_int, [C.POINTER(NrnRayLossBwdArgs)]),
    "nrn_adam_step": (C.c_int, [C.POINTER(NrnAdamArgs)]),
    "nrn_peer_window_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "nrn_peer_alloc": (C.c_int, [C.c_size_t, C.POINTER(_vp), C.c_char_p]),
    "nrn_peer_open": (C.c_int, [C.c_char_p, C.POINTER(_vp)]),
    "nrn_peer_close": (C.c_int, [_vp]),
    "nrn_peer_free": (C.c_int, [_vp]),
    "nrn_peer_reduce_adam": (C.c_int, [C.POINTER(NrnPeerCtx), C.POINTER(NrnAdamArgs)]),
    "nrn_peer_gather_rows": (C.c_int, [C.POINTER(NrnPeerCtx), _vp, C.c_int, _vp, _vp]),
    "nrn_timing_enable": (C.c_int, [C.c_int]),
    "nrn_timing_read": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_int]),
}

KERNEL_KINDS = ("field_fwd", "field_dgrad", "wgrad", "composite", "composite_bwd", "divergence")


def timing_enable(on: bool) -> None:
    check(load().nrn_timing_enable(1 if on else 0), "timing_enable")


def timing_read():
    """{kind: (total_ms, launches)} for the launches recorded since timing_enable(True)."""
    n = len(KERNEL_KINDS)
    ms = (C.c_double * n)()
    cnt = (C.c_int * n)()
    check(load().nrn_timing_read(ms, cnt, n), "timing_read")
    return {k: (ms[i], cnt[i]) for i, k in enumerate(KERNEL_KINDS)}

_lib = None
_lock = threading.Lock()


def load() -> C.CDLL:
    """Load the extension once; fail loudly when it is absent or of the wrong ABI version."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"nonrigid_nerf_b200: CUDA extension not found at {LIB_PATH}. There is no CPU/PyTorch fallback; "
                "build it with `make -C nonrigid_nerf_b200/csrc` (needs nvcc, sm_90a).")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError => symbol missing => broken build
            fn.restype = res
            fn.argtypes = args
        v = lib.nrn_abi_version()
        if v != ABI_VERSION:
            raise RuntimeError(f"nonrigid_nerf_b200: ABI version mismatch (library {v}, bindings {ABI_VERSION})")
        _lib = lib
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().nrn_last_error()
        raise RuntimeError(f"nrnerf_b200 {what} failed (code {rc}): {msg.decode() if msg else '?'}")


def device_error_check() -> None:
    """Synchronise and raise if any fused kernel recorded a device-side protocol error."""
    code = C.c_int(0)
    check(load().nrn_device_error(C.byref(code)), "device check")
