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
ABI_VERSION = 4

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
        ("relu_mask", _vp),
    ]


class NrnViewArgs(C.Structure):
    _fields_ = [
        ("views_packed", _vp), ("viewdirs", _vp), ("viewdirs_stride", C.c_int64), ("workspace", _vp),
    ]


class NrnViewTrainArgs(C.Structure):
    _fields_ = [("views_stash", _vp), ("hv_mask", _vp)]


class NrnViewBwdArgs(C.Structure):
    _fields_ = [("views_t_packed", _vp), ("views_stash", _vp), ("views_grad_stash", _vp), ("hv_mask", _vp)]


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
        ("relu_mask", _vp),
    ]


class NrnTcBwdArgs(C.Structure):
    _fields_ = [
        ("latents", _vp), ("latent_stride", C.c_int64), ("w0", _vp), ("w5", _vp), ("d_latents", _vp), ("workspace", _vp),
    ]


class NrnDivArgs(C.Structure):
    _fields_ = [
        ("n_rays", C.c_int32), ("n_samples", C.c_int32),
        ("relu_mask", _vp), ("e", _vp), ("unmasked_offsets", _vp), ("rigidity_mask", _vp), ("weights", _vp),
        ("weights_are_opacity_alpha", C.c_int32),
        ("bender_packed", _vp),
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


class NrnImageScoreArgs(C.Structure):
    _fields_ = [
        ("gt", _vp), ("generated", _vp), ("mask", _vp),
        ("n_frames", C.c_int32), ("height", C.c_int32), ("width", C.c_int32),
        ("psnr", _vp), ("ssim", _vp), ("ssim_map", _vp), ("error_rgb", _vp), ("error_ssim", _vp),
        ("workspace", _vp), ("stream", _vp),
    ]


class NrnFrameImageArgs(C.Structure):
    _fields_ = [
        ("rgb", _vp), ("disp", _vp), ("surface_pts", _vp), ("surface_rigidity", _vp),
        ("min_point", _vp), ("max_point", _vp),
        ("n_frames", C.c_int32), ("height", C.c_int32), ("width", C.c_int32),
        ("disp_max", _vp),
        ("out_rgb", _vp), ("out_disp", _vp), ("out_disp_video", _vp), ("out_disp_jet", _vp), ("out_disp_phong", _vp),
        ("out_correspondences", _vp), ("out_rigidity", _vp), ("out_rigidity_jet", _vp),
        ("stream", _vp),
    ]


class NrnMeshSlabArgs(C.Structure):
    _fields_ = [
        ("sigma0", _vp), ("sigma1", _vp), ("min_point", _vp), ("max_point", _vp),
        ("threshold", C.c_float),
        ("nx", C.c_int32), ("ny", C.c_int32), ("nz", C.c_int32), ("k", C.c_int32),
        ("workspace", _vp), ("totals", _vp),
        ("vertex_base_prev", C.c_int64), ("vertex_base", C.c_int64), ("face_base", C.c_int64),
        ("vertices", _vp), ("faces", _vp),
        ("stream", _vp),
    ]


class NrnLpipsArgs(C.Structure):
    _fields_ = [
        ("gt", _vp), ("generated", _vp), ("mask", _vp),
        ("n_frames", C.c_int32), ("height", C.c_int32), ("width", C.c_int32),
        ("packed", _vp), ("lpips", _vp), ("per_layer", _vp),
        ("workspace", _vp), ("workspace_bytes", C.c_size_t), ("stream", _vp),
    ]


class NrnLpipsMapArgs(C.Structure):
    _fields_ = [("map", _vp), ("layer_maps", _vp), ("error_image", _vp)]


class NrnMatchArgs(C.Structure):
    _fields_ = [
        ("query", _vp), ("target", _vp), ("query_mask", _vp), ("target_mask", _vp),
        ("n_query_frames", C.c_int32), ("query_height", C.c_int32), ("query_width", C.c_int32),
        ("n_target_frames", C.c_int32), ("target_height", C.c_int32), ("target_width", C.c_int32),
        ("max_distance", C.c_float), ("round_trip", C.c_int32), ("round_trip_pixels", C.c_float),
        ("index", _vp), ("distance", _vp), ("flow", _vp), ("consistent", _vp),
        ("workspace", _vp), ("workspace_bytes", C.c_size_t), ("stream", _vp),
    ]


class NrnOccupancyGrid(C.Structure):
    _fields_ = [
        ("bits", _vp), ("nx", C.c_int32), ("ny", C.c_int32), ("nz", C.c_int32),
        ("min_point", C.c_float * 3), ("max_point", C.c_float * 3),
    ]


class NrnTerminationArgs(C.Structure):
    _fields_ = [("threshold", C.c_float), ("noise", _vp), ("termination_index", _vp)]


class NrnDeformArgs(C.Structure):
    _fields_ = [
        ("points", _vp), ("n_points", C.c_int64),
        ("latents", _vp), ("n_latents", C.c_int32), ("latent_stride", C.c_int64),
        ("bender_packed", _vp),
        ("use_cutoff", C.c_int32), ("rigidity_cutoff", C.c_float), ("use_scaling", C.c_int32), ("scaling", C.c_float),
        ("iterations", C.c_int32), ("tol", C.c_float),
        ("out", _vp), ("residual", _vp), ("converged", _vp), ("rigidity", _vp),
        ("stream", _vp),
    ]


class NrnDensityGradArgs(C.Structure):
    _fields_ = [
        ("points", _vp), ("n_points", C.c_int64), ("points_stride", C.c_int64),
        ("latents", _vp), ("latent_stride", C.c_int64),
        ("nerf_packed", _vp), ("bender_packed", _vp),
        ("tc_w0", _vp), ("tc_b0", _vp), ("tc_w5", _vp), ("tc_b5", _vp),
        ("use_cutoff", C.c_int32), ("rigidity_cutoff", C.c_float), ("use_scaling", C.c_int32), ("scaling", C.c_float),
        ("use_removal", C.c_int32), ("removal_threshold", C.c_float),
        ("grad", _vp), ("workspace", _vp), ("workspace_bytes", C.c_size_t),
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
    "nrn_relu_mask_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_wgrad_scratch_bytes": (C.c_size_t, []),
    "nrn_nerf_grad_floats": (C.c_int, [C.c_int]),
    "nrn_bender_grad_floats": (C.c_int, []),
    "nrn_field_backward": (C.c_int, [C.POINTER(NrnFieldBwdArgs)]),
    "nrn_tc_latent_bias": (C.c_int, [_vp, C.c_int64, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nrn_field_forward_tc": (C.c_int, [C.POINTER(NrnFieldArgs), _vp]),
    "nrn_nerf_tc_grad_floats": (C.c_int, [C.c_int]),
    "nrn_tc_workspace_bytes": (C.c_size_t, [C.c_int]),
    "nrn_packed_views_bytes": (C.c_size_t, []),
    "nrn_pack_views": (C.c_int, [C.POINTER(_vp), C.POINTER(_vp), _vp, _vp]),
    "nrn_views_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_field_forward_views": (C.c_int, [C.POINTER(NrnFieldArgs), C.POINTER(NrnViewArgs)]),
    "nrn_field_backward_tc": (C.c_int, [C.POINTER(NrnFieldBwdArgs), C.POINTER(NrnTcBwdArgs)]),
    "nrn_packed_views_t_bytes": (C.c_size_t, []),
    "nrn_pack_views_t": (C.c_int, [C.POINTER(_vp), _vp, _vp]),
    "nrn_views_stash_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_views_grad_stash_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_hv_mask_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_nerf_views_grad_floats": (C.c_int, []),
    "nrn_field_forward_views_train": (C.c_int, [C.POINTER(NrnFieldArgs), C.POINTER(NrnViewArgs), C.POINTER(NrnViewTrainArgs)]),
    "nrn_field_backward_views": (C.c_int, [C.POINTER(NrnFieldBwdArgs), C.POINTER(NrnViewBwdArgs)]),
    "nrn_div_stash_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_div_grad_stash_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_divergence_forward": (C.c_int, [C.POINTER(NrnDivArgs)]),
    "nrn_divergence_backward": (C.c_int, [C.POINTER(NrnDivArgs)]),
    "nrn_latent_rows_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_div_loss_rows_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_field_backward_det": (C.c_int, [C.POINTER(NrnFieldBwdArgs), _vp]),
    "nrn_divergence_forward_det": (C.c_int, [C.POINTER(NrnDivArgs), _vp]),
    "nrn_field_backward_held_out": (C.c_int, [C.POINTER(NrnFieldBwdArgs), _vp]),
    "nrn_field_backward_det_held_out": (C.c_int, [C.POINTER(NrnFieldBwdArgs), _vp, _vp]),
    "nrn_divergence_backward_held_out": (C.c_int, [C.POINTER(NrnDivArgs), _vp]),
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
    "nrn_jet_colormap": (C.c_int, [_vp, _vp]),
    "nrn_image_scores_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "nrn_image_scores": (C.c_int, [C.POINTER(NrnImageScoreArgs)]),
    "nrn_disparity_images": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    "nrn_frame_std_image": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    "nrn_frame_images": (C.c_int, [C.POINTER(NrnFrameImageArgs)]),
    "nrn_mesh_grid_points": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp]),
    "nrn_mesh_sigma": (C.c_int, [_vp, C.c_longlong, C.c_int, _vp, _vp]),
    "nrn_mesh_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "nrn_mesh_count": (C.c_int, [C.POINTER(NrnMeshSlabArgs)]),
    "nrn_mesh_emit": (C.c_int, [C.POINTER(NrnMeshSlabArgs)]),
    "nrn_mesh_colors": (C.c_int, [_vp, C.c_longlong, C.c_int, _vp, _vp]),
    "nrn_mesh_cube_table": (C.c_int, [_vp, _vp]),
    "nrn_lpips_packed_bytes": (C.c_size_t, []),
    "nrn_lpips_pack": (C.c_int, [C.POINTER(_vp), _vp, _vp]),
    "nrn_lpips_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "nrn_lpips": (C.c_int, [C.POINTER(NrnLpipsArgs)]),
    "nrn_lpips_maps_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "nrn_lpips_maps": (C.c_int, [C.POINTER(NrnLpipsArgs), C.POINTER(NrnLpipsMapArgs)]),
    "nrn_match_workspace_bytes": (C.c_size_t, [C.c_int] * 7),
    "nrn_match": (C.c_int, [C.POINTER(NrnMatchArgs)]),
    "nrn_occupancy_words": (C.c_size_t, [C.c_int] * 3),
    "nrn_occupancy_build_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "nrn_occupancy_build": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, _vp, _vp, _vp]),
    "nrn_occupancy_compact_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "nrn_occupancy_compact": (C.c_int, [C.POINTER(NrnOccupancyGrid), _vp, C.c_int64, C.c_int64, _vp, _vp, _vp, _vp, _vp]),
    "nrn_occupancy_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "nrn_field_forward_occupancy": (C.c_int, [C.POINTER(NrnFieldArgs), C.POINTER(NrnOccupancyGrid), _vp, C.c_size_t]),
    "nrn_termination_segment": (C.c_int, []),
    "nrn_termination_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "nrn_field_forward_terminate": (C.c_int, [C.POINTER(NrnFieldArgs), C.POINTER(NrnOccupancyGrid), C.POINTER(NrnTerminationArgs), _vp,
                                              C.c_size_t]),
    "nrn_deform_points": (C.c_int, [C.POINTER(NrnDeformArgs)]),
    "nrn_density_gradient_chunk": (C.c_int64, []),
    "nrn_density_gradient_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "nrn_field_density_gradient": (C.c_int, [C.POINTER(NrnDensityGradArgs)]),
    "nrn_timing_enable": (C.c_int, [C.c_int]),
    "nrn_timing_read": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_int]),
}

KERNEL_KINDS = ("field_fwd", "field_dgrad", "wgrad", "composite", "composite_bwd", "divergence")
# the time-conditioned baseline's own kernels (ray bias; per-ray sums, d z and latent weight columns), timing kinds 6 and 7
TC_KERNEL_KINDS = ("tc_latent_bias", "tc_latent_bwd")
# the view-dependent head's kernels (bend pass, view-head field kernel), timing kinds 8 and 9
VIEW_KERNEL_KINDS = ("views_bend", "views_field")
# training the view-dependent head (training forward, its DGRAD, its WGRAD + reduce), timing kinds 10 to 12
VIEW_TRAIN_KERNEL_KINDS = ("views_field_train", "views_dgrad", "views_wgrad")
# deterministic mode's fixed-order per-ray reductions (latent gradient, divergence loss), timing kinds 13 and 14
DET_KERNEL_KINDS = ("latent_reduce", "div_loss_reduce")
# the held-out variants of DGRAD and of the divergence backward (render(..., held_out=)), timing kinds 15 and 16
HELD_OUT_KERNEL_KINDS = ("field_dgrad_held_out", "div_bwd_held_out")
# evaluation of rendered frames (image scores, disparity images, background stability), timing kinds 17 to 19
EVAL_KERNEL_KINDS = ("image_scores", "disparity_images", "frame_std_image")
# the saved 8-bit images of rendered frames (disparity maxima + every image), timing kind 20
FRAME_IMAGE_KERNEL_KINDS = ("frame_images",)
# triangle meshes (grid points + density, counts + scans, vertices + faces, vertex colours), timing kinds 21 to 24
MESH_KERNEL_KINDS = ("mesh_points", "mesh_count", "mesh_emit", "mesh_colors")
# LPIPS (mask + input scaling, convolutions, max-pools, distances + per-frame sums), timing kinds 25 to 28
LPIPS_KERNEL_KINDS = ("lpips_input", "lpips_conv", "lpips_pool", "lpips_distance")
# frame correspondences (grid builds, queries with their round trips), timing kinds 29 and 30
MATCH_KERNEL_KINDS = ("match_build", "match_query")
# occupancy grids (grid build; of a render pass: bend pass, lookup + compaction, trunk on the kept points, scatter),
# timing kinds 31 to 35
OCCUPANCY_KERNEL_KINDS = ("occupancy_build", "occupancy_bend", "occupancy_compact", "occupancy_field", "occupancy_scatter")
# early-terminating render passes (bend pass, lookups + compactions, trunk on the kept points, scatters, transmittance
# updates), timing kinds 36 to 40
TERMINATION_KERNEL_KINDS = ("termination_bend", "termination_compact", "termination_field", "termination_scatter",
                            "termination_transmittance")
# the inverse of the ray bender (geometry.deform_points), timing kind 41
DEFORM_KERNEL_KINDS = ("deform",)
# the density gradient (geometry.density_gradient: point-gradient forward, its DGRAD), timing kinds 42 and 43
NORMAL_KERNEL_KINDS = ("density_grad_fwd", "density_grad_dgrad")
# spatial LPIPS maps (evaluation.lpips_maps: the upsampling of the tap maps into per-pixel maps and error images), timing
# kind 44; the rest of the call is timed as LPIPS_KERNEL_KINDS
LPIPS_MAP_KERNEL_KINDS = ("lpips_upsample",)


def timing_enable(on: bool) -> None:
    check(load().nrn_timing_enable(1 if on else 0), "timing_enable")


def timing_read(kinds=KERNEL_KINDS):
    """{kind: (total_ms, launches)} for the launches recorded since timing_enable(True); `kinds` is KERNEL_KINDS,
    KERNEL_KINDS + TC_KERNEL_KINDS, KERNEL_KINDS + TC_KERNEL_KINDS + VIEW_KERNEL_KINDS, that + VIEW_TRAIN_KERNEL_KINDS,
    that + DET_KERNEL_KINDS, that + HELD_OUT_KERNEL_KINDS, that + EVAL_KERNEL_KINDS, that + FRAME_IMAGE_KERNEL_KINDS, that + MESH_KERNEL_KINDS, that + LPIPS_KERNEL_KINDS, that + MATCH_KERNEL_KINDS, that
    + OCCUPANCY_KERNEL_KINDS, that + TERMINATION_KERNEL_KINDS, that + DEFORM_KERNEL_KINDS, that + NORMAL_KERNEL_KINDS or
    that + LPIPS_MAP_KERNEL_KINDS."""
    n = len(kinds)
    ms = (C.c_double * n)()
    cnt = (C.c_int * n)()
    check(load().nrn_timing_read(ms, cnt, n), "timing_read")
    return {k: (ms[i], cnt[i]) for i, k in enumerate(kinds)}

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
