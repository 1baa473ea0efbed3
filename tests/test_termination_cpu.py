"""CPU tests of early ray termination: the numpy restatement (tests/termination_reference.py) against an fp64 brute force,
the workspace sizes, the C entry point's argument checks on host pointers (no kernel is launched), and the refusals of
render(..., early_termination=), raised before anything is launched."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import termination_reference as R


def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


def _brute_force(alpha, K, t):
    """fp64: the first segment end at which the product of (1 - alpha + 1e-10) is below t, and how close to t any segment
    end came (relative)."""
    n, S = alpha.shape
    out = np.full(n, S, np.int32)
    margin = np.full(n, np.inf)
    for r in range(n):
        T = 1.0
        for s0 in range(0, S, K):
            s1 = min(s0 + K, S)
            for i in range(s0, s1):
                T *= (1.0 - float(alpha[r, i])) + 1e-10
            margin[r] = min(margin[r], abs(T - t) / t)
            if T < t:
                out[r] = s1
                break
    return out, margin


@pytest.mark.parametrize("S,K", [(64, 16), (100, 16), (192, 32), (5, 16), (1, 16), (67, 8)])
def test_restatement_matches_fp64_away_from_ties(S, K):
    rs = np.random.RandomState(S * 31 + K)
    n = 400
    alpha = (rs.rand(n, S) * rs.choice([0.02, 0.2, 0.6], size=(n, 1))).astype(np.float32)
    alpha[rs.rand(n, S) < 0.02] = 1.0
    for t in (1e-4, 1e-2, 0.5):
        got = R.termination_index(alpha, K, t)
        want, margin = _brute_force(alpha, K, t)
        far = margin > 1e-4
        assert far.mean() > 0.9
        assert np.array_equal(got[far], want[far]), (t, np.nonzero(got[far] != want[far]))
        assert np.all((got == S) | ((got % K == 0) | (got == S)))


def test_restatement_edge_cases():
    alpha = np.array([[0.0] * 8, [1.0] * 8, [np.nan] + [0.9] * 7, [0.5] * 8], np.float32)
    assert R.termination_index(alpha, 4, 0.0).tolist() == [8, 8, 8, 8]      # t = 0 never terminates
    assert R.termination_index(alpha, 4, 1.0).tolist() == [8, 4, 8, 4]      # T = 1 is not < 1; NaN never dies
    assert R.termination_index(alpha, 4, 1e-3).tolist() == [8, 4, 8, 8]     # 0.5^4 = 0.0625, 0.5^8 = 0.0039
    assert R.termination_index(alpha, 3, 0.1).tolist() == [8, 3, 8, 6]      # ragged last segment [6, 8)
    T = R.transmittance_at_death(alpha, 4, 0.1)
    assert T[3] == np.float32(0.5) ** 4 and T[0] == 1.0   # ray 3 died after the first segment


def test_workspace_sizes():
    L, lib = _lib()
    K = lib.nrn_termination_segment()
    assert K in (8, 16, 32, 64)
    a = lambda n: (n + 255) // 256 * 256
    n, S = 1000, 64
    P, Pk = n * S, n * K
    blocks = a(4 * ((Pk + 1023) // 1024 + 1))
    assert lib.nrn_termination_workspace_bytes(n, S, 5, 1) == a(16 * P) + a(12 * Pk) + a(4 * Pk) + a(20 * Pk) + 256 + blocks + a(4 * n)
    assert lib.nrn_termination_workspace_bytes(n, S, 4, 0) == a(12 * Pk) + a(4 * Pk) + a(16 * Pk) + 256 + blocks + a(4 * n)
    # S < K: a round holds the whole ray
    assert lib.nrn_termination_workspace_bytes(10, 3, 4, 0) == a(12 * 30) + a(4 * 30) + a(16 * 30) + 256 + 256 + a(40)
    assert lib.nrn_termination_workspace_bytes(0, 64, 4, 0) == 256 + 256
    assert lib.nrn_termination_workspace_bytes(10, 64, 6, 0) == 0
    assert lib.nrn_termination_workspace_bytes(10, 0, 4, 0) == 0
    assert lib.nrn_termination_workspace_bytes(2 ** 25, 64, 4, 0) == 0   # 2^31 points


def _grid(L, **kw):
    g = L.NrnOccupancyGrid()
    g.bits, g.nx, g.ny, g.nz = kw.get("bits", 4096), kw.get("nx", 4), kw.get("ny", 4), kw.get("nz", 4)
    g.min_point[:] = [-1.0, -1.0, -1.0]
    g.max_point[:] = [1.0, 1.0, 1.0]
    return g


def test_c_argument_checks():
    L, lib = _lib()
    err = lambda: lib.nrn_last_error().decode()
    ws = C.c_void_p(4096)
    a = L.NrnFieldArgs()
    a.rays, a.z_vals, a.n_rays, a.n_samples, a.out_ch, a.nerf_packed, a.raw = 4096, 4096, 10, 64, 5, 4096, 4096
    t = L.NrnTerminationArgs()
    t.threshold, t.termination_index = 1e-4, 4096
    need = lib.nrn_termination_workspace_bytes(10, 64, 5, 0)
    call = lambda g=None, tt=t, w=ws, nb=need: lib.nrn_field_forward_terminate(C.byref(a), g, tt, w, nb)
    assert call(tt=None) == -1 and "null termination args" in err()
    for bad in (-0.5, 1.5, float("nan"), float("inf"), -float("inf")):
        t.threshold = bad
        assert call(tt=C.byref(t)) == -1 and "threshold" in err(), bad
    t.threshold = 1e-4
    assert call(tt=C.byref(t), nb=need - 1) == -1 and "workspace" in err()
    assert call(tt=C.byref(t), w=C.c_void_p(4096 + 16)) == -1 and "workspace" in err()
    assert call(tt=C.byref(t), w=None) == -1 and "workspace" in err()
    assert call(C.byref(_grid(L, nx=0)), C.byref(t)) == -1 and "out of range" in err()
    assert call(C.byref(_grid(L, bits=None)), C.byref(t)) == -1 and "bits" in err()
    t.termination_index = None
    assert call(tt=C.byref(t)) == -1 and "termination_index" in err()
    t.termination_index = 4096
    a.stash, a.relu_mask = 4096, 4096
    assert call(tt=C.byref(t)) == -1 and "inference only" in err()
    a.stash = a.relu_mask = None
    a.points, a.points_stride = 4096, 3
    assert call(tt=C.byref(t)) == -1 and "ray mode" in err()
    a.points = None
    a.raw = None
    assert call(tt=C.byref(t)) == -1 and "raw" in err()
    a.raw, a.out_ch = 4096, 6
    assert call(tt=C.byref(t)) == -1 and "out_ch" in err()
    a.out_ch = 5
    a.n_rays, a.n_samples = 2 ** 25, 64
    assert call(tt=C.byref(t)) == -1 and "2^31 - 1" in err()
    a.n_rays = 0   # an empty batch: nothing to check further, nothing launched
    assert call(tt=C.byref(t), w=None, nb=0) == 0


def _nets(**kw):
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    embed_fn, input_ch = H.get_embedder(10, 0)
    base = dict(D=8, W=256, input_ch=input_ch, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False, ray_bender=None,
                ray_bending_latent_size=32)
    base.update(kw)
    return H.NeRF(**base)


def test_refusals_before_launch():
    from nonrigid_nerf_b200 import _lib, train as T
    views = _nets(use_viewdirs=True, input_ch_views=27, output_ch=4)
    tc = _nets(time_conditioned_baseline=True)
    plain = _nets()
    rays_o, rays_d = torch.zeros(4, 3), torch.ones(4, 3)
    kw = dict(near=0.0, far=1.0, ndc=False, N_samples=8, N_importance=0, network_query_fn=None, perturb=0.0, white_bkgd=False,
              raw_noise_std=0.0, lindisp=False, additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
    kinds = (_lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + _lib.DET_KERNEL_KINDS
             + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + _lib.MESH_KERNEL_KINDS
             + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS + _lib.OCCUPANCY_KERNEL_KINDS + _lib.TERMINATION_KERNEL_KINDS)
    assert len(kinds) == 41
    _lib.timing_enable(True)
    try:
        with torch.no_grad():
            with pytest.raises(RuntimeError, match="use_viewdirs=True"):
                T.render(rays_o, rays_d, use_viewdirs=True, network_fn=views, early_termination=1e-4, **kw)
            with pytest.raises(RuntimeError, match="time_conditioned_baseline=True"):
                T.render(rays_o, rays_d, network_fn=tc, early_termination=1e-4, **kw)
            for bad in (True, False, np.bool_(True), torch.tensor(0.5), -0.1, 1.0001, float("nan"), float("inf"), "0.1", 1j):
                with pytest.raises(RuntimeError, match="early_termination"):
                    T.render(rays_o, rays_d, network_fn=plain, early_termination=bad, **kw)
            with pytest.raises(RuntimeError, match="early_termination"):
                T.render_rays(torch.zeros(4, 8), plain, None, 8, early_termination=2.0,
                              additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
        with pytest.raises(RuntimeError, match="early_termination is inference only"):   # parameters that require a gradient
            T.render(rays_o, rays_d, network_fn=plain, early_termination=1e-4, **kw)
        with pytest.raises(RuntimeError, match="early_termination is inference only"):
            T.render_rays(torch.zeros(4, 8), plain, None, 8, early_termination=0.0,
                          additional_pixel_information={"ray_bending_latents": torch.zeros(4, 32)})
        counts = _lib.timing_read(kinds)
    finally:
        _lib.timing_enable(False)
    assert all(c == 0 for _, c in counts.values()), counts   # nothing reached a kernel
