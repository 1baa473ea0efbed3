"""Time-conditioned baseline (NeRF(time_conditioned_baseline=True), run_nerf_helpers.py:206-209, 273-282) without a GPU:
the fp32 restatement (tests/tc_reference.py) against golden case L of the executed reference, the module's shapes and
checkpoint keys, the configurations that must raise, and the argument validation of the new C entry points (which
returns before any CUDA call)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import tc_reference as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load():
    return np.load(os.path.join(GOLD, "caseL_time_conditioned.npz"), allow_pickle=False)


def _close(a, b, atol, rtol, name):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    assert a.shape == np.asarray(b).shape, (name, a.shape, np.asarray(b).shape)
    np.testing.assert_allclose(a, b, atol=atol, rtol=rtol, equal_nan=True, err_msg=name)


def test_caseL_render_and_point_mode_match_executed_reference():
    g = _load()
    seed, n = int(g["seed"]), int(g["n"])
    cp, fp = R.make_params(seed)
    r = R.O.make_rays(seed, n)
    with torch.no_grad():
        ret = R.render_rays(cp, fp, r["rays_o"], r["rays_d"], r["near"], r["far"], torch.from_numpy(g["latents"]))
        raw_pts = R.query(cp, torch.from_numpy(g["pts"]), torch.from_numpy(g["pts_latents"]))
    for k in ("rgb_map", "acc_map", "rgb0"):
        _close(ret[k], g[k], 2e-6, 2e-5, k)
    _close(ret["raw"][:16], g["raw"], 2e-5, 2e-5, "raw")
    _close(raw_pts, g["pts_raw"], 2e-5, 2e-5, "pts_raw")


def test_caseL_training_loss_and_gradients_match_executed_reference():
    """training_wrapper_class.forward without bender and regularisers (train.py:574-578), at case H's tolerances."""
    g = _load()
    cp, fp = (R.O.clone_params(p, True) for p in R.make_params(int(g["seed"])))
    table = torch.from_numpy(g["latent_table"]).clone().requires_grad_(True)
    loss = R.training_loss(g, cp, fp, table)
    _close(loss, g["loss"], 2e-6, 2e-5, "loss")
    loss.mean().backward()
    _close(table.grad, g["latent_grads"], 1e-8, 2e-3, "latent_grads")
    for net, p in {"coarse": cp, "fine": fp}.items():
        for i in (0, 4, 5, 7):
            nm = f"{net}.pts_linears.{i}.weight"
            gr = p["pts_w"][i].grad.reshape(-1)
            _close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, 2e-3, nm)
        _close(p["pts_w"][0].grad[:, 63:95], g[net + ".w0_latent_grad"], 1e-9, 2e-3, net + ".w0_latent_grad")
        _close(p["pts_w"][5].grad[:, 63:95], g[net + ".w5_latent_grad"], 1e-7, 2e-3, net + ".w5_latent_grad")


def _tc_nerf(**kw):
    from nonrigid_nerf_b200.run_nerf_helpers import NeRF
    args = dict(D=8, W=256, input_ch=63, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False, ray_bender=None,
                ray_bending_latent_size=32, time_conditioned_baseline=True)
    args.update(kw)
    return NeRF(**args)


def test_constructor_shapes_keys_and_parameter_count():
    from nonrigid_nerf_b200.run_nerf_helpers import NeRF
    net = _tc_nerf()
    assert net.pts_linears[0].weight.shape == (256, 95) and net.pts_linears[5].weight.shape == (256, 351)
    for i in (1, 2, 3, 4, 6, 7):
        assert net.pts_linears[i].weight.shape == (256, 256)
    assert sum(p.numel() for p in net.parameters()) == 543621
    plain = NeRF(D=8, W=256, input_ch=63, output_ch=5, skips=[4], input_ch_views=0, ray_bending_latent_size=32)
    assert list(net.state_dict().keys()) == list(plain.state_dict().keys())   # reference baseline checkpoints load
    # the flat gradient layout of the backward is the parameter order of nerf_param_list
    from nonrigid_nerf_b200 import ops
    ws, bs = ops.nerf_param_list(net)
    assert sum(w.numel() + b.numel() for w, b in zip(ws, bs)) == 510725


def test_latent_size_other_than_32_and_a_seated_bender_raise():
    with pytest.raises(RuntimeError, match="time_conditioned_baseline"):
        _tc_nerf(ray_bending_latent_size=16)
    with pytest.raises(RuntimeError, match="time_conditioned"):
        _tc_nerf(ray_bending_latent_size=0)
    from nonrigid_nerf_b200 import autograd as ag
    net = _tc_nerf()
    net.ray_bender = (torch.nn.Linear(1, 1),)   # seated by a training wrapper that was given a bender
    with pytest.raises(RuntimeError, match="ray bending to be turned off"):
        ag.field(net, torch.zeros(2, 8), torch.zeros(2, 4), torch.zeros(2, 32), False)
    with pytest.raises(RuntimeError, match="ray bending to be turned off"):
        net(torch.zeros(4, 63 + 32))


def _lib():
    from nonrigid_nerf_b200 import _lib as L
    return L, L.load()


def test_tc_gradient_buffer_size():
    _, lib = _lib()
    assert lib.nrn_nerf_tc_grad_floats(5) == 510725
    assert lib.nrn_nerf_tc_grad_floats(4) == 510725 - 257
    assert lib.nrn_nerf_grad_floats(5) == 494341
    assert lib.nrn_tc_workspace_bytes(10) == (10 * 512 + 16384) * 4


def test_new_entry_points_validate_arguments_without_a_gpu():
    L, lib = _lib()
    fake = C.c_void_p(4096)   # never dereferenced: validation fails before any CUDA call

    def err():
        return lib.nrn_last_error().decode()

    # nrn_tc_latent_bias
    assert lib.nrn_tc_latent_bias(fake, 32, -1, fake, fake, fake, fake, fake, None) == -1 and "bad sizes" in err()
    assert lib.nrn_tc_latent_bias(fake, -5, 4, fake, fake, fake, fake, fake, None) == -1 and "bad sizes" in err()
    assert lib.nrn_tc_latent_bias(fake, 32, 4, fake, None, fake, fake, fake, None) == -1 and "null argument" in err()
    assert lib.nrn_tc_latent_bias(None, 32, 0, None, None, None, None, None, None) == 0   # nothing to do
    # nrn_field_forward_tc
    assert lib.nrn_field_forward_tc(None, fake) == -1 and "null args" in err()
    a = L.NrnFieldArgs()
    a.n_rays, a.n_samples, a.out_ch = 4, 8, 5
    a.rays, a.z_vals, a.nerf_packed, a.raw = 4096, 4096, 4096, 4096
    a.bender_packed = 4096
    assert lib.nrn_field_forward_tc(C.byref(a), fake) == -1 and "no bender" in err()
    a.bender_packed = None
    assert lib.nrn_field_forward_tc(C.byref(a), None) == -1 and "ray_bias" in err()
    a.latent_stride = -1
    assert lib.nrn_field_forward_tc(C.byref(a), fake) == -1 and "latent_stride" in err()
    a.latent_stride = 32
    a.out_ch = 7
    assert lib.nrn_field_forward_tc(C.byref(a), fake) == -1 and "nrn_field_forward_tc: out_ch=7" in err()
    a.out_ch, a.stash = 5, 4096
    assert lib.nrn_field_forward_tc(C.byref(a), fake) == -1 and "relu_mask" in err()
    # nrn_field_backward_tc
    b = L.NrnFieldBwdArgs()
    b.n_rays, b.n_samples, b.out_ch = 4, 8, 5
    b.nerf_packed, b.nerf_grad, b.relu_mask = 4096, 4096, 4096
    t = L.NrnTcBwdArgs()
    t.latents, t.latent_stride, t.w0, t.w5, t.d_latents, t.workspace = 4096, 32, 4096, 4096, 4096, 4096
    assert lib.nrn_field_backward_tc(None, C.byref(t)) == -1 and "null args" in err()
    assert lib.nrn_field_backward_tc(C.byref(b), None) == -1 and "null args" in err()
    b.bender_packed = 4096
    assert lib.nrn_field_backward_tc(C.byref(b), C.byref(t)) == -1 and "no bender" in err()
    b.bender_packed = None
    t.w5 = None
    assert lib.nrn_field_backward_tc(C.byref(b), C.byref(t)) == -1 and "w5" in err()
    t.w5, t.latent_stride = 4096, -1
    assert lib.nrn_field_backward_tc(C.byref(b), C.byref(t)) == -1 and "latent_stride" in err()
    t.latent_stride, b.out_ch = 32, 3
    assert lib.nrn_field_backward_tc(C.byref(b), C.byref(t)) == -1 and "nrn_field_backward_tc: out_ch=3" in err()
    b.out_ch, b.relu_mask = 5, None
    assert lib.nrn_field_backward_tc(C.byref(b), C.byref(t)) == -1 and "relu_mask" in err()
    # nrn_pack_nerf accepts input_ch = 95 (63 + 32) and still refuses the other widths above 63
    ptrs = (C.c_void_p * 9)(*([4096] * 9))
    assert lib.nrn_pack_nerf(ptrs, ptrs, 94, 5, fake, None) == -1 and "input_ch=94" in err()
    assert lib.nrn_pack_nerf(ptrs, ptrs, 96, 5, fake, None) == -1 and "input_ch=96" in err()
    assert lib.nrn_pack_nerf(ptrs, ptrs, 95, 17, fake, None) == -1 and "out_ch=17" in err()
