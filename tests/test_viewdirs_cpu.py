"""CPU-only tests of the view-dependent head (NeRF(use_viewdirs=True)): the module layout of the reference, every
configuration that raises, and the argument checks of its C entry points.  No kernel is launched here."""
import ctypes

import pytest
import torch

# NeRF(D=8, W=256, input_ch=63, input_ch_views=27, use_viewdirs=True) of the reference (run_nerf_helpers.py:217-236):
# state_dict keys in registration order and their shapes
REFERENCE_LAYOUT = [("pts_linears.0.weight", (256, 63)), ("pts_linears.0.bias", (256,))] + [
    item for i in range(1, 8) for item in ((f"pts_linears.{i}.weight", (256, 319 if i == 5 else 256)), (f"pts_linears.{i}.bias", (256,)))
] + [("views_linears.0.weight", (128, 283)), ("views_linears.0.bias", (128,)),
     ("feature_linear.weight", (256, 256)), ("feature_linear.bias", (256,)),
     ("alpha_linear.weight", (1, 256)), ("alpha_linear.bias", (1,)),
     ("rgb_linear.weight", (3, 128)), ("rgb_linear.bias", (3,))]


def _net(**kw):
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    args = dict(D=8, W=256, input_ch=63, output_ch=5, skips=[4], input_ch_views=27, use_viewdirs=True, ray_bender=None,
                ray_bending_latent_size=32, embeddirs_fn=None, num_ray_samples=64, approx_nonrigid_viewdirs=True)
    args.update(kw)
    return H.NeRF(**args)


def _bender():
    from nonrigid_nerf_b200 import run_nerf_helpers as H
    return H.ray_bending(63, 32, "simple_neural", None)


def test_module_layout_matches_the_reference_checkpoints():
    net = _net()
    sd = net.state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == REFERENCE_LAYOUT
    assert sum(v.numel() for v in sd.values()) == 595844
    assert not hasattr(net, "output_linear")
    # default nn.Linear init in the reference's registration order: the same seed gives the same weights
    torch.manual_seed(3)
    a = _net().state_dict()
    torch.manual_seed(3)
    ref = {}
    lin = lambda i, o: torch.nn.Linear(i, o)
    mods = [lin(63, 256)] + [lin(319 if i == 4 else 256, 256) for i in range(7)] + [lin(283, 128), lin(256, 256), lin(256, 1), lin(128, 3)]
    names = [f"pts_linears.{i}" for i in range(8)] + ["views_linears.0", "feature_linear", "alpha_linear", "rgb_linear"]
    for nm, m in zip(names, mods):
        ref[nm + ".weight"], ref[nm + ".bias"] = m.weight, m.bias
    for k in a:
        assert torch.equal(a[k], ref[k]), k


@pytest.mark.parametrize("kw", [dict(input_ch_views=3), dict(time_conditioned_baseline=True),
                                dict(ray_bender="bender", approx_nonrigid_viewdirs=False),
                                dict(ray_bender="bender", num_ray_samples=None), dict(ray_bender="bender", num_ray_samples=1)])
def test_unsupported_view_configurations_raise_at_construction(kw):
    if kw.get("ray_bender") == "bender":
        kw = dict(kw, ray_bender=_bender())
    with pytest.raises(RuntimeError, match="use_viewdirs"):
        _net(**kw)


def test_seated_bender_is_checked_at_call_time():
    from nonrigid_nerf_b200 import autograd as ag
    for kw in (dict(approx_nonrigid_viewdirs=False), dict(num_ray_samples=None)):
        net = _net(**kw)              # no bender yet: accepted
        net.ray_bender = (_bender(),)
        with torch.no_grad(), pytest.raises(RuntimeError, match="use_viewdirs"):
            ag.views_check(net)


def test_mismatched_batches_and_viewdirs_raise():
    from nonrigid_nerf_b200 import run_nerf_helpers as H, train as T
    plain = H.NeRF(D=8, W=256, input_ch=63, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False, ray_bending_latent_size=32)
    views = _net()
    info = {"ray_bending_latents": torch.zeros(4, 32)}
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="use_viewdirs"):
            T.run_network(torch.zeros(4, 64, 3), torch.zeros(4, 3), info, plain, None, None)
        with pytest.raises(RuntimeError, match="use_viewdirs"):
            T.run_network(torch.zeros(4, 64, 3), None, info, views, None, None)
        with pytest.raises(RuntimeError, match="use_viewdirs"):
            T.render_rays(torch.zeros(4, 11), plain, None, 64, additional_pixel_information=info)
        with pytest.raises(RuntimeError, match="use_viewdirs"):
            T.render_rays(torch.zeros(4, 8), views, None, 64, additional_pixel_information=info)
        with pytest.raises(RuntimeError, match="use_viewdirs"):
            T.render(torch.zeros(4, 3), torch.ones(4, 3), ndc=False, use_viewdirs=True, network_fn=plain, N_samples=64,
                     additional_pixel_information=info)


def test_differentiable_calls_raise_before_any_launch():
    """CPU tensors: a launch would fail with a different message, so the error proves nothing ran first."""
    from nonrigid_nerf_b200 import parallel, train as T
    views = _net(ray_bender=_bender())
    info = {"ray_bending_latents": torch.zeros(4, 32)}
    with pytest.raises(RuntimeError, match="training with the view-dependent head is not implemented"):
        T.render(torch.zeros(4, 3), torch.ones(4, 3), ndc=False, use_viewdirs=True, network_fn=views, N_samples=64,
                 additional_pixel_information=info)
    with pytest.raises(RuntimeError, match="training with the view-dependent head is not implemented"):
        T.render_rays(torch.zeros(4, 11), views, None, 64, additional_pixel_information=info)
    lat = [torch.zeros(32, requires_grad=True)]
    wrapper = parallel.training_wrapper_class(views, lat, ray_bender=views.ray_bender[0])
    with pytest.raises(RuntimeError, match="training with the view-dependent head is not implemented"):
        wrapper.forward(None, None, None, 0, {}, torch.zeros(4, 3), 0, 0, {"imageid_to_timestepid": [0]}, torch.zeros(4, 3))


def _fake(n=16):
    buf = ctypes.create_string_buffer(n + 16)
    return ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15), buf   # 16-byte aligned, never dereferenced


def test_view_entry_points_validate_their_arguments():
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    assert lib.nrn_packed_views_bytes() == 210496
    assert lib.nrn_views_workspace_bytes(10, 64) == 10 * 64 * 16 and lib.nrn_views_workspace_bytes(-1, 64) == 0
    p, keep = _fake()
    arr = (ctypes.c_void_p * 3)(p.value, p.value, p.value)
    assert lib.nrn_pack_views(None, arr, p, None) == -1 and b"null" in lib.nrn_last_error()
    assert lib.nrn_pack_views(arr, arr, ctypes.c_void_p(p.value + 4), None) == -1 and b"aligned" in lib.nrn_last_error()

    def args(bender=True):
        a, v = _lib.NrnFieldArgs(), _lib.NrnViewArgs()
        a.n_rays, a.n_samples, a.out_ch = 4, 64, 4
        a.rays = a.z_vals = a.nerf_packed = a.raw = p
        v.views_packed = p
        if bender:
            a.bender_packed = a.latents = p
            v.workspace = p
        else:
            v.viewdirs, v.viewdirs_stride = p, 3
        return a, v

    call = lambda a, v: lib.nrn_field_forward_views(ctypes.byref(a), ctypes.byref(v))
    assert lib.nrn_field_forward_views(None, None) == -1
    cases = [("out_ch", lambda a, v: setattr(a, "out_ch", 5), True),
             ("inference only", lambda a, v: setattr(a, "stash", p), True),
             ("inference only", lambda a, v: setattr(a, "relu_mask", p), True),
             ("n_samples >= 2", lambda a, v: setattr(a, "n_samples", 1), True),
             ("needs viewdirs", lambda a, v: setattr(v, "viewdirs", None), False),
             ("workspace", lambda a, v: setattr(v, "workspace", None), True),
             ("workspace", lambda a, v: setattr(v, "workspace", p.value + 4), True),
             ("aligned", lambda a, v: setattr(a, "nerf_packed", p.value + 4), True),
             ("aligned", lambda a, v: setattr(v, "views_packed", p.value + 8), False),
             ("null", lambda a, v: setattr(v, "views_packed", None), False)]
    for msg, spoil, bender in cases:
        a, v = args(bender)
        spoil(a, v)
        assert call(a, v) == -1, msg
        assert msg.encode() in lib.nrn_last_error(), (msg, lib.nrn_last_error())
