"""CPU tests of LPIPS: the fp64 restatement (tests/lpips_reference.py) against torchvision's AlexNet features and, where
the lpips package is importable, against lpips.LPIPS itself; the state-dict parsing and its refusals; the packed-block and
workspace sizes; and the C entry points' argument checks on host pointers (no kernel is launched)."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import lpips_reference as R


def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


def test_restatement_taps_are_torchvision_alexnet_features():
    torchvision = pytest.importorskip("torchvision")
    sd = R.random_state_dict(3)
    net = torchvision.models.alexnet(weights=None).features.double().eval()
    for i, (key, *_rest) in zip((0, 3, 6, 8, 10), R.CONVS):
        net[i].weight.data.copy_(sd[key + ".weight"])
        net[i].bias.data.copy_(sd[key + ".bias"])
    gt, _ = R.frames(0, 1, 67, 91)
    x = R.scaled(torch.from_numpy(gt), sd)
    ours = R.taps(x, sd)
    with torch.no_grad():
        theirs, h = [], x
        for i, layer in enumerate(net):
            h = layer(h)
            if i in (1, 4, 7, 9, 11):   # the five ReLU outputs
                theirs.append(h)
    assert len(ours) == 5
    for a, b in zip(ours, theirs):
        assert a.shape == b.shape and torch.equal(a, b)


def test_restatement_properties():
    sd = R.random_state_dict(1)
    gt, gen = R.frames(2, 6, 40, 45)
    total, per = R.lpips(gt, gen, sd)
    assert per.shape == (6, 5) and np.allclose(total, per.sum(axis=1), rtol=0, atol=0)
    assert total[0] == 0.0                                   # perturbation 0: the render is the ground truth
    assert np.all(np.diff(total[:5]) > 0)                    # larger perturbations score higher
    back, _ = R.lpips(gen, gt, sd)
    assert np.allclose(back, total, rtol=1e-12, atol=0)
    assert R.taps(R.scaled(torch.zeros(1, 31, 31, 3), sd), sd)[-1].shape[-2:] == (1, 1)   # 31 x 31: one pixel per tap


def test_restatement_against_lpips_package():
    try:
        import lpips
    except ImportError as e:
        pytest.skip(f"the lpips package is not importable ({e}); the restatement stands on the specification")
    net = lpips.LPIPS(net="alex", pretrained=False, pnet_rand=True, verbose=False).eval().double()
    sd = {k: v.float() for k, v in net.state_dict().items()}
    gt, gen = R.frames(4, 3, 48, 64)
    ours, _ = R.lpips(gt, gen, sd)
    with torch.no_grad():
        to = lambda a: 2 * torch.from_numpy(a).double().permute(0, 3, 1, 2) - 1
        theirs = net(to(gt), to(gen)).reshape(-1).numpy()
    assert np.allclose(ours, theirs, rtol=1e-9, atol=1e-12)


def test_state_parsing_and_defaults():
    from nonrigid_nerf_b200 import evaluation as E
    sd = R.random_state_dict(5)
    st = E.lpips_state(sd)
    assert len(st) == 17 and all(t.dtype == torch.float32 for t in st)
    assert [tuple(t.shape) for t in st[:10:2]] == [(64, 3, 11, 11), (192, 64, 5, 5), (384, 192, 3, 3), (256, 384, 3, 3), (256, 256, 3, 3)]
    assert [t.numel() for t in st[10:15]] == [64, 192, 384, 256, 256]
    assert torch.equal(st[10], sd["lin0.model.1.weight"].reshape(-1))
    del sd["scaling_layer.shift"], sd["scaling_layer.scale"]
    st = E.lpips_state(sd)
    assert torch.equal(st[15], torch.tensor(E.LPIPS_SHIFT)) and torch.equal(st[16], torch.tensor(E.LPIPS_SCALE))


class _Module(torch.nn.Module):
    def __init__(self, sd, **attrs):
        super().__init__()
        for k, v in attrs.items():
            setattr(self, k, v)
        self._sd = sd

    def state_dict(self, *a, **k):
        return dict(self._sd)


def test_state_refusals():
    from nonrigid_nerf_b200 import evaluation as E
    sd = R.random_state_dict(6)
    E.lpips_state(_Module(sd))   # a module is read through its state dict
    cases = []
    missing = dict(sd)
    del missing["net.slice3.6.bias"]
    cases.append((missing, "lacks net.slice3.6.bias"))
    vgg = dict(sd)
    vgg["net.slice1.0.weight"] = torch.zeros(64, 3, 3, 3)   # VGG's and SqueezeNet's first convolution
    cases.append((vgg, "VGG and SqueezeNet"))
    squeeze = dict(sd)
    squeeze["lin5.model.1.weight"] = torch.zeros(1, 512, 1, 1)
    cases.append((squeeze, "SqueezeNet"))
    lin = dict(sd)
    lin["lin2.model.1.weight"] = torch.zeros(1, 256, 1, 1)
    cases.append((lin, "lin2.model.1.weight must be"))
    nan = dict(sd)
    nan["net.slice2.3.weight"] = sd["net.slice2.3.weight"].clone()
    nan["net.slice2.3.weight"][0, 0, 0, 0] = float("nan")
    cases.append((nan, "non-finite"))
    cases += [(_Module(sd, version="0.0"), "version 0.0"), (_Module(sd, spatial=True), "spatial"),
              (_Module(sd, pnet_type="vgg"), "vgg backbone"), ([1, 2], "state dict")]
    for source, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            E.lpips_state(source)


def test_packed_and_workspace_sizes():
    _, lib = _lib()
    assert lib.nrn_lpips_packed_bytes() == 131072 + 614400 + 1327104 + 1769472 + 1179648 + 2 * 1152 * 4 + 24
    a256 = lambda v: (v + 255) // 256 * 256

    def frame_bytes(h, w):
        dims = [(h, w)]
        c1 = ((h + 4 - 11) // 4 + 1, (w + 4 - 11) // 4 + 1)
        p1 = ((c1[0] - 3) // 2 + 1, (c1[1] - 3) // 2 + 1)
        c2 = p1
        p2 = ((c2[0] - 3) // 2 + 1, (c2[1] - 3) // 2 + 1)
        dims += [c1, p1, c2, p2, p2, p2, p2]
        chans = (8, 64, 64, 192, 192, 384, 256, 256)
        b = sum(a256(2 * hh * ww * c * 2) for (hh, ww), c in zip(dims, chans))
        blocks = max((dims[s][0] * dims[s][1] + 255) // 256 for s in (1, 3, 5, 6, 7))
        return b + a256(5 * blocks * 8 + 2 * 4)   # the distance partials, then the two images' saturation words

    for h, w in ((378, 504), (756, 1008), (31, 31), (37, 53)):
        fb = frame_bytes(h, w)
        mask = a256(h * w)
        assert lib.nrn_lpips_workspace_bytes(0, h, w) == mask
        assert lib.nrn_lpips_workspace_bytes(1, h, w) == mask + fb
        fc = max(1, min((256 << 20) // fb, 4096))
        assert lib.nrn_lpips_workspace_bytes(1000, h, w) == mask + min(fc, 1000) * fb
    assert lib.nrn_lpips_workspace_bytes(37, 378, 504) == a256(378 * 504) + 18 * frame_bytes(378, 504)   # chunks of 18, 18 and 1
    for f, h, w in ((-1, 40, 40), (1, 30, 40), (1, 40, 30), (1, 16385, 40)):
        assert lib.nrn_lpips_workspace_bytes(f, h, w) == 0


def _fake(n=64):
    buf = C.create_string_buffer(n + 256)
    return C.c_void_p((C.addressof(buf) + 255) & ~255), buf   # 256-byte aligned, never dereferenced


def _args(p, f=2, h=40, w=50, ws=1 << 40):
    L, _ = _lib()
    a = L.NrnLpipsArgs()
    a.gt = a.generated = a.packed = a.lpips = a.workspace = p
    a.n_frames, a.height, a.width = f, h, w
    a.workspace_bytes = ws
    return a


def test_lpips_rejects_bad_arguments_before_any_cuda_call():
    L, lib = _lib()
    p, keep = _fake()
    assert lib.nrn_lpips(None) == -1 and b"null args" in lib.nrn_last_error()
    for field, value, msg in (("n_frames", -1, b"bad sizes"), ("height", -2, b"bad sizes"),
                              ("height", 30, b"at least 31"), ("width", 7, b"at least 31"), ("width", 16385, b"at most 16384"),
                              ("gt", None, b"null"), ("generated", None, b"null"), ("packed", None, b"null"),
                              ("lpips", None, b"null"), ("workspace", None, b"null"),
                              ("gt", p.value + 2, b"4-byte aligned"), ("per_layer", p.value + 1, b"4-byte aligned"),
                              ("packed", p.value + 8, b"16-byte"), ("workspace", p.value + 16, b"256-byte aligned"),
                              ("workspace_bytes", 1000, b"holds no frame")):
        a = _args(p)
        setattr(a, field, value)
        assert lib.nrn_lpips(C.byref(a)) == -1, field
        assert msg in lib.nrn_last_error(), (field, lib.nrn_last_error())
    # the bound is in the message, for either side
    a = _args(p, h=31, w=30)
    assert lib.nrn_lpips(C.byref(a)) == -1 and b"31 x 30" in lib.nrn_last_error()
    # no frames: valid, nothing launched, every pointer may be NULL; small frames are refused even then
    a = L.NrnLpipsArgs()
    a.n_frames, a.height, a.width = 0, 31, 31
    assert lib.nrn_lpips(C.byref(a)) == 0
    a.height = 30
    assert lib.nrn_lpips(C.byref(a)) == -1


def test_pack_rejects_bad_arguments_before_any_cuda_call():
    _, lib = _lib()
    p, keep = _fake()
    ptrs = (C.c_void_p * 17)(*([p.value] * 17))
    assert lib.nrn_lpips_pack(None, p, None) == -1 and b"null" in lib.nrn_last_error()
    assert lib.nrn_lpips_pack(ptrs, None, None) == -1 and b"null" in lib.nrn_last_error()
    assert lib.nrn_lpips_pack(ptrs, C.c_void_p(p.value + 4), None) == -1 and b"16-byte" in lib.nrn_last_error()
    for i, value, msg in ((7, None, b"null tensor 7"), (16, None, b"null tensor 16"), (3, p.value + 2, b"tensor 3 must be 4-byte")):
        bad = (C.c_void_p * 17)(*([p.value] * 17))
        bad[i] = value
        assert lib.nrn_lpips_pack(bad, p, None) == -1 and msg in lib.nrn_last_error(), i


def test_python_entry_points_refuse_host_tensors_and_small_frames():
    from nonrigid_nerf_b200 import evaluation as E
    x = torch.zeros(1, 40, 40, 3)
    with pytest.raises(RuntimeError, match="lpips_weights"):
        E.lpips(x, x, object())
    with pytest.raises(RuntimeError, match="CPU path"):
        E.lpips_weights(R.random_state_dict(0), device="cpu")


def test_timing_kinds():
    from nonrigid_nerf_b200 import _lib as L
    assert L.LPIPS_KERNEL_KINDS == ("lpips_input", "lpips_conv", "lpips_pool", "lpips_distance")
    kinds = L.KERNEL_KINDS + L.TC_KERNEL_KINDS + L.VIEW_KERNEL_KINDS + L.VIEW_TRAIN_KERNEL_KINDS + L.DET_KERNEL_KINDS + \
        L.HELD_OUT_KERNEL_KINDS + L.EVAL_KERNEL_KINDS + L.FRAME_IMAGE_KERNEL_KINDS + L.MESH_KERNEL_KINDS
    assert len(kinds) == 25   # the LPIPS kinds are 25 to 28
