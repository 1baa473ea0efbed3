"""CPU tests of spatial LPIPS maps (evaluation.lpips_maps, nrn_lpips_maps): the fp64 and fp32 upsampling restatements
(tests/lpips_maps_reference.py) against PyTorch's index rule and each other, the restated tap distances against
tests/lpips_reference.py's tap scores, the error-image rule, the workspace sizes against the layout mirror, and the entry
points' argument checks on host pointers (no kernel is launched)."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import lpips_layout as L
from tests import lpips_maps_reference as M
from tests import lpips_reference as R


def _lib():
    from nonrigid_nerf_b200 import _lib
    return _lib, _lib.load()


@pytest.mark.parametrize("src,dst", [((1, 1), (31, 31)), ((7, 5), (33, 47)), ((9, 13), (9, 13)), ((13, 17), (50, 71)),
                                     ((47, 62), (189, 251)), ((5, 8), (31, 32))])
def test_interpolate_follows_the_index_rule(src, dst):
    rng = np.random.default_rng(src[0] * 100 + dst[1])
    d = rng.random(src)
    loop = M.upsample_loop(d, *dst)
    ref = M.upsample64(torch.from_numpy(d)[None], *dst)[0].numpy()
    # the same indices and weights; the weights' fp64 rounding (about |src| 2^-52) and the order of the products differ
    assert np.abs(loop - ref).max() <= 2.0 ** -52 * 8 * (max(src) + 2) * max(1.0, np.abs(ref).max())
    if src == dst:
        assert np.array_equal(ref, d)   # equal sizes: the identity
    if src == (1, 1):   # l0 x + l1 x: constant up to the rounding of the two products
        assert np.abs(ref - d[0, 0]).max() <= 2.3e-16


@pytest.mark.parametrize("h,w", [(31, 31), (32, 33), (47, 64), (127, 255), (378, 504), (756, 1008)])
def test_fp32_rule_against_fp64_interpolate(h, w):
    rng = np.random.default_rng(h * w)
    worst = []
    for tap in range(L.TAPS):
        hh, ww = L.dims(h, w)[L.TAP_STAGES[tap]]
        d = rng.random((2, hh, ww)).astype(np.float32)
        a = M.upsample32(d, h, w).astype(np.float64)
        b = M.upsample64(torch.from_numpy(d), h, w).numpy()
        bound = M.fp32_bound(float(d.max()), hh, ww)
        assert np.abs(a - b).max() <= bound, (tap, np.abs(a - b).max(), bound)
        worst.append(np.abs(a - b).max() / bound)
    print(f"\n{h}x{w}: worst |fp32 - fp64| / bound per tap {np.array2string(np.array(worst), precision=3)}")


def test_maps32_sums_in_tap_order_and_propagates_nan():
    rng = np.random.default_rng(3)
    h, w = 40, 45
    taps = [rng.random((3,) + L.dims(h, w)[s]).astype(np.float32) for s in L.TAP_STAGES]
    total, ups = M.maps32(taps, h, w)
    acc = ups[:, 0]
    for k in range(1, 5):
        acc = acc + ups[:, k]
    assert total.dtype == np.float32 and np.array_equal(total, acc)
    total, ups = M.maps32(taps, h, w, first=[5, 2, 0])
    assert np.isfinite(total[0]).all() and np.isfinite(ups[0]).all()
    assert np.isfinite(ups[1, :2]).all() and np.isnan(ups[1, 2:]).all() and np.isnan(total[1]).all()
    assert np.isnan(ups[2]).all() and np.isnan(total[2]).all()


def test_restated_distances_average_to_the_tap_scores():
    sd = R.random_state_dict(2)
    gt, gen = R.frames(5, 3, 48, 61)
    explicit = np.zeros((48, 61), dtype=bool)
    explicit[10:20, 5:30] = True
    for mask in (None, explicit):
        _, per = R.lpips(gt, gen, sd, mask=mask)
        d = M.distances(gt, gen, sd, mask=mask)
        assert [tuple(x.shape[1:]) for x in d] == [L.dims(48, 61)[s] for s in L.TAP_STAGES]
        means = np.stack([x.mean(dim=(1, 2)).numpy() for x in d], axis=1)
        assert np.allclose(means, per, rtol=1e-12, atol=1e-15)
        assert np.all(means[0] == 0.0)   # frame 0's render is its ground truth
    total, layers = M.maps64(gt, gen, sd)
    assert total.shape == (3, 48, 61) and layers.shape == (3, 5, 48, 61)
    assert torch.allclose(total, layers.sum(dim=1), rtol=1e-14, atol=0)


def test_error_image_rule():
    jet = M.jet8()
    from nonrigid_nerf_b200 import evaluation as E
    assert np.array_equal(jet, (255.0 * E.jet_colormap()).astype(np.uint8))
    v = np.array([0.0, 1.0, 2.5, np.nan, -1.0, 0.5, 1.0 / 255, np.inf], dtype=np.float32)
    assert M.lut_index(v).tolist() == [0, 255, 255, 0, 0, 127, 1, 255]
    img = M.error_image(v.reshape(1, 2, 4))
    assert img.shape == (1, 2, 4, 3) and img.dtype == np.uint8
    assert np.array_equal(img[0, 0, 0], jet[0]) and np.array_equal(img[0, 0, 3], jet[0]) and np.array_equal(img[0, 0, 1], jet[255])


def test_workspace_bytes():
    _, lib = _lib()
    for f, h, w in ((0, 378, 504), (1, 378, 504), (37, 378, 504), (1000, 756, 1008), (1, 31, 31), (5, 37, 53), (3, 127, 255)):
        got = lib.nrn_lpips_maps_workspace_bytes(f, h, w)
        assert got == M.workspace_bytes(f, h, w), (f, h, w)
        assert got >= lib.nrn_lpips_workspace_bytes(min(f, 1), h, w)
    # one frame's share: nrn_lpips's frame plus the five tap maps, each rounded up to 256 bytes
    h, w = 756, 1008
    one = lib.nrn_lpips_maps_workspace_bytes(1, h, w) - lib.nrn_lpips_maps_workspace_bytes(0, h, w)
    assert one == L.frame_bytes(h, w) + sum(L.a256(L.px(h, w, s) * 4) for s in L.TAP_STAGES)
    # chunks are sized from the larger frame: 37 frames of 504 x 378 go in chunks of 17 here, 18 for the scores alone
    assert M.workspace_bytes(37, 378, 504) == L.mask_bytes(378, 504) + 17 * M.map_frame_bytes(378, 504)
    for f, h, w in ((-1, 40, 40), (1, 30, 40), (1, 40, 30), (1, 16385, 40)):
        assert lib.nrn_lpips_maps_workspace_bytes(f, h, w) == 0
    # the tap maps of a chunk lie after its nrn_lpips buffers and inside its share of the workspace
    for fc in (1, 2, 17):
        end = M.tap_map_offset(fc, 378, 504, 4) + fc * M.tap_map_bytes(378, 504, 4)
        assert M.tap_map_offset(fc, 378, 504, 0) >= L.chunk(fc, 378, 504)["end"]
        assert end <= L.mask_bytes(378, 504) + fc * M.map_frame_bytes(378, 504)
        assert all(M.tap_map_offset(fc, 378, 504, k) % 256 == 0 for k in range(5))


def _fake(n=64):
    buf = C.create_string_buffer(n + 256)
    return C.c_void_p((C.addressof(buf) + 255) & ~255), buf   # 256-byte aligned, never dereferenced


def _args(p, f=2, h=40, w=50, ws=1 << 40):
    Lb, _ = _lib()
    a = Lb.NrnLpipsArgs()
    a.gt = a.generated = a.packed = a.lpips = a.workspace = p
    a.n_frames, a.height, a.width = f, h, w
    a.workspace_bytes = ws
    m = Lb.NrnLpipsMapArgs()
    m.map = p
    return a, m


def test_maps_reject_bad_arguments_before_any_cuda_call():
    Lb, lib = _lib()
    p, keep = _fake()
    a, m = _args(p)
    assert lib.nrn_lpips_maps(None, C.byref(m)) == -1 and b"null args" in lib.nrn_last_error()
    assert lib.nrn_lpips_maps(C.byref(a), None) == -1 and b"nrn_lpips_maps: null args" in lib.nrn_last_error()
    one = M.workspace_bytes(1, 40, 50)
    for field, value, msg in (("n_frames", -1, b"bad sizes"), ("height", -2, b"bad sizes"),
                              ("height", 30, b"at least 31"), ("width", 7, b"at least 31"), ("width", 16385, b"at most 16384"),
                              ("height", 16385, b"at most 16384"),
                              ("gt", None, b"null"), ("generated", None, b"null"), ("packed", None, b"null"),
                              ("lpips", None, b"null"), ("workspace", None, b"null"),
                              ("gt", p.value + 2, b"4-byte aligned"), ("per_layer", p.value + 1, b"4-byte aligned"),
                              ("packed", p.value + 8, b"16-byte"), ("workspace", p.value + 16, b"256-byte aligned"),
                              ("workspace_bytes", 1000, b"holds no frame"),
                              # enough for one frame of nrn_lpips, not for one with its tap maps
                              ("workspace_bytes", L.mask_bytes(40, 50) + L.frame_bytes(40, 50), b"holds no frame"),
                              ("workspace_bytes", one - 1, b"holds no frame")):
        a, m = _args(p)
        setattr(a, field, value)
        assert lib.nrn_lpips_maps(C.byref(a), C.byref(m)) == -1, field
        assert msg in lib.nrn_last_error() and b"nrn_lpips_maps" in lib.nrn_last_error(), (field, lib.nrn_last_error())
    for field, value, msg in (("map", None, b"null argument"), ("map", p.value + 2, b"4-byte aligned"),
                              ("layer_maps", p.value + 1, b"4-byte aligned")):
        a, m = _args(p)
        setattr(m, field, value)
        assert lib.nrn_lpips_maps(C.byref(a), C.byref(m)) == -1, field
        assert msg in lib.nrn_last_error(), (field, lib.nrn_last_error())
    # the error image is uint8: any address
    a, m = _args(p, ws=1000)
    m.error_image = p.value + 1
    assert lib.nrn_lpips_maps(C.byref(a), C.byref(m)) == -1 and b"holds no frame" in lib.nrn_last_error()
    # no frames: valid, nothing launched, every output may be NULL; small frames are refused even then
    a, m = Lb.NrnLpipsArgs(), Lb.NrnLpipsMapArgs()
    a.n_frames, a.height, a.width = 0, 31, 31
    assert lib.nrn_lpips_maps(C.byref(a), C.byref(m)) == 0
    a.height = 30
    assert lib.nrn_lpips_maps(C.byref(a), C.byref(m)) == -1


def test_python_entry_point_refusals():
    from nonrigid_nerf_b200 import evaluation as E
    x = torch.zeros(1, 40, 40, 3)
    with pytest.raises(RuntimeError, match="lpips_weights"):
        E.lpips_maps(x, x, object())
    # the checks lpips() makes, in the same order and words
    with pytest.raises(RuntimeError, match="lpips_weights"):
        E.lpips_maps(x, x, None, chunk_frames=0)
    wt = E.LpipsWeights(torch.zeros(16, dtype=torch.uint8), [])
    with pytest.raises(RuntimeError, match="CPU path"):
        E.lpips_maps(x, x, wt)
    with pytest.raises(RuntimeError, match="CPU path"):
        E.lpips(x, x, wt)


def test_timing_kind():
    from nonrigid_nerf_b200 import _lib as Lb
    assert Lb.LPIPS_MAP_KERNEL_KINDS == ("lpips_upsample",)
    kinds = Lb.KERNEL_KINDS + Lb.TC_KERNEL_KINDS + Lb.VIEW_KERNEL_KINDS + Lb.VIEW_TRAIN_KERNEL_KINDS + Lb.DET_KERNEL_KINDS + \
        Lb.HELD_OUT_KERNEL_KINDS + Lb.EVAL_KERNEL_KINDS + Lb.FRAME_IMAGE_KERNEL_KINDS + Lb.MESH_KERNEL_KINDS + \
        Lb.LPIPS_KERNEL_KINDS + Lb.MATCH_KERNEL_KINDS + Lb.OCCUPANCY_KERNEL_KINDS + Lb.TERMINATION_KERNEL_KINDS + \
        Lb.DEFORM_KERNEL_KINDS + Lb.NORMAL_KERNEL_KINDS
    assert len(kinds) == 44   # the upsampling is kind 44
