"""GPU tests of spatial LPIPS maps (evaluation.lpips_maps, nrn_lpips_maps) against tests/lpips_maps_reference.py:

- the maps and per-tap maps against the fp64 restatement (lpips.LPIPS(net='alex', spatial=True)) within the score
  tolerance, per pixel, from the smallest frame to 1008 x 756 and 1 to 37 frames, with the default and explicit masks;
- the upsampling bit for bit: the tap maps read back from a workspace the test owns, then the numpy fp32 rule of them,
  and against F.interpolate in fp64 within the fp32 coordinate-rounding bound; the tap maps' means are the tap scores;
- scores bit-identical to lpips(), identity, symmetry, chunk independence, reruns and CUDA-graph replay;
- saturation (NaN maps exactly where lpips() gives NaN tap scores), error images bit for bit, and outputs past 2^31 bytes.

`pytest -s` prints the worst errors."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import lpips_layout as L
from tests import lpips_maps_reference as M
from tests import lpips_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 5e-4   # per pixel, the score tolerance of tests/test_lpips_gpu.py


@pytest.fixture(scope="module")
def setup():
    from nonrigid_nerf_b200 import evaluation as E
    sd = R.random_state_dict(0)
    return E, sd, E.lpips_weights(sd)


def _frames(seed, f, h, w):
    """R.frames with a default mask in gt[0] (zeroed in gen[0] too, so that frame 0 of several stays its own render under
    an explicit mask); a single frame is a render with noise of 0.1, not the ground truth itself"""
    gt, gen = R.frames(seed, f, h, w, perturb=(0.1,) if f == 1 else (0.0, 0.01, 0.03, 0.1, 0.3))
    gt[0, h // 3:h // 3 + 9, w // 4:w // 4 + 13] = 0   # a default mask
    gen[0, h // 3:h // 3 + 9, w // 4:w // 4 + 13] = 0
    return gt, gen


def _cuda(*a):
    return [torch.from_numpy(x).to(DEV) for x in a]


CASES = [(31, 31, 1), (31, 31, 5), (32, 33, 2), (47, 64, 1), (47, 64, 37), (127, 255, 2), (127, 255, 5), (378, 504, 2),
         (756, 1008, 1)]


@pytest.mark.parametrize("h,w,f", CASES, ids=[f"{h}x{w}-{f}f" for h, w, f in CASES])
def test_maps_against_fp64(setup, h, w, f):
    E, sd, wt = setup
    gt, gen = _frames(200 + h + f, f, h, w)
    mask = None
    if f == 2:   # the 2-frame runs take an explicit mask
        mask = np.zeros((h, w), dtype=bool)
        mask[-7:, : w // 2] = True
    g, r = _cuda(gt, gen)
    out = E.lpips_maps(g, r, wt, None if mask is None else torch.from_numpy(mask).to(DEV), per_layer=True)
    ref_map, ref_layers = M.maps64(gt, gen, sd, mask, device=DEV)
    err = (out.map.double() - ref_map).abs().max().item()
    err_l = (out.layer_maps.double() - ref_layers).abs().amax(dim=(0, 2, 3)).cpu().numpy()
    print(f"\n{h}x{w} x {f}: map max {ref_map.max().item():.3f}, max |err| {err:.2e}, per tap {np.array2string(err_l, precision=2)}")
    assert err <= TOL and err_l.max() <= TOL
    scores, per = E.lpips(g, r, wt, None if mask is None else torch.from_numpy(mask).to(DEV), per_layer=True)
    assert torch.equal(out.lpips, scores) and torch.equal(out.per_layer, per)
    if f > 1:   # frame 0's render is its ground truth
        assert torch.all(out.map[0] == 0) and torch.all(out.layer_maps[0] == 0)
    assert float(out.map[-1].max()) > 0


def _run(gt, gen, wt, mask=None, fc=None):
    """nrn_lpips_maps with a workspace of fc frames (default: all) filled with 0xFF: (workspace, LpipsMaps)"""
    from nonrigid_nerf_b200 import _lib, evaluation as E
    lib = _lib.load()
    f, h, w, _ = gt.shape
    fc = f if fc is None else fc
    nbytes = L.mask_bytes(h, w) + fc * M.map_frame_bytes(h, w)
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
    out = E.LpipsMaps(torch.empty(f, device=DEV), torch.empty((f, 5), device=DEV), torch.empty((f, h, w), device=DEV),
                      torch.empty((f, 5, h, w), device=DEV), torch.empty((f, h, w, 3), dtype=torch.uint8, device=DEV))
    a = _lib.NrnLpipsArgs()
    a.gt, a.generated, a.mask = gt.data_ptr(), gen.data_ptr(), None if mask is None else mask.data_ptr()
    a.n_frames, a.height, a.width = f, h, w
    a.packed, a.lpips, a.per_layer = wt.packed.data_ptr(), out.lpips.data_ptr(), out.per_layer.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
    a.stream = torch.cuda.current_stream().cuda_stream
    m = _lib.NrnLpipsMapArgs()
    m.map, m.layer_maps, m.error_image = out.map.data_ptr(), out.layer_maps.data_ptr(), out.error_image.data_ptr()
    _lib.check(lib.nrn_lpips_maps(C.byref(a), C.byref(m)), "lpips_maps")
    torch.cuda.synchronize()
    _lib.device_error_check()
    return ws, out


def _first_nan_tap(per):
    """[F] the first tap whose score is NaN (5: none)"""
    nan = torch.isnan(per).cpu().numpy()
    return [int(np.argmax(row)) if row.any() else 5 for row in nan]


@pytest.mark.parametrize("h,w,f", [(31, 31, 2), (32, 33, 1), (47, 64, 5), (127, 255, 2), (378, 504, 2), (756, 1008, 1)])
def test_upsampling_bit_for_bit(setup, h, w, f):
    E, sd, wt = setup
    gt, gen = _frames(300 + h, f, h, w)
    ws, out = _run(*_cuda(gt, gen), wt)
    taps = [M.tap_map(ws, f, h, w, k) for k in range(L.TAPS)]
    assert all(bool(torch.isfinite(t).all()) for t in taps)   # every tap pixel was written
    total, ups = M.maps32([t.cpu().numpy() for t in taps], h, w)
    assert np.array_equal(out.layer_maps.cpu().numpy(), ups) and np.array_equal(out.map.cpu().numpy(), total)
    assert np.array_equal(out.error_image.cpu().numpy(), M.error_image(total))
    worst = []
    for k, t in enumerate(taps):
        hh, ww = t.shape[1:]
        ref = M.upsample64(t.double(), h, w)
        bound = M.fp32_bound(float(t.max()), hh, ww)
        d = (out.layer_maps[:, k].double() - ref).abs().max().item()
        assert d <= bound, (k, d, bound)
        worst.append(d / max(bound, 1e-300))
        # the tap map's mean is the tap score: the same fp32 distances, summed in fp64 in another order
        mean = t.double().mean(dim=(1, 2))
        assert torch.allclose(mean, out.per_layer[:, k].double(), rtol=1e-6, atol=0), (k, mean, out.per_layer[:, k])
    print(f"\n{h}x{w} x {f}: |up - F.interpolate fp64| / bound per tap {np.array2string(np.array(worst), precision=3)}")
    scores, per = E.lpips(*_cuda(gt, gen), wt, per_layer=True)
    assert torch.equal(out.lpips, scores) and torch.equal(out.per_layer, per)


def test_identity_and_symmetry(setup):
    E, sd, wt = setup
    gt, gen = _frames(41, 5, 96, 128)
    g, r = _cuda(gt, gen)
    one = torch.zeros((96, 128), dtype=torch.uint8, device=DEV)
    same = E.lpips_maps(g, g, wt, one, per_layer=True, error_images=True)
    assert torch.all(same.map == 0) and torch.all(same.layer_maps == 0) and torch.all(same.lpips == 0)
    assert torch.equal(same.error_image.cpu(), torch.from_numpy(M.jet8()[0]).expand(5, 96, 128, 3))
    fwd = E.lpips_maps(g, r, wt, one, per_layer=True, error_images=True)
    back = E.lpips_maps(r, g, wt, one, per_layer=True, error_images=True)
    for a, b in zip(fwd, back):
        assert torch.equal(a, b)
    assert float(fwd.map.max()) > 0


def _all(x):
    return [t for t in x if t is not None]


def test_chunk_independence_and_repeatability(setup):
    E, sd, wt = setup
    f, h, w = 37, 127, 255
    gt, gen = _frames(77, f, h, w)
    g, r = _cuda(gt, gen)
    one = torch.zeros((h, w), dtype=torch.uint8, device=DEV)
    one[5:40, 60:90] = 1
    ref = E.lpips_maps(g, r, wt, one, per_layer=True, error_images=True)
    for chunk in (1, 2, 5):
        got = E.lpips_maps(g, r, wt, one, per_layer=True, error_images=True, chunk_frames=chunk)
        assert all(torch.equal(a, b) for a, b in zip(_all(got), _all(ref))), chunk
    for i in (0, 4, 17, 36):
        got = E.lpips_maps(g[i:i + 1], r[i:i + 1], wt, one, per_layer=True, error_images=True)
        assert all(torch.equal(a[0], b[i]) for a, b in zip(_all(got), _all(ref))), i
    again = E.lpips_maps(g, r, wt, one, per_layer=True, error_images=True)
    assert all(torch.equal(a, b) for a, b in zip(_all(again), _all(ref)))
    # without the optional outputs: the same map and scores
    bare = E.lpips_maps(g, r, wt, one)
    assert bare.per_layer is None and bare.layer_maps is None and bare.error_image is None
    assert torch.equal(bare.map, ref.map) and torch.equal(bare.lpips, ref.lpips)


def test_graph_replay_equals_eager(setup):
    E, sd, wt = setup
    g, r = _cuda(*_frames(44, 5, 96, 128))
    eager = E.lpips_maps(g, r, wt, per_layer=True, error_images=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        E.lpips_maps(g, r, wt, per_layer=True, error_images=True)   # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = E.lpips_maps(g, r, wt, per_layer=True, error_images=True)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(_all(out), _all(eager)))


def _scale_frames():
    """as tests/test_lpips_stages_gpu.py: 3 frames of 224 x 224 and frame 2 again at one tenth the contrast"""
    gt, gen = R.frames(61, 3, 224, 224)
    lo_gt, lo_gen = 0.5 + 0.05 * (gt[2:3] - 0.5), 0.5 + 0.05 * (gen[2:3] - 0.5)
    return np.concatenate([gt, lo_gt]).astype(np.float32), np.concatenate([gen, lo_gen]).astype(np.float32)


@pytest.mark.parametrize("gain", [8.0, 24.0])
def test_saturated_frames_have_nan_maps(gain):
    from nonrigid_nerf_b200 import evaluation as E
    wt = E.lpips_weights(R.he_state_dict(0, gain))
    gt, gen = _scale_frames()
    f, h, w, _ = gt.shape
    g, r = _cuda(gt, gen)
    ws, out = _run(g, r, wt)
    scores, per = E.lpips(g, r, wt, per_layer=True)
    assert torch.equal(out.lpips.isnan(), scores.isnan()) and torch.equal(out.per_layer.isnan(), per.isnan())
    finite = torch.isfinite(scores)
    assert torch.equal(out.lpips[finite], scores[finite]) and torch.equal(out.per_layer[finite], per[finite])
    first = _first_nan_tap(per)
    assert any(k < 5 for k in first), first
    for i, k in enumerate(first):
        assert bool(torch.isnan(out.layer_maps[i, k:]).all()) and bool(torch.isfinite(out.layer_maps[i, :k]).all()), (i, k)
        assert bool(torch.isnan(out.map[i]).all()) == (k < 5) and (k < 5 or bool(torch.isfinite(out.map[i]).all()))
    # the same rule in the fp32 restatement of the kernel's own tap maps, NaN error pixels at jet index 0
    total, ups = M.maps32([M.tap_map(ws, f, h, w, k).cpu().numpy() for k in range(5)], h, w, first)
    assert np.array_equal(out.layer_maps.cpu().numpy(), ups, equal_nan=True)
    assert np.array_equal(out.map.cpu().numpy(), total, equal_nan=True)
    assert np.array_equal(out.error_image.cpu().numpy(), M.error_image(total))
    print(f"\ngain {gain}: first NaN tap per frame {first}")


def test_error_images_bit_for_bit():
    """Tap weights 40 times the default: maps from 0 (frame 0) to well above 1, against the numpy rule on the kernel's map"""
    from nonrigid_nerf_b200 import evaluation as E
    wt = E.lpips_weights(R.random_state_dict(0, lin_scale=40.0))
    gt, gen = _frames(91, 6, 120, 160)
    out = E.lpips_maps(*_cuda(gt, gen), wt, error_images=True)
    mp = out.map.cpu().numpy()
    assert np.any(mp == 0) and np.any(mp >= 1) and np.any((mp > 0) & (mp < 1)), (mp.min(), mp.max())
    assert np.array_equal(out.error_image.cpu().numpy(), M.error_image(mp))
    print(f"\nerror images: map range [{mp.min():.3g}, {mp.max():.3g}], share >= 1: {np.mean(mp >= 1):.3f}")


def _gpu_frames(seed, n, h, w, step=20):
    """[n, h, w, 3] fp32 on the GPU, every frame different (as tests/test_lpips_stages_gpu.py)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    gt = torch.empty((n, h, w, 3), device=DEV)
    gen = torch.empty_like(gt)
    for i in range(0, n, step):
        k = min(step, n - i)
        base = F.interpolate(torch.rand((k, 3, 6, 8), generator=g, device=DEV), size=(h, w), mode="bilinear", align_corners=False)
        x = 0.8 * base + 0.2 * torch.rand((k, 3, h, w), generator=g, device=DEV)
        gt[i:i + k] = x.permute(0, 2, 3, 1)
        gen[i:i + k] = (x + 0.05 * torch.randn((k, 3, h, w), generator=g, device=DEV)).clamp(0, 1).permute(0, 2, 3, 1)
        del base, x
    return gt, gen


def test_outputs_past_2_to_the_31_bytes(setup):
    E, sd, wt = setup
    f, h, w = 180, 756, 1008
    g, r = _gpu_frames(9, f, h, w)
    out = E.lpips_maps(g, r, wt, per_layer=True, error_images=True)
    assert out.layer_maps.numel() * 4 > 2 ** 31 and 179 * 5 * h * w * 4 > 2 ** 31
    scores, per = E.lpips(g, r, wt, per_layer=True)
    assert torch.equal(out.lpips, scores) and torch.equal(out.per_layer, per)
    mask = R.mask_from(g[0].cpu().numpy())
    for i in (0, 1, 178, 179):
        ref_map, ref_layers = M.maps64(g[i:i + 1], r[i:i + 1], sd, mask, device=DEV)
        err = max((out.map[i].double() - ref_map[0]).abs().max().item(), (out.layer_maps[i].double() - ref_layers[0]).abs().max().item())
        assert err <= TOL, (i, err)
        one = E.lpips_maps(g[i:i + 1], r[i:i + 1], wt, torch.from_numpy(mask.astype(np.uint8)).to(DEV), per_layer=True, error_images=True)
        assert all(torch.equal(a[0], b[i]) for a, b in zip(_all(one), _all(out))), i
        print(f"\n180 x 1008 x 756, frame {i}: max |err| {err:.2e}")


def test_empty_batch_and_refusals(setup):
    E, sd, wt = setup
    x = torch.zeros((0, 40, 40, 3), device=DEV)
    out = E.lpips_maps(x, x, wt, per_layer=True, error_images=True)
    assert out.lpips.shape == (0,) and out.map.shape == (0, 40, 40) and out.layer_maps.shape == (0, 5, 40, 40)
    assert out.error_image.shape == (0, 40, 40, 3)
    a = torch.zeros((1, 40, 40, 3), device=DEV)
    for args, kw, msg in (((a, torch.zeros((1, 40, 41, 3), device=DEV), wt), {}, "differ"),
                          ((a, a.cpu(), wt), {}, "CUDA tensor"),
                          ((torch.zeros((1, 30, 64, 3), device=DEV),) * 2 + (wt,), {}, "at least 31"),
                          ((a, a, wt, torch.zeros((40, 41), device=DEV)), {}, "mask must be"),
                          ((a, a, wt, torch.zeros((40, 40))), {}, "mask must be"),
                          ((a, a, wt), {"chunk_frames": 0}, "chunk_frames must be at least 1"),
                          ((a, a, object()), {}, "lpips_weights")):
        with pytest.raises(RuntimeError, match=msg):
            E.lpips_maps(*args, **kw)
        with pytest.raises(RuntimeError, match=msg):   # lpips() refuses the same arguments in the same words
            E.lpips(*args, **kw)
