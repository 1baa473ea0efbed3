"""Every stage of the LPIPS kernels (csrc/lpips.cu) against a reference of that one stage fed with the kernel's own
operands, read back from a workspace the test owns (layout: tests/lpips_layout.py; references and bounds:
tests/lpips_stages.py): the input stage and the max-pools bit for bit, the five implicit-GEMM convolutions per element
against fp64 of their own fp16 input stage, the distance partials against fp64 per 256-pixel block, the reduce bit for
bit.  The workspace is filled with 0xFF first, so a stage a kernel did not write reads as NaN.

- shapes: lpips_stages.SHAPES, each an edge of the 128-pixel tiles at some stage, with 1, 2 and 5 frames (ground truth
  first, then renders, so the image index of the tiles and of the distances' fc + f is exercised), one run in chunks;
- a chunk of 180 frames at 1008 x 756: its input stage spans 4.4 GB and conv1 2.2 GB, so images 179 and 359 lie past
  2^31 and 2^32 bytes; the stages of images 0, 179, 180 and 359 are checked, and the scores equal chunk_frames=1's;
- activation scale: He-normal weights times a per-layer gain of 0.25 (fp16 subnormals), 1, 2 and 4, and PyTorch's
  default initialisation: every stage and the score against tests/lpips_reference.py;
- saturation: gains 8 and 24 take some convolution outputs past 65504; those frames score NaN from the first such tap
  on, and the words that flag them match the fp64 outputs of the kernel's own inputs.

`pytest -s` prints each stage's worst error over its bound, the median error in fp16 ulps and each weight set's
activation range."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import lpips_layout as L
from tests import lpips_reference as R
from tests import lpips_stages as S
from tests.parity import poison_f32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 5e-4   # end to end, as tests/test_lpips_gpu.py


def _run(gt, gen, wt, mask=None, fc=None):
    """nrn_lpips on device frames gt, gen [F, H, W, 3] with a workspace of fc frames (default: all), filled with 0xFF:
    (workspace bytes, lpips [F], per_layer [F, 5], frames in the last chunk)"""
    from nonrigid_nerf_b200 import _lib
    lib = _lib.load()
    f, h, w, _ = gt.shape
    fc = f if fc is None else fc
    nbytes = L.mask_bytes(h, w) + fc * L.frame_bytes(h, w)
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
    out, per = poison_f32(f), poison_f32(f, 5)
    a = _lib.NrnLpipsArgs()
    a.gt, a.generated, a.mask = gt.data_ptr(), gen.data_ptr(), None if mask is None else mask.data_ptr()
    a.n_frames, a.height, a.width = f, h, w
    a.packed, a.lpips, a.per_layer = wt.packed.data_ptr(), out.data_ptr(), per.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
    a.stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.nrn_lpips(C.byref(a)), "lpips")
    torch.cuda.synchronize()
    _lib.device_error_check()
    return ws, out, per, f - (f - 1) // fc * fc


def _check_stages(ws, sd, sel, mask, h, w, fcl, images, log, tag, in_range=None):
    """Every stage of the listed images of the last chunk of fcl frames (image i < fcl: ground truth of its frame i, else
    the render of frame i - fcl), whose numpy frames are sel [len(images), H, W, 3].  in_range(layer, z, m) -> bool
    [len(images)]: the images whose conv outputs are checked (default: those whose fp64 outputs stay in fp16's range).
    Returns {layer: the largest fp64 output of each image}."""
    weights = [(w_.to(DEV), b_.to(DEV)) for w_, b_ in S.conv_weights(sd)]
    shift, scale = sd["scaling_layer.shift"].reshape(-1).numpy(), sd["scaling_layer.scale"].reshape(-1).numpy()
    stage = lambda s: L.stage_images(ws, fcl, h, w, s, images)
    S.check_input(stage(0), sel, sel[:0], mask, shift, scale)
    S.check_pool(stage(2), stage(1), f"pool1{tag}")
    S.check_pool(stage(4), stage(3), f"pool2{tag}")
    zmax = {}
    for layer in range(L.TAPS):
        z, m = S.conv_reference(stage(L.IN_STAGE[layer]), layer, weights)
        zmax[layer] = z.flatten(1).max(1).values.cpu()
        keep = zmax[layer] <= S.F16_MAX if in_range is None else in_range(layer, z, m)
        if bool(keep.any()):
            k = keep.nonzero().flatten().to(DEV)
            S.check_conv(stage(L.TAP_STAGES[layer]).index_select(0, k), z.index_select(0, k), m.index_select(0, k), layer, log, tag)
    return zmax


def _check_distances(ws, sd, h, w, fcl, frames, log, tag):
    """The distance partials of the listed frames of the last chunk"""
    lins = [x.to(DEV) for x in S.lin_weights(sd)]
    part = L.partials(ws, fcl, h, w)
    images = list(frames) + [fcl + f for f in frames]
    for tap in range(L.TAPS):
        taps = L.stage_images(ws, fcl, h, w, L.TAP_STAGES[tap], images)
        p = part[tap, list(frames), :L.dist_blocks(h, w, tap)]
        S.check_distance(p, taps, lins[tap], len(frames), tap, log, tag)


def _frames(seed, f, h, w):
    gt, gen = R.frames(seed, f, h, w, perturb=(0.1,) if f == 1 else (0.0, 0.01, 0.03, 0.1, 0.3))
    gt[0, h // 3:h // 3 + 9, w // 4:w // 4 + 13] = 0   # a default mask (for the runs without an explicit one)
    return gt, gen


CASES = [(s, f) for s in S.SHAPES for f in ((1, 2, 5) if S.SHAPES[s][0] * S.SHAPES[s][1] < 100000 else (1, 2))]


@pytest.fixture(scope="module")
def default_weights():
    from nonrigid_nerf_b200 import evaluation as E
    sd = R.random_state_dict(0)
    return sd, E.lpips_weights(sd)


@pytest.mark.parametrize("shape,f", CASES, ids=[f"{s}-{f}f" for s, f in CASES])
def test_stages_against_fp64(default_weights, shape, f):
    sd, wt = default_weights
    h, w = S.SHAPES[shape]
    gt, gen = _frames(100 + f + list(S.SHAPES).index(shape), f, h, w)
    explicit = f == 2   # the 2-frame runs take an explicit mask, the others the default one
    if explicit:
        mask = np.zeros((h, w), dtype=bool)
        mask[-7:, : w // 2] = True
    else:
        mask = R.mask_from(gt[0])
        assert mask.sum() == 9 * 13
    g, r = torch.from_numpy(gt).to(DEV), torch.from_numpy(gen).to(DEV)
    # 5 frames in one chunk, or (every other shape) in chunks of 3 and 2: the last chunk's stages are read
    fc = 3 if f == 5 and list(S.SHAPES).index(shape) % 2 else None
    ws, out, per, fcl = _run(g, r, wt, torch.from_numpy(mask.astype(np.uint8)).to(DEV) if explicit else None, fc)
    if not explicit:
        assert np.array_equal(L.mask(ws, h, w).cpu().numpy() != 0, mask)   # the mask kernel's output
    f0 = f - fcl
    log = []
    _check_stages(ws, sd, np.concatenate([gt[f0:], gen[f0:]]), mask, h, w, fcl, list(range(2 * fcl)), log, "")
    _check_distances(ws, sd, h, w, fcl, range(fcl), log, "")
    assert torch.equal(L.sat_words(ws, fcl, h, w).cpu(), torch.zeros(2 * fcl, dtype=torch.int32))
    S.check_reduce(out[f0:], per[f0:], L.partials(ws, fcl, h, w), L.sat_words(ws, fcl, h, w), fcl, h, w)
    ref, ref_per = R.lpips(gt, gen, sd, mask=mask)
    assert np.abs(out.cpu().double().numpy() - ref).max() <= TOL and np.abs(per.cpu().double().numpy() - ref_per).max() <= TOL
    print(f"\n{shape} x {f} frames (last chunk {fcl}): " + "; ".join(log))


def _gpu_frames(seed, n, h, w, step=20):
    """[n, h, w, 3] fp32 on the GPU: a smooth field (bilinear from 6 x 8) plus noise per ground truth frame, the render its
    ground truth plus noise of 0.05; every frame different"""
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


def test_chunk_past_2_to_the_32_bytes(default_weights):
    from nonrigid_nerf_b200 import evaluation as E
    sd, wt = default_weights
    f, h, w = 180, 756, 1008
    g, r = _gpu_frames(7, f, h, w)
    ws, out, per, fcl = _run(g, r, wt, fc=f)
    assert fcl == f and ws.numel() > 10 * 2 ** 30
    # byte offsets inside the stage buffers: image 179 of the input stage past 2^31, image 359 past 2^32; in conv1 past 2^31
    ib0, ib1 = L.image_bytes(h, w, 0), L.image_bytes(h, w, 1)
    assert 179 * ib0 > 2 ** 31 and 359 * ib0 > 2 ** 32 and 359 * ib1 > 2 ** 31
    images = [0, 179, 180, 359]   # ground truth 0 and 179, renders 0 and 179 (the last image of the chunk)
    frames = [0, 179]
    sel = torch.stack([g[0], g[179], r[0], r[179]]).cpu().numpy()
    mask = R.mask_from(g[0].cpu().numpy())
    log = []
    _check_stages(ws, sd, sel, mask, h, w, f, images, log, " 180f")
    _check_distances(ws, sd, h, w, f, frames, log, " 180f")
    sat = L.sat_words(ws, f, h, w)
    assert int(sat.abs().sum()) == 0
    S.check_reduce(out, per, L.partials(ws, f, h, w), sat, f, h, w)
    del ws
    torch.cuda.empty_cache()
    one, one_per = E.lpips(g, r, wt, per_layer=True, chunk_frames=1)
    assert torch.equal(one, out) and torch.equal(one_per, per)
    assert bool(torch.isfinite(out).all()) and float(out.min()) > 0
    print("\n180 x 1008 x 756 in one chunk: " + "; ".join(log))


# ---- activation scale ------------------------------------------------------------------------------------------------
SETS = {"default": lambda: R.random_state_dict(0), "he x0.25": lambda: R.he_state_dict(0, 0.25),
        "he x1": lambda: R.he_state_dict(0, 1.0), "he x2": lambda: R.he_state_dict(0, 2.0), "he x4": lambda: R.he_state_dict(0, 4.0)}
SATURATING = {"he x8": lambda: R.he_state_dict(0, 8.0), "he x24": lambda: R.he_state_dict(0, 24.0)}


def _scale_frames():
    """3 frames of 224 x 224 and a fourth, frame 2 at one tenth the contrast (its activations about 5x smaller)"""
    gt, gen = R.frames(61, 3, 224, 224)
    lo_gt, lo_gen = 0.5 + 0.05 * (gt[2:3] - 0.5), 0.5 + 0.05 * (gen[2:3] - 0.5)
    return np.concatenate([gt, lo_gt]).astype(np.float32), np.concatenate([gen, lo_gen]).astype(np.float32)


def _ranges(ws, fcl, h, w, zmax, name):
    parts = []
    for s in range(1, L.STAGES):
        x = L.stage(ws, fcl, h, w, s).float().abs()
        nz = x[x > 0]
        tiny = float(nz.min()) if nz.numel() else 0.0
        line = f"{['in', 'conv1', 'pool1', 'conv2', 'pool2', 'conv3', 'conv4', 'conv5'][s]} max {float(x.max()):.4g} min>0 {tiny:.3g}"
        if s in L.TAP_STAGES:
            line += f" (fp64 max {float(zmax[L.TAP_STAGES.index(s)].max()):.4g})"
        parts.append(line)
    return f"{name}: " + ", ".join(parts)


@pytest.mark.parametrize("name", list(SETS))
def test_activation_scale(name):
    from nonrigid_nerf_b200 import evaluation as E
    sd = SETS[name]()
    wt = E.lpips_weights(sd)
    gt, gen = _scale_frames()
    f, h, w, _ = gt.shape
    ws, out, per, fcl = _run(torch.from_numpy(gt).to(DEV), torch.from_numpy(gen).to(DEV), wt)
    mask = R.mask_from(gt[0])
    log = []
    zmax = _check_stages(ws, sd, np.concatenate([gt, gen]), mask, h, w, fcl, list(range(2 * f)), log, f" {name}")
    assert all(float(zmax[k].max()) <= S.F16_MAX for k in zmax), "this weight set leaves fp16's range"
    _check_distances(ws, sd, h, w, fcl, range(f), log, f" {name}")
    S.check_reduce(out, per, L.partials(ws, f, h, w), L.sat_words(ws, f, h, w), f, h, w)
    assert int(L.sat_words(ws, f, h, w).abs().sum()) == 0
    ref, ref_per = R.lpips(gt, gen, sd)
    err = max(np.abs(out.cpu().double().numpy() - ref).max(), np.abs(per.cpu().double().numpy() - ref_per).max())
    assert err <= TOL, (name, err)
    if name == "he x0.25":   # outputs below 2^-14 (fp16 subnormals) occur, and were checked with the subnormal spacing
        smallest = [L.stage(ws, f, h, w, s).float() for s in L.TAP_STAGES]
        assert min(float(x[x > 0].min()) for x in smallest) < 2 ** -14
    print(f"\n{_ranges(ws, f, h, w, zmax, name)}; LPIPS max |err| {err:.2e}\n  " + "\n  ".join(log))


@pytest.mark.parametrize("name", list(SATURATING))
def test_saturated_frames_score_nan(name):
    """A convolution output above 65504 makes its frame's score NaN, and its tap scores from that tap on; the words that
    flag it are set exactly where an fp64 output of the kernel's own inputs exceeds 65504 (outside the accumulation
    bound of it); the other frames and taps are unaffected."""
    from nonrigid_nerf_b200 import evaluation as E
    sd = SATURATING[name]()
    wt = E.lpips_weights(sd)
    gt, gen = _scale_frames()
    f, h, w, _ = gt.shape
    ws, out, per, fcl = _run(torch.from_numpy(gt).to(DEV), torch.from_numpy(gen).to(DEV), wt)
    mask = R.mask_from(gt[0])
    words = L.sat_words(ws, f, h, w).cpu()
    expect = torch.zeros(2 * f, dtype=torch.int64)
    clear = torch.ones(2 * f, dtype=torch.bool)

    def in_range(layer, z, m):
        acc = S.C_CONV * (S.gemm_depth(layer) + 1) * S.U * m
        over = ((z - acc) > S.F16_MAX).flatten(1).any(1).cpu()
        near = ((z + acc) > S.F16_MAX).flatten(1).any(1).cpu() & ~over
        expect.add_(over.long() << layer)
        clear.logical_and_(~near)
        return ~(over | near)

    log = []
    zmax = _check_stages(ws, sd, np.concatenate([gt, gen]), mask, h, w, fcl, list(range(2 * f)), log, f" {name}", in_range)
    assert bool(clear.all()), "an fp64 output lies within rounding of 65504: the flag may go either way"
    assert torch.equal(words.long() & 0xFFFFFFFF, expect), (words, expect)
    S.check_reduce(out, per, L.partials(ws, f, h, w), words, f, h, w)
    flagged = (expect[:f] | expect[f:]).tolist()
    firsts = [(bits & -bits).bit_length() - 1 if bits else L.TAPS for bits in flagged]
    assert any(flagged) and len(set(firsts)) > 1, firsts   # frames differ in their first NaN tap, or have none
    ref, ref_per = R.lpips(gt, gen, sd)
    o, p = out.cpu().double().numpy(), per.cpu().double().numpy()
    for i, (bits, first) in enumerate(zip(flagged, firsts)):
        assert np.all(np.isnan(p[i, first:])) and np.all(np.abs(p[i, :first] - ref_per[i, :first]) <= TOL), (i, p[i], ref_per[i])
        assert (np.isnan(o[i]) if bits else abs(o[i] - ref[i]) <= TOL), (i, o[i], ref[i])
    print(f"\n{_ranges(ws, f, h, w, zmax, name)}\n  first NaN tap per frame {firsts}; fp64 LPIPS {np.round(ref, 4).tolist()}\n  " +
          "\n  ".join(log))
