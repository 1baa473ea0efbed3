"""Stage-by-stage references of the LPIPS kernels (csrc/lpips.cu), each fed with the kernel's own operands as read back
from the workspace (tests/lpips_layout.py), and the checks that compare a stage with them.  Torch and numpy, on any
device: tests/test_lpips_stages_gpu.py runs them on the stages the kernels wrote, tests/test_lpips_stages_cpu.py shows
that each check rejects a stage with a known implicit-GEMM bug.

  input (stage 0)  numpy fp32 in the kernel's order: mask, 2x - 1, - shift, / scale, fp16 round-to-nearest; channels
                   3..7 +0.  Bit for bit.
  pool1, pool2     3 x 3 / 2 floor max of the kernel's own previous stage.  Bit for bit (a max of fp16 values is one of
                   them; only the sign of a zero is left open).
  conv1 .. conv5   z = conv(x, fp16(w)) + b in fp64 on the kernel's own fp16 input stage x, with the weights rounded to
                   fp16 as nrn_lpips_pack rounds them.  Per element
                       |y - relu(z)| <= ulp16(max(|y|, relu(z))) / 2 + 2 (K + 1) 2^-24 (conv(|x|, |w|) + |b|)
                   K is the GEMM depth the kernel runs (ks^2 cin, conv1 with its 8 input channels).  Products of fp16
                   operands are exact in fp32; what is left is their sum with the bias.  Hopper's tensor cores align
                   the terms of an MMA step to its largest exponent and truncate instead of rounding to nearest, so
                   each of the K + 1 additions may lose a whole fp32 unit in the last place (2^-23 relative, twice
                   round-to-nearest's 2^-24): c = 2.  ulp16 has the subnormal spacing 2^-24 below 2^-14.  ReLU is
                   1-Lipschitz, so an output whose z lies within the accumulation term of 0 (the kink) passes on
                   either side.  Also the median of |y - relu(z)| / ulp16 over the outputs clear of the kink must
                   stay below MEDIAN_ULP: rounding to nearest alone gives about 0.25, and a bias of half an ulp or
                   more that the per-element bound would still admit does not.
  distances        per pixel in fp64 from the kernel's own fp16 taps, summed per 256-pixel block: |P - P64| <=
                   64 2^-24 sum_px sum_c w_c (|g_c| / |g| + |r_c| / |r|)^2.  The kernel's per-pixel fp32 chain (see
                   distance_partials) loses at most about 2 m + 12 units of 2^-24 of that sum, m <= 21 the sequential
                   fp32 additions of a channel sum (8 per lane and chunk, then 5 shuffle levels).
  reduce           the tap means (partials in block order, fp64) and their sum in tap order, restated from the
                   read-back partials and saturation words: bit for bit, NaN from the first flagged tap on.
"""
import numpy as np
import torch
import torch.nn.functional as F

from tests import lpips_layout as L
from tests import lpips_reference as R
from tests.parity import half_ulp

U = 2.0 ** -24
C_CONV = 2
C_DIST = 64
MEDIAN_ULP = 0.45
F16_MAX = 65504.0


def conv_weights(sd, device="cpu"):
    """[(w, b)] per layer in fp64: w the fp16 rounding of the fp32 weights (as packed), b the fp32 biases"""
    return [(sd[key + ".weight"].float().half().double().to(device), sd[key + ".bias"].float().double().to(device))
            for key, *_ in R.CONVS]


def lin_weights(sd, device="cpu"):
    return [sd[f"lin{k}.model.1.weight"].float().reshape(-1).double().to(device) for k in range(L.TAPS)]


def gemm_depth(layer):
    cin_real, cin, cout, ks, *_ = L.CONVS[layer]
    return ks * ks * cin


# ---- input -------------------------------------------------------------------------------------------------------------
def input_stage(gt, gen, mask, shift, scale):
    """numpy fp32 gt, gen [F, H, W, 3], mask bool [H, W], shift / scale fp32 [3] -> fp16 [2F, H, W, 8]"""
    x = np.concatenate([gt, gen]).astype(np.float32)
    x = np.where(mask[None, :, :, None], np.float32(0), x)
    t = np.float32(2) * x - np.float32(1)
    s = (t - np.asarray(shift, np.float32)) / np.asarray(scale, np.float32)
    out = np.zeros(s.shape[:3] + (8,), dtype=np.float16)
    out[..., :3] = s.astype(np.float16)
    return out


def check_input(got, gt, gen, mask, shift, scale):
    """got: the kernel's stage 0 [2F, H, W, 8] fp16 (any device)"""
    want = input_stage(gt, gen, mask, shift, scale)
    g = got.cpu().numpy()
    assert g.shape == want.shape, (g.shape, want.shape)
    assert np.all(g[..., 3:].view(np.uint16) == 0), "input channels 3..7 must be +0"
    bad = g.view(np.uint16) != want.view(np.uint16)
    assert not bad.any(), f"input stage: {int(bad.sum())} values differ (first at {np.argwhere(bad)[0].tolist()})"


# ---- pools -------------------------------------------------------------------------------------------------------------
def pool_stage(x):
    """3 x 3 / 2 floor max of fp16 NHWC x -> fp16 NHWC (in fp32, which holds every fp16 value exactly)"""
    y = F.max_pool2d(x.float().permute(0, 3, 1, 2), kernel_size=3, stride=2)
    return y.permute(0, 2, 3, 1).half()


def _bits(x):
    return (x + 0.0).contiguous().view(torch.int16)   # + 0 makes -0 into +0, and nothing else changes


def check_pool(got, prev, name="pool"):
    want = pool_stage(prev)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    bad = _bits(got) != _bits(want)
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} values differ (first at {bad.nonzero()[0].tolist()})"


# ---- convolutions ------------------------------------------------------------------------------------------------------
def conv_reference(x, layer, weights, w_override=None, b_override=None, x_padded=None):
    """fp64 (z, m) [N, ho, wo, cout] of layer `layer` on the fp16 NHWC stage x: z = conv(x, w) + b, m = conv(|x|, |w|) +
    |b|.  w_override / b_override replace the layer's weights; x_padded [N, C, h + 2p, w + 2p] replaces x's zero padding
    (both for the mutations of test_lpips_stages_cpu.py)."""
    cin_real, cin, cout, ks, stride, pad, split = L.CONVS[layer]
    w, b = weights[layer]
    w = w if w_override is None else w_override
    b = b if b_override is None else b_override
    xd = x[..., :cin_real].double().permute(0, 3, 1, 2)
    if x_padded is None:
        z = F.conv2d(xd, w, b, stride=stride, padding=pad)
    else:
        z = F.conv2d(x_padded, w, b, stride=stride)
    m = F.conv2d(xd.abs(), w.abs(), b.abs(), stride=stride, padding=pad)
    return z.permute(0, 2, 3, 1), m.permute(0, 2, 3, 1)


def conv_errors(y, z, m, layer):
    """(worst err / bound, median err / ulp16 clear of the kink, count of outputs clear of the kink) of fp16 outputs y
    against the fp64 pre-activation z with absolute-value sum m"""
    y = y.double()
    r = z.clamp_min(0.0)
    acc = C_CONV * (gemm_depth(layer) + 1) * U * m
    err = (y - r).abs()
    bound = half_ulp(torch.maximum(y.abs(), r)) + acc
    worst = float((err / bound).max()) if err.numel() else 0.0
    clear = r > acc
    ulp = 2 * half_ulp(r[clear])
    med = float((err[clear] / ulp).median()) if bool(clear.any()) else 0.0
    return worst, med, int(clear.sum())


def conv_passes(y, z, m, layer):
    worst, med, _ = conv_errors(y, z, m, layer)
    return worst <= 1.0 and med <= MEDIAN_ULP


def check_conv(y, z, m, layer, log=None, tag=""):
    assert y.shape == z.shape, (layer, y.shape, z.shape)
    finite = torch.isfinite(y)
    assert bool(finite.all()), f"conv{layer + 1}{tag}: {int((~finite).sum())} non-finite outputs"
    worst, med, n = conv_errors(y, z, m, layer)
    line = f"conv{layer + 1}{tag}: max err/bound {worst:.3f}, median err/ulp16 {med:.3f} over {n} outputs clear of the kink"
    if log is not None:
        log.append(line)
    assert worst <= 1.0 and med <= MEDIAN_ULP, line
    return worst, med


# ---- distances and reduce ----------------------------------------------------------------------------------------------
def distance_partials(taps, lin, fc, tap):
    """The kernel's per-pixel distance (lpips_distance_kernel) of its own fp16 tap images taps [2 fc, h, w, C] in fp64,
    summed per 256-pixel block: (P64, B) [fc, blocks], B the absolute-value sum the bound scales with.

    Kernel per pixel, fp32: |g|^2 and |r|^2 as fmaf chains of 8 per lane and 8-channel chunk, a 5-level shuffle sum,
    sqrt, + 1e-10; each channel's g_c / |g| - r_c / |r|, squared, times w_c, again per lane and over the shuffles."""
    x = taps.double()
    g, r = x[:fc], x[fc:]
    ng = torch.sqrt((g * g).sum(-1, keepdim=True)) + 1e-10
    nr = torch.sqrt((r * r).sum(-1, keepdim=True)) + 1e-10
    v = (lin * (g / ng - r / nr) ** 2).sum(-1).reshape(fc, -1)
    s = (lin * (g.abs() / ng + r.abs() / nr) ** 2).sum(-1).reshape(fc, -1)
    n = v.shape[1]
    blocks = -(-n // L.DIST_PIXELS)
    pad = blocks * L.DIST_PIXELS - n
    v, s = F.pad(v, (0, pad)), F.pad(s, (0, pad))
    return v.view(fc, blocks, L.DIST_PIXELS).sum(-1), s.view(fc, blocks, L.DIST_PIXELS).sum(-1)


def distance_errors(p, p64, b):
    err = (p.double() - p64).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / (C_DIST * U * b))
    return float(ratio.max()) if ratio.numel() else 0.0


def check_distance(p, taps, lin, fc, tap, log=None, tag=""):
    """p: the kernel's partials of one tap [fc, blocks]"""
    p64, b = distance_partials(taps, lin, fc, tap)
    assert p.shape == p64.shape, (tap, p.shape, p64.shape)
    assert bool(torch.isfinite(p).all()), f"tap {tap}{tag}: non-finite partials"
    worst = distance_errors(p, p64, b)
    line = f"distance tap {tap}{tag}: max err/bound {worst:.3g}"
    if log is not None:
        log.append(line)
    assert worst <= 1.0, line
    return worst


def reduce_restated(partials, sat, fc, h, w):
    """lpips_reduce_kernel restated from read-back partials [5, fc, max blocks] fp64 and saturation words [2 fc]:
    (lpips [fc], per_layer [fc, 5]) fp32"""
    part = partials.cpu().numpy()
    words = sat.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    out = np.empty(fc, np.float32)
    per = np.empty((fc, L.TAPS), np.float32)
    for f in range(fc):
        clamped = int(words[f] | words[fc + f])
        first = (clamped & -clamped).bit_length() - 1 if clamped else L.TAPS
        total = 0.0
        for k in range(L.TAPS):
            s = 0.0
            for b in range(L.dist_blocks(h, w, k)):
                s += float(part[k, f, b])
            mean = s / float(L.px(h, w, L.TAP_STAGES[k])) if k < first else float("nan")
            per[f, k] = np.float32(mean)
            total += mean
        out[f] = np.float32(total)
    return out, per


def same_bits(a, b):
    """fp32 arrays equal bit for bit, except that any NaN matches any NaN (the GPU's canonical NaN is not numpy's)"""
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def check_reduce(out, per, partials, sat, fc, h, w):
    want, want_per = reduce_restated(partials, sat, fc, h, w)
    got, got_per = out.cpu().numpy(), per.cpu().numpy()
    assert same_bits(got, want), (got, want)
    assert same_bits(got_per, want_per), (got_per, want_per)


# ---- shapes and a rounding-exact simulation of the pipeline --------------------------------------------------------------
# (h, w): each targets an edge of the implicit GEMMs' 128-pixel tiles (two 64-row warpgroups) at some stage
SHAPES = {
    "31x31": (31, 31),          # the smallest frame: conv3-5 are 1 x 1, one valid row of a tile
    "35x35": (35, 35),          # conv1: 64 px, exactly one warpgroup
    "35x67": (35, 67),          # conv1: 128 px, exactly one tile
    "47x143": (47, 143),        # conv1: 385 px, one row past three tiles
    "63x71": (63, 71),          # conv1: 255 px, one short of two tiles
    "63x191": (63, 191),        # conv1: 705 px, 65 into a tile: the second warpgroup has one row
    "71x135": (71, 135),        # pool1 / conv2: 128 px (0 mod 128)
    "127x143": (127, 143),      # pool1 / conv2: 255 px (127 mod 128)
    "31x1000": (31, 1000),      # extreme aspect ratios: conv3-5 one pixel high / wide
    "1000x31": (1000, 31),
    "378x504": (378, 504),      # the example sequence's frame sizes
    "756x1008": (756, 1008),
}


def simulate(sd, gt, gen, mask):
    """The stages an exact kernel would write (every conv output the fp16 rounding of its fp64 value, clamped to 65504
    as the kernels' satfinite convert clamps it) for numpy gt, gen [F, H, W, 3]: (stages [8] fp16 NHWC, {layer: (z, m)}
    of each conv on its simulated input)."""
    weights = conv_weights(sd)
    shift = sd["scaling_layer.shift"].reshape(-1).numpy()
    scale = sd["scaling_layer.scale"].reshape(-1).numpy()
    stages = [torch.from_numpy(input_stage(gt, gen, mask, shift, scale))]
    refs = {}
    for layer in range(L.TAPS):
        s_in = L.IN_STAGE[layer]
        if layer in (1, 2):   # conv2, conv3 read the max-pool of the stage before theirs
            stages.append(pool_stage(stages[s_in - 1]))
        x = stages[s_in]
        z, m = conv_reference(x, layer, weights)
        refs[layer] = (z, m)
        stages.append(z.clamp(0.0, F16_MAX).half())
    return stages, refs
