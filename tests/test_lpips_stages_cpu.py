"""The stage checks of tests/lpips_stages.py can fail: at every shape of lpips_stages.SHAPES, a rounding-exact simulation
of the kernels (every stage the fp16 rounding of its fp64 value) passes them, and the conv check of the affected stage
rejects each of four implicit-GEMM bugs applied to that simulation wherever the bug changes the stage:

  conv2 right pad   the first right padding column of conv2 reads the last real column instead of zero
  conv1 last tap    conv1's ragged last K slab, filter tap ky = kx = 10 (the only real tap of its slab), is dropped
  conv3 half bias   conv3's second N half (channels 192..383) adds the first half's bias
  row 64            output pixel 64 of every 128-pixel tile, the first row of the second warpgroup, holds pixel 63's
                    outputs (each conv layer in turn)

Each mutated stage exceeds its bound by a factor of about 80 or more somewhere (printed with -s)."""
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import lpips_layout as L
from tests import lpips_reference as R
from tests import lpips_stages as S


@functools.lru_cache(maxsize=None)
def _pipeline(shape):
    h, w = S.SHAPES[shape]
    sd = R.random_state_dict(0)
    gt, gen = R.frames(3 + list(S.SHAPES).index(shape), 1, h, w, perturb=(0.1,))
    gt[0, : h // 4, : w // 5] = 0   # a default mask
    mask = R.mask_from(gt[0])
    stages, refs = S.simulate(sd, gt, gen, mask)
    return sd, gt, gen, mask, stages, refs, S.conv_weights(sd)


@pytest.mark.parametrize("shape", list(S.SHAPES))
def test_exact_pipeline_passes_every_check(shape):
    sd, gt, gen, mask, stages, refs, weights = _pipeline(shape)
    h, w = S.SHAPES[shape]
    assert [tuple(s.shape[1:3]) for s in stages] == L.dims(h, w)
    assert [s.shape[3] for s in stages] == list(L.STAGE_CHANNELS)
    S.check_input(stages[0], gt, gen, mask, sd["scaling_layer.shift"].reshape(-1).numpy(), sd["scaling_layer.scale"].reshape(-1).numpy())
    S.check_pool(stages[2], stages[1], "pool1")
    S.check_pool(stages[4], stages[3], "pool2")
    log = []
    for layer in range(L.TAPS):
        _, med = S.check_conv(stages[L.TAP_STAGES[layer]], *refs[layer], layer, log)
        assert 0.2 <= med <= 0.3, log[-1]   # rounding to nearest alone: about 1/4 of an ulp
    lins = S.lin_weights(sd)
    for tap in range(L.TAPS):
        p64, _ = S.distance_partials(stages[L.TAP_STAGES[tap]], lins[tap], 1, tap)
        assert p64.shape == (1, L.dist_blocks(h, w, tap))
        assert S.check_distance(p64.float().double(), stages[L.TAP_STAGES[tap]], lins[tap], 1, tap) <= 1.0
    print(f"\n{shape}: " + "; ".join(log))


def _conv2_right_pad(x, weights):
    _, _, _, ks, stride, pad, _ = L.CONVS[1]
    xd = x.double().permute(0, 3, 1, 2)
    xp = F.pad(xd, (pad, pad, pad, pad))
    hh, ww = xd.shape[-2:]
    xp[:, :, pad:pad + hh, pad + ww] = xd[:, :, :, ww - 1]
    return S.conv_reference(x, 1, weights, x_padded=xp)[0]


def _conv1_last_tap(x, weights):
    w = weights[0][0].clone()
    w[:, :, 10, 10] = 0
    return S.conv_reference(x, 0, weights, w_override=w)[0]


def _conv3_half_bias(x, weights):
    b = weights[2][1].clone()
    b[192:] = b[:192]
    return S.conv_reference(x, 2, weights, b_override=b)[0]


def _row64(z):
    n, hh, ww, c = z.shape
    flat = z.reshape(n, hh * ww, c).clone()
    rows = torch.arange(64, hh * ww, 128)
    flat[:, rows] = flat[:, rows - 1]
    return flat.view(n, hh, ww, c)


MUTATIONS = {"conv2_right_pad": (1, _conv2_right_pad), "conv1_last_tap": (0, _conv1_last_tap),
             "conv3_half_bias": (2, _conv3_half_bias)}


def _rejects(shape, layer, z_mut, name):
    _, _, _, _, stages, refs, _ = _pipeline(shape)
    y, (z, m) = stages[L.TAP_STAGES[layer]], refs[layer]
    y_mut = z_mut.clamp_min(0.0).half()
    if torch.equal(y_mut, y):
        return None
    worst, med, _ = S.conv_errors(y_mut, z, m, layer)
    assert not S.conv_passes(y_mut, z, m, layer), (shape, name, worst, med)
    return worst


@pytest.mark.parametrize("mutation", list(MUTATIONS))
@pytest.mark.parametrize("shape", list(S.SHAPES))
def test_conv_check_rejects_mutation(shape, mutation):
    layer, fn = MUTATIONS[mutation]
    _, _, _, _, stages, _, weights = _pipeline(shape)
    worst = _rejects(shape, layer, fn(stages[L.IN_STAGE[layer]], weights), mutation)
    # each of these changes its stage at every shape: a border column, a tap that reaches into the image, a bias
    assert worst is not None, (shape, mutation)
    print(f"\n{shape} {mutation}: conv{layer + 1} max err/bound {worst:.3g}")


@pytest.mark.parametrize("shape", list(S.SHAPES))
def test_conv_check_rejects_row_64(shape):
    _, _, _, _, stages, refs, _ = _pipeline(shape)
    h, w = S.SHAPES[shape]
    seen = []
    for layer in range(L.TAPS):
        if L.px(h, w, L.TAP_STAGES[layer]) <= 64:
            continue
        worst = _rejects(shape, layer, _row64(refs[layer][0]), f"row 64 conv{layer + 1}")
        if worst is not None:
            seen.append(f"conv{layer + 1} {worst:.3g}")
    # conv1 has more than 64 pixels at every shape but 31 x 31 and 35 x 35, and pixel 64 differs from pixel 63 there
    assert seen or max(L.px(h, w, s) for s in L.TAP_STAGES) <= 64, shape
    print(f"\n{shape} row 64: max err/bound " + ", ".join(seen))


def test_reduce_restatement_flags_nan_from_the_first_saturated_tap():
    h, w, fc = 63, 71, 3
    mb = L.max_blocks(h, w)
    part = torch.rand(L.TAPS, fc, mb, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    sat = torch.tensor([0, 0b10100, 0, 0, 0, 0b01000], dtype=torch.int32)   # frame 1: gt conv3 and conv5; frame 2: render conv4
    out, per = S.reduce_restated(part, sat, fc, h, w)
    assert np.all(np.isfinite(per[0])) and np.isfinite(out[0])
    assert np.all(np.isfinite(per[1, :2])) and np.all(np.isnan(per[1, 2:])) and np.isnan(out[1])
    assert np.all(np.isfinite(per[2, :3])) and np.all(np.isnan(per[2, 3:])) and np.isnan(out[2])
    s = sum(float(part[0, 0, b]) for b in range(L.dist_blocks(h, w, 0))) / L.px(h, w, 1)
    assert per[0, 0] == np.float32(s)
