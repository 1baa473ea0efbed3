"""Helpers of the density gradient's stage tests (tests/test_normals_stages_gpu.py, tests/test_normals_stages_cpu.py): the
launch sizes that make every persistent CTA of field_grad.cu run several tiles, the chunks of a call, the per-point
rounding bound over row blocks, the kernel's bent point restated in fp32, and the fp64 trunk forward at a given point
(its ReLU masks, pre-activations and their magnitudes).  Plain torch; no kernel code."""
import torch

import oracle.nrnerf_oracle as O
from tests import normals_reference as R
from tests import stash_layout as S

# Per-point bound: |g - g64| <= SLACK * bound + ATOL (tests/test_normals_gpu.py explains both)
SLACK, ATOL = 2.0, 1e-6
# fp16's largest finite value: pack_h2_sat clamps the trunk gradients to it
F16_MAX = 65504.0
# fp16's smallest normal value
F16_MIN_NORMAL = 2.0 ** -14
# the fixed scale of the trunk's gradients: loss_scale(1) (field_grad.cu, kUnitAmax)
TRUNK_SCALE = 2.0 ** 9
# a trunk ReLU decided differently from fp64 must sit this close to its kink, relative to its layer: |z| <= 2^-6 |h| |W|
KINK_REL = 2.0 ** -6
TRUNK_STAGES = [f"Y{l}" for l in range(7, -1, -1)]


def tiles(n):
    """Tiles of a launch of n points (tile_count)."""
    return -(-n // S.TILE_M)


def tiles_per_cta(n, num_sms):
    """(fewest, most) tiles a persistent CTA runs: launch_field starts min(tiles, num_sms) CTAs, CTA b runs tiles
    b, b + grid, b + 2 grid, ..."""
    t = tiles(n)
    grid = min(t, num_sms)
    return t // grid, -(-t // grid)


def wave_sizes(num_sms, chunk):
    """Point counts of one launch that make CTAs run several tiles: one full chunk; num_sms + 1 full tiles (CTA 0 runs
    two); 2 num_sms + 1 tiles whose last tile holds one row; chunk - 1."""
    return [chunk, (num_sms + 1) * S.TILE_M, 2 * num_sms * S.TILE_M + 1, chunk - 1]


def chunks(n, chunk):
    """[(first point, points)] of the launches of an n-point call."""
    return [(c0, min(chunk, n - c0)) for c0 in range(0, n, chunk)]


def chunk_of_byte(byte, bytes_per_point, chunk):
    """The chunk whose points' rows of a [P][bytes_per_point] array hold byte `byte`."""
    return byte // bytes_per_point // chunk


def rounding_bound_rows(npar, bp, masks, E, unmasked=None, rigidity=None, block=16384, **kw):
    """R.rounding_bound over row blocks of `block` points, concatenated: the chain and its bound are row-local, so this is
    the same computation with bounded memory."""
    n = E.shape[0]
    out = []
    for a in range(0, n, block):
        b = min(n, a + block)
        out.append(R.rounding_bound(npar, bp, {k: v[a:b] for k, v in masks.items()}, E[a:b],
                                    None if unmasked is None else unmasked[a:b], None if rigidity is None else rigidity[a:b], **kw))
    return tuple(torch.cat([o[i] for o in out]) for i in range(3))


def trunk_capture(npar, bp, masks, E, unmasked=None, rigidity=None, **knobs):
    """The fixed-mask chain's trunk operands y (fp64, true units, as R.fixed_mask_chain captures them) -> {stage: [P, 256]}."""
    cap = {}
    R.fixed_mask_chain(npar, bp, masks, E, unmasked, rigidity, capture=cap, **knobs)
    return {k: cap[k][0] for k in TRUNK_STAGES}


def saturation_step(amax):
    """The smallest k >= 0 at which the largest trunk operand amax (true units) passes fp16's range at the trunk scale
    2^(9 + k): amax 2^(9 + k) > 65504."""
    assert amax > 0.0
    k = 0
    while amax * TRUNK_SCALE * 2.0 ** k <= F16_MAX:
        k += 1
    return k


def near_subnormal(trunk):
    """bool [P]: points with a nonzero trunk operand within 2x of fp16's subnormal range: 0 < |y| 2^9 < 2 * 2^-14.  At a
    scale 2^(9 + k) with k >= 0 the operand is larger, so the unscaled one decides.  Rounded there, fp16 is not
    scale-equivariant."""
    y0 = next(iter(trunk.values()))
    bad = torch.zeros(y0.shape[0], dtype=torch.bool, device=y0.device)
    for y in trunk.values():
        a = y.abs() * TRUNK_SCALE
        bad |= ((a > 0) & (a < 2 * F16_MIN_NORMAL)).any(1)
    return bad


def bent_point(x, unmasked, rigidity, scaling=None):
    """The kernel's bent point in fp32 (field_grad.cu, B4 epilogue): fl(x + fl(fl(rig * un) * s)), fp32 [P, 3]."""
    m = rigidity[:, None] * unmasked
    if scaling is not None:
        m = m * torch.tensor(scaling, dtype=torch.float32, device=m.device)
    return x + m


def encoding64(p):
    """The exact encoding [P, 64] of points p in the kernels' layout: [xyz, sin / cos of 2^k xyz (k = 0..9), 1]."""
    p = p.double()
    return torch.cat([O.positional_encoding(p), torch.ones(p.shape[0], 1, dtype=p.dtype, device=p.device)], 1)


def trunk_forward64(npar, p, z=None, tc=False):
    """fp64 trunk forward (L0 .. L7, no head) at the points p with npar's weights; tc: the latent z [P, 32] enters L0 and
    L5 as NeRF.forward concatenates it.  -> (E [P, 64], {"H1".."H8": mask}, [pre-activation z], [|h_prev| |W|])."""
    E = encoding64(p)
    emb = E[:, :63]
    if tc:
        emb = torch.cat([emb, z.double().expand(p.shape[0], -1)], 1)
    W, b = npar["pts_w"], npar["pts_b"]
    h, masks, pre, mag = emb, {}, [], []
    for l in range(8):
        zl = h @ W[l].T + b[l]
        pre.append(zl)
        mag.append(h.abs() @ W[l].abs().T)
        masks[f"H{l + 1}"] = zl > 0
        h = torch.relu(zl)
        if l == 4:
            h = torch.cat([emb, h], 1)
    return E, masks, pre, mag


def relative(a, b, floor=1e-6):
    """|a - b| / |b| per point (rows), |b| floored."""
    return (a - b).norm(dim=1) / b.norm(dim=1).clamp_min(floor)
