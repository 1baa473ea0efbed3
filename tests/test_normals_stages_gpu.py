"""The density-gradient kernels (csrc/field_grad.cu) against fp64 on every tile of launches in which each persistent CTA
runs several tiles, on every chunk of multi-chunk calls and past 2^31 bytes, with latents per point; the point-mode
forward pinned to the training forward and checked stage by stage; the exact power-of-two scaling of the chain and the
fp16 headroom of its trunk; and the forward's share of the free-running error, point by point.

Each check reads back the workspace of a call (mask bits, encoding E, offsets, rigidity) and evaluates the same chain in
fp64 on those (tests/normals_reference.py).  The lines printed with -s are profiles/r24_*_normals_stages.txt."""
import copy
import math

import pytest
import torch

from nonrigid_nerf_b200 import _lib, geometry, ops
from nonrigid_nerf_b200 import autograd as _ag
from tests import normals_reference as R, normals_stages as NS, stage_reference as SR, stash_layout as S
from tests import test_normals_gpu as T
from tests.parity import Report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KINDS = T.KINDS
# kinds that take a latent per point in the multi-chunk and multi-wave checks; the others with a bender take one latent
PER_POINT = ("bender", "views_bender", "tc")


@pytest.fixture(scope="module")
def chunk():
    return int(_lib.load().nrn_density_gradient_chunk())


@pytest.fixture(scope="module")
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def nets():
    cache = {}

    def get(kind):
        if kind not in cache:
            cache[kind] = T._model(kind)
        return cache[kind]
    return get


def _latents(kind, n, per_point=None, seed=5):
    """None without a latent input; [n, 32] for PER_POINT kinds (or per_point=True), else one [32] latent."""
    if kind in ("canonical", "views"):
        return None
    if per_point if per_point is not None else kind in PER_POINT:
        return (torch.randn(n, 32, generator=torch.Generator().manual_seed(seed)) * 0.3).to(DEV)
    return T._latent(kind)


def _workspace(kind, n, z):
    per_point_bias = int(kind == "tc" and z is not None and z.dim() == 2)
    return torch.empty(_lib.load().nrn_density_gradient_workspace_bytes(n, per_point_bias), dtype=torch.uint8, device=DEV)


def _bound_check(net, kind, x, z, g, ws, tag, report):
    """g of a call of x.shape[0] <= chunk points against R.rounding_bound on its workspace, on every component of every
    point: |g - g64| <= 2 bound + 1e-6, median err / sigma <= 3."""
    n = x.shape[0]
    masks, E, un, rig, _ = T._readback(ws, n)
    npar, bp = R.params(net, fp16=True, device=DEV)
    bent = bp is not None and z is not None
    kn = T._knobs(net) if bent else {}
    ref, bound, sigma = NS.rounding_bound_rows(npar, bp if bent else None, masks, E, un, rig, **kn)
    err = (g.double() - ref).abs()
    lim = NS.SLACK * bound + NS.ATOL
    ratio = float((err / lim).max())
    zs = float((err / (sigma + NS.ATOL)).median())
    report.append(f"{tag}: max err / bound {ratio:.3f}, median err / sigma {zs:.2f}")
    out = ~(err <= lim).all(1)
    assert not bool(out.any()), f"{report[-1]}; {int(out.sum())} points out of bound, first rows {out.nonzero()[:8, 0].tolist()}"
    assert zs <= 3.0, report[-1]


def _print(report):
    for line in report:
        print(line)


# ---- 1. every tile of multi-wave launches --------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_every_tile_of_multi_wave_launches_within_the_bound(kind, nets, chunk, num_sms):
    net, report = nets(kind), []
    for n in NS.wave_sizes(num_sms, chunk):
        x, z = T._points(n, seed=n % 97), _latents(kind, n)
        ws = _workspace(kind, n, z)
        g = geometry._density_gradient(net, x, z, ws)
        _lib.device_error_check()
        lo, hi = NS.tiles_per_cta(n, num_sms)
        _bound_check(net, kind, x, z, g, ws, f"{kind} P={n} ({NS.tiles(n)} tiles, {lo}-{hi} per CTA on {num_sms} SMs)", report)
    _print(report)


# ---- 2. across chunks ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_every_chunk_of_a_multi_chunk_call_is_its_standalone_call(kind, nets, chunk):
    net, report = nets(kind), []
    n = 3 * chunk + 77
    x, z = T._points(n, seed=8), _latents(kind, n)
    g = geometry.density_gradient(net, x, z)
    _lib.device_error_check()
    for c0, m in NS.chunks(n, chunk):
        xs = x[c0:c0 + m].clone()
        zs = z[c0:c0 + m].clone() if z is not None and z.dim() == 2 else z
        ws = _workspace(kind, m, zs)
        gs = geometry._density_gradient(net, xs, zs, ws)
        assert torch.equal(g[c0:c0 + m], gs), (kind, c0, m)
        _bound_check(net, kind, xs, zs, gs, ws, f"{kind} P={n} chunk at {c0} ({m} points) alone", report)
    _print(report)


# ---- 3. the forward with latents per point: pinned to the training forward, and stage by stage ---------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_forward_with_per_point_latents_matches_the_training_forward(kind, nets, chunk):
    """field_fwd_grad_kernel's mask bits, E, offsets and rigidity equal the training forward's (field_fwd.cu) for the
    same points and latents per point, at a full chunk; tc with a ray bias per point."""
    net, n = nets(kind), chunk
    x, z = T._points(n, seed=12), _latents(kind, n, per_point=True, seed=13)
    lib = _lib.load()
    ws = _workspace(kind, n, z)
    geometry._density_gradient(net, x, z, ws)
    _, _, un, rig, (e_off, _, _) = T._readback(ws, n)
    tc = _ag._tc_net(net)
    bent = net.ray_bender[0] is not None and z is not None
    rays = torch.cat([x, torch.zeros(n, 3, device=DEV), torch.full((n, 1), 0.5, device=DEV), torch.full((n, 1), 2.0, device=DEV)], 1)
    zv = torch.ones(n, 1, device=DEV)   # o + 0 * z = o: the same points
    stash = torch.empty(lib.nrn_stash_bytes(n, 1), dtype=torch.uint8, device=DEV)
    mask = torch.empty(lib.nrn_relu_mask_bytes(n, 1), dtype=torch.uint8, device=DEV)
    kn = T._knobs(net) if bent else dict(cutoff=None, scaling=None, removal=None)
    out_ch = 4 if getattr(net, "use_viewdirs", False) else net.output_linear.weight.shape[0]
    _, det = ops.field_forward(rays, zv, z, ops.pack_nerf(net), ops.pack_bender(net.ray_bender[0]) if bent else None, out_ch,
                               kn["cutoff"], kn["scaling"], kn["removal"], want_details=True, stash=stash, relu_mask=mask, tc_net=tc)
    torch.cuda.synchronize()
    t = T._tiles(n)
    used = S.MASK_TILE if bent else S.MK_HB1[0]   # without a bender the Hb images are written by neither kernel
    mk_ws, mk_tr = ws[:t * S.MASK_TILE].view(t, S.MASK_TILE), mask[:t * S.MASK_TILE].view(t, S.MASK_TILE)
    assert torch.equal(mk_ws[:, :used], mk_tr[:, :used])
    assert torch.equal(S.image(ws[e_off:], S.E_BYTES, 0, 8, t).view(torch.int16),
                       S.image(stash, S.STASH_TILE, S.ST_E[0], 8, t).view(torch.int16))
    if bent:
        assert torch.equal(un, det["unmasked_offsets"].reshape(n, 3))
        assert torch.equal(rig, det["rigidity_mask"].reshape(n))


@pytest.mark.parametrize("mode", ["bender", "canonical", "tc"])
def test_forward_at_the_gradients_points_stage_by_stage_with_per_point_latents(mode, chunk):
    """The training forward at the density gradient's points, one latent per point, every stage against fp64 of its own
    fp16 operands (stage_reference.check_forward); the test above ties the density gradient's forward to it bit for bit.
    The training stash is written in ray mode only, so each point is a ray of one sample with o = x, d = 0, z = 1, whose
    sample is exactly x (test_field_variants_gpu: point mode equals this ray mode)."""
    cs = SR.Case(chunk, 1, bender=mode == "bender", tc=mode == "tc")
    x = T._points(chunk, seed=12).contiguous()
    cs.rays[:, :3], cs.rays[:, 3:6] = x, 0.0
    cs.z = torch.ones_like(cs.z)
    if mode != "canonical":
        cs.lat = (torch.randn(chunk, 32, generator=torch.Generator().manual_seed(13)) * 0.3).to(DEV).contiguous()
    o = SR.run_forward(cs)
    assert torch.equal(o["init"], x)
    rep = Report(f"points {mode} P={chunk}", quiet=True)
    SR.check_forward(cs, o, rep)
    rep.worst()


# ---- 4. past 2^31 bytes ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["bender", "canonical"])
def test_past_2_31_bytes(kind, nets, chunk):
    """bender: latents per point past 2^31 bytes (128 B per point); canonical: points and output past 2^31 bytes (12 B per
    point).  The first chunk, the chunks on either side of byte 2^31 and the last equal their standalone calls and are
    within the bound."""
    net, report = nets(kind), []
    if kind == "bender":
        n, per_point_bytes = 2 ** 24 + 300, 128
    else:
        n, per_point_bytes = math.ceil(2 ** 31 / 12) + 300, 12
    gen = torch.Generator(device=DEV).manual_seed(21)
    x = torch.rand(n, 3, device=DEV, generator=gen) * 2.4 - 1.2
    z = torch.randn(n, 32, device=DEV, generator=gen) * 0.3 if kind == "bender" else None
    try:
        g = geometry.density_gradient(net, x, z)
        _lib.device_error_check()
        last = (n - 1) // chunk
        at = NS.chunk_of_byte(2 ** 31, per_point_bytes, chunk)
        for c in sorted({0, at - 1, at, last}):
            c0 = c * chunk
            m = min(chunk, n - c0)
            xs = x[c0:c0 + m].clone()
            zs = z[c0:c0 + m].clone() if z is not None else None
            ws = _workspace(kind, m, zs)
            gs = geometry._density_gradient(net, xs, zs, ws)
            assert torch.equal(g[c0:c0 + m], gs), (kind, c)
            _bound_check(net, kind, xs, zs, gs, ws, f"{kind} P={n} chunk {c} (points {c0}..{c0 + m - 1}, bytes "
                         f"{c0 * per_point_bytes}..{(c0 + m) * per_point_bytes - 1})", report)
        _print(report)
    finally:
        del x, z
        g = None
        torch.cuda.empty_cache()


# ---- 5. exact power-of-two scaling and the fp16 headroom ---------------------------------------------------------------
def _scaled(net, k):
    """A copy of net whose density head row is scaled by 2^k: output_linear.weight[3], or alpha_linear for a
    view-dependent trunk.  The row is first rounded to fp16 values, so that its fp16 image scales exactly too."""
    out = copy.deepcopy(net)
    with torch.no_grad():
        row = out.alpha_linear.weight[0] if getattr(out, "use_viewdirs", False) else out.output_linear.weight[3]
        row.copy_(row.half().float() * 2.0 ** k)
    return out


@pytest.mark.parametrize("kind", KINDS)
def test_power_of_two_head_scaling_is_exact_below_saturation(kind, nets):
    """The point-mode forward has no head, so 2^k on the density head row leaves masks, E, offsets and rigidity alone,
    scales every fp16 trunk operand exactly and is cancelled in the bender chain by its row scale: g(2^k) = 2^k g(1) bit
    for bit while no operand saturates (k < k_sat) and none is fp16-subnormal; past k_sat the clamp breaks it."""
    n = 8192
    base = _scaled(nets(kind), 0)
    x, z = T._points(n, seed=31), _latents(kind, n)
    ws = _workspace(kind, n, z)
    g1 = geometry._density_gradient(base, x, z, ws)
    masks, E, un, rig, _ = T._readback(ws, n)
    npar, bp = R.params(base, fp16=True, device=DEV)
    bent = bp is not None and z is not None
    trunk = NS.trunk_capture(npar, bp if bent else None, masks, E, un, rig, **(T._knobs(base) if bent else {}))
    amax = max(float(y.abs().max()) for y in trunk.values())
    k_sat = NS.saturation_step(amax)
    excl = NS.near_subnormal(trunk)
    keep = ~excl
    line = (f"{kind} P={n}: largest trunk operand {amax * NS.TRUNK_SCALE:.4g} at 2^9, k_sat {k_sat} (headroom 2^{k_sat}); "
            f"points excluded near fp16 subnormals {int(excl.sum())} ({float(excl.double().mean()):.2%})")
    assert float(excl.double().mean()) <= 0.05, line
    # A kernel operand can sit in fp16's subnormal range where the fp64 one does not.  Rounded there it moves g by far
    # less than an fp32 ulp, so a point outside the band may still differ, by a few ulps at most; those are counted.
    ulps = 0
    for k in range(k_sat):
        gk = geometry._density_gradient(_scaled(base, k), x, z, ws)
        want = g1 * 2.0 ** k
        diff = ~(gk == want).all(1) & keep
        far = ~((gk - want).abs() <= 2.0 ** -21 * want.abs().amax(1, keepdim=True)).all(1) & keep
        ulps = max(ulps, int(diff.sum()))
        assert not bool(far.any()), f"{line}; k={k}: {int(far.sum())} points differ from 2^k g(1) by more than 4 ulps"
    line += f"; outside it, points off 2^k g(1) by at most 4 ulps {ulps}"
    assert float((excl.double().sum() + ulps) / n) <= 0.05, line
    gk = geometry._density_gradient(_scaled(base, k_sat + 1), x, z, ws)
    broken = ~(gk == g1 * 2.0 ** (k_sat + 1)).all(1) & keep
    line += f"; at k_sat + 1 the identity breaks at {int(broken.sum())} points"
    print(line)
    assert bool(broken.any()), line
    assert k_sat >= 4, f"{line}: less than 2^4 of headroom at the fixed trunk scale"


# ---- 6. the forward's share of the free-running error ------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_free_running_error_split_into_bent_point_and_mask_flips(kind, nets):
    """g_b: fp64 at the kernel's own fp32 bent point (and its bender path), with its own encoding and trunk masks.
    (a) where every trunk mask of g_b is the kernel's, g is within the rounding bound plus the encoding's fp16 rounding;
    (b) every trunk mask bit that differs sits at a unit near its kink, |z64| <= 2^-6 |h_prev| |W|;
    (c) the free-running error g - g_free splits into g_b - g_free (the bent point) and g - g_b (mask flips)."""
    net, n = nets(kind), 16384
    x, z = T._points(n, seed=41), _latents(kind, n)
    ws = _workspace(kind, n, z)
    g = geometry._density_gradient(net, x, z, ws).double()
    masks, E, un, rig, _ = T._readback(ws, n)
    npar, bp = R.params(net, fp16=True, device=DEV)
    bent = bp is not None and z is not None
    kn = T._knobs(net) if bent else {}
    bpb = bp if bent else None
    xb = NS.bent_point(x, un, rig, kn.get("scaling")) if bent else x
    assert torch.equal(E[:, :3], xb.half().double()), "E's xyz columns are not fp16 of the restated bent point"
    tc = kind == "tc"
    zz = None if z is None else z.expand(n, 32)
    E_b, m_b, pre, mag = NS.trunk_forward64(npar, xb, zz, tc=tc)
    g_b = R.fixed_mask_chain(npar, bpb, {**masks, **m_b}, E_b, un, rig, **kn)
    flip = torch.zeros(n, dtype=torch.bool, device=DEV)
    worst = 0.0
    for l in range(8):
        d = m_b[f"H{l + 1}"] != masks[f"H{l + 1}"]
        flip |= d.any(1)
        if bool(d.any()):
            worst = max(worst, float((pre[l].abs() / mag[l])[d].max()))
    # (a)
    _, bound_e, _ = NS.rounding_bound_rows(npar, bpb, masks, E, un, rig, e_term=True, **kn)
    err = (g - g_b).abs()
    lim = NS.SLACK * bound_e + NS.ATOL
    same = ~flip
    ratio = float((err / lim)[same].max())
    # (c)
    g_free = R.density_gradient(npar, bpb, x, zz if (bent or tc) else None, tc=tc, **kn)
    e_bent, e_flip = (g_b - g_free).norm(dim=1), (g - g_b).norm(dim=1)
    off = NS.relative(g, g_free) > 2e-2
    mass = float(e_bent.sum() / (e_bent.sum() + e_flip.sum()).clamp_min(1e-300))
    n_off = max(int(off.sum()), 1)
    line = (f"{kind} P={n}: free-running rel > 2e-2 at {float(off.double().mean()):.2%} of points; of those, bent point "
            f"dominant {int((off & (e_bent >= e_flip)).sum()) / n_off:.1%}, trunk mask flips dominant "
            f"{int((off & (e_bent < e_flip)).sum()) / n_off:.1%}; error mass: bent point {mass:.1%}, mask flips {1 - mass:.1%}; "
            f"points with a trunk mask flip {float(flip.double().mean()):.2%}, largest |z64| / (|h| |W|) at a flip {worst:.2e}; "
            f"without flips max err / (bound + E term) {ratio:.3f}")
    print(line)
    assert bool((err <= lim).all(1)[same].all()), line
    assert worst <= NS.KINK_REL, line
