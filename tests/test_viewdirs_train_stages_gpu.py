"""Training the view-dependent head without a bender, stage by stage: every buffer is filled with NaN first, then the
training forward and backward run through the C ABI, and each new stage is checked against fp64 of the kernel's own fp16
operands (read back from its stashes), with the per-element bound c 2^-24 (|A| |W|) (+ 0.5 ulp of fp16 where the result is
stored as fp16), c = K + 2 for a product of depth K:

    dYv = fp16(d_raw . rgb_linear) * [hv > 0]                 (K = 16)
    dF  = fp16(dYv . views_linears.0[:, :256])                (K = 128)
    dY7 = fp16(dF . feature_linear + d_alpha alpha_linear) * [h8 > 0]   (K = 256 + 16)
    the head block of the flat gradient: feature_linear, views_linears.0 (feature and direction columns), alpha_linear
    (row 3 of the head job), rgb_linear, weights and biases, as sums over all points / loss scale (c = P + 2)

Which wrong implementation each check catches: the Hv mask not applied (dYv), ViewsF^T reading the direction columns (dF),
the alpha term dropped (dY7), a head block in the wrong order or a wrong partial layout in the reduce (the flat head
block), a row of a ragged tile left unwritten or non-finite (every row of every tile is finite after the NaN fill).
Shapes: a ragged single tile, 1023 x 64, S = 100, 1024 x 128; the loss-scale edges (upstream 0, 1e-15, 1e10)."""
import ctypes as C

import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import stash_layout as SL
from tests.parity import DEV, F64, U, half_ulp
from tests.viewdirs_reference import build_view_models

pytestmark = pytest.mark.gpu

V_STASH_TILE, V_GRAD_TILE, HV_MASK_TILE = 106496, 98304, 2048
VS_DIR, VS_F, VS_HV = (0, 4), (4 * SL.CHUNK, 32), (36 * SL.CHUNK, 16)
VG_YV, VG_F = (0, 16), (16 * SL.CHUNK, 32)
TRUNK_FLOATS = 493056
HEAD_SHAPES = [("views_linears.0.weight", (128, 283)), ("views_linears.0.bias", (128,)), ("feature_linear.weight", (256, 256)),
               ("feature_linear.bias", (256,)), ("alpha_linear.weight", (1, 256)), ("alpha_linear.bias", (1,)),
               ("rgb_linear.weight", (3, 128)), ("rgb_linear.bias", (3,))]


def _nan(nbytes):
    return torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)   # every fp16 / fp32 a NaN


def _run(net, n, s, seed, factor):
    from nonrigid_nerf_b200 import _lib, ops
    lib = _lib.load()
    r = O.make_rays(seed, n)
    g = torch.Generator().manual_seed(seed)
    t = torch.sort(torch.rand(n, s, generator=g), -1).values
    z = (r["near"] * (1.0 - t) + r["far"] * t).float().to(DEV)
    rays = helpers.rays8(r, DEV)
    vd = torch.nn.functional.normalize(rays[:, 3:6], dim=-1).contiguous()
    nerf_pack, views_pack, views_t = ops.pack_nerf(net), ops.pack_views(net), ops.pack_views_t(net)
    b = {k: _nan(f(n, s)) for k, f in (("stash", lib.nrn_stash_bytes), ("relu_mask", lib.nrn_relu_mask_bytes),
                                        ("views_stash", lib.nrn_views_stash_bytes), ("hv_mask", lib.nrn_hv_mask_bytes),
                                        ("grad_stash", lib.nrn_grad_stash_bytes), ("views_grad_stash", lib.nrn_views_grad_stash_bytes))}
    raw = torch.full((n, s, 4), float("nan"), device=DEV)
    a, v, tr = _lib.NrnFieldArgs(), _lib.NrnViewArgs(), _lib.NrnViewTrainArgs()
    a.rays, a.z_vals, a.n_rays, a.n_samples, a.out_ch, a.nerf_packed, a.raw = rays.data_ptr(), z.data_ptr(), n, s, 4, nerf_pack.data_ptr(), raw.data_ptr()
    a.stash, a.relu_mask = b["stash"].data_ptr(), b["relu_mask"].data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    v.views_packed, v.viewdirs, v.viewdirs_stride = views_pack.data_ptr(), vd.data_ptr(), 3
    tr.views_stash, tr.hv_mask = b["views_stash"].data_ptr(), b["hv_mask"].data_ptr()
    _lib.check(lib.nrn_field_forward_views_train(C.byref(a), C.byref(v), C.byref(tr)), "forward")
    d_raw = (torch.randn(n, s, 4, generator=torch.Generator().manual_seed(seed + 1)) * factor).float().to(DEV)
    flat = torch.full((lib.nrn_nerf_views_grad_floats(),), float("nan"), device=DEV)
    scratch = torch.empty(lib.nrn_wgrad_scratch_bytes(), dtype=torch.uint8, device=DEV)
    ba, bv = _lib.NrnFieldBwdArgs(), _lib.NrnViewBwdArgs()
    ba.n_rays, ba.n_samples, ba.out_ch = n, s, 4
    ba.d_raw, ba.stash, ba.grad_stash, ba.wgrad_scratch = d_raw.data_ptr(), b["stash"].data_ptr(), b["grad_stash"].data_ptr(), scratch.data_ptr()
    ba.nerf_packed, ba.nerf_grad, ba.relu_mask = nerf_pack.data_ptr(), flat.data_ptr(), b["relu_mask"].data_ptr()
    ba.stream = torch.cuda.current_stream().cuda_stream
    bv.views_t_packed, bv.views_stash, bv.views_grad_stash, bv.hv_mask = (views_t.data_ptr(), b["views_stash"].data_ptr(),
                                                                         b["views_grad_stash"].data_ptr(), b["hv_mask"].data_ptr())
    _lib.check(lib.nrn_field_backward_views(C.byref(ba), C.byref(bv)), "backward")
    _lib.device_error_check()
    return raw, d_raw, flat, b


def _h16(t):
    return t.detach().half().to(F64)


def _check(name, got, exact, bound):
    err = (got - exact).abs()
    pos = bound > 0   # where the bound is 0 (masked elements, exact zeros) the error must be 0
    ratio = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
    print(f"  {name}: max |kernel - exact| / bound {ratio:.3f}")
    assert bool(torch.isfinite(got).all()), name
    assert bool((err <= bound).all()), (name, int((err > bound).sum()), ratio)


@pytest.mark.parametrize("n,s,factor", [(1, 64, 1.0), (1023, 64, 1.0), (40, 100, 1.0), (1024, 128, 1.0), (1023, 64, 0.0),
                                        (1023, 64, 1e-15), (1023, 64, 1e10)])
def test_stages_against_fp64_of_their_own_operands(n, s, factor):
    net, _, _, _ = build_view_models(O, 7100 + s, DEV, with_bender=False, s_coarse=s)
    raw, d_raw, flat, b = _run(net, n, s, 7100 + s, factor)
    P, T = n * s, (n * s + 127) // 128
    rows = T * 128
    assert bool(torch.isfinite(raw).all())
    # every row of every tile written and finite, rows past P of a ragged tile included
    img = lambda buf, tile, im: SL.image(buf, tile, im[0], im[1], T).to(F64)
    Dir, F, Hv = img(b["views_stash"], V_STASH_TILE, VS_DIR), img(b["views_stash"], V_STASH_TILE, VS_F), img(b["views_stash"], V_STASH_TILE, VS_HV)
    H8 = img(b["stash"], SL.STASH_TILE, SL.ST_H[7])
    A = img(b["grad_stash"], SL.GRAD_TILE, SL.GS_RAW)            # the scaled fp16 d_raw, zero rows past P
    dYv, dF = img(b["views_grad_stash"], V_GRAD_TILE, VG_YV), img(b["views_grad_stash"], V_GRAD_TILE, VG_F)
    dY7 = img(b["grad_stash"], SL.GRAD_TILE, SL.GS_Y[7])
    for nm, x in (("Dir", Dir), ("F", F), ("Hv", Hv), ("d_raw image", A), ("dYv", dYv), ("dF", dF), ("dY7", dY7)):
        assert x.shape[0] == rows and bool(torch.isfinite(x).all()), nm
    assert torch.equal(SL.relu_bits(b["hv_mask"], 0, 128, T, tile_bytes=HV_MASK_TILE), Hv > 0)
    # the loss scale of the run: a power of two from max |d_raw| over the four channels
    amax = float(d_raw.abs().max())
    scale = SL.loss_scale(amax)
    assert torch.equal(A[:P, :4], _h16((d_raw.reshape(P, 4).double() * scale).clamp(-65504, 65504)))
    wr, wv, wf, wa = (_h16(net.rgb_linear.weight), _h16(net.views_linears[0].weight), _h16(net.feature_linear.weight),
                      _h16(net.alpha_linear.weight))
    Wr = wr.to(DEV)                 # [3][128]
    WvF = wv[:, :256].to(DEV)       # [128][256]
    Wf, Wa = wf.to(DEV), wa.to(DEV)  # [256][256], [1][256]
    c = lambda k: (k + 2) * U
    # dYv
    x = A[:, :3] @ Wr
    e = c(16) * (A[:, :3].abs() @ Wr.abs())
    _check("dYv", dYv, x * (Hv > 0), (e + half_ulp(x.abs() + e)) * (Hv > 0))
    # dF from the kernel's own dYv
    x = dYv @ WvF
    e = c(128) * (dYv.abs() @ WvF.abs())
    _check("dF", dF, x, e + half_ulp(x.abs() + e))
    # dY7 from the kernel's own dF and d_alpha, with the alpha term
    x = dF @ Wf + A[:, 3:4] @ Wa
    e = c(256 + 16) * (dF.abs() @ Wf.abs() + A[:, 3:4].abs() @ Wa.abs())
    m = H8 > 0
    _check("dY7", dY7, x * m, (e + half_ulp(x.abs() + e)) * m)
    # the head block of the flat gradient, per parameter shape, from all points' operands
    head = flat[TRUNK_FLOATS:].double()
    assert head.numel() == sum(torch.Size(sh).numel() for _, sh in HEAD_SHAPES)
    assert bool(torch.isfinite(flat).all())
    parts, o = {}, 0
    for nm, sh in HEAD_SHAPES:
        k = torch.Size(sh).numel()
        parts[nm] = head[o:o + k].view(sh)
        o += k
    cw = (rows + 2) * U / scale
    ones = torch.ones(rows, 1, dtype=F64, device=DEV)
    XvB = torch.cat([F, Dir[:, :27]], 1)
    refs = {
        "views_linears.0.weight": (dYv.T @ XvB, dYv.abs().T @ XvB.abs()),
        "views_linears.0.bias": ((dYv.T @ ones)[:, 0], (dYv.abs().T @ ones)[:, 0]),
        "feature_linear.weight": (dF.T @ H8, dF.abs().T @ H8.abs()),
        "feature_linear.bias": ((dF.T @ ones)[:, 0], (dF.abs().T @ ones)[:, 0]),
        "alpha_linear.weight": (A[:, 3:4].T @ H8, A[:, 3:4].abs().T @ H8.abs()),
        "alpha_linear.bias": ((A[:, 3:4].T @ ones)[:, 0], (A[:, 3:4].abs().T @ ones)[:, 0]),
        "rgb_linear.weight": (A[:, :3].T @ Hv, A[:, :3].abs().T @ Hv.abs()),
        "rgb_linear.bias": ((A[:, :3].T @ ones)[:, 0], (A[:, :3].abs().T @ ones)[:, 0]),
    }
    for nm, (x, mag) in refs.items():
        _check(nm, parts[nm], x / scale, cw * mag + 1e-300)
    if factor == 0.0:
        assert bool((flat == 0).all()), "a zero upstream gives zero gradients"
