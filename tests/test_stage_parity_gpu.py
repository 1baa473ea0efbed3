"""Every stage of the fused training kernels against an fp64 reference of that one stage, fed with the kernel's own
fp16 operands read back from the stashes (tests/stash_layout.py) and the packed weights' own rounding fp16(w).

What is left between kernel and reference is fp32 accumulation and one final rounding, bounded per element by

    |kernel - exact| <= 0.5 ulp_fp16(kernel)        (only where the output is stored as fp16)
                        + c * 2^-24 * (|A| @ |W|)   (the same product on absolute values)

c is the accumulation depth of the step: K + 2 for one tensor-core GEMM of depth K (K products, the bias add and the
final fp32 rounding).  Where a check spans several fp32 stages (PE backward, bend, latent reduction) the absolute-value
product is propagated through those stages and c is the sum of their depths.  The weight gradients use c = 16 T + 64
(8 wgmma k-steps per tile over T tiles, plus the split reduction) and, because that per-element bound grows with the batch,
also a relative L2 bound of 1.5e-4 per tensor (the worst measured, 3.5e-5, is L0's at 1024 x 128, whose sin / cos inputs
cancel strongly); a weight gradient missing one tile of 1024 moves by about 1e-3.
The divergence kernels are checked against the full tangent / adjoint chains in fp64 with the UNROUNDED fp32 bender
weights at c = 64 (eta = 2^-18): their hi/lo split is meant to be fp32-accurate, and plain fp16 operands (about 4e-4)
fail this by orders of magnitude.

The time-conditioned baseline (TC: no bender, the latent z enters L0 and L5 as a per-ray bias) adds these checks:
  ray bias rb[ray][l] = b_l + W_l[:, 63:95] z    fp32 weights and latents, c = 34 on |b| + |W||z|
  H1, H6 (L0, L5)      each accumulator row adds rb of its own ray, min(row, P - 1) // S; c_mma(K) on |A||W| + |rb|
  per-ray sums         sum of the decoded dY0 / dY5 over the ray's samples / loss scale, c = S + 2
  d z                  from the kernel's own sums and the fp32 W0 / W5 latent columns, c = 514
  dW0 / dW5[:, 63:95]  from the kernel's own sums, c = 4 (n + 2): n fp32 FMAs, whose worst case few rays nearly reach
and WGRAD checks the whole TC gradient layout (W0 [256][95], W5 [256][351]) as above.

Measured on one H100 80GB HBM3 (700 W power limit): the worst observed ratio of each stage (|kernel - exact| - rounding)
/ (2^-24 |A||W|) is printed with `pytest -s` ("c_obs"); every c above has at least 4x margin over the largest c_obs of its
stage.  The worst TC c_obs: ray bias 4.48 (1023 x 64), H1 1.55 and H6 8.30 (1024 x 128), per-ray sums 0.69 (37 x 3),
d z 6.49 (1024 x 128), latent columns 2.24 of c = 20 (3 x 100); H2 .. H8, raw and dY0 .. dY6 at most 3.70 of c = 258,
dY7 1.99 of 18, the other weight gradients 5.43 of 80 (37 x 3).

Every caller-owned buffer (stashes, masks, scratch, outputs) is filled with 0xFF (fp16 / fp32 NaN) before the calls, so a
read of memory no kernel wrote shows up as a NaN in a checked value.
"""
import ctypes as C

import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import stash_layout as SL
from tests import tc_reference as TR
from tests.parity import DEV, F64, U, Report, half_ulp, poison_bytes, poison_f32, ptr

pytestmark = pytest.mark.gpu
SEED = 5150
C_DIV = 64                 # eta = 2^-18 for the fp32-accurate divergence chains
LOSS_REL_DIV = 1e-5        # per-ray divergence loss, relative
C_CLOSED = 16              # closed forms of a few fp32 operations (G, d_unmasked, d_rigidity): two per operation
WGRAD_REL_L2 = 1.5e-4      # weight gradients, relative L2 per tensor
# The hi / lo split of the divergence kernels resolves an operand x to about 2^-22 |x| only while its residual stays in
# fp16's normal range; below that (|x - fp16(x)| * 2048 < 2^-14) it carries x to 2^-36 absolute.  The divergence checks
# therefore add that floor, propagated through one or two rows of at most 128 weights |w| < 1: 2^-36 * 128.
DIV_FLOOR = 2.0 ** -29
C_RAY_BIAS = 34            # time-conditioned ray bias: 32 fp32 FMAs, the bias add and the rounding
C_DZ = 514                 # time-conditioned d z: 512 fp32 FMAs over both layers' per-ray sums


def c_mma(k):
    return k + 2


def c_wgrad(n_tiles):
    return 16 * n_tiles + 64


def c_latent_columns(n_rays):
    """The n + 2 of an n-ray fp32 FMA chain with the 4x margin applied up front: with few rays that worst case is nearly
    reached (c_obs 2.24 at n = 3)."""
    return 4 * (n_rays + 2)


# ----------------------------------------------------------------------------------------------------------------------
# checking (Report, half_ulp: tests/parity.py)
# ----------------------------------------------------------------------------------------------------------------------
def mm(a, w):
    """a @ w^T and |a| @ |w|^T"""
    return a @ w.T, a.abs() @ w.abs().T


def dmm(a, w):
    """DGRAD step a @ w and |a| @ |w|"""
    return a @ w, a.abs() @ w.abs()


def wsum(dy, x):
    """sum_p dy[p] (x) x[p] and its absolute value"""
    return dy.T @ x, dy.abs().T @ x.abs()


# ----------------------------------------------------------------------------------------------------------------------
# the kernels, called through the C ABI as autograd._FieldTrainFn / _DivergenceFn do
# ----------------------------------------------------------------------------------------------------------------------
def _lib():
    from nonrigid_nerf_b200 import _lib as L
    return L


_MODELS = {}


def models(bender, tc=False):
    """(coarse NeRF, bender); tc: the time-conditioned baseline's NeRF (W0 [256][95], W5 [256][351]), no bender."""
    key = "tc" if tc else bender
    if key not in _MODELS:
        if tc:
            from nonrigid_nerf_b200 import run_nerf_helpers as H
            cp, _ = TR.make_params(SEED)
            kw = dict(D=8, W=256, input_ch=63, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False, ray_bender=None,
                      ray_bending_latent_size=32, time_conditioned_baseline=True)
            _MODELS[key] = (helpers.load_nerf_module(H.NeRF(num_ray_samples=64, **kw), cp).to(DEV), None)
        else:
            coarse, _, bend, _ = helpers.build_models(O, SEED, DEV, with_bender=bender)
            _MODELS[key] = (coarse, bend)
    return _MODELS[key]


def pack_nerf(ws, bs, out_ch, input_ch=63):
    from nonrigid_nerf_b200 import ops
    L = _lib()
    lib = L.load()
    ws = [w.detach().contiguous() for w in ws[:8]] + [ws[8][:out_ch].detach().contiguous()]
    bs = [b.detach().contiguous() for b in bs[:8]] + [bs[8][:out_ch].detach().contiguous()]
    buf = torch.empty(lib.nrn_packed_nerf_bytes(), dtype=torch.uint8, device=DEV)
    L.check(lib.nrn_pack_nerf(ops._ptr_array(ws), ops._ptr_array(bs), input_ch, out_ch, C.c_void_p(buf.data_ptr()),
                              C.c_void_p(torch.cuda.current_stream().cuda_stream)), "pack_nerf")
    torch.cuda.synchronize()
    return buf, ws, bs


class Case:
    """tc: the time-conditioned baseline (no bender); lat_stride0: one latent row for every ray (latent_stride 0)."""
    def __init__(self, n, s, bender=True, out_ch=5, cutoff=None, scaling=None, draw_mag=1.0, reg_mag=0.05, ch4=0.0,
                 seed=0, tc=False, lat_stride0=False):
        assert not (tc and bender), "the time-conditioned baseline has no bender"
        self.n, self.s, self.bender, self.out_ch, self.tc = n, s, bender, out_ch, tc
        self.cutoff, self.scaling = cutoff, scaling
        self.P = n * s
        self.T = -(-self.P // SL.TILE_M)
        self.R = self.T * SL.TILE_M
        g = torch.Generator().manual_seed(1000 + 7 * n + s + seed)
        r = O.make_rays(SEED + n, n)
        self.rays = helpers.rays8(r, DEV).contiguous()
        u = (torch.arange(s, dtype=torch.float32) + torch.rand(n, s, generator=g)) / s
        self.z = (r["near"] + (r["far"] - r["near"]) * u).to(DEV).contiguous()
        self.lat = r["latents"].to(DEV).contiguous()
        if lat_stride0:
            self.lat = self.lat[:1].expand(n, 32)
        mags = torch.tensor([0.3, 0.3, 0.3, 2.0, 0.0][:out_ch])
        d = torch.randn(self.P, out_ch, generator=g) * mags * draw_mag
        if out_ch == 5:
            d[:, 4] = ch4
        self.d_raw = d.to(DEV).contiguous()
        self.d_un_up = self.d_rig_up = None
        if bender and reg_mag:
            self.d_un_up = (torch.randn(self.P, 3, generator=g) * reg_mag).to(DEV).contiguous()
            self.d_rig_up = (torch.randn(self.P, generator=g) * reg_mag).to(DEV).contiguous()
        self.e = torch.randn(self.P, 3, generator=g).to(DEV).contiguous()
        self.w = torch.rand(self.P, generator=g).to(DEV).contiguous()
        self.g_ray = (torch.randn(n, generator=g) * 3.0).to(DEV).contiguous()


def run_forward(cs, train=True, removal=None, points=None):
    """The training kernel (stash and ReLU masks), or with train=False the inference kernel render() runs; `removal`: its
    object-removal threshold; `points` [P, stride >= 3]: point mode (NeRF.forward(x)) instead of cs.rays / cs.z."""
    from nonrigid_nerf_b200 import ops
    L = _lib()
    lib = L.load()
    coarse, bend = models(cs.bender, cs.tc)
    ws, bs = ops.nerf_param_list(coarse)
    npk, ws, bs = pack_nerf(ws, bs, cs.out_ch, 95 if cs.tc else 63)
    bpk = ops.pack_bender(bend) if cs.bender else None
    o = {"npk": npk, "bpk": bpk, "ws": ws, "bs": bs, "bend": bend}
    a = L.NrnFieldArgs()
    if points is None:
        a.rays, a.z_vals = cs.rays.data_ptr(), cs.z.data_ptr()
    else:
        a.points, a.points_stride = points.data_ptr(), points.stride(0)
    a.n_rays, a.n_samples = cs.n, cs.s
    a.nerf_packed, a.out_ch = npk.data_ptr(), cs.out_ch
    o["raw"] = poison_f32(cs.P, cs.out_ch)
    o["init"], o["bent"] = poison_f32(cs.P, 3), poison_f32(cs.P, 3)
    a.raw, a.initial_input_pts, a.input_pts = o["raw"].data_ptr(), o["init"].data_ptr(), o["bent"].data_ptr()
    if cs.bender:
        a.latents, a.latent_stride, a.bender_packed = cs.lat.data_ptr(), cs.lat.stride(0), bpk.data_ptr()
        o["un"], o["masked"], o["rig"] = poison_f32(cs.P, 3), poison_f32(cs.P, 3), poison_f32(cs.P)
        a.unmasked_offsets, a.masked_offsets, a.rigidity_mask = o["un"].data_ptr(), o["masked"].data_ptr(), o["rig"].data_ptr()
    if cs.cutoff is not None:
        a.use_cutoff, a.rigidity_cutoff = 1, cs.cutoff
    if cs.scaling is not None:
        a.use_scaling, a.scaling = 1, cs.scaling
    if removal is not None:
        a.use_removal, a.removal_threshold = 1, removal
    if train:
        o["stash"] = poison_bytes(lib.nrn_stash_bytes(cs.n, cs.s))
        o["mask"] = poison_bytes(lib.nrn_relu_mask_bytes(cs.n, cs.s))
        a.stash, a.relu_mask = o["stash"].data_ptr(), o["mask"].data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    if cs.tc:
        # the ray bias [rows][L0, L5][256] from the fp32 weights; one row when the latent stride is 0
        stride = cs.lat.stride(0)
        rows = cs.n if stride else 1
        o["rb"] = poison_f32(rows, 2, 256)
        L.check(lib.nrn_tc_latent_bias(cs.lat.data_ptr(), stride, rows, ws[0].data_ptr(), bs[0].data_ptr(), ws[5].data_ptr(),
                                       bs[5].data_ptr(), o["rb"].data_ptr(), a.stream), "tc_latent_bias")
        a.latents, a.latent_stride = cs.lat.data_ptr(), stride
        L.check(lib.nrn_field_forward_tc(C.byref(a), o["rb"].data_ptr()), "field_forward_tc")
    else:
        L.check(lib.nrn_field_forward(C.byref(a)), "field_forward")
    L.device_error_check()
    return o


def run_backward(cs, o, d_raw=None, nerf_grad=None, nerf_head=None, bender_grad=None, accumulate=False):
    L = _lib()
    lib = L.load()
    d_raw = cs.d_raw if d_raw is None else d_raw
    a = L.NrnFieldBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = cs.n, cs.s, cs.out_ch
    a.d_raw, a.stash, a.relu_mask, a.nerf_packed = d_raw.data_ptr(), o["stash"].data_ptr(), o["mask"].data_ptr(), o["npk"].data_ptr()
    b = {"gstash": poison_bytes(lib.nrn_grad_stash_bytes(cs.n, cs.s)), "scratch": poison_bytes(lib.nrn_wgrad_scratch_bytes())}
    n_nerf = lib.nrn_nerf_tc_grad_floats(cs.out_ch) if cs.tc else lib.nrn_nerf_grad_floats(cs.out_ch)
    b["nerf_grad"] = poison_f32(n_nerf) if nerf_grad is None else nerf_grad
    b["nerf_head"] = nerf_head
    a.grad_stash, a.wgrad_scratch, a.nerf_grad = b["gstash"].data_ptr(), b["scratch"].data_ptr(), b["nerf_grad"].data_ptr()
    if nerf_head is not None:
        a.nerf_grad_head = nerf_head.data_ptr()
    if cs.bender:
        b["bender_grad"] = poison_f32(lib.nrn_bender_grad_floats()) if bender_grad is None else bender_grad
        b["d_lat"] = poison_f32(cs.n, 32)
        a.bender_packed = o["bpk"].data_ptr()
        a.unmasked_offsets, a.rigidity_mask = o["un"].data_ptr(), o["rig"].data_ptr()
        a.d_unmasked_offsets, a.d_rigidity_mask = ptr(cs.d_un_up), ptr(cs.d_rig_up)
        a.bender_grad, a.d_latents = b["bender_grad"].data_ptr(), b["d_lat"].data_ptr()
        if cs.cutoff is not None:
            a.use_cutoff, a.rigidity_cutoff = 1, cs.cutoff
        if cs.scaling is not None:
            a.use_scaling, a.scaling = 1, cs.scaling
    a.accumulate_nerf = a.accumulate_bender = 1 if accumulate else 0
    a.stream = torch.cuda.current_stream().cuda_stream
    if cs.tc:
        t = L.NrnTcBwdArgs()
        b["d_lat"] = poison_f32(cs.n, 32)
        b["tc_ws"] = poison_f32(lib.nrn_tc_workspace_bytes(cs.n) // 4)   # per-ray sums [n][2][256] | latent columns [2][256][32]
        t.latents, t.latent_stride = cs.lat.data_ptr(), cs.lat.stride(0)
        t.w0, t.w5 = o["ws"][0].data_ptr(), o["ws"][5].data_ptr()
        t.d_latents, t.workspace = b["d_lat"].data_ptr(), b["tc_ws"].data_ptr()
        L.check(lib.nrn_field_backward_tc(C.byref(a), C.byref(t)), "field_backward_tc")
    else:
        L.check(lib.nrn_field_backward(C.byref(a)), "field_backward")
    L.device_error_check()
    return b


def run_divergence(cs, o):
    L = _lib()
    lib = L.load()
    a = L.NrnDivArgs()
    a.n_rays, a.n_samples = cs.n, cs.s
    a.relu_mask, a.e, a.unmasked_offsets, a.rigidity_mask, a.weights = (
        o["mask"].data_ptr(), cs.e.data_ptr(), o["un"].data_ptr(), o["rig"].data_ptr(), cs.w.data_ptr())
    a.bender_packed = o["bpk"].data_ptr()
    d = {"tan": poison_bytes(lib.nrn_div_stash_bytes(cs.n, cs.s)), "scal": poison_f32(4, cs.P), "loss": poison_f32(cs.n)}
    a.tangent_stash = d["tan"].data_ptr()
    a.d, a.alpha, a.beta, a.tau_c = (d["scal"][i].data_ptr() for i in range(4))
    a.loss = d["loss"].data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    L.check(lib.nrn_divergence_forward(C.byref(a)), "divergence_forward")
    d["G"], d["adj"] = poison_f32(cs.P), poison_bytes(lib.nrn_div_grad_stash_bytes(cs.n, cs.s))
    d["scratch"] = poison_bytes(lib.nrn_wgrad_scratch_bytes())
    d["d_un"], d["d_rig"], d["grad"] = poison_f32(cs.P, 3), poison_f32(cs.P), poison_f32(lib.nrn_bender_grad_floats())
    a.g_ray, a.G_workspace = cs.g_ray.data_ptr(), d["G"].data_ptr()
    a.adjoint_stash, a.wgrad_scratch = d["adj"].data_ptr(), d["scratch"].data_ptr()
    a.d_unmasked_offsets, a.d_rigidity_mask, a.bender_grad = d["d_un"].data_ptr(), d["d_rig"].data_ptr(), d["grad"].data_ptr()
    L.check(lib.nrn_divergence_backward(C.byref(a)), "divergence_backward")
    L.device_error_check()
    return d


# ----------------------------------------------------------------------------------------------------------------------
# fp64 references
# ----------------------------------------------------------------------------------------------------------------------
def bender_blocks(bend, rnd):
    """The block-diagonal bender steps B0..B4 of csrc/pack.cu (rows = outputs) and their biases, weights through rnd."""
    from nonrigid_nerf_b200 import ops
    nw, nb, rw, rb = ops.bender_param_list(bend)
    nw = [rnd(w.detach()) for w in nw]
    rw = [rnd(w.detach()) for w in rw]
    nb = [b.detach().to(F64) for b in nb]
    rb = [b.detach().to(F64) for b in rb]
    z = lambda *s: torch.zeros(*s, dtype=F64, device=DEV)
    B0 = z(96, 48)
    B0[:64, 0:3] = nw[0][:, :3]
    B0[:64, 3:6] = nw[0][:, :3]
    B0[:64, 6:38] = nw[0][:, 3:]
    B0[64:, 0:3] = rw[0]
    B0[64:, 3:6] = rw[0]
    B1 = z(96, 96)
    B1[:64, :64] = nw[1]
    B1[64:, 64:] = rw[1]
    B2 = z(80, 96)
    B2[:64, :64] = nw[2]
    B2[64, 64:] = rw[2][0]
    B3 = nw[3].clone()
    B4 = z(16, 64)
    B4[:3] = nw[4]
    bias = [torch.cat([nb[0], rb[0]]), torch.cat([nb[1], rb[1]]), torch.cat([nb[2], rb[2], z(15)]), nb[3]]
    return [B0, B1, B2, B3, B4], bias


def h16(t):
    return t.detach().half().to(F64)


def pe_backward(de, de_abs, E):
    """dx_d = dE[d] + sum_k 2^k (dE[sin_kd] cos_kd - dE[cos_kd] sin_kd) with the stashed fp16 sin / cos, and its
    absolute-value counterpart."""
    R = E.shape[0]
    sc = E[:, 3:63].reshape(R, 10, 2, 3)
    d = de[:, 3:63].reshape(R, 10, 2, 3)
    da = de_abs[:, 3:63].reshape(R, 10, 2, 3)
    f = (2.0 ** torch.arange(10, dtype=F64, device=E.device)).view(1, 10, 1)
    dx = de[:, :3] + (f * (d[:, :, 0] * sc[:, :, 1] - d[:, :, 1] * sc[:, :, 0])).sum(1)
    ax = de_abs[:, :3] + (f * (da[:, :, 0] * sc[:, :, 1].abs() + da[:, :, 1] * sc[:, :, 0].abs())).sum(1)
    return dx, ax


C_PE = 32   # the fp32 operations of one pe_backward call per coordinate


def check_forward(cs, o, rep):
    T, R, P = cs.T, cs.R, cs.P
    st = o["stash"]
    img = lambda oc: SL.image(st, SL.STASH_TILE, *oc, T).to(F64)
    E = img(SL.ST_E)
    H = [img(oc) for oc in SL.ST_H]
    init, bent = o["init"].to(F64), o["bent"].to(F64)
    if cs.bender:
        Bin, Hb = img(SL.ST_BIN), [img(SL.ST_HB1), img(SL.ST_HB2), img(SL.ST_HB3), img(SL.ST_HB4)]
        Bh, bias = bender_blocks(o["bend"], h16)
        hi, lo = Bin[:P, 0:3], Bin[:P, 3:6]
        assert torch.equal(hi, h16(o["init"])), "bender input: xyz hi column is not fp16(x)"
        assert bool(((hi + lo - init).abs() <= 2.0 ** -22 * init.abs() + 2.0 ** -25).all()), "bender input: hi + lo != x"
        lat = cs.lat.repeat_interleave(cs.s, 0)
        assert torch.equal(Bin[:P, 6:38], h16(lat)), "bender input: latent columns are not fp16(latent)"
        assert bool((Bin[:, 38:] == 0).all()) and bool((Bin[P:] == 0).all()), "bender input: padding is not zero"
        v, a = mm(Bin, Bh[0])
        rep.check("Hb1", Hb[0], torch.relu(v + bias[0]), a + bias[0].abs(), c_mma(48), True)
        v, a = mm(Hb[0], Bh[1])
        rep.check("Hb2", Hb[1], torch.relu(v + bias[1]), a + bias[1].abs(), c_mma(96), True)
        v, a = mm(Hb[1], Bh[2])
        v, a = v + bias[2], a + bias[2].abs()
        rep.check("Hb3", Hb[2], torch.relu(v[:, :64]), a[:, :64], c_mma(96), True)
        # rigidity = (tanh(pre) + 1) / 2: |dr/dpre| <= 1/2, plus tanhf (2 ulp) and the fp32 arithmetic around it
        pre, pre_a = v[:P, 64], a[:P, 64]
        r = (torch.tanh(pre) + 1.0) / 2.0
        r_bound = 0.5 * c_mma(96) * U * pre_a + 2.0 ** -21
        got_r = o["rig"].to(F64)
        keep = torch.ones_like(r, dtype=torch.bool)
        if cs.cutoff is not None:
            keep = (r - cs.cutoff).abs() > r_bound   # the cut-off decision itself is only defined up to the bound
            r = torch.where(r <= cs.cutoff, torch.zeros_like(r), r)
            assert bool(keep.float().mean() > 0.9) and bool((got_r[keep] == 0).any()), "cut-off case does not cut"
        err = (got_r - r).abs()[keep]
        assert bool((err <= r_bound[keep]).all()), f"rigidity: max err {float(err.max()):.3e}"
        v4, a4 = mm(Hb[2], Bh[3])
        rep.check("Hb4", Hb[3], torch.relu(v4 + bias[3]), a4 + bias[3].abs(), c_mma(64), True)
        v, a = mm(Hb[3], Bh[4])
        rep.check("unmasked_offsets", o["un"], v[:P, :3], a[:P, :3], c_mma(64))
        masked = o["rig"][:, None] * o["un"]
        if cs.scaling is not None:
            masked = masked * cs.scaling
        assert torch.equal(o["masked"], masked), "masked offsets are not fp32(rigidity * unmasked)"
        assert torch.equal(o["bent"], o["init"] + o["masked"]), "bent point is not fp32(x + masked)"
    else:
        assert torch.equal(o["bent"], o["init"])
    # embedding of the bent point
    assert torch.equal(E[:P, :3], h16(o["bent"])), "E columns 0-2 are not fp16(bent xyz)"
    k = 2.0 ** torch.arange(10, dtype=F64, device=DEV)
    arg = bent[:, None, :] * k[None, :, None]                                        # [P, 10, 3]
    sc = torch.stack([torch.sin(arg), torch.cos(arg)], 2).reshape(P, 60)
    got = E[:P, 3:63]
    err = (got - sc).abs() - half_ulp(got)
    assert bool((err <= 1e-6).all()), f"PE sin / cos: max excess {float(err.max()):.3e}"
    assert bool((E[:, 63] == 1.0).all()), "E column 63 is not 1.0"
    assert bool(torch.isfinite(E).all()), "E is not finite past P"
    # L0 .. L7 from their own input images
    W = [h16(w) for w in o["ws"]]
    b = [x.detach().to(F64) for x in o["bs"]]
    if cs.tc:
        # the ray bias rb[ray][l] = b_l + W_l[:, 63:95] z[ray] from the fp32 weights; then L0 / L5 add, per row, the kernel's
        # own row of the row's ray (rows past P: the last point's ray)
        z = cs.lat[:o["rb"].shape[0]].to(F64)
        ref, ref_a = [], []
        for l in (0, 5):
            wl = o["ws"][l][:, 63:95].to(F64)
            ref.append(b[l] + z @ wl.T)
            ref_a.append(b[l].abs() + z.abs() @ wl.abs().T)
        rep.check("ray bias", o["rb"], torch.stack(ref, 1), torch.stack(ref_a, 1), C_RAY_BIAS)
        ray = torch.arange(R, device=DEV).clamp(max=P - 1) // cs.s
        rb = o["rb"].to(F64)[ray if o["rb"].shape[0] > 1 else torch.zeros_like(ray)]
        b[0], b[5] = rb[:, 0], rb[:, 1]
    zc = torch.zeros(256, 1, dtype=F64, device=DEV)
    W0p = torch.cat([W[0][:, :63], zc], 1)
    W5p = torch.cat([W[5][:, :63], zc, W[5][:, -256:]], 1)
    for l in range(8):
        inp = E if l == 0 else (torch.cat([E, H[4]], 1) if l == 5 else H[l - 1])
        Wl = W0p if l == 0 else (W5p if l == 5 else W[l])
        v, a = mm(inp, Wl)
        rep.check(f"H{l + 1}", H[l], torch.relu(v + b[l]), a + b[l].abs(), c_mma(Wl.shape[1]), True)
    v, a = mm(H[7][:P], W[8])
    rep.check("raw", o["raw"], v + b[8], a + b[8].abs(), c_mma(256))
    # ReLU mask bits: the encoding of stash image > 0, every bit of every word, rows past P included
    imgs = [SL.image(st, SL.STASH_TILE, *oc, T) for oc in SL.ST_H]
    names = [f"H{l + 1}" for l in range(8)]
    if cs.bender:
        imgs += [SL.image(st, SL.STASH_TILE, *oc, T) for oc in (SL.ST_HB1, SL.ST_HB2, SL.ST_HB3, SL.ST_HB4)]
        names += ["Hb1", "Hb2", "Hb3", "Hb4"]
    for nm, im, (off, ncols) in zip(names, imgs, SL.MASK_IMAGES):
        enc = SL.encode_relu_bits(im[:, :ncols] > 0)
        got = o["mask"][:T * SL.MASK_TILE].view(T, SL.MASK_TILE)[:, off:off + enc.shape[1]]
        assert torch.equal(got, enc), f"ReLU mask of {nm}: {int((got != enc).sum())} bytes differ from stash > 0"


def dgrad_reference(cs, o, b, rep, scale):
    """Checks DGRAD stage by stage; returns the decoded images the WGRAD check needs."""
    T, R, P = cs.T, cs.R, cs.P
    img = lambda oc: SL.image(o["stash"], SL.STASH_TILE, *oc, T).to(F64)
    gimg = lambda oc: SL.image(b["gstash"], SL.GRAD_TILE, *oc, T).to(F64)
    mbits = lambda oc: SL.relu_bits(o["mask"], oc[0], oc[1], T).to(F64)
    E = img(SL.ST_E)
    H = [img(oc) for oc in SL.ST_H]
    W = [h16(w) for w in o["ws"]]
    Draw = gimg(SL.GS_RAW)
    exp_raw = (cs.d_raw[:, :4] * scale).clamp(-65504.0, 65504.0).half().to(F64)
    assert torch.equal(Draw[:P, :4], exp_raw), "d_raw image is not fp16(clamp(d_raw[:, :4] * scale))"
    assert bool((Draw[:P, 4:] == 0).all()) and bool((Draw[P:] == 0).all()), "d_raw image: padding is not zero"
    dY = [gimg(oc) for oc in SL.GS_Y]
    m = [mbits(oc) for oc in SL.MK_H]
    v, a = dmm(Draw[:, :cs.out_ch], W[8])
    rep.check("dY7", dY[7], v * m[7], a * m[7], c_mma(16), True)
    for l in (6, 5):
        v, a = dmm(dY[l + 1], W[l + 1])
        rep.check(f"dY{l}", dY[l], v * m[l], a * m[l], c_mma(256), True)
    dE5, dE5a = dmm(dY[5], W[5][:, :63])
    v, a = dmm(dY[5], W[5][:, -256:])   # W5 = [embedding (| latent) | h]
    rep.check("dY4", dY[4], v * m[4], a * m[4], c_mma(256), True)
    for l in (3, 2, 1, 0):
        v, a = dmm(dY[l + 1], W[l + 1])
        rep.check(f"dY{l}", dY[l], v * m[l], a * m[l], c_mma(256), True)
    dE0, dE0a = dmm(dY[0], W[0][:, :63])
    pad = lambda t: torch.cat([t, torch.zeros(R, 1, dtype=F64, device=DEV)], 1)
    dx5, ax5 = pe_backward(pad(dE5), pad(dE5a), E)
    dx0, ax0 = pe_backward(pad(dE0), pad(dE0a), E)
    dx, adx = dx5 + dx0, ax5 + ax0
    c_dx = c_mma(256) + C_PE
    out = {"E": E, "H": H, "Draw": Draw, "dY": dY}
    if cs.tc:
        # per-ray sums of the stashed dY0 / dY5 over the ray's samples, in fp32 and divided by the loss scale
        ds = [dY[l][:P].view(cs.n, cs.s, 256) for l in (0, 5)]
        sums = b["tc_ws"][:cs.n * 512].view(cs.n, 2, 256)
        rep.check("tc per-ray sums", sums, torch.stack([d.sum(1) for d in ds], 1) / scale,
                  torch.stack([d.abs().sum(1) for d in ds], 1) / scale, cs.s + 2)
        # d z from the kernel's own sums and the fp32 latent columns of W0 / W5
        s = sums.to(F64)
        w0, w5 = o["ws"][0][:, 63:95].to(F64), o["ws"][5][:, 63:95].to(F64)
        rep.check("tc d_latents", b["d_lat"], s[:, 0] @ w0 + s[:, 1] @ w5, s[:, 0].abs() @ w0.abs() + s[:, 1].abs() @ w5.abs(),
                  C_DZ)
    if not cs.bender:
        return out
    Bin, Hb = img(SL.ST_BIN), [img(SL.ST_HB1), img(SL.ST_HB2), img(SL.ST_HB3), img(SL.ST_HB4)]
    Bh, _ = bender_blocks(o["bend"], h16)
    Yb4, Yb3, Yb2, Yb1, Yb0 = (gimg(oc) for oc in (SL.GS_YB4, SL.GS_YB3, SL.GS_YB2, SL.GS_YB1, SL.GS_YB0))
    rig, un = o["rig"].to(F64)[:, None], o["un"].to(F64)
    s = 1.0 if cs.scaling is None else float(torch.tensor(cs.scaling, dtype=torch.float32))
    dm, adm = dx[:P] * s, adx[:P] * abs(s)
    up_u = torch.zeros_like(un) if cs.d_un_up is None else cs.d_un_up.to(F64) * scale
    up_r = torch.zeros_like(rig[:, 0]) if cs.d_rig_up is None else cs.d_rig_up.to(F64) * scale
    dun = rig * dm + up_u
    a_dun = rig * adm + up_u.abs()
    rep.check("dYb4 (d unmasked)", Yb4[:P, :3], dun, a_dun, c_dx + 4, True)
    assert bool((Yb4[:P, 3:] == 0).all()) and bool((Yb4[P:] == 0).all()), "dYb4: padding is not zero"
    g = 2.0 * rig[:, 0] * (1.0 - rig[:, 0])
    drpre = (up_r + (un * dm).sum(1)) * g
    a_dr = (up_r.abs() + (un.abs() * adm).sum(1)) * g
    if cs.cutoff is not None:
        cut = rig[:, 0] <= cs.cutoff
        drpre, a_dr = torch.where(cut, 0.0, drpre), torch.where(cut, 0.0, a_dr)
    rep.check("dYb2[64] (d rig. pre)", Yb2[:P, 64], drpre, a_dr, c_dx + 8, True)
    assert bool((Yb2[:, 65:] == 0).all()) and bool((Yb2[P:, 64] == 0).all()), "dYb2: padding is not zero"
    mb = [mbits(oc) for oc in (SL.MK_HB1, SL.MK_HB2, SL.MK_HB3, SL.MK_HB4)]
    v, a = dmm(Yb4, Bh[4])
    rep.check("dYb3", Yb3, v * mb[3], a * mb[3], c_mma(16), True)
    v, a = dmm(Yb3, Bh[3])
    rep.check("dYb2", Yb2[:, :64], v * mb[2], a * mb[2], c_mma(64), True)
    v, a = dmm(Yb2, Bh[2])
    rep.check("dYb1", Yb1, v * mb[1], a * mb[1], c_mma(80), True)
    v, a = dmm(Yb1, Bh[1])
    rep.check("dYb0", Yb0, v * mb[0], a * mb[0], c_mma(96), True)
    v, a = dmm(Yb0[:P], Bh[0][:, 6:38])
    ray = torch.arange(P, device=DEV) // cs.s
    lat = torch.zeros(cs.n, 32, dtype=F64, device=DEV).index_add_(0, ray, v) / scale
    lat_a = torch.zeros(cs.n, 32, dtype=F64, device=DEV).index_add_(0, ray, a) / scale
    rep.check("d_latents", b["d_lat"], lat, lat_a, c_mma(96) + cs.s + 8)
    out.update(Bin=Bin, Hb=Hb, Yb=[Yb0, Yb1, Yb2, Yb3, Yb4])
    return out


def bender_wgrad_reference(Yb, X):
    """Bender weight gradients sum_p dY (x) X over the images: Yb = [dYb0..dYb4] (or adjoints), X = [input, h1..h4]
    (or tangents); (value, abs) per parameter of SL.bender_param_shapes()."""
    Y0, Y1, Y2, Y3, Y4 = Yb
    Xin, X1, X2, X3, X4 = X
    ref = {}
    v1, a1 = wsum(Y0[:, :64], Xin[:, 0:3])
    v2, a2 = wsum(Y0[:, :64], Xin[:, 3:6])
    v3, a3 = wsum(Y0[:, :64], Xin[:, 6:38])
    ref["net_w0"] = (torch.cat([v1 + v2, v3], 1), torch.cat([a1 + a2, a3], 1))
    ref["net_b0"] = (Y0[:, :64].sum(0), Y0[:, :64].abs().sum(0))
    ref["net_w1"] = wsum(Y1[:, :64], X1[:, :64])
    ref["net_b1"] = (Y1[:, :64].sum(0), Y1[:, :64].abs().sum(0))
    ref["net_w2"] = wsum(Y2[:, :64], X2[:, :64])
    ref["net_b2"] = (Y2[:, :64].sum(0), Y2[:, :64].abs().sum(0))
    ref["net_w3"] = wsum(Y3, X3)
    ref["net_b3"] = (Y3.sum(0), Y3.abs().sum(0))
    ref["net_w4"] = wsum(Y4[:, :3], X4)
    v1, a1 = wsum(Y0[:, 64:96], Xin[:, 0:3])
    v2, a2 = wsum(Y0[:, 64:96], Xin[:, 3:6])
    ref["rig_w0"] = (v1 + v2, a1 + a2)
    ref["rig_b0"] = (Y0[:, 64:96].sum(0), Y0[:, 64:96].abs().sum(0))
    ref["rig_w1"] = wsum(Y1[:, 64:96], X1[:, 64:96])
    ref["rig_b1"] = (Y1[:, 64:96].sum(0), Y1[:, 64:96].abs().sum(0))
    ref["rig_w2"] = wsum(Y2[:, 64:65], X2[:, 64:96])
    ref["rig_b2"] = (Y2[:, 64].sum(0, keepdim=True), Y2[:, 64].abs().sum(0, keepdim=True))
    return ref


def check_wgrad(cs, b, imgs, rep, scale, nerf_flat=None, bend_flat=None, base_nerf=None, base_bend=None):
    E, H, Draw, dY = imgs["E"], imgs["H"], imgs["Draw"], imgs["dY"]
    c = c_wgrad(cs.T)
    # the inputs of W0 and of W5's first columns: [E[:, :63] | the row's latent (time-conditioned; 0 past P)]
    X = E[:, :63]
    if cs.tc:
        Z = torch.zeros(cs.R, 32, dtype=F64, device=DEV)
        Z[:cs.P] = cs.lat.to(F64).repeat_interleave(cs.s, 0)
        X = torch.cat([X, Z], 1)
    ref = {}
    ref["w0"], ref["b0"] = wsum(dY[0], X), (dY[0].sum(0), dY[0].abs().sum(0))
    for l in range(1, 8):
        if l == 5:
            v1, a1 = wsum(dY[5], X)
            v2, a2 = wsum(dY[5], H[4])
            ref["w5"] = (torch.cat([v1, v2], 1), torch.cat([a1, a2], 1))
        else:
            ref[f"w{l}"] = wsum(dY[l], H[l - 1])
        ref[f"b{l}"] = (dY[l].sum(0), dY[l].abs().sum(0))
    v, a = wsum(Draw[:, :4], H[7])
    z = torch.zeros(cs.out_ch - 4, 256, dtype=F64, device=DEV)
    ref["w_out"] = (torch.cat([v, z]), torch.cat([a, z]))
    zb = torch.zeros(cs.out_ch - 4, dtype=F64, device=DEV)
    ref["b_out"] = (torch.cat([Draw[:, :4].sum(0), zb]), torch.cat([Draw[:, :4].abs().sum(0), zb]))
    shapes = SL.nerf_param_shapes(cs.out_ch, cs.tc)
    got = SL.split_flat(b["nerf_grad"] if nerf_flat is None else nerf_flat, shapes)
    if b["nerf_head"] is not None:
        got.update(SL.split_flat(b["nerf_head"], shapes[-2:]))
    base = SL.split_flat(base_nerf, shapes) if base_nerf is not None else None
    for name, (v, a) in ref.items():
        g = got[name].to(F64) - (base[name].to(F64) if base is not None else 0.0)
        rep.check(f"WGRAD {name}", g, v / scale, a / scale + (base[name].to(F64).abs() if base is not None else 0.0), c)
        if base is None:
            rep.rel_l2(f"WGRAD {name}", g, v / scale, WGRAD_REL_L2)
    if cs.tc:
        # the latent columns of W0 / W5 from the kernel's own per-ray sums: one fp32 FMA per ray, c_latent_columns(n)
        s = b["tc_ws"][:cs.n * 512].view(cs.n, 2, 256).to(F64)
        z = cs.lat.to(F64)
        for l, name in ((0, "w0"), (1, "w5")):
            g = got[name][:, 63:95].to(F64)
            a = s[:, l].abs().T @ z.abs()
            if base is not None:
                g, a = g - base[name][:, 63:95].to(F64), a + base[name][:, 63:95].to(F64).abs()
            rep.check(f"WGRAD {name}[:, 63:95]", g, s[:, l].T @ z, a, c_latent_columns(cs.n))
    if cs.out_ch == 5 and base is None:
        assert bool((got["w_out"][4] == 0).all()) and float(got["b_out"][4]) == 0.0, "head row 4 gradient is not exactly 0"
    if not cs.bender:
        return
    ref = bender_wgrad_reference(imgs["Yb"], [imgs["Bin"]] + imgs["Hb"])
    got = SL.split_flat(b["bender_grad"] if bend_flat is None else bend_flat, SL.bender_param_shapes())
    base = SL.split_flat(base_bend, SL.bender_param_shapes()) if base_bend is not None else None
    for name, (v, a) in ref.items():
        g = got[name].to(F64) - (base[name].to(F64) if base is not None else 0.0)
        rep.check(f"WGRAD {name}", g, v / scale, a / scale + (base[name].to(F64).abs() if base is not None else 0.0), c)


def expected_scale(cs, d_raw=None):
    d_raw = cs.d_raw if d_raw is None else d_raw
    amax = float(d_raw[:, :4].abs().max())
    for t in (cs.d_un_up, cs.d_rig_up):
        if t is not None:
            amax = max(amax, float(t.abs().max()))
    return SL.loss_scale(amax)


def check_divergence(cs, o, d, rep):
    T, R, P = cs.T, cs.R, cs.P
    Bf, _ = bender_blocks(o["bend"], lambda t: t.to(F64))
    mb = [SL.relu_bits(o["mask"], oc[0], oc[1], T).to(F64) for oc in (SL.MK_HB1, SL.MK_HB2, SL.MK_HB3, SL.MK_HB4)]
    tan = lambda oc: SL.image(d["tan"], SL.TAN_TILE, *oc, T).to(F64)
    adj = lambda oc: SL.image(d["adj"], SL.ADJ_TILE, *oc, T).to(F64)
    zpad = lambda t: torch.cat([t, torch.zeros(R - P, *t.shape[1:], dtype=F64, device=DEV)])
    e = zpad(cs.e.to(F64))
    TE = tan(SL.T_E)
    e_hi = cs.e.half()
    assert torch.equal(TE[:P, 0:3], e_hi.to(F64)) and torch.equal(TE[:P, 3:6], (cs.e - e_hi.float()).half().to(F64)), \
        "tangent input is not [fp16(e) | fp16(e - fp16(e))]"
    assert bool((TE[:, 6:] == 0).all()) and bool((TE[P:] == 0).all()), "tangent input: padding is not zero"
    # tangent chain, fp64 with the fp32 weights and the primal pass's mask bits
    W0x = Bf[0][:, 0:3]
    t1, t1a = mm(e, W0x)
    t1, t1a = t1 * mb[0], t1a * mb[0]
    t2, t2a = mm(t1, Bf[1])
    t2, t2a = t2 * mb[1], (t1a @ Bf[1].abs().T) * mb[1]
    v, a = mm(t2, Bf[2])
    a = t2a @ Bf[2].abs().T
    t3, t3a, tc, tca = v[:, :64] * mb[2], a[:, :64] * mb[2], v[:, 64], a[:, 64]
    v, _ = mm(t3, Bf[3])
    t4, t4a = v * mb[3], (t3a @ Bf[3].abs().T) * mb[3]
    tau, taua = t4 @ Bf[4][:3].T, t4a @ Bf[4][:3].abs().T
    for nm, oc, x, xa in (("tangent t1", SL.T_1, t1, t1a), ("tangent t2", SL.T_2, t2, t2a), ("tangent t3", SL.T_3, t3, t3a),
                          ("tangent t4", SL.T_4, t4, t4a)):
        rep.check(nm, tan(oc), x, xa, C_DIV, True, floor=DIV_FLOOR)
    r, un, ek = o["rig"].to(F64), o["un"].to(F64), cs.e.to(F64)
    alpha, alpha_a = (ek * tau[:P]).sum(1), (ek.abs() * taua[:P]).sum(1)
    beta, beta_a = (ek * un).sum(1), (ek.abs() * un.abs()).sum(1)
    g = 2.0 * r * (1.0 - r)
    dd = r * alpha + beta * g * tc[:P]
    dd_a = r * alpha_a + beta_a * g * tca[:P].abs() + beta.abs() * g * tca[:P]
    scal = d["scal"]
    rep.check("div tau_c", scal[3], tc[:P], tca[:P], C_DIV, floor=DIV_FLOOR)
    rep.check("div alpha", scal[1], alpha, alpha_a, C_DIV, floor=DIV_FLOOR)
    rep.check("div beta", scal[2], beta, beta_a, C_DIV, floor=DIV_FLOOR)
    rep.check("div d", scal[0], dd, dd_a, C_DIV, floor=DIV_FLOOR)
    ray = torch.arange(P, device=DEV) // cs.s
    loss = torch.zeros(cs.n, dtype=F64, device=DEV).index_add_(0, ray, cs.w.to(F64) * dd * dd) / cs.s
    lerr = float(((d["loss"].to(F64) - loss).abs() / loss.abs().clamp_min(1e-30)).max())
    print(f"  [{rep.tag}] {'div loss per ray':<24s} rel err {lerr:.3e}   bound {LOSS_REL_DIV:.0e}")
    assert lerr <= LOSS_REL_DIV, lerr
    # backward: G = g_ray * 2 / S * w * d (from the kernel's d), the loss scale of max |G|, the adjoint chain
    dk = scal[0].to(F64)
    G = cs.g_ray.to(F64)[ray] * 2.0 / cs.s * cs.w.to(F64) * dk
    rep.check("div G", d["G"], G, G.abs(), C_CLOSED)
    scale = SL.loss_scale(float(d["G"].abs().max()))
    Gk = d["G"].to(F64)
    alpha_k, beta_k, tc_k = scal[1].to(F64), scal[2].to(F64), scal[3].to(F64)
    tau_r = g * tc_k
    rep.check("div d_unmasked", d["d_un"], Gk[:, None] * tau_r[:, None] * ek, (Gk * tau_r)[:, None].abs() * ek.abs(), C_CLOSED)
    dr = Gk * (alpha_k + 2.0 * beta_k * tc_k * (1.0 - 2.0 * r))
    dr_a = Gk.abs() * (alpha_k.abs() + (2.0 * beta_k * tc_k * (1.0 - 2.0 * r)).abs())
    rep.check("div d_rigidity", d["d_rig"], dr, dr_a, C_CLOSED)
    Gs = zpad(Gk * scale)
    rr = zpad(r)
    tb = Gs[:, None] * rr[:, None] * e
    tba = tb.abs()
    A4 = adj(SL.A_4)
    rep.check("adjoint taubar_off", A4[:, :3], tb, tba, C_DIV, True, floor=DIV_FLOOR)
    a4, a4a = tb @ Bf[4][:3], tba @ Bf[4][:3].abs()
    a4, a4a = a4 * mb[3], a4a * mb[3]
    a3, a3a = (a4 @ Bf[3]) * mb[2], (a4a @ Bf[3].abs()) * mb[2]
    tbc = Gs * zpad(beta_k) * zpad(g)
    a2in, a2ina = torch.cat([a3, tbc[:, None]], 1), torch.cat([a3a, tbc.abs()[:, None]], 1)
    a2, a2a = (a2in @ Bf[2][:65]) * mb[1], (a2ina @ Bf[2][:65].abs()) * mb[1]
    a1, a1a = (a2 @ Bf[1]) * mb[0], (a2a @ Bf[1].abs()) * mb[0]
    A3, A2, A1, A0 = adj(SL.A_3), adj(SL.A_2), adj(SL.A_1), adj(SL.A_0)
    rep.check("adjoint abar4", A3, a4, a4a, C_DIV, True, floor=DIV_FLOOR)
    rep.check("adjoint abar3 | taubar_c", A2[:, :65], a2in, a2ina, C_DIV, True, floor=DIV_FLOOR)
    rep.check("adjoint abar2", A1, a2, a2a, C_DIV, True, floor=DIV_FLOOR)
    rep.check("adjoint abar1", A0, a1, a1a, C_DIV, True, floor=DIV_FLOOR)
    assert bool((A4[:, 3:] == 0).all()) and bool((A2[:, 65:] == 0).all()), "adjoint images: padding is not zero"
    # compact WGRAD over the decoded stashes: sum adj (x) tan / scale, no bias
    ref = bender_wgrad_reference([A0, A1, A2, A3, A4], [TE, tan(SL.T_1), tan(SL.T_2), tan(SL.T_3), tan(SL.T_4)])
    got = SL.split_flat(d["grad"], SL.bender_param_shapes())
    for name, (v, a) in ref.items():
        if "_b" in name:
            assert bool((got[name] == 0).all()), f"divergence WGRAD {name}: the tangent chain has no bias"
            continue
        rep.check(f"div WGRAD {name}", got[name], v / scale, a / scale, c_wgrad(T))


def grad_stash_images(cs, b):
    """Every gradient-stash image DGRAD writes, side by side: d_raw and dY0..dY7, and with a bender its dYb images."""
    return SL.image(b["gstash"], SL.GRAD_TILE, 0, (SL.GRAD_TILE if cs.bender else SL.GS_YB4[0]) // SL.CHUNK, cs.T)


def run_all(cs, tag, divergence=True):
    rep = Report(tag)
    o = run_forward(cs)
    check_forward(cs, o, rep)
    b = run_backward(cs, o)
    scale = expected_scale(cs)
    imgs = dgrad_reference(cs, o, b, rep, scale)
    check_wgrad(cs, b, imgs, rep, scale)
    d = None
    if cs.bender and divergence:
        d = run_divergence(cs, o)
        check_divergence(cs, o, d, rep)
    return o, b, d


# ----------------------------------------------------------------------------------------------------------------------
# shapes
# ----------------------------------------------------------------------------------------------------------------------
SHAPES = {
    "1x7": dict(n=1, s=7),                     # one ragged tile, odd tile count
    "2x64": dict(n=2, s=64),                   # exactly one tile
    "3x100": dict(n=3, s=100),                 # rays straddle tiles
    "11x100": dict(n=11, s=100),               # 9 tiles: WGRAD plan with empty trailing splits (see below)
    "1023x64": dict(n=1023, s=64),             # several tiles per CTA everywhere, ragged
    "1024x128": dict(n=1024, s=128),           # the benchmark's fine pass, full WGRAD plan
    "3x100_nobender": dict(n=3, s=100, bender=False),
    "2x64_out4": dict(n=2, s=64, out_ch=4),
    "3x100_out4_nobender": dict(n=3, s=100, out_ch=4, bender=False),
    "3x100_cutoff_scaling": dict(n=3, s=100, cutoff="median", scaling=0.7),
    # time-conditioned baseline: L0 / L5 take each accumulator row's bias from its own ray
    "37x3_tc": dict(n=37, s=3, bender=False, tc=True),          # rows r0 and r0 + 8 on different rays; one ragged tile
    "5x1_tc": dict(n=5, s=1, bender=False, tc=True),            # every row its own ray
    "1x7_tc": dict(n=1, s=7, bender=False, tc=True),            # one ray, rows past P
    "3x100_tc": dict(n=3, s=100, bender=False, tc=True),        # rays straddle tiles
    "3x100_tc_stride0": dict(n=3, s=100, bender=False, tc=True, lat_stride0=True),   # one latent row for every ray
    "3x100_out4_tc": dict(n=3, s=100, out_ch=4, bender=False, tc=True),
    "11x100_tc": dict(n=11, s=100, bender=False, tc=True),      # 9 tiles: empty trailing WGRAD splits without a bender
    "1023x64_tc": dict(n=1023, s=64, bender=False, tc=True),
    "1024x128_tc": dict(n=1024, s=128, bender=False, tc=True),
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_every_stage_matches_its_fp64_reference(name):
    kw = dict(SHAPES[name])
    if kw.get("cutoff") == "median":
        # a cut-off that removes about half of the points: the median rigidity of the same points without one
        kw["cutoff"] = float(run_forward(Case(**dict(kw, cutoff=None)))["rig"].median())
    cs = Case(**kw)
    o, b, _ = run_all(cs, name)
    if kw.get("lat_stride0"):
        # a broadcast latent row computes exactly what the same row repeated for every ray does
        ex = Case(**kw)
        ex.lat = cs.lat.contiguous()
        oe = run_forward(ex)
        for k in ("stash", "mask", "raw"):
            assert torch.equal(o[k], oe[k]), f"latent stride 0 vs repeated rows: {k} differs"
    if cs.T >= 500:
        # the fp16 gradient chain must not saturate at the benchmark's shapes
        g = grad_stash_images(cs, b).float().abs()
        assert float(g.max()) < 65504.0, f"gradient stash saturates: max {float(g.max())}"
        print(f"  [{name}] max |gradient stash| {float(g.max()):.1f}")


# ---- WGRAD's split plan (wgrad.cu, launch_wgrad), replicated to find a tile count whose plan has an empty split ----
_JOB_CHUNKS = [46, 48, 48, 48, 48, 48, 48, 48, 32, 32, 54, 42]


def wgrad_plan(n_tiles, max_ctas, has_bender=True):
    jobs = range(12 if has_bender else 10)
    splits = {j: 1 for j in jobs}
    halves = {j: 2 if 1 <= j <= 9 else 1 for j in jobs}
    used, tiles = sum(halves.values()), max(n_tiles, 1)
    while True:
        best, best_load = -1, -1
        for j in jobs:
            if splits[j] >= tiles or used + halves[j] > max_ctas:
                continue
            load = _JOB_CHUNKS[j] * -(-tiles // splits[j])
            if load > best_load:
                best, best_load = j, load
        if best < 0:
            return splits
        splits[best] += 1
        used += halves[best]


def empty_splits(n_tiles, splits):
    out = {}
    for j, ns in splits.items():
        per = -(-n_tiles // ns)
        n_valid = min(ns, -(-n_tiles // per))
        if n_valid < ns:
            out[j] = ns - n_valid
    return out


def test_the_9_tile_shape_has_an_empty_trailing_wgrad_split():
    """wgrad_reduce_kernel skips splits that own no tiles (n_valid).  The 11 x 100 shape above covers that path only if
    the plan for this device leaves such a split; a cluster-limited device can run fewer CTAs than SMs, so every even
    CTA budget down to 3/4 of the SMs is checked.  The same holds for the bender-less plan of 11 x 100_tc."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    for name, has_bender in (("11x100", True), ("11x100_tc", False)):
        n_tiles = SHAPES[name]["n"] * SHAPES[name]["s"] // SL.TILE_M + 1
        assert n_tiles == 9
        for max_ctas in range(sms & ~1, (3 * sms // 4) & ~1, -2):
            assert empty_splits(n_tiles, wgrad_plan(n_tiles, max_ctas, has_bender)), (name, max_ctas)


# ---- loss-scale edges: the bending model and the time-conditioned baseline (TC) ----
def edge_case(mode, **kw):
    return Case(3, 100, bender=False, tc=True, **kw) if mode == "tc" else Case(3, 100, **kw)


MODES = ["bender", "tc"]


def test_zero_upstream_gives_exactly_zero_gradients():
    for mode in MODES:
        cs = edge_case(mode, draw_mag=0.0, reg_mag=0.0)
        o = run_forward(cs)
        b = run_backward(cs, o)
        # every float of each buffer (nerf_grad: the TC layout's full length), the TC per-ray sums and latent columns included
        for k in ("nerf_grad", "d_lat") + (("tc_ws",) if cs.tc else ("bender_grad",)):
            assert bool((b[k] == 0).all()), (mode, k)
        assert bool((grad_stash_images(cs, b) == 0).all()), (mode, "gradient stash")


@pytest.mark.parametrize("mag", [1e-15, 1e10])
def test_extreme_upstream_magnitudes_keep_every_stage_bound(mag):
    for mode in MODES:
        cs = edge_case(mode, draw_mag=mag, reg_mag=0.05 * mag)
        run_all(cs, f"{mode} |d_raw| x {mag:g}", divergence=False)


def test_regulariser_upstream_sets_the_loss_scale():
    cs = Case(3, 100, draw_mag=1e-3, reg_mag=40.0)
    assert float(cs.d_un_up.abs().max()) > 100 * float(cs.d_raw[:, :4].abs().max())
    run_all(cs, "regulariser-dominated", divergence=False)


def test_channel_4_of_d_raw_changes_nothing():
    """Channel 4 never reaches the loss (the head's row 4 gets a zero gradient), so a large d_raw[..., 4] must not move
    the loss scale: every gradient equals the channel-4-zero run bit for bit (the bender's latent gradient up to the order
    of its fp32 atomics; the TC latent sums run in a fixed order, so there the latent gradient too)."""
    for mode in MODES:
        cs = edge_case(mode)
        o = run_forward(cs)
        b0 = run_backward(cs, o)
        d4 = cs.d_raw.clone()
        d4[:, 4] = 3.0e4 * torch.sign(torch.randn(cs.P, device=DEV))
        b4 = run_backward(cs, o, d_raw=d4)
        assert torch.equal(b0["gstash"], b4["gstash"]), f"{mode}: gradient stash differs"
        assert torch.equal(b0["nerf_grad"], b4["nerf_grad"]), f"{mode}: NeRF weight gradients differ"
        if cs.tc:
            assert torch.equal(b0["tc_ws"], b4["tc_ws"]), "tc: per-ray sums or latent weight columns differ"
            assert torch.equal(b0["d_lat"], b4["d_lat"]), "tc: latent gradients differ"
        else:
            assert torch.equal(b0["bender_grad"], b4["bender_grad"]), "bender weight gradients differ"
            # the latent gradient's fp32 atomics add in no fixed order: equal up to that rounding
            torch.testing.assert_close(b0["d_lat"], b4["d_lat"], rtol=0.0, atol=1e-5 * float(b0["d_lat"].abs().max()))


def test_head_redirection_and_accumulation():
    """nerf_grad_head puts the output layer's gradient in its own buffer; accumulate_nerf / accumulate_bender add the
    gradients onto what the destination holds (optim.Adam's gradient arena)."""
    lib = _lib().load()
    for mode in MODES:
        cs = edge_case(mode)
        rep = Report(f"{mode} accumulate + head redirect")
        o = run_forward(cs)
        g = torch.Generator(device=DEV).manual_seed(3)
        n_head = cs.out_ch * 257
        pre_n = torch.randn(lib.nrn_nerf_tc_grad_floats(cs.out_ch) if cs.tc else lib.nrn_nerf_grad_floats(cs.out_ch),
                            generator=g, device=DEV)
        pre_n[-n_head:] = float("nan")        # the head part lives elsewhere: this tail must stay untouched
        pre_h = torch.randn(n_head, generator=g, device=DEV)
        pre_b = torch.randn(lib.nrn_bender_grad_floats(), generator=g, device=DEV)
        nerf, head, bend = pre_n.clone(), pre_h.clone(), pre_b.clone()
        b = run_backward(cs, o, nerf_grad=nerf, nerf_head=head, bender_grad=bend, accumulate=True)
        assert bool(torch.isnan(nerf[-n_head:]).all()), f"{mode}: the head's slot of nerf_grad was written despite nerf_grad_head"
        imgs = dgrad_reference(cs, o, b, rep, expected_scale(cs))
        full = torch.cat([nerf[:-n_head], head])
        base = torch.cat([pre_n[:-n_head], pre_h])
        b["nerf_head"] = None
        check_wgrad(cs, b, imgs, rep, expected_scale(cs), nerf_flat=full, bend_flat=bend, base_nerf=base, base_bend=pre_b)


@pytest.mark.parametrize("head", [False, True])
def test_empty_tc_batch_zeroes_the_whole_gradient_layout(head):
    """n_rays = 0 (an empty shard) contributes zero gradients: every float of the time-conditioned layout, the latent
    columns of W0 / W5 included, is overwritten with 0; with nerf_grad_head the head's slot of nerf_grad stays untouched."""
    from nonrigid_nerf_b200 import ops
    L = _lib()
    lib = L.load()
    npk, _, _ = pack_nerf(*ops.nerf_param_list(models(False, tc=True)[0]), 5, 95)
    n_nerf, n_head = lib.nrn_nerf_tc_grad_floats(5), 5 * 257
    grad, head_buf = poison_f32(n_nerf), poison_f32(n_head)
    a, t = L.NrnFieldBwdArgs(), L.NrnTcBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = 0, 64, 5
    a.nerf_packed, a.nerf_grad = npk.data_ptr(), grad.data_ptr()
    if head:
        a.nerf_grad_head = head_buf.data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    L.check(lib.nrn_field_backward_tc(C.byref(a), C.byref(t)), "field_backward_tc")
    L.device_error_check()
    if head:
        assert bool((grad[:-n_head] == 0).all()) and bool((head_buf == 0).all())
        assert bool(torch.isnan(grad[-n_head:]).all()), "the head's slot of nerf_grad was written despite nerf_grad_head"
    else:
        assert bool((grad == 0).all())


def test_forward_is_deterministic_past_p():
    """Rows past P of a ragged last tile are computed from x = 0 and a zero latent: finite (checked with the stages) and
    the same on every run, masks included."""
    cs = Case(1, 7)
    o1, o2 = run_forward(cs), run_forward(cs)
    n = cs.T
    assert torch.equal(o1["stash"][:n * SL.STASH_TILE], o2["stash"][:n * SL.STASH_TILE])
    assert torch.equal(o1["mask"][:n * SL.MASK_TILE], o2["mask"][:n * SL.MASK_TILE])
