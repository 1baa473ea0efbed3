"""The fused training kernels called through the C ABI (autograd._FieldTrainFn / _DivergenceFn's calling pattern), and an
fp64 reference of every stage fed with the kernel's own fp16 operands read back from the stashes (tests/stash_layout.py).
The bounds are explained in tests/test_stage_parity_gpu.py.

Every check takes a tile subset (Tiles): forward, DGRAD and the divergence chains are row-local, so a check on some tiles
restates exactly the check on all of them.  Per-ray quantities (the latent gradient, the divergence loss) are checked on
the rays whose samples all lie in the chosen tiles.  The weight gradients sum over every tile: checked on a subset they
equal the subset's sum only when every other tile's upstream is zero (tests/test_scale_gpu.py's coverage sweep).
"""
import ctypes as C

import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests import stash_layout as SL
from tests import tc_reference as TR
from tests.parity import DEV, F64, U, Report, half_ulp, poison_bytes, poison_f32, ptr

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


class Tiles:
    """The rows a check covers: every tile of the case (tiles=None) or the listed ones, in ascending order.  Only the last
    tile holds rows past P, so the rows of points are the first `n` rows of every decoded image, and `points` their point
    indices into the per-point arrays [P, ...]."""
    def __init__(self, cs, tiles=None):
        self.T, self.P, self.s, self.n_rays = cs.T, cs.P, cs.s, cs.n
        if tiles is None:
            self.idx, self.count, self.R, self.n = None, cs.T, cs.R, cs.P
            self.rows = torch.arange(cs.R, device=DEV)
        else:
            t = sorted(set(int(x) for x in tiles))
            assert t and 0 <= t[0] and t[-1] < cs.T, (t[:3], t[-3:], cs.T)
            self.idx = torch.tensor(t, dtype=torch.long, device=DEV)
            self.count, self.R = len(t), len(t) * SL.TILE_M
            self.rows = (self.idx[:, None] * SL.TILE_M + torch.arange(SL.TILE_M, device=DEV)).flatten()
            self.n = int((self.rows < cs.P).sum())
        self.points = self.rows[:self.n]

    def pt(self, x, dim=0):
        """The covered points of a per-point array (points along `dim`)."""
        return x if self.idx is None else x.index_select(dim, self.points)

    def ray_rows(self, lat):
        """The latent row of each covered point."""
        return lat.repeat_interleave(self.s, 0) if self.idx is None else lat.index_select(0, self.points // self.s)

    def complete_rays(self):
        """Rays whose samples all lie in the covered tiles (None: every ray)."""
        if self.idx is None:
            return None
        cnt = torch.zeros(self.n_rays, dtype=torch.long, device=DEV).index_add_(0, self.points // self.s,
                                                                                 torch.ones_like(self.points))
        return (cnt == self.s).nonzero().flatten()

    def img(self, buf, tile_bytes, oc):
        return SL.image(buf, tile_bytes, *oc, self.T, tiles=self.idx)

    def bits(self, buf, oc):
        return SL.relu_bits(buf, oc[0], oc[1], self.T, tiles=self.idx)


def on_rays(x, rays):
    return x if rays is None else x.index_select(0, rays)


# ----------------------------------------------------------------------------------------------------------------------
# the kernels, called through the C ABI as autograd._FieldTrainFn / _DivergenceFn do
# ----------------------------------------------------------------------------------------------------------------------
def _lib():
    from nonrigid_nerf_b200 import _lib as L
    return L


_MODELS = {}


def models(bender, tc=False, views=False):
    """(coarse NeRF, bender); tc: the time-conditioned baseline's NeRF (W0 [256][95], W5 [256][351]), no bender; views:
    NeRF(use_viewdirs=True) with tests/viewdirs_reference's weights, no bender."""
    key = "views" if views else ("tc" if tc else bender)
    if key not in _MODELS:
        if views:
            from tests.viewdirs_reference import build_view_models
            _MODELS[key] = (build_view_models(O, SEED, DEV, with_bender=False)[0], None)
        elif tc:
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
    """tc: the time-conditioned baseline (no bender); lat_stride0: one latent row for every ray (latent_stride 0);
    views: the view-dependent head without a bender (out_ch 4), fed the normalised ray directions `vd`."""
    def __init__(self, n, s, bender=True, out_ch=5, cutoff=None, scaling=None, draw_mag=1.0, reg_mag=0.05, ch4=0.0,
                 seed=0, tc=False, lat_stride0=False, views=False):
        assert not (tc and bender), "the time-conditioned baseline has no bender"
        if views:
            bender, out_ch = False, 4
        self.n, self.s, self.bender, self.out_ch, self.tc, self.views = n, s, bender, out_ch, tc, views
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
        self.vd = torch.nn.functional.normalize(self.rays[:, 3:6], dim=-1).contiguous() if views else None
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
    if cs.views:
        assert train and removal is None and points is None
        return run_forward_views(cs)
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


def run_forward_views(cs):
    """nrn_field_forward_views_train (autograd._ViewsTrainFn's forward): the trunk's stash and masks, the view stash and
    the Hv masks; o["ws"] / o["bs"] are the trunk's and alpha_linear's parameters, o["net"] the module."""
    from nonrigid_nerf_b200 import ops
    L = _lib()
    lib = L.load()
    net, _ = models(False, views=True)
    ws, bs = ops._views_trunk_params(net)
    o = {"npk": ops.pack_nerf(net), "vpk": ops.pack_views(net), "vtpk": ops.pack_views_t(net), "net": net, "bend": None,
         "ws": [w.detach() for w in ws], "bs": [b.detach() for b in bs]}
    a, v, t = L.NrnFieldArgs(), L.NrnViewArgs(), L.NrnViewTrainArgs()
    a.rays, a.z_vals, a.n_rays, a.n_samples, a.out_ch = cs.rays.data_ptr(), cs.z.data_ptr(), cs.n, cs.s, 4
    a.nerf_packed = o["npk"].data_ptr()
    o["raw"], o["init"], o["bent"] = poison_f32(cs.P, 4), poison_f32(cs.P, 3), poison_f32(cs.P, 3)
    a.raw, a.initial_input_pts, a.input_pts = o["raw"].data_ptr(), o["init"].data_ptr(), o["bent"].data_ptr()
    for k, f in (("stash", lib.nrn_stash_bytes), ("mask", lib.nrn_relu_mask_bytes), ("vstash", lib.nrn_views_stash_bytes),
                 ("hv_mask", lib.nrn_hv_mask_bytes)):
        o[k] = poison_bytes(f(cs.n, cs.s))
    a.stash, a.relu_mask = o["stash"].data_ptr(), o["mask"].data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    v.views_packed, v.viewdirs, v.viewdirs_stride = o["vpk"].data_ptr(), cs.vd.data_ptr(), cs.vd.stride(0)
    t.views_stash, t.hv_mask = o["vstash"].data_ptr(), o["hv_mask"].data_ptr()
    L.check(lib.nrn_field_forward_views_train(C.byref(a), C.byref(v), C.byref(t)), "field_forward_views_train")
    L.device_error_check()
    return o


def run_backward_views(cs, o, d_raw=None, nerf_grad=None, nerf_head=None, accumulate=False):
    """nrn_field_backward_views into poisoned buffers: b["nerf_grad"] the flat layout (or the trunk, with `nerf_head` the
    head block's own destination), b["gstash"] / b["vgstash"] the trunk's and the head's gradient stashes."""
    L = _lib()
    lib = L.load()
    d_raw = cs.d_raw if d_raw is None else d_raw
    a, v = L.NrnFieldBwdArgs(), L.NrnViewBwdArgs()
    a.n_rays, a.n_samples, a.out_ch = cs.n, cs.s, 4
    a.d_raw, a.stash, a.relu_mask, a.nerf_packed = d_raw.data_ptr(), o["stash"].data_ptr(), o["mask"].data_ptr(), o["npk"].data_ptr()
    b = {"gstash": poison_bytes(lib.nrn_grad_stash_bytes(cs.n, cs.s)), "vgstash": poison_bytes(lib.nrn_views_grad_stash_bytes(cs.n, cs.s)),
         "scratch": poison_bytes(lib.nrn_wgrad_scratch_bytes())}
    b["nerf_grad"] = poison_f32(lib.nrn_nerf_views_grad_floats()) if nerf_grad is None else nerf_grad
    b["nerf_head"] = nerf_head
    a.grad_stash, a.wgrad_scratch, a.nerf_grad = b["gstash"].data_ptr(), b["scratch"].data_ptr(), b["nerf_grad"].data_ptr()
    if nerf_head is not None:
        a.nerf_grad_head = nerf_head.data_ptr()
    a.accumulate_nerf = 1 if accumulate else 0
    a.stream = torch.cuda.current_stream().cuda_stream
    v.views_t_packed, v.views_stash, v.views_grad_stash, v.hv_mask = (o["vtpk"].data_ptr(), o["vstash"].data_ptr(),
                                                                     b["vgstash"].data_ptr(), o["hv_mask"].data_ptr())
    L.check(lib.nrn_field_backward_views(C.byref(a), C.byref(v)), "field_backward_views")
    L.device_error_check()
    return b


def run_backward(cs, o, d_raw=None, nerf_grad=None, nerf_head=None, bender_grad=None, accumulate=False):
    if cs.views:
        return run_backward_views(cs, o, d_raw, nerf_grad, nerf_head, accumulate)
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


def _div_args(cs, o, d):
    L = _lib()
    a = L.NrnDivArgs()
    a.n_rays, a.n_samples = cs.n, cs.s
    a.relu_mask, a.e, a.unmasked_offsets, a.rigidity_mask, a.weights = (
        o["mask"].data_ptr(), cs.e.data_ptr(), o["un"].data_ptr(), o["rig"].data_ptr(), cs.w.data_ptr())
    a.bender_packed = o["bpk"].data_ptr()
    a.tangent_stash = d["tan"].data_ptr()
    a.d, a.alpha, a.beta, a.tau_c = (d["scal"][i].data_ptr() for i in range(4))
    a.loss = d["loss"].data_ptr()
    a.stream = torch.cuda.current_stream().cuda_stream
    return a


def run_divergence_forward(cs, o):
    """The divergence forward; it reads the forward pass's ReLU masks, per-point outputs and packed bender, not its stash."""
    L = _lib()
    lib = L.load()
    d = {"tan": poison_bytes(lib.nrn_div_stash_bytes(cs.n, cs.s)), "scal": poison_f32(4, cs.P), "loss": poison_f32(cs.n)}
    L.check(lib.nrn_divergence_forward(C.byref(_div_args(cs, o, d))), "divergence_forward")
    L.device_error_check()
    return d


def run_divergence_backward(cs, o, d):
    """The divergence backward with the upstream cs.g_ray, into fresh poisoned buffers in d."""
    L = _lib()
    lib = L.load()
    a = _div_args(cs, o, d)
    d["G"], d["adj"] = poison_f32(cs.P), poison_bytes(lib.nrn_div_grad_stash_bytes(cs.n, cs.s))
    d["scratch"] = poison_bytes(lib.nrn_wgrad_scratch_bytes())
    d["d_un"], d["d_rig"], d["grad"] = poison_f32(cs.P, 3), poison_f32(cs.P), poison_f32(lib.nrn_bender_grad_floats())
    a.g_ray, a.G_workspace = cs.g_ray.data_ptr(), d["G"].data_ptr()
    a.adjoint_stash, a.wgrad_scratch = d["adj"].data_ptr(), d["scratch"].data_ptr()
    a.d_unmasked_offsets, a.d_rigidity_mask, a.bender_grad = d["d_un"].data_ptr(), d["d_rig"].data_ptr(), d["grad"].data_ptr()
    L.check(lib.nrn_divergence_backward(C.byref(a)), "divergence_backward")
    L.device_error_check()
    return d


def run_divergence(cs, o):
    return run_divergence_backward(cs, o, run_divergence_forward(cs, o))


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


def check_forward(cs, o, rep, tiles=None):
    sub = Tiles(cs, tiles)
    R, P = sub.R, sub.n
    st = o["stash"]
    img = lambda oc: sub.img(st, SL.STASH_TILE, oc).to(F64)
    E = img(SL.ST_E)
    H = [img(oc) for oc in SL.ST_H]
    init, bent = sub.pt(o["init"]).to(F64), sub.pt(o["bent"]).to(F64)
    if cs.bender:
        Bin, Hb = img(SL.ST_BIN), [img(SL.ST_HB1), img(SL.ST_HB2), img(SL.ST_HB3), img(SL.ST_HB4)]
        Bh, bias = bender_blocks(o["bend"], h16)
        hi, lo = Bin[:P, 0:3], Bin[:P, 3:6]
        assert torch.equal(hi, h16(sub.pt(o["init"]))), "bender input: xyz hi column is not fp16(x)"
        assert bool(((hi + lo - init).abs() <= 2.0 ** -22 * init.abs() + 2.0 ** -25).all()), "bender input: hi + lo != x"
        lat = sub.ray_rows(cs.lat)
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
        got_r = sub.pt(o["rig"]).to(F64)
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
        rep.check("unmasked_offsets", sub.pt(o["un"]), v[:P, :3], a[:P, :3], c_mma(64))
        masked = sub.pt(o["rig"])[:, None] * sub.pt(o["un"])
        if cs.scaling is not None:
            masked = masked * cs.scaling
        assert torch.equal(sub.pt(o["masked"]), masked), "masked offsets are not fp32(rigidity * unmasked)"
        assert torch.equal(sub.pt(o["bent"]), sub.pt(o["init"]) + sub.pt(o["masked"])), "bent point is not fp32(x + masked)"
    else:
        assert torch.equal(sub.pt(o["bent"]), sub.pt(o["init"]))
    # embedding of the bent point
    assert torch.equal(E[:P, :3], h16(sub.pt(o["bent"]))), "E columns 0-2 are not fp16(bent xyz)"
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
        ray = sub.rows.clamp(max=cs.P - 1) // cs.s
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
    if cs.views:
        check_view_head(cs, o, rep, sub, H[7])
    else:
        v, a = mm(H[7][:P], W[8])
        rep.check("raw", sub.pt(o["raw"]), v + b[8], a + b[8].abs(), c_mma(256))
    # ReLU mask bits: the encoding of stash image > 0, every bit of every word, rows past P included
    imgs = [sub.img(st, SL.STASH_TILE, oc) for oc in SL.ST_H]
    names = [f"H{l + 1}" for l in range(8)]
    if cs.bender:
        imgs += [sub.img(st, SL.STASH_TILE, oc) for oc in (SL.ST_HB1, SL.ST_HB2, SL.ST_HB3, SL.ST_HB4)]
        names += ["Hb1", "Hb2", "Hb3", "Hb4"]
    for nm, im, (off, ncols) in zip(names, imgs, SL.MASK_IMAGES):
        enc = SL.encode_relu_bits(im[:, :ncols] > 0)
        got = SL.tile_slices(o["mask"], SL.MASK_TILE, off, enc.shape[1], sub.T, sub.idx)
        assert torch.equal(got, enc), f"ReLU mask of {nm}: {int((got != enc).sum())} bytes differ from stash > 0"


# The direction encoding's sin / cos: the phase 2^k d / 2 pi is reduced exactly to [-1/2, 1/2) turns (field_fwd.cu,
# encode_octaves); the reduced phase (one fp32 add), its product with fl(2 pi) (one fp32 multiply, fl(2 pi) itself within
# 2^-24 relative) put the angle in [-pi, pi] within 2^-22 absolute, and __sinf / __cosf err by at most 2^-21.41 / 2^-21.19
# there (CUDA C++ Programming Guide, intrinsic functions).  |d sin / d angle| <= 1, so the fp32 value lies within
# 2^-21.19 + 2^-22 (6.6e-7; DESIGN section 2: about 4e-7 for MUFU alone) of the exact encoding of the fp32 direction,
# and its fp16 image within half an ulp more.
E_DIR_ENC = 2.0 ** -21.19 + 2.0 ** -22


def direction_encoding64(d):
    """[d, sin(2^k d), cos(2^k d)] (k = 0..3, embeddirs_fn's order) of fp64 directions [R, 3] -> [R, 27]."""
    k = 2.0 ** torch.arange(4, dtype=F64, device=d.device)
    arg = d[:, None, :] * k[None, :, None]
    return torch.cat([d, torch.stack([torch.sin(arg), torch.cos(arg)], 2).reshape(d.shape[0], 24)], 1)


def view_head_weights(net):
    """fp16(w) of the head as the kernels hold it, fp32 biases; fp64 on DEV."""
    g = lambda m: (h16(m.weight), m.bias.detach().to(F64))
    wv, bv = g(net.views_linears[0])
    wf, bf = g(net.feature_linear)
    wa, ba = g(net.alpha_linear)
    wr, br = g(net.rgb_linear)
    return dict(wvf=wv[:, :256], wve=wv[:, 256:], bv=bv, wf=wf, bf=bf, wa=wa, ba=ba, wr=wr, br=br)


def check_view_head(cs, o, rep, sub, H8):
    """The view stash and the head's outputs on sub's tiles, each from the kernel's own operands:
        Dir  = fp16 of the encoding of the fp32 direction, within 0.5 ulp + E_DIR_ENC; rows past P encode d = 0 (the
               kernel keeps every stashed row finite); columns 27..31 exactly 0
        F    = fp16(H8 Wf^T + bf)                                      c_mma(256) + 0.5 ulp
        Hv   = relu(fp16(F WvF^T + Dir WvE^T + bv))                    c_mma(256 + 32): one N = 128 accumulator
        raw  = [Hv Wr^T + br | H8 Wa^T + ba]                           c_mma(128) / c_mma(256), fp32
    and the Hv mask bits equal the encoding of Hv > 0 byte for byte."""
    R, P = sub.R, sub.n
    img = lambda oc: sub.img(o["vstash"], SL.V_STASH_TILE, oc).to(F64)
    Dir, F, Hv = img(SL.VS_DIR), img(SL.VS_F), img(SL.VS_HV)
    w = view_head_weights(o["net"])
    d = torch.zeros(R, 3, dtype=F64, device=DEV)
    d[:P] = sub.ray_rows(cs.vd).to(F64)
    assert torch.equal(Dir[:, :3], d.half().to(F64)), "Dir columns 0-2 are not fp16(direction)"
    assert bool((Dir[:, 27:] == 0).all()), "Dir columns 27-31 are not 0"
    enc = direction_encoding64(d)
    rep.check("Dir (sin / cos)", Dir[:, 3:27], enc[:, 3:], torch.full_like(enc[:, 3:], E_DIR_ENC / U), 1.0, True)
    v, a = mm(H8, w["wf"])
    rep.check("F", F, v + w["bf"], a + w["bf"].abs(), c_mma(256), True)
    v1, a1 = mm(F, w["wvf"])
    v2, a2 = mm(Dir[:, :27], w["wve"])
    rep.check("Hv", Hv, torch.relu(v1 + v2 + w["bv"]), a1 + a2 + w["bv"].abs(), c_mma(256 + 32), True)
    rgb, rgb_a = mm(Hv[:P], w["wr"])
    alpha, alpha_a = mm(H8[:P], w["wa"])
    raw = sub.pt(o["raw"])
    rep.check("raw rgb", raw[:, :3], rgb + w["br"], rgb_a + w["br"].abs(), c_mma(128))
    rep.check("raw alpha", raw[:, 3:], alpha + w["ba"], alpha_a + w["ba"].abs(), c_mma(256))
    enc_bits = SL.encode_relu_bits(sub.img(o["vstash"], SL.V_STASH_TILE, SL.VS_HV) > 0)
    got = SL.tile_slices(o["hv_mask"], SL.HV_MASK_TILE, 0, SL.HV_MASK_TILE, sub.T, sub.idx)
    assert torch.equal(got, enc_bits), f"Hv mask: {int((got != enc_bits).sum())} bytes differ from Hv > 0"


def wgrad_images(cs, o, b, sub):
    """The decoded fp16 operands of WGRAD on the tiles of sub: E, H1..H8, d_raw, dY0..dY7, and with a bender its input,
    Hb1..Hb4 and dYb0..dYb4."""
    img = lambda oc: sub.img(o["stash"], SL.STASH_TILE, oc).to(F64)
    gimg = lambda oc: sub.img(b["gstash"], SL.GRAD_TILE, oc).to(F64)
    out = {"E": img(SL.ST_E), "H": [img(oc) for oc in SL.ST_H], "Draw": gimg(SL.GS_RAW), "dY": [gimg(oc) for oc in SL.GS_Y]}
    if cs.views:
        vimg = lambda oc: sub.img(o["vstash"], SL.V_STASH_TILE, oc).to(F64)
        vgimg = lambda oc: sub.img(b["vgstash"], SL.V_GRAD_TILE, oc).to(F64)
        out.update(Dir=vimg(SL.VS_DIR), F=vimg(SL.VS_F), Hv=vimg(SL.VS_HV), dYv=vgimg(SL.VG_YV), dF=vgimg(SL.VG_F))
    if cs.bender:
        out.update(Bin=img(SL.ST_BIN), Hb=[img(SL.ST_HB1), img(SL.ST_HB2), img(SL.ST_HB3), img(SL.ST_HB4)],
                   Yb=[gimg(oc) for oc in (SL.GS_YB0, SL.GS_YB1, SL.GS_YB2, SL.GS_YB3, SL.GS_YB4)])
    return out


def dgrad_reference(cs, o, b, rep, scale, tiles=None):
    """Checks DGRAD stage by stage; returns the decoded images the WGRAD check needs and the Tiles they cover."""
    sub = Tiles(cs, tiles)
    R, P = sub.R, sub.n
    mbits = lambda oc: sub.bits(o["mask"], oc).to(F64)
    out = wgrad_images(cs, o, b, sub)
    out["sub"] = sub
    E, Draw, dY = out["E"], out["Draw"], out["dY"]
    W = [h16(w) for w in o["ws"]]
    exp_raw = (sub.pt(cs.d_raw)[:, :4] * scale).clamp(-65504.0, 65504.0).half().to(F64)
    assert torch.equal(Draw[:P, :4], exp_raw), "d_raw image is not fp16(clamp(d_raw[:, :4] * scale))"
    assert bool((Draw[:P, 4:] == 0).all()) and bool((Draw[P:] == 0).all()), "d_raw image: padding is not zero"
    m = [mbits(oc) for oc in SL.MK_H]
    if cs.views:
        # Rgb^T, ViewsF^T, then Feature^T and alpha's column into one accumulator, each from the kernel's own operands
        w = view_head_weights(o["net"])
        mv = SL.relu_bits(o["hv_mask"], 0, 128, sub.T, tile_bytes=SL.HV_MASK_TILE, tiles=sub.idx).to(F64)
        dYv, dF = out["dYv"], out["dF"]
        v, a = dmm(Draw[:, :3], w["wr"])
        rep.check("dYv", dYv, v * mv, a * mv, c_mma(16), True)
        v, a = dmm(dYv, w["wvf"])
        rep.check("dF", dF, v, a, c_mma(128), True)
        v1, a1 = dmm(dF, w["wf"])
        v2, a2 = dmm(Draw[:, 3:4], w["wa"])
        rep.check("dY7", dY[7], (v1 + v2) * m[7], (a1 + a2) * m[7], c_mma(256 + 16), True)
    else:
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
    if cs.views:
        return out            # no L5e^T / L0^T: the embedding gradient has no consumer without a bender
    dE0, dE0a = dmm(dY[0], W[0][:, :63])
    pad = lambda t: torch.cat([t, torch.zeros(R, 1, dtype=F64, device=DEV)], 1)
    dx5, ax5 = pe_backward(pad(dE5), pad(dE5a), E)
    dx0, ax0 = pe_backward(pad(dE0), pad(dE0a), E)
    dx, adx = dx5 + dx0, ax5 + ax0
    c_dx = c_mma(256) + C_PE
    if cs.tc:
        # per-ray sums of the stashed dY0 / dY5 over the ray's samples, in fp32 and divided by the loss scale
        rays = sub.complete_rays()
        sums = b["tc_ws"][:cs.n * 512].view(cs.n, 2, 256)
        if rays is None:
            ds = [dY[l][:P].view(cs.n, cs.s, 256) for l in (0, 5)]
            ref, ref_a = torch.stack([d.sum(1) for d in ds], 1), torch.stack([d.abs().sum(1) for d in ds], 1)
        else:
            ray = sub.points // cs.s
            acc = lambda x: torch.zeros(cs.n, 256, dtype=F64, device=DEV).index_add_(0, ray, x)
            ref = torch.stack([acc(dY[l][:P]) for l in (0, 5)], 1)[rays]
            ref_a = torch.stack([acc(dY[l][:P].abs()) for l in (0, 5)], 1)[rays]
        rep.check("tc per-ray sums", on_rays(sums, rays), ref / scale, ref_a / scale, cs.s + 2)
        # d z from the kernel's own sums and the fp32 latent columns of W0 / W5
        s = sums.to(F64)
        w0, w5 = o["ws"][0][:, 63:95].to(F64), o["ws"][5][:, 63:95].to(F64)
        rep.check("tc d_latents", b["d_lat"], s[:, 0] @ w0 + s[:, 1] @ w5, s[:, 0].abs() @ w0.abs() + s[:, 1].abs() @ w5.abs(),
                  C_DZ)
    if not cs.bender:
        return out
    Yb0, Yb1, Yb2, Yb3, Yb4 = out["Yb"]
    Bh, _ = bender_blocks(o["bend"], h16)
    rig, un = sub.pt(o["rig"]).to(F64)[:, None], sub.pt(o["un"]).to(F64)
    s = 1.0 if cs.scaling is None else float(torch.tensor(cs.scaling, dtype=torch.float32))
    dm, adm = dx[:P] * s, adx[:P] * abs(s)
    up_u = torch.zeros_like(un) if cs.d_un_up is None else sub.pt(cs.d_un_up).to(F64) * scale
    up_r = torch.zeros_like(rig[:, 0]) if cs.d_rig_up is None else sub.pt(cs.d_rig_up).to(F64) * scale
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
    ray = sub.points // cs.s
    lat = torch.zeros(cs.n, 32, dtype=F64, device=DEV).index_add_(0, ray, v) / scale
    lat_a = torch.zeros(cs.n, 32, dtype=F64, device=DEV).index_add_(0, ray, a) / scale
    rays = sub.complete_rays()
    rep.check("d_latents", on_rays(b["d_lat"], rays), on_rays(lat, rays), on_rays(lat_a, rays), c_mma(96) + cs.s + 8)
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


def wgrad_reference(cs, imgs):
    """(NeRF, bender) weight-gradient sums over the decoded images of wgrad_images, before the loss scale: {name: (value,
    abs)}; the bender dict is None without a bender."""
    sub = imgs["sub"]
    E, H, Draw, dY = imgs["E"], imgs["H"], imgs["Draw"], imgs["dY"]
    # the inputs of W0 and of W5's first columns: [E[:, :63] | the row's latent (time-conditioned; 0 past P)]
    X = E[:, :63]
    if cs.tc:
        Z = torch.zeros(sub.R, 32, dtype=F64, device=DEV)
        Z[:sub.n] = sub.ray_rows(cs.lat.to(F64))
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
    if cs.views:
        # the head block; job 0 (the trunk's head job) contributes alpha_linear only: d_raw column 3 (x) H8
        bsum = lambda y: (y.sum(0), y.abs().sum(0))
        Dir, F, Hv, dYv, dF = imgs["Dir"], imgs["F"], imgs["Hv"], imgs["dYv"], imgs["dF"]
        ref["views_linears.0.weight"] = wsum(dYv, torch.cat([F, Dir[:, :27]], 1))
        ref["views_linears.0.bias"] = bsum(dYv)
        ref["feature_linear.weight"], ref["feature_linear.bias"] = wsum(dF, H[7]), bsum(dF)
        ref["alpha_linear.weight"], ref["alpha_linear.bias"] = wsum(Draw[:, 3:4], H[7]), bsum(Draw[:, 3:4])
        ref["rgb_linear.weight"], ref["rgb_linear.bias"] = wsum(Draw[:, :3], Hv), bsum(Draw[:, :3])
        return ref, None
    v, a = wsum(Draw[:, :4], H[7])
    z = torch.zeros(cs.out_ch - 4, 256, dtype=F64, device=DEV)
    ref["w_out"] = (torch.cat([v, z]), torch.cat([a, z]))
    zb = torch.zeros(cs.out_ch - 4, dtype=F64, device=DEV)
    ref["b_out"] = (torch.cat([Draw[:, :4].sum(0), zb]), torch.cat([Draw[:, :4].abs().sum(0), zb]))
    bend = bender_wgrad_reference(imgs["Yb"], [imgs["Bin"]] + imgs["Hb"]) if cs.bender else None
    return ref, bend


def check_wgrad(cs, b, imgs, rep, scale, nerf_flat=None, bend_flat=None, base_nerf=None, base_bend=None, refs=None,
                n_tiles=None, rel_l2=WGRAD_REL_L2):
    """WGRAD against the sums over imgs' tiles (or precomputed `refs` over n_tiles tiles) at c_wgrad of that tile count,
    and at relative L2 `rel_l2` per NeRF tensor."""
    ref, bref = wgrad_reference(cs, imgs) if refs is None else refs
    c = c_wgrad(imgs["sub"].count if refs is None else n_tiles)
    shapes = SL.views_param_shapes() if cs.views else SL.nerf_param_shapes(cs.out_ch, cs.tc)
    got = SL.split_flat(b["nerf_grad"] if nerf_flat is None else nerf_flat, shapes)
    if b["nerf_head"] is not None:
        got.update(SL.split_flat(b["nerf_head"], SL.HEAD_SHAPES if cs.views else shapes[-2:]))
    assert set(got) == set(ref), set(got) ^ set(ref)
    base = SL.split_flat(base_nerf, shapes) if base_nerf is not None else None
    for name, (v, a) in ref.items():
        g = got[name].to(F64) - (base[name].to(F64) if base is not None else 0.0)
        rep.check(f"WGRAD {name}", g, v / scale, a / scale + (base[name].to(F64).abs() if base is not None else 0.0), c)
        if base is None:
            rep.rel_l2(f"WGRAD {name}", g, v / scale, rel_l2)
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
            # the worst case c_latent_columns(n) grows with n faster than one ray's share of the sum shrinks: at 8,192 rays
            # one ray dropped stays inside it, but moves these 8,192 elements by about 1 / sqrt(n) in relative L2
            if base is None:
                rep.rel_l2(f"WGRAD {name}[:, 63:95]", g, s[:, l].T @ z, rel_l2)
    if cs.out_ch == 5 and base is None:
        assert bool((got["w_out"][4] == 0).all()) and float(got["b_out"][4]) == 0.0, "head row 4 gradient is not exactly 0"
    if not cs.bender:
        return
    got = SL.split_flat(b["bender_grad"] if bend_flat is None else bend_flat, SL.bender_param_shapes())
    base = SL.split_flat(base_bend, SL.bender_param_shapes()) if base_bend is not None else None
    for name, (v, a) in bref.items():
        g = got[name].to(F64) - (base[name].to(F64) if base is not None else 0.0)
        rep.check(f"WGRAD {name}", g, v / scale, a / scale + (base[name].to(F64).abs() if base is not None else 0.0), c)


def expected_scale(cs, d_raw=None):
    d_raw = cs.d_raw if d_raw is None else d_raw
    amax = float(d_raw[:, :4].abs().max())
    for t in (cs.d_un_up, cs.d_rig_up):
        if t is not None:
            amax = max(amax, float(t.abs().max()))
    return SL.loss_scale(amax)


def check_divergence(cs, o, d, rep, tiles=None, wgrad=True):
    """The divergence chains on the tiles given; with `wgrad` the compact WGRAD against their sum (which is all of it only
    when every other tile's G is zero)."""
    sub = Tiles(cs, tiles)
    R, P = sub.R, sub.n
    Bf, _ = bender_blocks(o["bend"], lambda t: t.to(F64))
    mb = [sub.bits(o["mask"], oc).to(F64) for oc in (SL.MK_HB1, SL.MK_HB2, SL.MK_HB3, SL.MK_HB4)]
    tan = lambda oc: sub.img(d["tan"], SL.TAN_TILE, oc).to(F64)
    adj = lambda oc: sub.img(d["adj"], SL.ADJ_TILE, oc).to(F64)
    zpad = lambda t: torch.cat([t, torch.zeros(R - P, *t.shape[1:], dtype=F64, device=DEV)])
    e_pts = sub.pt(cs.e)
    e = zpad(e_pts.to(F64))
    TE = tan(SL.T_E)
    e_hi = e_pts.half()
    assert torch.equal(TE[:P, 0:3], e_hi.to(F64)) and torch.equal(TE[:P, 3:6], (e_pts - e_hi.float()).half().to(F64)), \
        "tangent input is not [fp16(e) | fp16(e - fp16(e))]"
    assert bool((TE[:, 6:] == 0).all()) and bool((TE[P:] == 0).all()), "tangent input: padding is not zero"
    # the probe as the tangent chain sees it, hi + lo: fp32-accurate (2^-22 |e|) only while e's residual is an fp16 normal;
    # below |e| of about 2^-3 it is resolved to 2^-25 absolute, as the bender input's hi / lo columns are
    e_op = TE[:, 0:3] + TE[:, 3:6]
    assert bool(((e_op - e).abs() <= 2.0 ** -22 * e.abs() + 2.0 ** -25).all()), "tangent input: hi + lo != e"
    # tangent chain, fp64 from the kernel's own input operand with the fp32 weights and the primal pass's mask bits
    W0x = Bf[0][:, 0:3]
    t1, t1a = mm(e_op, W0x)
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
    r, un, ek = sub.pt(o["rig"]).to(F64), sub.pt(o["un"]).to(F64), e_pts.to(F64)
    alpha, alpha_a = (ek * tau[:P]).sum(1), (ek.abs() * taua[:P]).sum(1)
    beta, beta_a = (ek * un).sum(1), (ek.abs() * un.abs()).sum(1)
    g = 2.0 * r * (1.0 - r)
    dd = r * alpha + beta * g * tc[:P]
    dd_a = r * alpha_a + beta_a * g * tca[:P].abs() + beta.abs() * g * tca[:P]
    scal = sub.pt(d["scal"], 1)
    rep.check("div tau_c", scal[3], tc[:P], tca[:P], C_DIV, floor=DIV_FLOOR)
    rep.check("div alpha", scal[1], alpha, alpha_a, C_DIV, floor=DIV_FLOOR)
    rep.check("div beta", scal[2], beta, beta_a, C_DIV, floor=DIV_FLOOR)
    rep.check("div d", scal[0], dd, dd_a, C_DIV, floor=DIV_FLOOR)
    ray = sub.points // cs.s
    w = sub.pt(cs.w).to(F64)
    loss = torch.zeros(cs.n, dtype=F64, device=DEV).index_add_(0, ray, w * dd * dd) / cs.s
    rays = sub.complete_rays()
    loss, got_loss = on_rays(loss, rays), on_rays(d["loss"], rays).to(F64)
    lerr = float(((got_loss - loss).abs() / loss.abs().clamp_min(1e-30)).max())
    if not rep.quiet:
        print(f"  [{rep.tag}] {'div loss per ray':<24s} rel err {lerr:.3e}   bound {LOSS_REL_DIV:.0e}")
    assert lerr <= LOSS_REL_DIV, lerr
    # backward: G = g_ray * 2 / S * w * d (from the kernel's d), the loss scale of max |G|, the adjoint chain
    dk = scal[0].to(F64)
    G = cs.g_ray.to(F64)[ray] * 2.0 / cs.s * w * dk
    Gk = sub.pt(d["G"]).to(F64)
    rep.check("div G", Gk, G, G.abs(), C_CLOSED)
    scale = SL.loss_scale(float(d["G"].abs().max()))
    alpha_k, beta_k, tc_k = scal[1].to(F64), scal[2].to(F64), scal[3].to(F64)
    tau_r = g * tc_k
    rep.check("div d_unmasked", sub.pt(d["d_un"]), Gk[:, None] * tau_r[:, None] * ek, (Gk * tau_r)[:, None].abs() * ek.abs(),
              C_CLOSED)
    dr = Gk * (alpha_k + 2.0 * beta_k * tc_k * (1.0 - 2.0 * r))
    dr_a = Gk.abs() * (alpha_k.abs() + (2.0 * beta_k * tc_k * (1.0 - 2.0 * r)).abs())
    rep.check("div d_rigidity", sub.pt(d["d_rig"]), dr, dr_a, C_CLOSED)
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
    if not wgrad:
        return
    # compact WGRAD over the decoded stashes: sum adj (x) tan / scale, no bias
    ref = bender_wgrad_reference([A0, A1, A2, A3, A4], [TE, tan(SL.T_1), tan(SL.T_2), tan(SL.T_3), tan(SL.T_4)])
    got = SL.split_flat(d["grad"], SL.bender_param_shapes())
    for name, (v, a) in ref.items():
        if "_b" in name:
            assert bool((got[name] == 0).all()), f"divergence WGRAD {name}: the tangent chain has no bias"
            continue
        rep.check(f"div WGRAD {name}", got[name], v / scale, a / scale, c_wgrad(sub.count))


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


# ---- WGRAD's split plan (wgrad.cu, launch_jobs), replicated ----
# kJobCost: per job id 0..15 (0 head, 1..9 NeRF layers, 10 / 11 bender, 12 feature_linear, 13 views_linears.0's feature
# columns, 14 rgb_linear, 15 views_linears.0's direction columns)
_JOB_COST = [46, 48, 48, 48, 48, 48, 48, 48, 32, 32, 54, 42, 48, 48, 24, 20]
VIEW_HEAD_JOBS = (12, 13, 14, 15)
WG_SCRATCH_FLOATS = 256 * 256 + 256   # one partial per (job, split, half): kWgScratchFloats


def wgrad_halves(has_bender=True, compact=False, views=False):
    """{job: CTAs per split}, in the launch's job order: the NeRF layer jobs 1..9 take two; the head (0) and bender jobs
    (10, 11) one.  The divergence kernels' compact launch runs the bender jobs only.  views: launch_wgrad_views' jobs,
    where feature_linear (12) takes two like a NeRF layer and the other head jobs one."""
    if views:
        return {j: 2 if 1 <= j <= 9 or j == 12 else 1 for j in (*range(10), *VIEW_HEAD_JOBS)}
    jobs = range(10, 12) if compact else range(12 if has_bender else 10)
    return {j: 2 if 1 <= j <= 9 else 1 for j in jobs}


def wgrad_rel_l2(split_tiles):
    """Relative L2 bound of a NeRF weight gradient whose largest split sums `split_tiles` tiles in one fp32 accumulator.
    Measured on an H100 at 1,024, 4,096 and 8,192 tiles, W0's error grows in step with the tiles of its split (about
    0.6 x 2^-22 per tile: the partial sums grow with the depth, and so does each k-step's rounding).  Those three sizes
    all give W0's job 4 splits, so depth per split and T were not varied apart.  2.5 x 2^-22 per tile keeps a 4x margin;
    the bound never drops below WGRAD_REL_L2."""
    return max(WGRAD_REL_L2, 2.5 * 2.0 ** -22 * split_tiles)


def wgrad_plan(n_tiles, max_ctas, has_bender=True, compact=False, views=False):
    halves = wgrad_halves(has_bender, compact, views)
    splits = {j: 1 for j in halves}
    used, tiles = sum(halves.values()), max(n_tiles, 1)
    while True:
        best, best_load = -1, -1
        for j in halves:
            if splits[j] >= tiles or used + halves[j] > max_ctas:
                continue
            load = _JOB_COST[j] * -(-tiles // splits[j])
            if load > best_load:
                best, best_load = j, load
        if best < 0:
            return splits
        splits[best] += 1
        used += halves[best]


def split_ranges(n_tiles, n_split):
    """[t_begin, t_end) of every split of a job that owns tiles (wgrad_kernel: ceil(T / splits) contiguous tiles each)."""
    per = -(-n_tiles // n_split)
    return [(t, min(t + per, n_tiles)) for t in range(0, n_tiles, per)]


def empty_splits(n_tiles, splits):
    out = {}
    for j, ns in splits.items():
        n_valid = len(split_ranges(n_tiles, ns))
        if n_valid < ns:
            out[j] = ns - n_valid
    return out
