"""The per-ray kernels of a training step -- compositing forward and backward, fused and stand-alone resampling, coarse
sampling, the ray loss and Adam -- against fp64 references of the same operation (tests/ray_reference.py) fed with the
kernel's own fp32 inputs, called through the C ABI.

Per element: |kernel - exact| <= c * 2^-24 * M (tests/parity.py), M the reference expression on absolute values and c
the depth of the kernel's fp32 evaluation:
  * alpha: absolute (M = 1), c = 10: the fp32 roundings of relu(sigma) dist reach alpha as exp(-x) x <= 1/e times their size.
  * weights and maps: the product T_i of i fp32 factors 1 - alpha + 1e-10 (two roundings each) and the strided warp sums,
    c = 3 S + 16 (disp: twice that); computed from the kernel's own alpha, because near alpha -> 1 the fp32 factor
    1 - alpha + 1e-10 has lost its digits and an fp64 alpha would compare against a different product.
  * composite backward: c = 4 S + 64 on M = |dalpha| terms of g_i T_i and sum_{k>=i} |g_k w_k| / om_i (the kernel forms the
    exclusive suffix sum as inclusive minus its own term, so |g_i w_i| belongs in M), times the dist exp(-x) (1 + x)
    derivative.
  * sample_pdf: per sample, no fraction allowance; where u or denom lies within the CDF's fp32 error bound of a CDF entry
    or of the 1e-5 threshold, either neighbouring branch is accepted (ray_reference.sample_pdf_accepts).
  * ray loss: c = ceil(S / 32) + 48 for the loss, 8 for the rgb gradients and 32 for the regularisers' (powf, logf and
    the schedule 0.01^(1 - step / N)); the backward is bit-exact (one product).
  * Adam: the update p_new - p_old within 0.5 ulp(p_new) + 16 * 2^-24 |update|, m and v with c = 8.
Bit-exact: fused resampling against the stand-alone sample_pdf kernel and torch.sort; sample_coarse against the reference
formula run by torch on CUDA (torch.linspace on the device); stride-3 against stride-8 rays_d; d_raw channels >= 4 are 0.

Every output buffer is filled with 0xFF (fp32 NaN) first, so a slot no kernel wrote shows up.  `pytest -s` prints c_obs.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import ray_reference as R
from tests.parity import DEV, F64, Report, poison_f32, ptr

pytestmark = pytest.mark.gpu
C_ALPHA = 10
C_PDF = 8
C_STD = 16
C_LOSS_RGB = 8               # (rgb - t) * (2 / 3): three roundings
C_LOSS_GRAD = 32
C_ADAM_UPD, C_ADAM_MOM = 16, 8
UNDERFLOW = 2.0 ** -126      # an fp32 product of transmittances may flush below the normal range where fp64 does not
BWD_UNDERFLOW = 2.0 ** -110  # the same, times the O(10^4) factors (g, dist, 1 / om) the backward applies after it


def c_scan(S):
    return 3 * S + 16


def c_bwd(S):
    return 4 * S + 64


def c_loss(S):
    return math.ceil(S / 32) + 48


def pdf_k(nb):
    """error of the kernel's fp32 CDF in units of 2^-24: the strided lane sums, the warp sum and the chunked scan"""
    return 3 * math.ceil((nb - 1) / 32) + 16


def _lib():
    from nonrigid_nerf_b200 import _lib as L
    return L, L.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def all_poison(t):
    return bool((bits(t) == -1).all())


# ----------------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------------
class Rays:
    """n rays of S samples: rays [n, 8] (d in columns 3-5, the layout training passes), z sorted in [2, 6], raw [n, S, ch]
    with densities around one optical depth per ray.  With `special`, ray 1 has zero density and ray 2 saturates at its
    third sample (when there are enough rays)."""

    def __init__(self, n, S, ch=5, noise=False, special=True, seed=0):
        g = torch.Generator().manual_seed(9000 + 31 * n + S + 7 * ch + seed)
        self.n, self.S, self.ch = n, S, ch
        rays = torch.randn(n, 8, generator=g)
        rays[:, 6], rays[:, 7] = 2.0, 6.0
        z = torch.sort(2.0 + 4.0 * torch.rand(n, S, generator=g), -1)[0]
        raw = torch.randn(n, S, ch, generator=g) * 2
        raw[..., 3] = (torch.randn(n, S, generator=g) + 0.5) * (S / 8.0)
        nz = torch.randn(n, S, generator=g) * (S / 8.0) if noise else None
        if special and n >= 2:
            raw[1, :, 3] = -raw[1, :, 3].abs()
            if nz is not None:
                nz[1] = 0.0
        if special and n >= 3 and S >= 3:
            raw[2, :, 3] = raw[2, :, 3].abs()
            raw[2, 2, 3] = 1e6
        self.rays, self.z, self.raw = rays.to(DEV), z.to(DEV), raw.to(DEV)
        self.noise = None if nz is None else nz.to(DEV)
        self.d8 = self.rays[:, 3:6]                 # row stride 8
        self.d3 = self.d8.contiguous()              # row stride 3


def composite(r, d, white=False, n_imp=0, u=None, raw=None):
    """nrn_composite of r (or of `raw` in place of r.raw) on poisoned outputs; rays_d `d` is read with its row stride"""
    L, lib = _lib()
    raw = r.raw if raw is None else raw
    n, S, ch = raw.shape
    a = L.NrnCompositeArgs()
    a.raw, a.z_vals, a.rays_d, a.rays_d_stride = raw.data_ptr(), r.z.data_ptr(), d.data_ptr(), d.stride(0)
    a.noise = ptr(r.noise)
    a.n_rays, a.n_samples, a.channels, a.white_bkgd = n, S, ch, int(white)
    o = {"rgb": poison_f32(n, 3), "disp": poison_f32(n), "acc": poison_f32(n), "depth": poison_f32(n),
         "weights": poison_f32(n, S), "alpha": poison_f32(n, S)}
    a.rgb_map, a.disp_map, a.acc_map, a.depth_map = (o[k].data_ptr() for k in ("rgb", "disp", "acc", "depth"))
    a.weights, a.alpha = o["weights"].data_ptr(), o["alpha"].data_ptr()
    a.n_importance = n_imp
    if n_imp:
        a.u = ptr(u)
        o["z_out_pad"] = poison_f32(n + 1, S + n_imp)      # one spare row: nothing may be written past the last ray
        o["z_std"] = poison_f32(n)
        a.z_vals_out, a.z_std = o["z_out_pad"].data_ptr(), o["z_std"].data_ptr()
    a.stream = _stream()
    L.check(lib.nrn_composite(C.byref(a)), "composite")
    torch.cuda.synchronize()
    if n_imp:
        o["z_out"] = o["z_out_pad"][:n]
    return o


class Window:
    """samples a..b-1 of every ray of r"""

    def __init__(self, r, a, b):
        self.raw, self.z = r.raw[:, a:b].contiguous(), r.z[:, a:b].contiguous()
        self.noise = None if r.noise is None else r.noise[:, a:b].contiguous()


def kernel_alpha(r, d):
    """the composite kernel's alpha for any S (the kernel takes at most 3000 samples): windows of at most 2049 samples
    overlapping by one, as sample i's alpha needs z_{i+1}; the last window ends with the ray, so its last alpha takes the
    1e10 distance like the full ray's"""
    if r.S <= 2048:
        return composite(r, d)["alpha"]
    parts = []
    for a in range(0, r.S, 2048):
        b = min(a + 2049, r.S)
        al = composite(Window(r, a, b), d)["alpha"]
        parts.append(al[:, :2048] if b < r.S else al)
    return torch.cat(parts, 1)


def sample_pdf(bins, weights, u, n_samp):
    L, lib = _lib()
    n, nb = bins.shape
    out = poison_f32(n, n_samp)
    L.check(lib.nrn_sample_pdf(bins.data_ptr(), weights.data_ptr(), ptr(u), n, nb, n_samp, out.data_ptr(), _stream()),
            "sample_pdf")
    torch.cuda.synchronize()
    return out


def det_u(n, n_samp):
    """the u a call without u uses: torch.linspace(0, 1, n_samp) on the device (0 for one sample)"""
    return torch.linspace(0.0, 1.0, n_samp, device=DEV).expand(n, n_samp).contiguous()


# ----------------------------------------------------------------------------------------------------------------------
# 1. composite forward
# ----------------------------------------------------------------------------------------------------------------------
S_SET = [1, 7, 31, 32, 33, 64, 100, 128, 192, 1000]
N_SET = [1, 5, 1023]


def check_composite(rep, r, o, white):
    S = r.S
    ones = torch.ones(r.n, S, dtype=F64, device=DEV)
    rep.check("alpha", o["alpha"], R.alpha_ref(r.raw, r.z, r.d3, r.noise), ones, C_ALPHA)
    ref = R.composite_ref(o["alpha"], r.raw, r.z, white)
    for k in ("weights", "rgb", "acc", "depth"):
        rep.check(k + (" white" if white and k == "rgb" else ""), o[k], *ref[k], c_scan(S), floor=UNDERFLOW)
    dk, (dr, dM) = o["disp"].to(F64), ref["disp"]
    assert torch.equal(dk.isnan(), dr.isnan()), "disp: NaN where acc = depth = 0, and only there"
    f = ~dr.isnan()
    rep.check("disp", dk[f], dr[f], dM[f], 2 * c_scan(S))


@pytest.mark.parametrize("n", N_SET)
@pytest.mark.parametrize("S", S_SET)
def test_composite_forward(S, n):
    for ch in (4, 5):
        for noise in (False, True):
            r = Rays(n, S, ch, noise)
            rep = Report(f"composite n={n} S={S} ch={ch} noise={int(noise)}")
            o8 = composite(r, r.d8)
            check_composite(rep, r, o8, False)
            o3 = composite(r, r.d3)
            for k in o8:
                assert same_bits(o8[k], o3[k]), f"{k}: rays_d with row stride 3 and 8 differ"
            ow = composite(r, r.d8, white=True)
            check_composite(rep, r, ow, True)
            for k in ("weights", "alpha", "acc", "depth", "disp"):
                assert same_bits(ow[k], o8[k]), k
            if n >= 2:
                assert bool((o8["alpha"][1] == 0).all()) and math.isnan(float(o8["disp"][1])), "zero-density ray"
            if n >= 3 and S >= 3:
                assert float(o8["acc"][2]) > 0.999 and bool((o8["weights"][2, 3:] < 1e-9).all()), "ray saturating early"


# ----------------------------------------------------------------------------------------------------------------------
# 2. fused resampling
# ----------------------------------------------------------------------------------------------------------------------
def make_u(kind, n, n_imp, seed):
    if kind == "none":
        return None
    g = torch.Generator().manual_seed(seed)
    u = torch.rand(n, n_imp, generator=g)
    if kind == "edges":
        u[::2, 0], u[1::2, -1] = 0.0, 1.0
        u[:, n_imp // 2] = torch.tensor([0.0, 1.0]).repeat(n)[:n]
    return u.to(DEV)


@pytest.mark.parametrize("u_kind", ["none", "rand", "edges"])
@pytest.mark.parametrize("n_imp", [1, 31, 64, 128])
@pytest.mark.parametrize("S", [64, 1000])
def test_fused_resampling(S, n_imp, u_kind):
    n = 37
    r = Rays(n, S, 5, noise=False)
    raw = r.raw.clone()
    raw[3, :, 3] = -1.0                       # all-zero weights: a uniform CDF
    raw[4, :, 3] = -1.0
    raw[4, S // 3, 3] = 1e6                   # a delta weight: every new sample in one or two bins
    u = make_u(u_kind, n, n_imp, S + n_imp)
    o = composite(r, r.d8, n_imp=n_imp, u=u, raw=raw)
    assert all_poison(o["z_out_pad"][n:]), "z_vals_out written past the last ray"
    bins = 0.5 * (r.z[:, 1:] + r.z[:, :-1])
    samples = sample_pdf(bins, o["weights"][:, 1:-1].contiguous(), u, n_imp)
    merged = torch.sort(torch.cat([r.z, samples], -1), -1)[0]
    assert same_bits(o["z_out"], merged), (
        f"z_vals_out != sort(cat(z, sample_pdf)): {int((bits(o['z_out']) != bits(merged)).sum())} slots differ")
    s64 = samples.to(F64)
    mean = s64.mean(-1, keepdim=True)
    std = ((s64 - mean) ** 2).mean(-1).sqrt()
    # sum (x - m~)^2 = sum (x - m)^2 + n (m - m~)^2: an fp32 mean m~ off by delta moves std by at most delta
    Report(f"resample S={S} n_imp={n_imp} u={u_kind}").check("z_std", o["z_std"], std, std + mean[:, 0].abs(), C_STD)


# ----------------------------------------------------------------------------------------------------------------------
# 3. stand-alone sample_pdf
# ----------------------------------------------------------------------------------------------------------------------
def check_pdf(tag, bins, w, u, n_samp):
    got = sample_pdf(bins, w, u, n_samp)
    uu = det_u(bins.shape[0], n_samp) if u is None else u
    ok, ratio = R.sample_pdf_accepts(bins, w, uu, got, pdf_k(bins.shape[1]), C_PDF)
    obs = float(ratio.max())
    print(f"  [{tag}] {'samples':<24s} c_obs {obs:10.3f}   c {C_PDF}")
    assert torch.isfinite(got).all(), tag
    assert bool(ok.all()), f"{tag}: {int((~ok).sum())} samples off the fp64 inverse CDF, worst c_obs {obs:.4g}"


@pytest.mark.parametrize("nb", [3, 33, 64, 1000, 4000])
def test_sample_pdf(nb):
    n, n_samp = 24, 64
    g = torch.Generator().manual_seed(nb)
    bins = torch.sort(2.0 + 4.0 * torch.rand(n, nb, generator=g), -1)[0]
    w = torch.rand(n, nb - 1, generator=g)
    w[0:4] = 0.0                                        # uniform CDF
    w[4:8] = 0.0
    for i in range(4, 8):
        w[i, (7 * i) % (nb - 1)] = 1.0                  # delta
    w[8:16] = 0.0                                       # flat spots of 1e-5 / 5: below the 1e-5 threshold, above 1e-6
    for i in range(8, 16):
        for j in range(3):
            w[i, (5 * i + 11 * j) % (nb - 1)] += 5.0 / 3
    u = torch.rand(n, n_samp, generator=g)
    u[:, 0], u[:, 1] = 0.0, 1.0
    cdf = R.cdf_ref(w)
    for i in range(8, 16):                             # u in the middle of flat CDF steps
        flat = (w[i] == 0).nonzero()[:, 0]
        pick = flat[torch.randperm(len(flat), generator=g)[:n_samp // 2]]
        u[i, 2:2 + len(pick)] = (0.5 * (cdf[i, pick] + cdf[i, pick + 1])).float()
    bins, w, u = bins.to(DEV), w.to(DEV), u.to(DEV)
    check_pdf(f"sample_pdf nb={nb} u", bins, w, u, n_samp)
    check_pdf(f"sample_pdf nb={nb} det", bins, w, None, n_samp)
    check_pdf(f"sample_pdf nb={nb} det 1", bins, w, None, 1)


def test_sample_pdf_golden_case_e():
    g = np.load("tests/golden/caseE_ops.npz")
    bins, w = torch.from_numpy(g["bins"]).to(DEV), torch.from_numpy(g["weights"]).to(DEV)
    check_pdf("sample_pdf case E rand", bins, w, torch.from_numpy(g["u_rand"]).to(DEV), 64)
    check_pdf("sample_pdf case E det", bins, w, None, 64)


# ----------------------------------------------------------------------------------------------------------------------
# 4. composite backward
# ----------------------------------------------------------------------------------------------------------------------
def composite_backward(r, d, white, d_rgb, d_acc):
    L, lib = _lib()
    a = L.NrnCompositeBwdArgs()
    a.raw, a.z_vals, a.rays_d, a.rays_d_stride = r.raw.data_ptr(), r.z.data_ptr(), d.data_ptr(), d.stride(0)
    a.noise = ptr(r.noise)
    a.n_rays, a.n_samples, a.channels, a.white_bkgd = r.n, r.S, r.ch, int(white)
    a.d_rgb_map, a.d_acc_map = d_rgb.data_ptr(), ptr(d_acc)
    out = poison_f32(r.n, r.S, r.ch)
    a.d_raw = out.data_ptr()
    a.stream = _stream()
    L.check(lib.nrn_composite_backward(C.byref(a)), "composite_backward")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("n", N_SET)
@pytest.mark.parametrize("S", S_SET + [4000])
def test_composite_backward(S, n):
    g = torch.Generator().manual_seed(77 + S + n)
    d_rgb = torch.randn(n, 3, generator=g).to(DEV)
    d_acc = torch.randn(n, generator=g).to(DEV)
    for ch, noise, white, acc in ((5, False, False, False), (5, True, True, True), (4, True, False, True), (4, False, True, False)):
        r = Rays(n, S, ch, noise, seed=1)
        alpha = kernel_alpha(r, r.d8)
        rep = Report(f"composite_bwd n={n} S={S} ch={ch} noise={int(noise)} white={int(white)} d_acc={int(acc)}")
        da = d_acc if acc else None
        got = composite_backward(r, r.d8, white, d_rgb, da)
        ref, M = R.composite_backward_ref(alpha, r.raw, r.z, r.d3, r.noise, white, d_rgb, da)
        rep.check("d_raw", got[..., :4], ref, M, c_bwd(S), floor=BWD_UNDERFLOW)
        assert bool((got[..., 4:] == 0).all()), "d_raw channels >= 4 must be 0"
        assert same_bits(got, composite_backward(r, r.d3, white, d_rgb, da)), "rays_d with row stride 3 and 8 differ"


# ----------------------------------------------------------------------------------------------------------------------
# 5. sample_coarse
# ----------------------------------------------------------------------------------------------------------------------
def coarse_ref(rays, S, t_rand, lindisp):
    """train.py:847-869 evaluated by torch on CUDA in fp32, one rounding per operation"""
    t = torch.linspace(0.0, 1.0, S, device=DEV)
    near, far = rays[:, 6:7], rays[:, 7:8]
    z = near * (1.0 - t) + far * t if not lindisp else 1.0 / (1.0 / near * (1.0 - t) + 1.0 / far * t)
    z = z.expand(rays.shape[0], S)
    if t_rand is not None:
        mids = 0.5 * (z[:, 1:] + z[:, :-1])
        upper = torch.cat([mids, z[:, -1:]], -1)
        lower = torch.cat([z[:, :1], mids], -1)
        z = lower + (upper - lower) * t_rand
    return z


@pytest.mark.parametrize("lindisp", [False, True])
@pytest.mark.parametrize("S", [1, 2, 3, 63, 64, 65, 200])
def test_sample_coarse(S, lindisp):
    L, lib = _lib()
    n = 37
    g = torch.Generator().manual_seed(S)
    rays = torch.randn(n, 8, generator=g)
    rays[:, 6] = 0.5 + 1.5 * torch.rand(n, generator=g)
    rays[:, 7] = rays[:, 6] + 1.0 + 4.0 * torch.rand(n, generator=g)
    rays = rays.to(DEV)
    t_rand = torch.rand(n, S, generator=g)
    t_rand[:, 0], t_rand[:, -1] = 0.0, 1.0
    t_rand[::2, S // 2] = 1.0
    t_rand = t_rand.to(DEV)
    for tr in (None, t_rand):
        out = poison_f32(n, S)
        L.check(lib.nrn_sample_coarse(rays.data_ptr(), ptr(tr), n, S, int(lindisp), out.data_ptr(), _stream()), "sample_coarse")
        torch.cuda.synchronize()
        ref = coarse_ref(rays, S, tr, lindisp)
        diff = int((bits(out) != bits(ref)).sum())
        print(f"  [sample_coarse S={S} lindisp={int(lindisp)} t_rand={int(tr is not None)}] {diff} of {n * S} differ from torch")
        assert diff == 0


# ----------------------------------------------------------------------------------------------------------------------
# 6. ray loss, forward and backward
# ----------------------------------------------------------------------------------------------------------------------
N_ITERS = 200000.0
LOSS_VARIANTS = [  # rgb0, offsets (None / "rand" / "zero"), divergence, sched step
    (True, "rand", True, 0.0),
    (True, "zero", False, N_ITERS / 2),
    (False, "rand", False, N_ITERS),
    (True, None, True, N_ITERS / 2),
    (False, None, False, None),
]


@pytest.mark.parametrize("S", [7, 64, 192])
@pytest.mark.parametrize("n", [1, 67, 2048])
def test_ray_loss(n, S):
    L, lib = _lib()
    g = torch.Generator().manual_seed(n * 1000 + S)
    mk = lambda *sh: torch.randn(*sh, generator=g)
    rgb, rgb0, tgt = torch.sigmoid(mk(n, 3)), torch.sigmoid(mk(n, 3)), torch.sigmoid(mk(n, 3))
    w = torch.rand(n, S, generator=g)
    off = mk(n, S, 3) * 0.05
    off[0, : min(S, 3)] = 0.0
    rig = torch.sigmoid(mk(n, S))
    div = torch.rand(n, generator=g) * 0.1
    gray = mk(n) * 2
    lam_o, lam_r, lam_div = 60.0, 5e-4, 3.0
    T = {k: v.to(DEV).contiguous() for k, v in dict(rgb=rgb, rgb0=rgb0, tgt=tgt, w=w, off=off, rig=rig, div=div, g=gray).items()}
    T["zero"] = torch.zeros(n, S, 3, device=DEV)
    for use_rgb0, offs, use_div, step in LOSS_VARIANTS:
        tag = f"ray_loss n={n} S={S} rgb0={int(use_rgb0)} off={offs} div={int(use_div)} step={step}"
        rep = Report(tag)
        a = L.NrnRayLossArgs()
        s_eff = S if offs else 1
        a.n_rays, a.n_samples = n, s_eff
        a.rgb, a.target = T["rgb"].data_ptr(), T["tgt"].data_ptr()
        o = {"loss": poison_f32(n), "u_rgb": poison_f32(n, 3)}
        if use_rgb0:
            o["u_rgb0"] = poison_f32(n, 3)
            a.rgb0, a.u_rgb0 = T["rgb0"].data_ptr(), o["u_rgb0"].data_ptr()
        off_t = {"rand": T["off"], "zero": T["zero"], None: None}[offs]
        if offs:
            o["u_off"], o["u_rig"] = poison_f32(n, S, 3), poison_f32(n, S)
            a.weights, a.unmasked_offsets, a.rigidity_mask = T["w"].data_ptr(), off_t.data_ptr(), T["rig"].data_ptr()
            a.u_unmasked_offsets, a.u_rigidity_mask = o["u_off"].data_ptr(), o["u_rig"].data_ptr()
        a.lam_offsets, a.lam_rigidity = lam_o, lam_r
        sched = 1.0
        if step is not None:
            st = torch.full((), step, dtype=torch.float32, device=DEV)
            a.sched_step, a.sched_n_iters = st.data_ptr(), N_ITERS
            sched = 0.01 ** (1.0 - step / N_ITERS)
        if use_div:
            o["u_div"] = poison_f32(n)
            a.divergence, a.lam_divergence, a.u_divergence = T["div"].data_ptr(), lam_div, o["u_div"].data_ptr()
        a.loss, a.u_rgb = o["loss"].data_ptr(), o["u_rgb"].data_ptr()
        a.stream = _stream()
        L.check(lib.nrn_ray_loss(C.byref(a)), "ray_loss")
        torch.cuda.synchronize()
        ref = R.ray_loss_ref(T["rgb"], T["rgb0"] if use_rgb0 else None, T["tgt"], T["w"] if offs else None, off_t,
                             T["rig"] if offs else None, lam_o, lam_r, sched, T["div"] if use_div else None, lam_div)
        for k in o:
            c = c_loss(S) if k == "loss" else (C_LOSS_RGB if k in ("u_rgb", "u_rgb0") else C_LOSS_GRAD)
            rep.check(k, o[k].reshape(ref[k][0].shape), *ref[k], c)
        # backward: d_k[i] = g[ray] * u_k[i], one fp32 product, so bit-exact with torch's
        b = L.NrnRayLossBwdArgs()
        b.n_rays, b.n_samples, b.g = n, s_eff, T["g"].data_ptr()
        d = {}
        for k, per in (("rgb", 3), ("rgb0", 3), ("unmasked_offsets", 3 * S), ("rigidity_mask", S), ("divergence", 1)):
            uk = {"rgb": "u_rgb", "rgb0": "u_rgb0", "unmasked_offsets": "u_off", "rigidity_mask": "u_rig", "divergence": "u_div"}[k]
            if uk in o:
                d[uk] = (poison_f32(*o[uk].shape), per)
                setattr(b, "u_" + k, o[uk].data_ptr())
                setattr(b, "d_" + k, d[uk][0].data_ptr())
        b.stream = _stream()
        L.check(lib.nrn_ray_loss_backward(C.byref(b)), "ray_loss_backward")
        torch.cuda.synchronize()
        for uk, (dk, per) in d.items():
            want = (T["g"][:, None] * o[uk].reshape(n, per)).reshape(dk.shape)
            assert same_bits(dk, want), f"{tag} backward {uk}: {int((bits(dk) != bits(want)).sum())} of {dk.numel()} differ"


# ----------------------------------------------------------------------------------------------------------------------
# 7. Adam
# ----------------------------------------------------------------------------------------------------------------------
def half_ulp32(x):
    """0.5 ulp of fp32 values x (float64 tensor)"""
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), torch.clamp(e - 1, min=-126) - 24)


def test_adam():
    L, lib = _lib()
    # size, steps taken before, gradient scale (None: no gradient this step)
    spec = [(1, 0, 1.0), (2047, 0, 1e-9), (2048, 3, 0.1), (3000, 2, None), (2049, 0, 1.0), (4097, 7, 1e-9), (5, 1, None)]
    b1, b2, eps = 0.9, 0.999, 1e-8
    b1f, b2f = float(np.float32(b1)), float(np.float32(b2))   # the ABI takes fp32 betas; the reference uses those values
    lr = 5e-4
    g = torch.Generator().manual_seed(123)
    sizes = [s for s, _, _ in spec]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    tot = int(offs[-1])
    p = torch.randn(tot, generator=g)
    m, v = torch.zeros(tot), torch.zeros(tot)
    for (sz, st, _), o in zip(spec, offs):
        if st:
            m[o:o + sz] = torch.randn(sz, generator=g) * 0.05
            v[o:o + sz] = torch.rand(sz, generator=g) * 1e-3
    grads = [None if sc is None else (torch.randn(sz, generator=g) * sc).to(DEV) for sz, _, sc in spec]
    blocks = [(i, s, min(2048, sz - s), int(o) + s) for i, ((sz, _, _), o) in enumerate(zip(spec, offs)) for s in range(0, sz, 2048)]
    P, Mm, V = p.to(DEV), m.to(DEV), v.to(DEV)
    p0, m0, v0 = P.clone(), Mm.clone(), V.clone()
    gp = torch.tensor([0 if x is None else x.data_ptr() for x in grads], dtype=torch.int64, device=DEV)
    bt = torch.tensor(blocks, dtype=torch.int32, device=DEV)
    steps = torch.tensor([st for _, st, _ in spec], dtype=torch.int64, device=DEV)
    lr_dev = torch.full((), lr, dtype=torch.float32, device=DEV)
    a = L.NrnAdamArgs()
    a.params, a.exp_avg, a.exp_avg_sq = P.data_ptr(), Mm.data_ptr(), V.data_ptr()
    a.grad_ptrs, a.blocks, a.n_tensors, a.n_blocks = gp.data_ptr(), bt.data_ptr(), len(spec), len(blocks)
    a.lr, a.step, a.beta1, a.beta2, a.eps = lr_dev.data_ptr(), steps.data_ptr(), b1, b2, eps
    a.stream = _stream()
    L.check(lib.nrn_adam_step(C.byref(a)), "adam_step")
    torch.cuda.synchronize()
    assert steps.tolist() == [st + (sc is not None) for _, st, sc in spec], "per-tensor step counts"
    for i, ((sz, st, sc), o) in enumerate(zip(spec, offs)):
        sl = slice(int(o), int(o) + sz)
        rep = Report(f"adam size={sz} step={st + 1 if sc is not None else st} g~{sc}")
        if sc is None:
            assert same_bits(P[sl], p0[sl]) and same_bits(Mm[sl], m0[sl]) and same_bits(V[sl], v0[sl]), "skipped tensor moved"
            continue
        upd, Mu, m_new, M_m, v_new, M_v = R.adam_ref(p0[sl], m0[sl], v0[sl], grads[i], st + 1, float(np.float32(lr)), b1f, b2f,
                                                    float(np.float32(eps)))
        got = P[sl].to(F64) - p0[sl].to(F64)
        rep.check("update", got, upd, Mu, C_ADAM_UPD, floor=half_ulp32(P[sl].to(F64)))
        rep.check("exp_avg", Mm[sl], m_new, M_m, C_ADAM_MOM)
        rep.check("exp_avg_sq", V[sl], v_new, M_v, C_ADAM_MOM)
