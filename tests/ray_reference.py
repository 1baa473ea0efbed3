"""fp64 restatements of the per-ray kernels (csrc/ray_ops.cu, csrc/loss.cu) and of torch.optim.Adam (csrc/adam.cu), for
test_ray_kernels_parity_gpu.py.  They run on any device; test_ray_reference_cpu.py checks them against the fp32 oracle.

Each function returns the exact value of the operation on the kernel's own fp32 inputs together with M, the same
expression evaluated on absolute values (with the sensitivity of exp / pow / log folded in where an fp32 rounding of an
argument is amplified).  A kernel is then held to |kernel - exact| <= c * 2^-24 * M per element (tests/parity.py).

Where 1 - alpha + 1e-10 is ill-conditioned (alpha -> 1) the compositing references take the kernel's own alpha: the
kernel's fp32 alpha is checked against raw -> alpha on its own, with an absolute bound.
"""
import torch

F64 = torch.float64


# ----------------------------------------------------------------------------------------------------------------------
# compositing (raw2outputs, train.py:724-789)
# ----------------------------------------------------------------------------------------------------------------------
def dists(z, rays_d):
    """z_{i+1} - z_i (1e10 after the last sample) times |d|, in fp64"""
    z, d = z.to(F64), rays_d.to(F64)
    dz = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], -1)
    return dz * d.norm(dim=-1, keepdim=True)


def sigma_of(raw, noise):
    s = raw[..., 3].to(F64)
    return s if noise is None else s + noise.to(F64)


def alpha_ref(raw, z, rays_d, noise=None):
    """alpha = 1 - exp(-relu(sigma) dist)"""
    return -torch.expm1(-torch.relu(sigma_of(raw, noise)) * dists(z, rays_d))


def transmittance(alpha):
    """om_i = 1 - alpha_i + 1e-10 and the exclusive product T_i = prod_{k<i} om_k"""
    om = 1.0 - alpha + 1e-10
    T = torch.cumprod(torch.cat([torch.ones_like(om[:, :1]), om[:, :-1]], -1), -1)
    return om, T


def composite_ref(alpha, raw, z, white_bkgd=False):
    """weights and maps from a given alpha (the kernel's).  Returns {name: (exact, M)}; all terms but z are >= 0."""
    alpha, raw, z = alpha.to(F64), raw.to(F64), z.to(F64)
    _, T = transmittance(alpha)
    w = alpha * T
    rgb = torch.sigmoid(raw[..., :3])
    rgb_map = (w[..., None] * rgb).sum(1)
    acc = w.sum(1)
    depth = (w * z).sum(1)
    out = {"weights": (w, w), "acc": (acc, acc), "depth": (depth, (w * z.abs()).sum(1))}
    if white_bkgd:
        bg = (1.0 - acc)[:, None]
        out["rgb"] = (rgb_map + bg, rgb_map + acc[:, None] + bg.abs() + (rgb_map + bg).abs())
    else:
        out["rgb"] = (rgb_map, rgb_map)
    disp = 1.0 / torch.maximum(torch.full_like(depth, 1e-10), depth / acc)   # NaN where acc = depth = 0, like torch.max
    out["disp"] = (disp, disp.abs())
    return out


def composite_backward_ref(alpha, raw, z, rays_d, noise, white_bkgd, d_rgb, d_acc=None):
    """dL/draw for L = <d_rgb, rgb_map> + <d_acc, acc>, by fp64 autograd of raw2outputs.  alpha enters with the given
    value (the kernel's) and the fp64 derivative of 1 - exp(-relu(sigma) dist).  Returns (d_raw[..., :4], M)."""
    raw64 = raw.to(F64).detach().requires_grad_(True)
    a64 = -torch.expm1(-torch.relu(sigma_of(raw64, noise)) * dists(z, rays_d))   # relu': 0 at sigma = 0, like the kernel
    a = a64 + (alpha.to(F64) - a64).detach()
    om, T = transmittance(a)
    w = a * T
    rgb = torch.sigmoid(raw64[..., :3])
    rgb_map = (w[..., None] * rgb).sum(1)
    acc = w.sum(1)
    if white_bkgd:
        rgb_map = rgb_map + (1.0 - acc)[:, None]
    g_rgb = d_rgb.to(F64)
    loss = (rgb_map * g_rgb).sum()
    g_acc = torch.zeros_like(acc) if d_acc is None else d_acc.to(F64)
    loss = loss + (acc * g_acc).sum()
    loss.backward()
    # M: dalpha_i = g_i T_i - (sum_{k>i} g_k w_k) / om_i with g_i = dL/dw_i, on absolute values; the exclusive suffix sum
    # is formed in the kernel as inclusive minus its own term, so |g_i w_i| is part of it
    with torch.no_grad():
        om, T, w, rgb = om.detach(), T.detach(), w.detach(), rgb.detach()
        g_white = -g_rgb.sum(-1, keepdim=True) if white_bkgd else torch.zeros_like(g_acc[:, None])
        Mg = (g_rgb.abs()[:, None, :] * rgb).sum(-1) + g_acc.abs()[:, None] + g_white.abs()
        Msuf = torch.flip(torch.cumsum(torch.flip(Mg * w, [1]), 1), [1])
        Mda = Mg * T + Msuf / om
        sig = sigma_of(raw, noise)
        x = torch.relu(sig) * dists(z, rays_d)
        dadsig = torch.where(sig > 0, dists(z, rays_d) * torch.exp(-x), torch.zeros_like(x))
        M = torch.empty(raw.shape[0], raw.shape[1], 4, dtype=F64, device=raw.device)
        M[..., :3] = w[..., None] * g_rgb.abs()[:, None, :] * rgb
        M[..., 3] = dadsig * Mda * (1.0 + x)          # exp(-x) of an fp32 argument x: relative error ~ x * 2^-24
    return raw64.grad[..., :4], M


# ----------------------------------------------------------------------------------------------------------------------
# inverse-CDF sampling (run_nerf_helpers.py:651-698)
# ----------------------------------------------------------------------------------------------------------------------
def cdf_ref(weights):
    w = weights.to(F64) + 1e-5
    pdf = w / w.sum(-1, keepdim=True)
    return torch.cat([torch.zeros_like(pdf[:, :1]), torch.cumsum(pdf, -1)], -1)


def sample_pdf_accepts(bins, weights, u, got, k, c):
    """Per-sample check of an fp32 inverse CDF `got` [N, n] against the fp64 one.  k bounds the fp32 CDF's error in units
    of 2^-24 (it depends on the summation order).  Where u lies within that bound of a CDF entry, or denom within it of
    1e-5, every branch the fp32 CDF could have taken is evaluated, and `got` must match one of them to
    c 2^-24 M, M = |out| + 3 |t (b_a - b_b)| + |b_a - b_b| k (1 + 2|t|) / denom (the last term: the CDF error carried
    through t).  Returns (accepted [N, n] bool, worst ratio of the closest branch)."""
    U = 2.0 ** -24
    bins, u, got = bins.to(F64), u.to(F64), got.to(F64)
    cdf = cdf_ref(weights)
    nb = cdf.shape[-1]
    E = k * U
    lo_min = torch.searchsorted(cdf + E, u.contiguous(), right=False)
    lo_max = torch.searchsorted(cdf - E, u.contiguous(), right=False)
    best = torch.full_like(u, float("inf"))
    for off in range(int((lo_max - lo_min).max()) + 1):
        lo = torch.minimum(lo_min + off, lo_max)
        below, above = (lo - 1).clamp_min(0), lo.clamp_max(nb - 1)
        cb, ca = cdf.gather(1, below), cdf.gather(1, above)
        bb, ba = bins.gather(1, below), bins.gather(1, above)
        d = ca - cb
        taken = d < 1e-5
        amb = ((d - 1e-5).abs() <= 2 * E + U * d) & (below != above)
        for flat in (taken, taken ^ amb):   # the branch taken; the other one where ambiguous
            denom = torch.where(flat, torch.ones_like(d), d)
            t = (u - cb) / denom
            out = bb + t * (ba - bb)
            M = out.abs() + 3 * (t * (ba - bb)).abs() + (ba - bb).abs() * k * (1 + 2 * t.abs()) / denom
            ratio = (got - out).abs() / (U * M)
            best = torch.minimum(best, torch.where(got == out, torch.zeros_like(ratio), ratio))
    return best <= c, best


# ----------------------------------------------------------------------------------------------------------------------
# per-ray training loss (csrc/loss.cu, train.py:208-242)
# ----------------------------------------------------------------------------------------------------------------------
def ray_loss_ref(rgb, rgb0, target, w=None, off=None, rig=None, lam_o=0.0, lam_r=0.0, sched=1.0, div=None, lam_div=0.0):
    """Loss per ray and its gradients per unit upstream gradient.  Returns {name: (exact, M)} for loss, u_rgb, u_rgb0,
    u_off, u_rig, u_div (those the inputs call for).  sched is the fp64 value of 0.01^(1 - step / N)."""
    o = {}
    t = target.to(F64)
    d1 = rgb.to(F64) - t
    loss, Mloss = (d1 * d1).sum(-1) / 3, (d1 * d1).sum(-1) / 3
    o["u_rgb"] = (d1 * (2.0 / 3.0), d1.abs() * (2.0 / 3.0))
    if rgb0 is not None:
        d0 = rgb0.to(F64) - t
        loss, Mloss = loss + (d0 * d0).sum(-1) / 3, Mloss + (d0 * d0).sum(-1) / 3
        o["u_rgb0"] = (d0 * (2.0 / 3.0), d0.abs() * (2.0 / 3.0))
    if off is not None:
        S = off.shape[1]
        w, off, r = w.to(F64), off.to(F64), rig.to(F64).reshape(w.shape)
        nrm = off.norm(dim=-1)
        pw = 2.0 - r
        pos = nrm > 0
        safe = torch.where(pos, nrm, torch.ones_like(nrm))
        f = torch.where(pos, safe ** pw, torch.where(pw == 0, torch.ones_like(nrm), torch.zeros_like(nrm)))
        ln = torch.where(pos, torch.log(safe), torch.zeros_like(nrm))
        L = 1.0 + ln.abs() * (1.0 + pw)                  # relative sensitivity of nrm^pw to fp32 roundings of nrm and pw
        lam = lam_o * sched
        loss = loss + lam * (w * (f + lam_r * r)).sum(-1) / S
        Mloss = Mloss + lam * (w * (f * L + lam_r * r)).sum(-1) / S
        cw = lam * w / S
        k = torch.where(pos, cw * pw * f / (safe * safe), torch.zeros_like(nrm))
        o["u_off"] = (k[..., None] * off, (k[..., None] * off).abs() * L[..., None])
        dr = -f * ln
        o["u_rig"] = (cw * (dr + lam_r), cw * (dr.abs() * L + f + lam_r))
    if div is not None:
        c = lam_div * sched
        loss = loss + c * div.to(F64)
        Mloss = Mloss + abs(c) * div.to(F64).abs()
        o["u_div"] = (torch.full_like(loss, c), torch.full_like(loss, abs(c)))
    o["loss"] = (loss, Mloss)
    return o


# ----------------------------------------------------------------------------------------------------------------------
# Adam (torch.optim.Adam, amsgrad=False, weight_decay=0)
# ----------------------------------------------------------------------------------------------------------------------
def adam_ref(p, m, v, g, step, lr, beta1, beta2, eps):
    """One update of one tensor after its step count became `step`.  Returns (update = p_new - p, |update|-bound M,
    m_new, M_m, v_new, M_v): p_new = p - lr / (1 - b1^t) * m_new / (sqrt(v_new) / sqrt(1 - b2^t) + eps)."""
    p, m, v, g = (x.to(F64) for x in (p, m, v, g))
    m_new = m + (g - m) * (1.0 - beta1)
    v_new = beta2 * v + (1.0 - beta2) * g * g
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    upd = -(lr / bc1) * m_new / (v_new.sqrt() / bc2 ** 0.5 + eps)
    return upd, upd.abs(), m_new, m.abs() + (g - m).abs() * (1.0 - beta1), v_new, v_new
