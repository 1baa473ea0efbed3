"""fp64 restatement of the density gradient (geometry.density_gradient, csrc/field_grad.cu): g = d raw[..., 3] / d x of
NeRF.forward in point mode, by torch.func.grad through the oracle's nerf_mlp and bender_forward, with the parameters of
the package's modules (optionally rounded to fp16 first, as the kernels' weight images are)."""
import torch
from torch.func import grad, vmap

import oracle.nrnerf_oracle as O
from tests.parity import half_ulp


def _t(p, fp16, device):
    p = p.detach().to(device)
    if fp16:
        p = p.half()
    return p.double()


def _w_pts(w, l, fp16, device):
    """A trunk weight as the kernels apply it: fp16 in the weight images, except the latent columns 63..94 of a
    time-conditioned L0 / L5, which fold into fp32 ray biases."""
    w64 = _t(w, fp16, device)
    if fp16 and l in (0, 5) and w.shape[1] in (95, 95 + 256):
        w64[:, 63:95] = _t(w[:, 63:95], False, device)
    return w64


def params(net, fp16=False, device="cpu"):
    """(npar, bp) fp64 dicts of a NeRF module and its bender (None without one).  A view-dependent model's head is
    [0, 0, 0, alpha_linear] (its density is the trunk's alpha).  fp16: the weights rounded as the kernels' weight images
    round them; biases stay fp32, as the kernels keep them."""
    npar = {"pts_w": [_w_pts(l.weight, i, fp16, device) for i, l in enumerate(net.pts_linears)],
            "pts_b": [_t(l.bias, False, device) for l in net.pts_linears]}
    if getattr(net, "use_viewdirs", False):
        w, b = _t(net.alpha_linear.weight, fp16, device), _t(net.alpha_linear.bias, False, device)
        npar["out_w"] = torch.cat([torch.zeros(3, w.shape[1], dtype=w.dtype, device=device), w], 0)
        npar["out_b"] = torch.cat([torch.zeros(3, dtype=b.dtype, device=device), b], 0)
    else:
        npar["out_w"], npar["out_b"] = _t(net.output_linear.weight, fp16, device), _t(net.output_linear.bias, False, device)
    bender = net.ray_bender[0]
    bp = None
    if bender is not None:
        bp = {"net_w": [_t(l.weight, fp16, device) for l in bender.network],
              "net_b": [_t(l.bias, False, device) for l in list(bender.network)[:4]],
              "rig_w": [_t(l.weight, fp16, device) for l in bender.rigidity_network],
              "rig_b": [_t(l.bias, False, device) for l in bender.rigidity_network]}
    return npar, bp


def raw3(npar, bp, x, z=None, tc=False, cutoff=None, scaling=None, removal=None):
    """raw[..., 3] of NeRF.forward in point mode at x [P, 3] (fp64) with latents z [P, 32] (bender or time-conditioned)."""
    rig = None
    if bp is not None and z is not None:
        out = O.bender_forward(bp, x, z, cutoff, scaling)
        x, rig = out["bent"], out["rigidity_mask"][:, 0]
    emb = O.positional_encoding(x)
    if tc:
        emb = torch.cat([emb, z], -1)
    r = O.nerf_mlp(npar, emb)[:, 3]
    if removal is not None and rig is not None:
        r = torch.where(rig >= removal, r * 0.0, r)
    return r


def density_gradient(npar, bp, x, z=None, tc=False, cutoff=None, scaling=None, removal=None):
    """g [P, 3] fp64 at x [P, 3]."""
    x = x.double()
    z = None if z is None else z.double().expand(x.shape[0], -1)

    def f(xi, zi):
        return raw3(npar, bp, xi[None], None if zi is None else zi[None], tc, cutoff, scaling, removal)[0]

    if z is None:
        return vmap(grad(lambda xi: f(xi, None)))(x)
    return vmap(grad(f), in_dims=(0, 0))(x, z)


def central_differences(npar, bp, x, z=None, tc=False, h=1e-6, **knobs):
    x = x.double()
    z = None if z is None else z.double().expand(x.shape[0], -1)
    cols = []
    for d in range(3):
        e = torch.zeros_like(x)
        e[:, d] = h
        cols.append((raw3(npar, bp, x + e, z, tc, **knobs) - raw3(npar, bp, x - e, z, tc, **knobs)) / (2 * h))
    return torch.stack(cols, 1)


def normals(g):
    """n = -g / |g|, 0 where |g| = 0 or g is not finite."""
    norm = g.norm(dim=-1, keepdim=True)
    ok = torch.isfinite(norm) & (norm > 0)
    return torch.where(ok, -g / torch.where(ok, norm, torch.ones_like(norm)), torch.zeros_like(g))


# fp16 rounding stages of the kernels' chain (field_grad.cu): the trunk gradients dY7 .. dY0 (8), and with a bender the
# A operands d unmasked, the rigidity pre-activation gradient, dYb3, dYb2, dYb1, dYb0 (6).  U16: fp16's unit roundoff;
# ACC: fp32 accumulation over K <= 256 terms, relative to the sum of the terms' magnitudes.
U16 = 2.0 ** -11
ACC = 256 * 2.0 ** -24


def fixed_mask_chain(npar, bp, masks, E, unmasked=None, rigidity=None, cutoff=None, scaling=None, removal=None, eps=None, capture=None):
    """d raw[3] / d x [P, 3] in fp64 along the kernels' own path: the ReLU masks `masks` (dict "H1".."H8", "Hb1".."Hb4" ->
    bool [P, cols]), the encoding E [P, 64] and, with a bender, unmasked [P, 3] and rigidity [P] (after the cutoff) as the
    forward kernel wrote them, and the weights of npar / bp.  eps: additive perturbations of the fp16 stages (by name);
    capture: a dict that receives each stage's value y and the magnitude |y_prev| |W| of its fp32 sum."""
    def st(name, y, mag):
        if capture is not None:
            capture[name] = (y.detach(), mag.detach())
        return y + eps[name] if eps is not None and name in eps else y

    W = npar["pts_w"]
    P = E.shape[0]
    m = {k: v.double() for k, v in masks.items()}
    E = E.double()
    if eps is not None and "E" in eps:
        E = E + eps["E"]
    in_ch = W[0].shape[1]
    w3 = npar["out_w"][3].expand(P, -1)
    dY = st("Y7", w3 * m["H8"], w3.abs() * m["H8"])
    demb = torch.zeros(P, 63, dtype=torch.float64, device=E.device)
    for L in (7, 6, 5, 4, 3, 2, 1):
        Wh = W[5][:, in_ch:] if L == 5 else W[L]
        if L == 5:
            demb = demb + dY @ W[5][:, :63]
        dY = st(f"Y{L - 1}", (dY @ Wh) * m[f"H{L}"], (dY.abs() @ Wh.abs()) * m[f"H{L}"])
    demb = demb + dY @ W[0][:, :63]
    dx = demb[:, :3].clone()
    for k in range(10):
        s, c = E[:, 3 + 6 * k:6 + 6 * k], E[:, 6 + 6 * k:9 + 6 * k]
        ds, dc = demb[:, 3 + 6 * k:6 + 6 * k], demb[:, 6 + 6 * k:9 + 6 * k]
        dx = dx + 2.0 ** k * (ds * c - dc * s)
    if bp is None:
        return dx
    un, rig = unmasked.double(), rigidity.double()
    dm = dx * (scaling if scaling is not None else 1.0)
    dun = st("Yb4", rig[:, None] * dm, torch.zeros_like(dm))
    drpre = (un * dm).sum(1) * (2.0 * rig * (1.0 - rig))
    if cutoff is not None:
        drpre = torch.where(rig <= cutoff, torch.zeros_like(drpre), drpre)
    drpre = st("R", drpre, torch.zeros_like(drpre))
    nw, rw = bp["net_w"], bp["rig_w"]
    dyb3 = st("Yb3", (dun @ nw[4]) * m["Hb4"], (dun.abs() @ nw[4].abs()) * m["Hb4"])
    dyb2 = st("Yb2", (dyb3 @ nw[3]) * m["Hb3"], (dyb3.abs() @ nw[3].abs()) * m["Hb3"])
    dyb1 = st("Yb1", torch.cat([dyb2 @ nw[2], drpre[:, None] * rw[2]], 1) * m["Hb2"],
              torch.cat([dyb2.abs() @ nw[2].abs(), drpre.abs()[:, None] * rw[2].abs()], 1) * m["Hb2"])
    dyb0 = st("Yb0", torch.cat([dyb1[:, :64] @ nw[1], dyb1[:, 64:] @ rw[1]], 1) * m["Hb1"],
              torch.cat([dyb1[:, :64].abs() @ nw[1].abs(), dyb1[:, 64:].abs() @ rw[1].abs()], 1) * m["Hb1"])
    g = dx + dyb0[:, :64] @ nw[0][:, :3] + dyb0[:, 64:] @ rw[0]
    if removal is not None:
        g = torch.where((rig >= removal)[:, None], torch.zeros_like(g), g)
    return g


# The encoding E's sin / cos (columns 3..62) as pe_backward reads them: fp16 of the fp32 MUFU value, within half an fp16
# ulp plus E_PE of the exact sin / cos of the fp32 point (stage_reference.check_forward's PE bound)
E_PE = 1e-6


def rounding_bound(npar, bp, masks, E, unmasked=None, rigidity=None, e_term=False, **knobs):
    """(g64, bound, sigma) [P, 3]: sigma is the standard deviation of the same first-order error when each rounding is an
    independent uniform error of at most U16 relative (variance U16^2 y^2 / 3), the scale of a typical error; fixed_mask_chain and, per component, the first-order effect of the kernels' roundings,
    sum over stages s and elements j of |d g_i / d y_sj| (U16 |y_sj| + ACC |y_prev| |W|_sj), with the derivatives of the
    chain's own (signed) linear map, taken by autograd through additive perturbations at every stage.  e_term: the bound
    also carries the stashed encoding's own error, sum_j |d g_i / d E_j| (half_ulp(E_j) + E_PE) over the sin / cos
    columns, for a comparison against a chain fed the exact encoding."""
    cap = {}
    g = fixed_mask_chain(npar, bp, masks, E, unmasked, rigidity, capture=cap, **knobs)
    eps = {k: torch.zeros_like(y, requires_grad=True) for k, (y, _) in cap.items()}
    if e_term:
        E = E.double()
        eps["E"] = torch.zeros_like(E, requires_grad=True)
        cap["E"] = (E, None)
    with torch.enable_grad():
        gp = fixed_mask_chain(npar, bp, masks, E, unmasked, rigidity, eps=eps, **knobs)
        bound, var = torch.zeros_like(g), torch.zeros_like(g)
        names = list(eps)
        for i in range(3):
            jac = torch.autograd.grad(gp[:, i].sum(), [eps[k] for k in names], retain_graph=True, allow_unused=True)
            for k, J in zip(names, jac):
                if J is None:
                    continue
                y, mag = cap[k]
                if k == "E":
                    bound[:, i] += (J[:, 3:63].abs() * (half_ulp(y[:, 3:63]) + E_PE)).sum(1)
                    continue
                J = J if J.dim() == y.dim() else J[:, None]
                yy, mm = (y, mag) if y.dim() == 2 else (y[:, None], mag[:, None])
                bound[:, i] += (J.abs() * (U16 * yy.abs() + ACC * mm)).sum(1)
                var[:, i] += ((J * U16 * yy) ** 2).sum(1) / 3.0
    return g, bound, var.sqrt()
