"""fp64 restatement of the inverse ray bender (geometry.deform_points, csrc/deform.cu) on oracle.bender_forward: the same
start x_0 = c - s r~(c) o(c, z), the same freezing rule (|b(x) - c|_2 <= tol), the same singular-J fallback and the same
last evaluation, with J from torch.func.jacfwd."""
import torch
import torch.nn.functional as F
from torch.func import jacfwd, vmap

import oracle.nrnerf_oracle as O

SINGULAR = 1e-6   # csrc/deform.cuh: kDeformSingular


def params64(bp, device=None):
    return {k: [t.to(device=device, dtype=torch.float64) for t in v] for k, v in bp.items()}


def bend(bp64, x, z, cutoff=None, scaling=None):
    """b(x; z) [N, 3], r~ [N] and s r~ o [N, 3] for x [N, 3], z [N, 32]."""
    out = O.bender_forward(bp64, x, z, cutoff, scaling)
    return out["bent"], out["rigidity_mask"][:, 0], out["masked_offsets"]


def jacobian(bp64, x, z, cutoff=None, scaling=None):
    """db/dx [N, 3, 3] (J[n, i, a] = d b_i / d x_a)."""
    def f(xi, zi):
        return O.bender_forward(bp64, xi[None], zi[None], cutoff, scaling)["bent"][0]
    return vmap(jacfwd(f, argnums=0))(x, z)


def kink_margin(bp64, x, z):
    """min over the bender's ReLU units of |pre-activation| at x [N, 3], z [N, 32]: J jumps where one of them crosses 0, so
    an fp32 and an fp64 evaluation within that distance of a kink may take different one-sided derivatives."""
    h, m = torch.cat([x, z], -1), []
    for i in range(4):
        h = F.linear(h, bp64["net_w"][i], bp64["net_b"][i])
        m.append(h.abs().min(1).values)
        h = F.relu(h)
    r = x
    for i in range(2):
        r = F.linear(r, bp64["rig_w"][i], bp64["rig_b"][i])
        m.append(r.abs().min(1).values)
        r = F.relu(r)
    return torch.stack(m, 1).min(1).values


def newton_step(J, g):
    """J^-1 g by Cramer's rule on J's columns, or g (the fixed-point step) where J is singular or the step is not finite."""
    j0, j1, j2 = J[..., 0], J[..., 1], J[..., 2]
    k = torch.stack([torch.cross(j1, j2, dim=-1), torch.cross(j2, j0, dim=-1), torch.cross(j0, j1, dim=-1)], -2)
    det = (j0 * k[..., 0, :]).sum(-1)
    had = j0.norm(dim=-1) * j1.norm(dim=-1) * j2.norm(dim=-1)
    st = (k @ g.unsqueeze(-1)).squeeze(-1) / det.unsqueeze(-1)
    ok = (det.abs() > SINGULAR * had) & torch.isfinite(st).all(-1)
    return torch.where(ok.unsqueeze(-1), st, g)


def deform(bp64, c, latents, iterations, tol, cutoff=None, scaling=None, with_margin=False):
    """x [F, P, 3], residual [F, P], converged [F, P] bool, rigidity [F, P] and the step at which each point froze
    (-1: never) [F, P], for canonical points c [P, 3] and latents [F, 32] (any device, fp64).  with_margin: also the
    smallest kink_margin [F, P] over the iterates at which J was taken (inf: none)."""
    c = c.to(torch.float64)
    latents = latents.to(torch.float64)
    F, P = latents.shape[0], c.shape[0]
    xs, rs, cs, rig, its, mg = [], [], [], [], [], []
    for f in range(F):
        z = latents[f].expand(P, latents.shape[1])
        bad = ~torch.isfinite(c).all(1) | ~torch.isfinite(latents[f]).all()
        cc = torch.where(bad.unsqueeze(1), torch.zeros_like(c), c)
        zz = torch.where(bad.unsqueeze(1), torch.zeros_like(z), z)
        _, _, m = bend(bp64, cc, zz, cutoff, scaling)
        x = cc - m
        frozen = torch.zeros(P, dtype=torch.bool, device=c.device)
        it_conv = torch.full((P,), -1, dtype=torch.int64, device=c.device)
        margin = torch.full((P,), float("inf"), dtype=torch.float64, device=c.device)
        for it in range(iterations + 1):
            b, r, _ = bend(bp64, x, zz, cutoff, scaling)
            g = b - cc
            res = g.norm(dim=1)
            it_conv = torch.where((res <= tol) & ~frozen, torch.full_like(it_conv, it), it_conv)
            frozen = frozen | (res <= tol)
            if it == iterations:
                break
            active = ~frozen & ~bad
            if not bool(active.any()):
                break
            idx = active.nonzero()[:, 0]
            J = jacobian(bp64, x[idx], zz[idx], cutoff, scaling)
            if with_margin:
                margin[idx] = torch.minimum(margin[idx], kink_margin(bp64, x[idx], zz[idx]))
            x = x.clone()
            x[idx] = x[idx] - newton_step(J, g[idx])
        nan = torch.full_like(res, float("nan"))
        xs.append(torch.where(bad.unsqueeze(1), nan.unsqueeze(1).expand(P, 3), x))
        rs.append(torch.where(bad, nan, res))
        cs.append((res <= tol) & ~bad)
        rig.append(torch.where(bad, nan, r))
        its.append(torch.where(bad, torch.full_like(it_conv, -1), it_conv))
        mg.append(margin)
    out = (torch.stack(xs), torch.stack(rs), torch.stack(cs), torch.stack(rig), torch.stack(its))
    return out + (torch.stack(mg),) if with_margin else out
