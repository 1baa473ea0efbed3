"""Checking helpers shared by the kernel-parity tests (test_stage_parity_gpu.py, test_ray_kernels_parity_gpu.py).

A kernel's output is compared per element with an fp64 reference of the same operation, fed with the kernel's own inputs:

    |kernel - exact| <= [0.5 ulp_fp16(kernel)] + c * 2^-24 * M

M is the reference expression evaluated on absolute values and c the depth of the fp32 evaluation.  Report.check prints
the worst observed ratio ("c_obs") with `pytest -s`.  poison_* allocate buffers filled with 0xFF (fp16 / fp32 NaN), so a
slot no kernel wrote shows up as a NaN in a checked value.
"""
import torch

DEV = "cuda:0"
U = 2.0 ** -24
F64 = torch.float64


def half_ulp(x):
    """0.5 ulp of fp16 values x (float64 tensor); subnormal spacing 2^-24 below 2^-14."""
    _, e = torch.frexp(x)
    u = torch.ldexp(torch.ones_like(x), torch.clamp(e - 1, min=-14) - 10)
    return torch.where(x == 0, torch.full_like(x, 2.0 ** -25), 0.5 * u)


class Report:
    """quiet: print nothing per check; worst() prints the largest c_obs / relative L2 of each stage seen so far."""
    def __init__(self, tag, quiet=False):
        self.tag, self.quiet = tag, quiet
        self.c_obs, self.l2 = {}, {}

    def worst(self):
        for stage, (obs, c) in self.c_obs.items():
            print(f"  [{self.tag}] {stage:<24s} worst c_obs {obs:10.3f}   c {c}")
        for stage, (d, tol) in self.l2.items():
            print(f"  [{self.tag}] {stage:<24s} worst rel L2 {d:.3e}   bound {tol:.0e}")

    def check(self, stage, got, exact, absb, c, fp16=False, floor=0.0):
        got = got.to(F64)
        assert got.shape == exact.shape == absb.shape, (stage, got.shape, exact.shape, absb.shape)
        bad = ~torch.isfinite(got)
        assert not bool(bad.any()), f"{self.tag} {stage}: {int(bad.sum())} non-finite values (first at {bad.nonzero()[0].tolist()})"
        err = (got - exact).abs()
        if fp16:
            err = (err - half_ulp(got)).clamp_min(0.0)
        if torch.is_tensor(floor) or floor:
            err = (err - floor).clamp_min(0.0)
        ratio = torch.where(err == 0, torch.zeros_like(err), err / (U * absb))
        obs = float(ratio.max()) if ratio.numel() else 0.0
        if obs >= self.c_obs.get(stage, (-1.0, c))[0]:
            self.c_obs[stage] = (obs, c)
        if not self.quiet:
            print(f"  [{self.tag}] {stage:<24s} c_obs {obs:10.3f}   c {c}")
        if not obs <= c:
            i = int(ratio.flatten().argmax())
            raise AssertionError(f"{self.tag} {stage}: |kernel - exact| exceeds the bound, c_obs {obs:.4g} > c {c}; worst element "
                                 f"{i}: kernel {float(got.flatten()[i]):.9g} exact {float(exact.flatten()[i]):.9g} "
                                 f"abs {float(absb.flatten()[i]):.4g}")
        return obs

    def rel_l2(self, stage, got, exact, tol):
        d = float((got.to(F64) - exact).norm() / (exact.norm() + 1e-300))
        if d >= self.l2.get(stage, (-1.0, tol))[0]:
            self.l2[stage] = (d, tol)
        if not self.quiet:
            print(f"  [{self.tag}] {stage:<24s} rel L2 {d:.3e}   bound {tol:.0e}")
        assert d <= tol, (self.tag, stage, d)


def poison_bytes(n, device=DEV):
    return torch.full((n,), 0xFF, dtype=torch.uint8, device=device)


def poison_f32(*shape, device=DEV):
    n = 1
    for s in shape:
        n *= s
    return poison_bytes(4 * n, device).view(torch.float32).view(*shape)


def ptr(t):
    return None if t is None else t.data_ptr()
