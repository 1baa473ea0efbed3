"""The fp64 references of tests/ray_reference.py against the fp32 oracle (golden case E and seeded inputs), so that a wrong
reference cannot make the GPU parity checks of test_ray_kernels_parity_gpu.py pass vacuously.  No GPU needed."""
import os

import numpy as np
import torch

import oracle.nrnerf_oracle as O
from tests import ray_reference as R

GOLD = os.path.join(os.path.dirname(__file__), "golden", "caseE_ops.npz")
F64 = torch.float64


def _case_e():
    g = np.load(GOLD)
    return {k: torch.from_numpy(g[k]) for k in g.files}


def _close(a, b, rtol, atol, name):
    np.testing.assert_allclose(a.detach().to(F64).numpy(), b.detach().to(F64).numpy(), rtol=rtol, atol=atol, equal_nan=True,
                               err_msg=name)


def test_composite_references_match_the_oracle_on_case_e():
    g = _case_e()
    raw, z, rd = g["raw"], g["z"], g["rays_d"]
    alpha = R.alpha_ref(raw, z, rd)
    _close(alpha, g["alpha"], 0, 1e-6, "alpha")
    for white, key in ((False, "rgb_map"), (True, "rgb_map_white")):
        ref = R.composite_ref(g["alpha"], raw, z, white)     # the oracle's own fp32 alpha, as the GPU test uses the kernel's
        _close(ref["rgb"][0], g[key], 1e-5, 1e-6, key)
        for k, gk in (("weights", "weights_out"), ("acc", "acc_map"), ("depth", "depth_map"), ("disp", "disp_map")):
            _close(ref[k][0], g[gk], 1e-5, 1e-6, k)
            assert bool(((ref[k][1] >= ref[k][0].abs()) | ref[k][0].isnan()).all()), k
    assert np.isnan(g["disp_map"][3]) and bool(torch.isnan(R.composite_ref(g["alpha"], raw, z)["disp"][0][3]))


def test_composite_backward_reference_matches_oracle_autograd():
    rs = np.random.RandomState(11)
    n, s = 9, 70
    raw = torch.from_numpy(rs.randn(n, s, 5).astype(np.float32) * 2)
    z = torch.from_numpy(np.sort(rs.uniform(0.1, 2.0, size=(n, s)).astype(np.float32), -1))
    rd = torch.from_numpy(rs.randn(n, 3).astype(np.float32))
    noise = torch.from_numpy(rs.randn(n, s).astype(np.float32))
    g_rgb = torch.from_numpy(rs.randn(n, 3).astype(np.float32))
    g_acc = torch.from_numpy(rs.randn(n).astype(np.float32))
    for white in (False, True):
        r64 = raw.to(F64).requires_grad_(True)
        rgb, _, acc, alpha, _, _ = O.raw2outputs(r64, z.to(F64), rd.to(F64), noise.to(F64), white)
        ((rgb * g_rgb.to(F64)).sum() + (acc * g_acc.to(F64)).sum()).backward()
        ref, M = R.composite_backward_ref(alpha.detach(), raw, z, rd, noise, white, g_rgb, g_acc)
        _close(ref, r64.grad[..., :4], 1e-9, 1e-12, f"d_raw white={white}")
        assert bool((M >= ref.abs() * (1 - 1e-12)).all())
        # the fp32 oracle, as a check of the conventions (white background, d_acc, the noise mask)
        r32 = raw.clone().requires_grad_(True)
        rgb, _, acc, _, _, _ = O.raw2outputs(r32, z, rd, noise, white)
        ((rgb * g_rgb).sum() + (acc * g_acc).sum()).backward()
        _close(ref, r32.grad[..., :4], 2e-4, 2e-6, f"d_raw vs fp32 white={white}")


def test_sample_pdf_reference_accepts_the_oracle_and_rejects_a_shift():
    g = _case_e()
    bins, w = g["bins"], g["weights"]
    nw = w.shape[1]
    for u, key in ((O.det_u(bins.shape[0], 64), "samples_det"), (g["u_rand"], "samples_rand")):
        ours = O.sample_pdf(bins, w, u)
        _close(ours, g[key], 0, 1e-6, key)
        # the oracle sums its CDF sequentially: error depth nw, not the kernel's parallel scan
        ok, ratio = R.sample_pdf_accepts(bins, w, u, ours, k=2 * nw + 16, c=8)
        assert bool(ok.all()), (key, float(ratio.max()))
        width = (bins[:, -1] - bins[:, 0])[:, None]
        ok, _ = R.sample_pdf_accepts(bins, w, u, ours + 1e-3 * width, k=2 * nw + 16, c=8)
        assert float(ok.float().mean()) < 0.05, key


def test_ray_loss_reference_matches_the_oracle():
    rs = np.random.RandomState(21)
    n, s = 13, 40
    mk = lambda *sh: torch.from_numpy(rs.randn(*sh).astype(np.float32))
    rgb, rgb0, tgt = torch.sigmoid(mk(n, 3)), torch.sigmoid(mk(n, 3)), torch.sigmoid(mk(n, 3))
    w = torch.from_numpy(rs.uniform(0, 1, size=(n, s)).astype(np.float32))
    off = mk(n, s, 3) * 0.05
    off[0, :5] = 0.0
    rig = torch.sigmoid(mk(n, s, 1))
    a = [t.to(F64).requires_grad_(True) for t in (rgb, rgb0, off, rig)]
    ret = {"rgb_map": a[0], "rgb0": a[1], "visibility_weights": w.to(F64), "unmasked_offsets": a[2], "rigidity_mask": a[3]}
    loss = O.training_loss(ret, tgt.to(F64), 60.0, 5e-4, 0.07)
    loss.sum().backward()
    ref = R.ray_loss_ref(rgb, rgb0, tgt, w, off, rig, 60.0, 5e-4, 0.07)
    _close(ref["loss"][0], loss, 1e-12, 0, "loss")
    for k, t in (("u_rgb", a[0]), ("u_rgb0", a[1]), ("u_off", a[2]), ("u_rig", a[3])):
        _close(ref[k][0], t.grad.reshape(ref[k][0].shape), 1e-12, 1e-300, k)
        assert bool((ref[k][1] >= ref[k][0].abs() * (1 - 1e-12)).all()), k


def test_adam_reference_matches_torch_adam():
    gen = torch.Generator().manual_seed(7)
    p0 = torch.randn(300, generator=gen, dtype=F64)
    for steps, gscale in ((1, 1.0), (4, 1e-9)):
        p = p0.clone().requires_grad_(True)
        opt = torch.optim.Adam([p], lr=5e-4, betas=(0.9, 0.999), eps=1e-8)
        for _ in range(steps):
            g = torch.randn(300, generator=gen, dtype=F64) * gscale
            st = opt.state.get(p)
            m = st["exp_avg"].clone() if st else torch.zeros_like(p0)
            v = st["exp_avg_sq"].clone() if st else torch.zeros_like(p0)
            before = p.detach().clone()
            t = int(st["step"]) + 1 if st else 1
            p.grad = g
            opt.step()
            upd, _, m_new, _, v_new, _ = R.adam_ref(before, m, v, g, t, 5e-4, 0.9, 0.999, 1e-8)
            _close(before + upd, p.detach(), 1e-13, 1e-15, "p")
            _close(m_new, opt.state[p]["exp_avg"], 1e-13, 0, "m")
            _close(v_new, opt.state[p]["exp_avg_sq"], 1e-13, 0, "v")
