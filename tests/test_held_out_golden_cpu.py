"""Pins the oracle's version of the reference loop's two backward passes for held-out frames (train.py:1595-1608) against
golden case N, which executed the unmodified reference (tests/golden/make_golden_held_out.py).  CPU only."""
import os

import numpy as np
import torch

import oracle.nrnerf_oracle as O
from tests.golden.make_golden_held_out import held_out_batch, held_out_probes
from tests.test_oracle_golden import _bender_grad_checks, close, models

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def case_n(n):
    """Case N's entries of the n-ray batch, without their "n<N>_" prefix, and the file's shared entries."""
    g = np.load(os.path.join(GOLD, "caseN_held_out.npz"), allow_pickle=False)
    p = f"n{n}_"
    out = {k[len(p):]: g[k] for k in g.files if k.startswith(p)}
    out.update({k: g[k] for k in g.files if not k.startswith("n")})
    return out


def oracle_two_pass(n, device="cpu"):
    """The oracle's training_wrapper_loss on case N's n-ray batch, then the reference loop's two backward passes.
    Returns (loss, latent table with its gradient, cp, fp, bp with the second pass's gradients)."""
    g = case_n(n)
    seed = int(g["seed"]) + n
    cp, fp, bp = (O.clone_params(p, True) for p in models(seed))
    r = O.make_rays(seed, n)
    rnd = O.make_randomness(seed, n, 64, 64)
    table_np, pix_np, i2t = held_out_batch(seed, n)
    table = torch.from_numpy(table_np).clone().requires_grad_(True)
    pix = torch.from_numpy(pix_np)
    loss, _ = O.training_wrapper_loss(cp, fp, bp, r, table, i2t, pix, rnd, held_out_probes(seed, n), int(g["global_step"]),
                                      int(g["N_iters"]), float(g["offsets_w"]), float(g["divergence_w"]), float(g["rigidity_w"]))
    test = torch.isin(pix[:, 0], torch.from_numpy(g["held_images"])).float()
    torch.mean(test * loss).backward(retain_graph=True)
    for p in (cp, fp, bp):
        for v in p.values():
            for t in (v if isinstance(v, list) else [v]):
                t.grad = None
    torch.mean((1 - test) * loss).backward()
    return loss, table, cp, fp, bp


def test_caseN_oracle_two_pass_matches_executed_reference():
    g = case_n(96)
    loss, table, cp, fp, bp = oracle_two_pass(96)
    close(loss, g["loss"], 2e-6, 2e-5, name="loss")
    close(table.grad, g["latent_grads"], 1e-8, 2e-3, name="latent_grads")
    held = np.isin(np.arange(7), g["held_images"])
    assert np.abs(g["latent_grads"][held]).max() > 0 and np.abs(g["latent_grads"][~held]).max() > 0
    for net, p in {"coarse": cp, "fine": fp}.items():
        for i in range(8):
            nm = f"{net}.pts_linears.{i}.weight"
            gr = p["pts_w"][i].grad.reshape(-1)
            close(gr[torch.from_numpy(g[nm + ".idx"])], g[nm + ".val"], 1e-7, 2e-3, name=nm)
    _bender_grad_checks(g, bp, 2e-3)
