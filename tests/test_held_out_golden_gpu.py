"""Held-out rays on the GPU against the executed reference and the fp32 oracle, and under CUDA-graph replay.

  golden case N   one backward of ((train + test) * loss).mean() with held_out=test, at 96, 1,024 and 8,192 rays, against
                  the unmodified reference's two backward passes (tests/golden/make_golden_held_out.py): the per-ray loss,
                  a sample of every parameter's gradient and the latent gradients of held-out and training frames, at
                  test_training_wrapper_gpu.py's bounds.
  fp32 oracle     the same step at 96 rays against the oracle's two passes, every parameter's whole gradient.
  graph replay    a deterministic one-pass step captured by GraphedStep with the mask as a static input, replayed with
                  other masks (one all zero): each replay equals the eager step with that mask bit for bit.
"""
import types

import numpy as np
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers
from tests.golden.make_golden_held_out import held_out_batch, held_out_probes
from tests.test_held_out_golden_cpu import case_n, oracle_two_pass

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


class _Golden(dict):
    """case_n's entries with the .files attribute the sampled-gradient check reads"""

    @property
    def files(self):
        return list(self.keys())


def _one_pass(n, g):
    """The port's one-pass step on case N's n-ray batch: (loss, coarse, fine, bender, latents)."""
    from nonrigid_nerf_b200 import _lib, parallel
    seed = int(g["seed"]) + n
    coarse, fine, bender, _ = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    rnd = dict(O.make_randomness(seed, n, 64, 64))
    rnd["e"] = held_out_probes(seed, n)
    table, pix_np, i2t = held_out_batch(seed, n)
    latents = [torch.from_numpy(row.copy()).to(DEV).requires_grad_(True) for row in table]
    pix = torch.from_numpy(pix_np).to(DEV)
    test = torch.isin(pix[:, 0], torch.from_numpy(g["held_images"]).to(DEV))
    targs = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=int(g["N_iters"]),
                                  offsets_loss_weight=float(g["offsets_w"]), divergence_loss_weight=float(g["divergence_w"]),
                                  rigidity_loss_weight=float(g["rigidity_w"]), ray_bending_latent_size=32)
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64,
          "network_fn": coarse, "ray_bender": bender, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": 1.0,
          "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"], "randomness": rnd}
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
    loss = wrapper(targs, r["rays_o"].to(DEV), r["rays_d"].to(DEV), 100, kw, r["target"].to(DEV), int(g["global_step"]), 0,
                   {"imageid_to_timestepid": i2t}, pix, held_out=test)
    (((~test).float() + test.float()) * loss).mean().backward()
    _lib.device_error_check()
    return loss.detach().cpu(), coarse, fine, bender, latents


@pytest.mark.parametrize("n", [96, 1024, 8192])
def test_one_pass_matches_the_executed_two_pass_loop_caseN(n):
    from tests.test_training_wrapper_gpu import _golden_grad_check
    g = _Golden(case_n(n))
    loss, coarse, fine, bender, latents = _one_pass(n, g)
    d = float(np.abs(loss.numpy() - g["loss"]).max())
    rel = _rel(loss, torch.from_numpy(g["loss"]))
    assert d <= 2e-3 and rel <= 2e-3, (d, rel)
    named = [("coarse." + k, v) for k, v in coarse.named_parameters()] + [("fine." + k, v) for k, v in fine.named_parameters()] + \
            [("bender." + k, v) for k, v in bender.named_parameters()]
    checked = [nm for nm, t in named if nm + ".val" in g and t.grad is not None]
    assert len(checked) == sum(t.grad is not None for _, t in named) >= 2 * 18 + 15   # every trained parameter
    worst = _golden_grad_check(g, named, 1.2e-1, f"caseN n={n}")
    lg = torch.stack([l.grad for l in latents]).cpu()
    ref = torch.from_numpy(g["latent_grads"])
    held = torch.from_numpy(np.isin(np.arange(len(latents)), g["held_images"]))
    e_test, e_train = _rel(lg[held], ref[held]), _rel(lg[~held], ref[~held])
    print(f"n={n}: loss L-inf {d:.2e}; worst sampled gradient {worst:.2e}; latents held out {e_test:.2e}, training {e_train:.2e}")
    assert e_test <= 8e-2 and e_train <= 8e-2, (e_test, e_train)


def _oracle_pairs(coarse, fine, bender, cp, fp, bp):
    """(name, port parameter, oracle tensor) for every trained parameter"""
    out = []
    for net, m, p in (("coarse", coarse, cp), ("fine", fine, fp)):
        for i in range(8):
            out += [(f"{net}.pts_linears.{i}.weight", m.pts_linears[i].weight, p["pts_w"][i]),
                    (f"{net}.pts_linears.{i}.bias", m.pts_linears[i].bias, p["pts_b"][i])]
        out += [(f"{net}.output_linear.weight", m.output_linear.weight, p["out_w"]),
                (f"{net}.output_linear.bias", m.output_linear.bias, p["out_b"])]
    for i in range(5):
        out.append((f"bender.network.{i}.weight", bender.network[i].weight, bp["net_w"][i]))
        if i < 4:
            out.append((f"bender.network.{i}.bias", bender.network[i].bias, bp["net_b"][i]))
    for i in range(3):
        out += [(f"bender.rigidity_network.{i}.weight", bender.rigidity_network[i].weight, bp["rig_w"][i]),
                (f"bender.rigidity_network.{i}.bias", bender.rigidity_network[i].bias, bp["rig_b"][i])]
    return out


def test_one_pass_matches_the_fp32_oracle_two_passes():
    n = 96
    g = _Golden(case_n(n))
    loss, coarse, fine, bender, latents = _one_pass(n, g)
    o_loss, o_table, cp, fp, bp = oracle_two_pass(n)
    assert _rel(loss, o_loss.detach()) <= 2e-3
    worst = 0.0
    for nm, t, ref in _oracle_pairs(coarse, fine, bender, cp, fp, bp):
        e = _rel(t.grad.cpu(), ref.grad)
        worst = max(worst, e)
        assert e <= 1.2e-1, (nm, e)
    lg = torch.stack([l.grad for l in latents]).cpu()
    held = torch.from_numpy(np.isin(np.arange(len(latents)), g["held_images"]))
    e_test, e_train = _rel(lg[held], o_table.grad[held]), _rel(lg[~held], o_table.grad[~held])
    print(f"vs fp32 oracle: worst whole-gradient rel err {worst:.2e}; latents held out {e_test:.2e}, training {e_train:.2e}")
    assert e_test <= 8e-2 and e_train <= 8e-2


def test_graph_replay_with_changing_masks_equals_eager():
    from nonrigid_nerf_b200 import parallel
    from nonrigid_nerf_b200.graphs import GraphedStep
    from tests.test_deterministic_gpu import _bits_equal, deterministic
    n, n_images, seed = 1024, 7, 4321
    coarse, fine, bender, _ = helpers.build_models(O, seed, DEV)
    r = O.make_rays(seed, n)
    gen = torch.Generator().manual_seed(seed)
    rnd = {k: v.to(DEV) for k, v in O.make_randomness(seed, n, 64, 64).items()}
    rnd["e"] = torch.randn(n, 64, 3, generator=gen).to(DEV)
    latents = [(0.1 * torch.randn(32, generator=gen)).to(DEV).requires_grad_(True) for _ in range(n_images)]
    pix = torch.stack([torch.randint(0, n_images, (n,), generator=gen), torch.zeros(n, dtype=torch.long),
                       torch.zeros(n, dtype=torch.long)], 1).to(DEV)
    masks = [torch.isin(pix[:, 0], torch.tensor(h, dtype=torch.long, device=DEV)) for h in ((2, 5), (), (0, 1, 6))]
    params = latents + list(bender.parameters()) + list(coarse.parameters()) + list(fine.parameters())
    targs = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=200000, offsets_loss_weight=60.0,
                                  divergence_loss_weight=3.0, rigidity_loss_weight=0.0005, ray_bending_latent_size=32)
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64,
          "network_fn": coarse, "ray_bender": bender, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": 1.0,
          "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"], "randomness": rnd}
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
    extras = {"imageid_to_timestepid": list(range(n_images))}
    inputs = [r["rays_o"].to(DEV), r["rays_d"].to(DEV), r["target"].to(DEV), pix]

    def step(rays_o, rays_d, target, pix, held):
        for p in params:
            p.grad = None
        losses = wrapper(targs, rays_o, rays_d, 100, kw, target, 1000, 0, extras, pix, held_out=held)
        (losses.sum() / n).backward()   # every ray is a training or a held-out ray: (train + test) = 1
        return [losses.detach()] + [p.grad for p in params if p.grad is not None]   # (the dead views_linears have none)

    with deterministic():
        eager = [[t.clone() for t in step(*inputs, m)] for m in masks]
        torch.cuda.synchronize()
        graphed = GraphedStep(step, inputs + [masks[0]], warmup=3)
        for order in ((1, 0, 2), (2, 1, 0)):
            for i in order:
                out = graphed(*inputs, masks[i])
                torch.cuda.synchronize()
                for j, (a, b) in enumerate(zip(eager[i], out)):
                    assert _bits_equal(a, b), f"mask {i}: output {j} of the replay differs from the eager step"
    # the masks matter: the weight gradients of the split steps differ from those of the all-zero mask
    assert not torch.equal(eager[0][-1], eager[1][-1]) and not torch.equal(eager[2][-1], eager[1][-1])
