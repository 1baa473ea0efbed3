"""The time-conditioned baseline's whole training step (NeRF(time_conditioned_baseline=True), no bender: the latent enters
L0 and L5 as a per-ray bias, nrn_field_forward_tc / nrn_field_backward_tc) at the benchmark's cfg4 batch: 8,192 rays,
64 + 64 samples, an 86-row trainable latent table, random (image, y, x) pixel indices, every random draw injected.  The
stage checks of this model at that batch and past 2^31 bytes of its masks are in tests/test_scale_gpu.py.

  cfg4 step     training_wrapper_class against tests/tc_reference.py's fp32 restatement run on the GPU with TF32 off, in
                chunks of 1,024 rays whose gradients add up: per-ray loss within 2e-3 (L-inf and relative L2), gradients
                within DESIGN section 2's bounds for 1,024 rays (NeRF layers 5e-2, heads 2e-2, the latent columns of
                W0 / W5 and the latent table 8e-2)
  graph replay  six steps under torch.use_deterministic_algorithms(True) (Adam over the table and both models, a
                device-scalar global step, set_lr between steps, one at lr = 0).  The only order-dependent sum of this
                path is the latent-table scatter, which is deterministic under the flag, so two eager runs must be
                bit-identical and GraphedStep's replays of steps 4..6 must equal them bit for bit

Measured on one H100 80GB HBM3 (700 W power limit, 132 SMs), printed with `pytest -s`; the two tests run in about 1 s
after the first CUDA initialisation.
  cfg4 step     per-ray loss 2.2e-6 L-inf, 2.8e-6 relative L2; gradients at most 2.5e-2 (coarse W0's latent columns),
                1.1e-2 for the other NeRF columns, 2.4e-4 for the heads, 9.6e-3 for the latent table
  graph replay  two eager runs and the replay bit-identical
"""
import pytest
import torch

import oracle.nrnerf_oracle as O
from tests import helpers, tc_reference as TR
from tests.parity import DEV
from tests.test_scale_gpu import f32_bits_equal

pytestmark = pytest.mark.gpu
SEED_STEP = 8194
N_IMAGES = 86


def tc_setup(seed, n, n_iters):
    """cfg4's step inputs for the time-conditioned baseline: coarse and fine NeRF(time_conditioned_baseline=True), an
    86-row trainable latent table, (image, y, x) pixel indices and render_rays' four random draws injected."""
    import types
    from nonrigid_nerf_b200 import optim
    torch.manual_seed(seed)   # the modules' dead weights (views_linears) keep nn.Linear's random initialisation
    coarse, fine, params = helpers.tc_models(seed, DEV)
    r = O.make_rays(seed, n)
    g = torch.Generator().manual_seed(seed)
    rnd = {k: v.to(DEV) for k, v in O.make_randomness(seed, n, 64, 64).items()}
    table = (torch.randn(N_IMAGES, 32, generator=g) * 0.1).to(DEV)
    pix = torch.stack([torch.randint(0, N_IMAGES, (n,), generator=g), torch.randint(0, 384, (n,), generator=g),
                       torch.randint(0, 512, (n,), generator=g)], 1).to(DEV)
    latents = [table[i].clone().requires_grad_(True) for i in range(N_IMAGES)]
    opt = optim.Adam(latents + list(coarse.parameters()) + list(fine.parameters()), lr=5e-4)
    targs = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=n_iters, offsets_loss_weight=0.0,
                                  divergence_loss_weight=0.0, rigidity_loss_weight=0.0, ray_bending_latent_size=32)
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64,
          "network_fn": coarse, "ray_bender": None, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": 1.0,
          "ndc": False, "lindisp": False, "near": r["near"], "far": r["far"], "randomness": rnd}
    inputs = [r["rays_o"].to(DEV), r["rays_d"].to(DEV), r["target"].to(DEV), pix]
    extras = {"imageid_to_timestepid": list(range(N_IMAGES))}
    return dict(models=(coarse, fine), params=params, r=r, rnd=rnd, table=table, latents=latents, opt=opt, targs=targs,
                kw=kw, inputs=inputs, extras=extras)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


LATENT_COLS = slice(63, 95)


def _layer_checks(nm, net, po):
    """(name, ours, oracle's, bound) of one model's layers: W0 / W5 split into their latent columns (8e-2) and the rest
    (5e-2), the other layers and every bias 5e-2, the head 2e-2."""
    out = []
    for i in range(8):
        got, exp = net.pts_linears[i].weight.grad, po["pts_w"][i].grad
        if i in (0, 5):
            rest = [c for c in range(got.shape[1]) if not 63 <= c < 95]
            out += [(f"{nm} W{i}[:, 63:95]", got[:, LATENT_COLS], exp[:, LATENT_COLS], 8e-2),
                    (f"{nm} W{i} other columns", got[:, rest], exp[:, rest], 5e-2)]
        else:
            out.append((f"{nm} W{i}", got, exp, 5e-2))
        out.append((f"{nm} b{i}", net.pts_linears[i].bias.grad, po["pts_b"][i].grad, 5e-2))
    out += [(f"{nm} head", net.output_linear.weight.grad, po["out_w"].grad, 2e-2),
            (f"{nm} head bias", net.output_linear.bias.grad, po["out_b"].grad, 2e-2)]
    return out


def test_cfg4_tc_training_step_matches_the_fp32_oracle():
    """training_wrapper_class at 8,192 rays against tc_reference.training_loss_rays on the GPU with TF32 off, in chunks of
    1,024 rays whose gradients add up: the per-ray loss, every layer's gradient and the latent table's."""
    from nonrigid_nerf_b200 import _lib as L, parallel
    n, global_step = 8192, 1000
    st = tc_setup(SEED_STEP, n, 200000)
    coarse, fine = st["models"]
    ro, rd, target, pix = st["inputs"]
    wrapper = parallel.training_wrapper_class(coarse, st["latents"], fine_model=fine, ray_bender=None)
    loss = wrapper(st["targs"], ro, rd, 100, st["kw"], target, global_step, 0, st["extras"], pix)
    loss.mean().backward()
    L.device_error_check()

    def dev_params(p):
        return {k: [t.to(DEV).requires_grad_(True) for t in v] if isinstance(v, list) else v.to(DEV).requires_grad_(True)
                for k, v in p.items()}

    cpo, fpo = (dev_params(O.clone_params(p)) for p in st["params"])
    table = st["table"].clone().requires_grad_(True)
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        ref = []
        for a in range(0, n, 1024):
            sl = slice(a, a + 1024)
            rays = {"rays_o": ro[sl], "rays_d": rd[sl], "near": st["r"]["near"], "far": st["r"]["far"], "target": target[sl]}
            rnd = {k: v[sl] for k, v in st["rnd"].items()}
            lo = TR.training_loss_rays(cpo, fpo, rays, table, st["extras"]["imageid_to_timestepid"], pix[sl], rnd)
            (lo.sum() / n).backward()
            ref.append(lo.detach())
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    ref = torch.cat(ref)
    d, rel = float((loss.detach() - ref).abs().max()), _rel(loss.detach(), ref)
    print(f"  [tc cfg4 step] per-ray loss vs fp32 oracle: L-inf {d:.3e}, rel L2 {rel:.3e}")
    assert d <= 2e-3 and rel <= 2e-3, (d, rel)
    checks = _layer_checks("coarse", coarse, cpo) + _layer_checks("fine", fine, fpo)
    checks.append(("latent table", torch.stack([l.grad for l in st["latents"]]), table.grad, 8e-2))
    worst = {}
    for nm, got, exp, tol in checks:
        assert got is not None and exp is not None, nm
        assert bool(torch.isfinite(got).all()), nm
        worst[nm] = _rel(got, exp)
        assert worst[nm] <= tol, (nm, worst[nm], tol)
    print(f"  [tc cfg4 step] gradient rel L2 vs fp32 oracle: worst {max(worst.values()):.2e} ({max(worst, key=worst.get)}); " +
          ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))


LRS_STEP = [5e-4, 5e-4, 5e-4, 2e-3, 0.0, 1e-3]   # steps 1..6; the graph's 3 warm-up steps run at the first value


def _tc_run(graph):
    """Six steps at 8,192 rays under torch.use_deterministic_algorithms(True) (Adam over the table and both models, a
    device-scalar global_step): eagerly, or 3 warm-up steps inside GraphedStep and 3 replays.  Returns per step (losses,
    parameters before, parameters after) for the steps run after the warm-up."""
    from nonrigid_nerf_b200 import _lib as L, parallel
    from nonrigid_nerf_b200.graphs import GraphedStep
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        st = tc_setup(SEED_STEP, 8192, 8)
        coarse, fine = st["models"]
        opt, inputs = st["opt"], st["inputs"]
        wrapper = parallel.training_wrapper_class(coarse, st["latents"], fine_model=fine, ray_bender=None)
        global_step = torch.zeros((), dtype=torch.float32, device=DEV)
        n = inputs[0].shape[0]

        def local_step(rays_o, rays_d, target, pix):
            opt.zero_grad()
            losses = wrapper(st["targs"], rays_o, rays_d, 100, st["kw"], target, global_step, 0, st["extras"], pix)
            (losses.sum() / n).backward()
            opt.step()
            global_step.add_(1.0)
            return losses.detach()

        first = 3 if graph else 0
        if graph:
            opt.set_lr(LRS_STEP[0])
            run = GraphedStep(local_step, inputs, warmup=3)
        else:
            run = local_step
        out = []
        for i in range(first, 6):
            opt.set_lr(LRS_STEP[i])
            p0 = opt._flat.clone()
            losses = run(*inputs)
            torch.cuda.synchronize()
            out.append((losses.clone(), p0, opt._flat.clone()))
        L.device_error_check()
        assert float(global_step) == 6
    finally:
        torch.use_deterministic_algorithms(prev)
    return out[-3:]


def test_cfg4_tc_graphed_step_equals_eager_bit_for_bit():
    """Two eager deterministic runs of steps 1..6 are bit-identical, and GraphedStep's replays of steps 4..6 equal them bit
    for bit: losses and every parameter, the latent table included; lr = 0 leaves the parameters untouched."""
    eager, eager2, graph = _tc_run(False), _tc_run(False), _tc_run(True)
    for j, ((le, pe0, pe1), (le2, _, pe12), (lg, pg0, pg1)) in enumerate(zip(eager, eager2, graph)):
        step = 4 + j
        assert f32_bits_equal(le, le2) and f32_bits_equal(pe1, pe12), \
            f"step {step}: two eager runs differ, loss rel L2 {_rel(le2, le):.3e}, parameters {_rel(pe12, pe1):.3e}"
        assert f32_bits_equal(lg, le), f"step {step}: replay vs eager per-ray loss differs, rel L2 {_rel(lg, le):.3e}"
        assert f32_bits_equal(pg0, pe0) and f32_bits_equal(pg1, pe1), \
            f"step {step}: replay vs eager parameters differ, rel L2 {_rel(pg1, pe1):.3e}"
        if LRS_STEP[step - 1] == 0.0:
            assert f32_bits_equal(pg1, pg0), f"step {step}: lr = 0 moved the parameters"
        else:
            assert not f32_bits_equal(pg1, pg0), f"step {step}: the replay did not move the parameters"
    print("  [tc cfg4 graph] steps 4..6: two eager runs and the replay are bit-identical in losses and parameters")
