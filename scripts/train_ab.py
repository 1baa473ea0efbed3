#!/usr/bin/env python3
"""Training-quality A/B (north_star: "PSNR within 0.1 dB of the reference"; SURVEY.md section 4 item 4).

Trains the SAME model from the SAME initialisation on the SAME ray batches with the SAME random draws, twice:
  A  this repository's path: fused fp16 tensor-core forward / DGRAD / WGRAD, gradient arena, one-launch Adam
  B  the oracle (oracle/nrnerf_oracle.py: the fp32 PyTorch restatement pinned to the executed reference), run on the GPU
     as the checker, with torch.optim.Adam
  B' the oracle again with TF32 matmuls allowed -- a second fp32-class run whose distance from B shows how much two
     numerically different but equally valid trainings drift apart (the noise floor of the comparison)
on a synthetic non-rigid scene (analytic density / colour blobs that move with time, rendered by quadrature), with all three
regularisers on, then renders held-out pixels of every frame with each trained model (deterministic sampling) and
reports the loss curves and the PSNR against the ground truth.  Writes one JSON document (stdout or --out).

    python scripts/train_ab.py --iters 1000 --out train_ab.json
"""
import argparse
import json
import math
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_FRAMES, H, W, FOCAL = 8, 48, 64, 60.0
NEAR, FAR = 0.2, 1.8


def scene_field(pts, t):
    """Analytic ground truth: three coloured Gaussian blobs; the first swings sideways with time t in [0, 1]."""
    centers = torch.tensor([[-0.25, 0.0, -1.0], [0.2, 0.15, -1.1], [0.05, -0.2, -0.85]], device=pts.device)
    colors = torch.tensor([[0.9, 0.2, 0.1], [0.1, 0.8, 0.3], [0.2, 0.3, 0.9]], device=pts.device)
    radii = torch.tensor([0.16, 0.13, 0.11], device=pts.device)
    shift = torch.zeros_like(centers)
    shift[0, 0] = 0.25 * math.sin(2 * math.pi * t)
    shift[0, 1] = 0.10 * math.cos(2 * math.pi * t)
    shift[2, 1] = 0.12 * t
    d2 = ((pts[..., None, :] - (centers + shift)) ** 2).sum(-1)
    dens = 40.0 * torch.exp(-d2 / (2 * radii ** 2))
    sigma = dens.sum(-1)
    rgb = (dens[..., None] * colors).sum(-2) / (sigma[..., None] + 1e-6)
    return sigma, rgb


def render_gt(rays_o, rays_d, t, n=384):
    z = torch.linspace(NEAR, FAR, n, device=rays_o.device)
    pts = rays_o[:, None, :] + rays_d[:, None, :] * z[None, :, None]
    sigma, rgb = scene_field(pts, t)
    delta = (z[1] - z[0]) * rays_d.norm(dim=-1, keepdim=True)
    alpha = 1 - torch.exp(-sigma * delta)
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], -1), -1)[:, :-1]
    w = alpha * trans
    return (w[..., None] * rgb).sum(-2)


def make_dataset(dev):
    from nonrigid_nerf_b200 import run_nerf_helpers as Hh
    intr = {"height": H, "width": W, "focal_x": FOCAL, "focal_y": FOCAL, "center_x": W * 0.5, "center_y": H * 0.5}
    poses, images = [], []
    for k in range(N_FRAMES):
        ang = 0.5 * (k / (N_FRAMES - 1) - 0.5)
        c2w = torch.tensor([[math.cos(ang), 0, math.sin(ang), 0.45 * math.sin(ang)], [0, 1, 0, 0.0],
                            [-math.sin(ang), 0, math.cos(ang), 0.1 * (1 - math.cos(ang))]], dtype=torch.float32, device=dev)
        ro, rd = Hh.get_rays(c2w, intr)
        images.append(render_gt(ro.reshape(-1, 3), rd.reshape(-1, 3), k / (N_FRAMES - 1)).reshape(H, W, 3))
        poses.append(c2w)
    return torch.stack(images), torch.stack(poses), [intr]


def psnr(a, b):
    return float(-10.0 * torch.log10(((a - b) ** 2).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--n-rand", type=int, default=1024)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-tf32-run", action="store_true")
    ap.add_argument("--seeds", type=int, default=1, help="ensemble: independent initialisations / batch sequences; two fp32-class trainings "
                    "of this scene drift apart chaotically (see the TF32 run), so a single pair of runs cannot resolve 0.1 dB")
    args = ap.parse_args()
    if args.seeds > 1:
        runs = []
        for k in range(args.seeds):
            runs.append(run_once(args, seed=12 + 101 * k, with_tf32=False, curves=False))
            print(f"[seed {k}] A {runs[-1]['psnr_held_out']['A_this_repo_fp16']:.3f} dB  B {runs[-1]['psnr_held_out']['B_oracle_fp32']:.3f} dB", file=sys.stderr, flush=True)
        d = np.array([r["delta_psnr_A_minus_B"] for r in runs])
        a = np.array([r["psnr_held_out"]["A_this_repo_fp16"] for r in runs])
        b = np.array([r["psnr_held_out"]["B_oracle_fp32"] for r in runs])
        la = np.array([r["mean_loss_last_tenth"]["A"] for r in runs])
        lb = np.array([r["mean_loss_last_tenth"]["B"] for r in runs])
        out = {"iters": args.iters, "n_rand": args.n_rand, "seeds": args.seeds,
               "psnr_A_mean": float(a.mean()), "psnr_B_mean": float(b.mean()), "psnr_B_std_over_seeds": float(b.std(ddof=1)),
               "delta_psnr_mean": float(d.mean()), "delta_psnr_stderr": float(d.std(ddof=1) / np.sqrt(len(d))),
               "delta_psnr_per_seed": d.tolist(), "psnr_A_per_seed": a.tolist(), "psnr_B_per_seed": b.tolist(),
               "final_loss_A_mean": float(la.mean()), "final_loss_B_mean": float(lb.mean()),
               "final_loss_rel_diff_mean": float(((la - lb) / lb).mean()), "final_loss_rel_diff_stderr": float(((la - lb) / lb).std(ddof=1) / np.sqrt(len(d))),
               "render_parity_on_B_weights_psnr_min": float(min(r["trained_weights_render_parity"]["psnr_this_repo_vs_oracle_on_B_weights"] for r in runs))}
        text = json.dumps(out, indent=1)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                f.write(text + "\n")
        print(text)
        return
    out = run_once(args, seed=12, with_tf32=not args.no_tf32_run, curves=True)
    text = json.dumps(out, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


def run_once(args, seed, with_tf32, curves):
    import oracle.nrnerf_oracle as O
    from nonrigid_nerf_b200 import _lib, optim, parallel, train as T
    from tests import helpers
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    images, poses, intr = make_dataset(dev)
    sampler = T.RayBatchSampler(images, poses, intr, None, dev)
    # held-out pixels: a fixed checkerboard of every frame never offered to the optimiser
    yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    held = ((yy + xx) % 4 == 0)
    train_pix = torch.stack([t.reshape(-1) for t in torch.meshgrid(torch.arange(N_FRAMES, device=dev), torch.arange(W, device=dev),
                                                                    torch.arange(H, device=dev), indexing="ij")], -1)
    keep = ~held[train_pix[:, 2], train_pix[:, 1]]
    train_pix = train_pix[keep]
    held_pix = torch.stack([t.reshape(-1) for t in torch.meshgrid(torch.arange(N_FRAMES, device=dev), torch.arange(W, device=dev),
                                                                   torch.arange(H, device=dev), indexing="ij")], -1)[~keep]

    targs = types.SimpleNamespace(chunk=32768, N_samples=64, N_importance=64, N_iters=args.iters, offsets_loss_weight=60.0,
                                  divergence_loss_weight=3.0, rigidity_loss_weight=0.0005, ray_bending_latent_size=32)
    i2t = list(range(N_FRAMES))
    gen = torch.Generator(device=dev).manual_seed(99 + seed)
    batches = []
    for it in range(args.iters):
        sel = torch.randint(train_pix.shape[0], (args.n_rand,), device=dev, generator=gen)
        batches.append(train_pix[sel])

    def draws(it):
        g = torch.Generator(device=dev).manual_seed(1000 * seed + it)
        n = args.n_rand
        return {"t_rand": torch.rand(n, 64, device=dev, generator=g), "noise_c": torch.randn(n, 64, device=dev, generator=g),
                "u": torch.rand(n, 64, device=dev, generator=g), "noise_f": torch.randn(n, 128, device=dev, generator=g),
                "e": torch.randn(n * 64, 3, device=dev, generator=g)}

    def lr_at(it):
        return 5e-4 * (0.1 ** (it / (250 * 1000)))

    # ------------------------------ A: this repository ------------------------------
    coarse, fine, bender, (cp0, fp0, bp0) = helpers.build_models(O, seed, dev, density_boost=1.0)
    latents = [torch.zeros(32, device=dev).requires_grad_(True) for _ in range(N_FRAMES)]
    opt = optim.Adam(latents + list(bender.parameters()) + list(coarse.parameters()) + list(fine.parameters()), lr=5e-4)
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": 64, "network_fine": fine, "N_samples": 64, "network_fn": coarse,
          "ray_bender": bender, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": 1.0, "ndc": False, "lindisp": False,
          "near": NEAR, "far": FAR}
    curve_a = []
    for it in range(args.iters):
        batch_rays, target, pix = sampler.rays_for(batches[it])
        kw["randomness"] = draws(it)
        opt.set_lr(lr_at(it))
        opt.zero_grad()
        losses = wrapper(targs, batch_rays[0], batch_rays[1], it, kw, target, it, 0, {"imageid_to_timestepid": i2t}, pix)
        losses.mean().backward()
        opt.step()
        curve_a.append(float(losses.mean().detach()))
    _lib.device_error_check()

    def eval_ours():
        rays, target, pix = sampler.rays_for(held_pix)
        kwt = dict(kw, perturb=0.0, raw_noise_std=0.0)
        kwt.pop("randomness", None)
        lat = torch.stack([l.detach() for l in latents])[pix[:, 0]]
        with torch.no_grad():
            rgb = T.render(rays[0], rays[1], chunk=32768, additional_pixel_information={"ray_bending_latents": lat}, **kwt)[0]
        return rgb, target

    rgb_a, target_h = eval_ours()

    # ------------------------------ B / B': the fp32 oracle on the GPU ------------------------------
    def run_oracle(allow_tf32):
        torch.backends.cuda.matmul.allow_tf32 = allow_tf32
        to = lambda p: {k: ([t.to(dev).clone().requires_grad_(True) for t in v] if isinstance(v, list) else v.to(dev).clone().requires_grad_(True))
                        for k, v in p.items()}
        cp, fp, bp = to(cp0), to(fp0), to(bp0)
        table = torch.zeros(N_FRAMES, 32, device=dev, requires_grad=True)
        opt_b = torch.optim.Adam([table] + O.flat_param_list(bp) + O.flat_param_list(cp) + O.flat_param_list(fp), lr=5e-4, betas=(0.9, 0.999))
        curve = []
        for it in range(args.iters):
            batch_rays, target, pix = sampler.rays_for(batches[it])
            rays = {"rays_o": batch_rays[0], "rays_d": batch_rays[1], "near": NEAR, "far": FAR, "target": target}
            d = draws(it)
            for grp in opt_b.param_groups:
                grp["lr"] = lr_at(it)
            opt_b.zero_grad()
            loss, _ = O.training_wrapper_loss(cp, fp, bp, rays, table, i2t, pix, d, d["e"], it, args.iters, 60.0, 3.0, 0.0005)
            loss.mean().backward()
            opt_b.step()
            curve.append(float(loss.mean().detach()))
        rays, target, pix = sampler.rays_for(held_pix)
        with torch.no_grad():
            ret = O.render_rays(cp, fp, bp, rays[0], rays[1], NEAR, FAR, table[pix[:, 0]], 64, 64)
        torch.backends.cuda.matmul.allow_tf32 = False
        return curve, ret["rgb_map"], (cp, fp, bp, table)

    curve_b, rgb_b, state_b = run_oracle(False)
    out = {"iters": args.iters, "n_rand": args.n_rand, "frames": N_FRAMES, "held_out_pixels": int(held_pix.shape[0]),
           "regularisers": {"offsets_loss_weight": 60.0, "divergence_loss_weight": 3.0, "rigidity_loss_weight": 0.0005},
           "psnr_held_out": {"A_this_repo_fp16": psnr(rgb_a, target_h), "B_oracle_fp32": psnr(rgb_b, target_h)},
           "psnr_A_vs_B_render": psnr(rgb_a, rgb_b)}
    out["delta_psnr_A_minus_B"] = out["psnr_held_out"]["A_this_repo_fp16"] - out["psnr_held_out"]["B_oracle_fp32"]
    # cross-check of the two renderers on identical (B's trained) weights: numerics of inference alone
    cpb, fpb, bpb, table_b = state_b
    with torch.no_grad():
        helpers.load_nerf_module(coarse, {k: ([t.detach() for t in v] if isinstance(v, list) else v.detach()) for k, v in cpb.items()})
        helpers.load_nerf_module(fine, {k: ([t.detach() for t in v] if isinstance(v, list) else v.detach()) for k, v in fpb.items()})
        helpers.load_bender_module(bender, {k: ([t.detach() for t in v] if isinstance(v, list) else v.detach()) for k, v in bpb.items()})
        for l, row in zip(latents, table_b.detach()):
            l.copy_(row)
    from nonrigid_nerf_b200 import ops
    ops.note_parameters_changed()
    rgb_ab, _ = eval_ours()
    out["trained_weights_render_parity"] = {"rgb_linf_this_repo_vs_oracle_on_B_weights": float((rgb_ab - rgb_b).abs().max()),
                                            "psnr_this_repo_vs_oracle_on_B_weights": psnr(rgb_ab, rgb_b)}
    if with_tf32:
        curve_c, rgb_c, _ = run_oracle(True)
        out["psnr_held_out"]["Bprime_oracle_tf32"] = psnr(rgb_c, target_h)
        out["delta_psnr_Bprime_minus_B (noise floor)"] = out["psnr_held_out"]["Bprime_oracle_tf32"] - out["psnr_held_out"]["B_oracle_fp32"]
        out["loss_curve_Bprime"] = curve_c[::max(1, args.iters // 50)]
    k = max(1, args.iters // 50)
    if curves:
        out["loss_curve_A"], out["loss_curve_B"] = curve_a[::k], curve_b[::k]
    else:
        out.pop("loss_curve_Bprime", None)
    tail = max(10, args.iters // 10)
    out["mean_loss_last_tenth"] = {"A": float(np.mean(curve_a[-tail:])), "B": float(np.mean(curve_b[-tail:]))}
    return out


if __name__ == "__main__":
    main()
