#!/usr/bin/env python3
"""Training-step throughput of the time-conditioned baseline beside the ray-bending model, in one process.

    python scripts/bench_tc.py --steps 20 --warmup 5 [--out result.json]

Both steps are bench.py's example_sequence step (N_rand = 1024, 64 coarse + 128 fine samples, optim.Adam, CUDA-graph
replay): "bending" with bench.py's models and regulariser weights, "time_conditioned" with
NeRF(time_conditioned_baseline=True), no bender and zero regulariser weights (train.py:574-578).  Afterwards a few eager
time-conditioned steps run with the library's per-kernel timing, which reports the two kernel kinds of the baseline
(ray bias; per-ray sums, d z and the latent weight columns) beside the fused field kernels.  Prints one JSON line."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as B  # noqa: E402


def build(dev, H, tc):
    if not tc:
        return B.build_models(dev, H)
    torch.manual_seed(0)
    kw = dict(D=8, W=256, input_ch=63, output_ch=5, skips=[4], input_ch_views=0, use_viewdirs=False, ray_bender=None,
              ray_bending_latent_size=32, time_conditioned_baseline=True)
    return (H.NeRF(num_ray_samples=B.N_SAMPLES, **kw).to(dev), H.NeRF(num_ray_samples=B.N_SAMPLES + B.N_IMPORTANCE, **kw).to(dev),
            None)


def run(tc, args, dev):
    from nonrigid_nerf_b200 import _lib, optim, parallel, run_nerf_helpers as H
    from nonrigid_nerf_b200.graphs import GraphedStep
    coarse, fine, bender = build(dev, H, tc)
    n_images = 86
    latents = [torch.zeros(32, device=dev).normal_(0, 0.1).requires_grad_(True) for _ in range(n_images)]
    params = latents + (list(bender.parameters()) if bender is not None else []) + list(coarse.parameters()) + list(fine.parameters())
    opt = optim.Adam(params, lr=5e-4, betas=(0.9, 0.999))
    kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": B.N_IMPORTANCE, "network_fine": fine, "N_samples": B.N_SAMPLES,
          "network_fn": coarse, "ray_bender": bender, "use_viewdirs": False, "white_bkgd": False, "raw_noise_std": 1.0, "ndc": False,
          "lindisp": False, "near": 0.0022, "far": 1.0024}
    targs = B.make_args()
    if tc:
        targs.offsets_loss_weight = targs.divergence_loss_weight = targs.rigidity_loss_weight = 0.0
    extras = {"imageid_to_timestepid": list(range(n_images))}
    wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
    rs = np.random.RandomState(1234)
    batches = [[torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in B.synth_batch(rs, args.n_rand, n_images)] for _ in range(4)]
    global_step = torch.full((), 1000.0, dtype=torch.float32, device=dev)

    def step(rays_o, rays_d, target, idx):
        opt.zero_grad()
        losses = wrapper(targs, rays_o, rays_d, 100, kw, target, global_step, 0, extras, idx)
        (losses.sum() / args.n_rand).backward()
        opt.step()
        global_step.add_(1.0)
        return losses.detach().mean()

    graphed = GraphedStep(step, batches[0], warmup=3)
    for i in range(args.warmup):
        graphed(*batches[i % 4])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        loss = graphed(*batches[i % 4])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    out = {"ms_per_step": ms, "rays_per_sec": args.n_rand / (ms / 1000.0), "loss": float(loss)}
    if tc:   # per-kernel times of eager steps (no graph: every launch is bracketed by the library's events)
        del graphed
        torch.cuda.synchronize()
        _lib.timing_enable(True)
        for i in range(args.steps):
            step(*batches[i % 4])
        kinds = _lib.timing_read(_lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS)
        _lib.timing_enable(False)
        out["eager_ms_per_step_by_kernel"] = {k: v[0] / args.steps for k, v in kinds.items()}
        out["launches_per_step"] = {k: v[1] / args.steps for k, v in kinds.items()}
    _lib.device_error_check()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--n-rand", type=int, default=B.N_RAND)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"workload": f"example_sequence training step, N_rand = {args.n_rand}, {B.N_SAMPLES}c + {B.N_SAMPLES + B.N_IMPORTANCE}f "
                       "samples, CUDA-graph replay", "gpu": torch.cuda.get_device_name(dev),
           "bending": run(False, args, dev), "time_conditioned": run(True, args, dev)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
