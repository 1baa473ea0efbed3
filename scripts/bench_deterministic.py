#!/usr/bin/env python3
"""Cost of deterministic mode (torch.use_deterministic_algorithms(True)) on the graph-replayed training step.

    python scripts/bench_deterministic.py --steps 50 --warmup 5 --runs 5 [--out results.jsonl]

bench.py's example_sequence step (64 coarse + 64 fine samples, bender and all three regularisers, optim.Adam, CUDA-graph
replay) at N_rand = 1024 and at cfg4's 8,192 rays, in three configurations: the flag off; the flag on with
torch.utils.deterministic.fill_uninitialized_memory True (PyTorch's default: every torch.empty is NaN-filled); the flag on
with it False.  Each configuration captures its own graph from fresh models; the configurations alternate within each of
`runs` rounds, so that drift of the shared machine spreads over all of them.  Prints one JSON line per (batch, round,
configuration), then one summary line per batch (median and spread over the rounds); the card's name and power limit are
read in the same process."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as B  # noqa: E402

CONFIGS = (("off", False, True), ("on_fill", True, True), ("on_nofill", True, False))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_config(n_rand, det, fill, args, dev):
    import torch.utils.deterministic as TD
    from nonrigid_nerf_b200 import _lib, optim, parallel, run_nerf_helpers as H
    from nonrigid_nerf_b200.graphs import GraphedStep
    prev = (torch.are_deterministic_algorithms_enabled(), TD.fill_uninitialized_memory)
    torch.use_deterministic_algorithms(det)
    TD.fill_uninitialized_memory = fill
    try:
        coarse, fine, bender = B.build_models(dev, H)
        n_images = 86
        latents = [torch.zeros(32, device=dev).normal_(0, 0.1).requires_grad_(True) for _ in range(n_images)]
        params = latents + list(bender.parameters()) + list(coarse.parameters()) + list(fine.parameters())
        opt = optim.Adam(params, lr=5e-4, betas=(0.9, 0.999))
        kw = {"network_query_fn": None, "perturb": 1.0, "N_importance": B.N_IMPORTANCE, "network_fine": fine,
              "N_samples": B.N_SAMPLES, "network_fn": coarse, "ray_bender": bender, "use_viewdirs": False, "white_bkgd": False,
              "raw_noise_std": 1.0, "ndc": False, "lindisp": False, "near": 0.0022, "far": 1.0024}
        targs = B.make_args()
        extras = {"imageid_to_timestepid": list(range(n_images))}
        wrapper = parallel.training_wrapper_class(coarse, latents, fine_model=fine, ray_bender=bender)
        rs = np.random.RandomState(1234)
        batches = [[torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in B.synth_batch(rs, n_rand, n_images)]
                   for _ in range(4)]
        global_step = torch.full((), 1000.0, dtype=torch.float32, device=dev)

        def step(rays_o, rays_d, target, idx):
            opt.zero_grad()
            losses = wrapper(targs, rays_o, rays_d, 100, kw, target, global_step, 0, extras, idx)
            (losses.sum() / n_rand).backward()
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
        _lib.device_error_check()
        out = {"ms_per_step": ms, "loss": float(loss)}
        del graphed
        torch.cuda.synchronize()
        return out
    finally:
        torch.use_deterministic_algorithms(prev[0])
        TD.fill_uninitialized_memory = prev[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--n-rand", type=int, nargs="+", default=[B.N_RAND, 8192])
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power = card()
    lines = []
    for n_rand in args.n_rand:
        ms = {c[0]: [] for c in CONFIGS}
        for r in range(args.runs):
            for label, det, fill in CONFIGS:
                res = time_config(n_rand, det, fill, args, dev)
                ms[label].append(res["ms_per_step"])
                lines.append({"n_rand": n_rand, "round": r, "config": label, **res, "gpu": name, "power_limit": power})
                print(json.dumps(lines[-1]), flush=True)
        summ = {k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))} for k, v in ms.items()}
        base = summ["off"]["median_ms"]
        for k in ("on_fill", "on_nofill"):
            summ[k]["overhead_vs_off"] = summ[k]["median_ms"] / base - 1.0
        lines.append({"n_rand": n_rand, "summary": summ, "steps": args.steps, "runs": args.runs, "gpu": name, "power_limit": power,
                      "workload": f"example_sequence training step, {B.N_SAMPLES}c + {B.N_SAMPLES + B.N_IMPORTANCE}f samples, "
                                  "CUDA-graph replay"})
        print(json.dumps(lines[-1]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
