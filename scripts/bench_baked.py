#!/usr/bin/env python3
"""Rendering time and accuracy with baked radiance grids (render(..., baked=scene)) beside the exact render, in one process.

    python scripts/bench_baked.py --steps 10 --warmup 3 [--out result.json]

Workload: scripts/bench_workloads.py's render workload -- a 504 x 378 full frame, fixed camera, one latent, 64 coarse + 64
importance samples (128 fine), deterministic sampling, chunk = 65536, under torch.no_grad() -- with the models bench.py
builds (create_nerf's default inits and one ray bender).  The coarse and the fine model are baked at 128^3, 256^3 and
512^3 vertices over the box of the exact frame's bent sample points (padded by 0.01), so nearly every sample is looked
up.  Reported: the median frame time per configuration (frames alternate between the exact render and every grid, so
drifting clocks hit all alike), one eager frame's per-kernel times from the library's timing, the time to bake both
models, and the accuracy of each baked frame against the exact one (PSNR, max, mean and 99th percentile of |d rgb|, rgb
in [0, 1], and the fraction of pixels off by more than 0.1).  The models are untrained, so the accuracy says how trilinear
lookup treats these networks' fields, not a trained scene's.  Prints one JSON line with the card's name and power limit,
read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as B  # noqa: E402

RESOLUTIONS = (128, 256, 512)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:   # the number is informative only
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from nonrigid_nerf_b200 import _lib, geometry as G, run_nerf_helpers as H, train as T

    coarse, fine, bender = B.build_models(dev, H)
    Hh, Ww, focal = 378, 504, 252.6
    near, far = 0.0022, 1.0024
    j, i = np.meshgrid(np.arange(Hh, dtype=np.float32), np.arange(Ww, dtype=np.float32), indexing="ij")
    dirs = np.stack([(i - Ww * 0.5) / focal, -(j - Hh * 0.5) / focal, -np.ones_like(i)], -1).reshape(-1, 3).astype(np.float32)
    rays_d = torch.from_numpy(dirs).to(dev)
    rays_o = torch.zeros_like(rays_d)
    n = rays_d.shape[0]
    lat = torch.from_numpy((np.random.RandomState(7).randn(32) * 0.1).astype(np.float32)).to(dev)

    def render(scene, detailed=False):
        kw = {} if scene is None else {"baked": scene}
        with torch.no_grad():
            out = T.render(rays_o, rays_d, chunk=65536, near=near, far=far, use_viewdirs=False, ndc=False,
                           additional_pixel_information={"ray_bending_latents": lat[None].expand(n, 32)},
                           network_query_fn=None, perturb=0.0, N_importance=64, network_fine=fine, N_samples=64, network_fn=coarse,
                           white_bkgd=False, raw_noise_std=0.0, lindisp=False, detailed_output=detailed, **kw)
        return out if detailed else out[0]

    exact_full = render(None, detailed=True)
    exact = exact_full[0]
    pts = torch.cat([exact_full[3]["input_pts"].reshape(-1, 3), exact_full[3]["fine_input_pts"].reshape(-1, 3)])
    lo = (pts.min(0)[0].cpu().numpy() - np.float32(0.01)).astype(np.float32)
    hi = (pts.max(0)[0].cpu().numpy() + np.float32(0.01)).astype(np.float32)
    del exact_full, pts

    scenes, bake_ms = {}, {}
    G.bake_radiance(coarse, lo, hi, 64)   # warm-up
    for res in RESOLUTIONS:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        scenes[res] = G.BakedScene(G.bake_radiance(coarse, lo, hi, res), G.bake_radiance(fine, lo, hi, res))
        torch.cuda.synchronize()
        bake_ms[res] = (time.perf_counter() - t0) * 1e3

    configs = [None] + list(RESOLUTIONS)
    name = lambda c: "exact" if c is None else f"baked_{c}"
    for _ in range(args.warmup):
        for c in configs:
            render(None if c is None else scenes[c])
    ms = {c: [] for c in configs}
    for _ in range(args.steps):
        for c in configs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            render(None if c is None else scenes[c])
            e1.record()
            torch.cuda.synchronize()
            ms[c].append(e0.elapsed_time(e1))

    acc = {}
    for res in RESOLUTIONS:
        d = (render(scenes[res]) - exact).double()
        mse = float((d * d).mean())
        a = d.abs()
        acc[name(res)] = {"psnr_db": -10.0 * np.log10(mse) if mse > 0 else float("inf"), "max_abs_drgb": float(a.max()),
                          "mean_abs_drgb": float(a.mean()), "p99_abs_drgb": float(torch.quantile(a.reshape(-1).float(), 0.99)),
                          "pixels_over_0.1": float((a.max(1)[0] > 0.1).double().mean())}

    kinds = (_lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + _lib.DET_KERNEL_KINDS
             + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + _lib.MESH_KERNEL_KINDS
             + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS + _lib.OCCUPANCY_KERNEL_KINDS + _lib.TERMINATION_KERNEL_KINDS
             + _lib.DEFORM_KERNEL_KINDS + _lib.NORMAL_KERNEL_KINDS + _lib.LPIPS_MAP_KERNEL_KINDS + _lib.BAKED_KERNEL_KINDS)
    per = {}
    for c in configs:
        torch.cuda.synchronize()
        _lib.timing_enable(True)
        render(None if c is None else scenes[c])
        t = _lib.timing_read(kinds)
        _lib.timing_enable(False)
        per[name(c)] = {k: round(v[0], 4) for k, v in t.items() if v[1]}

    med = {c: float(np.median(ms[c])) for c in configs}
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "steps": args.steps, "warmup": args.warmup,
           "workload": "504x378 frame, 64c+64 importance (128f), det sampling, chunk=65536, untrained bench.py models, ray bender on",
           "grid_box": {"min": lo.tolist(), "max": hi.tolist()},
           "ms_median": {name(c): med[c] for c in configs},
           "speedup_vs_exact": {name(c): med[None] / med[c] for c in configs if c is not None},
           "accuracy_vs_exact": acc,
           "bake_ms_coarse_and_fine": {name(r): bake_ms[r] for r in RESOLUTIONS},
           "kernel_ms": per}
    _lib.device_error_check()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
