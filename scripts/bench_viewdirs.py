#!/usr/bin/env python3
"""Rendering throughput of the view-dependent head (use_viewdirs=True) beside the same render without it, in one process.

    python scripts/bench_viewdirs.py --steps 10 --warmup 3 [--out result.json]

Two workloads, each run with use_viewdirs=False and =True alternately (frame by frame), under torch.no_grad():
  frame: scripts/bench_workloads.py's render workload, a 504 x 378 full frame, fixed camera, one latent, 64 coarse + 128 fine
         samples, deterministic sampling, chunk = 65536;
  rays:  1024 rays of the same camera, 64 coarse + 128 fine.
Both models are built like bench.py's (create_nerf with default inits, one shared ray bender), the view-dependent one as
NeRF(use_viewdirs=True, input_ch_views=27).  Afterwards one eager frame of each runs with the library's per-kernel timing
(field kernel; bend pass and view-head kernel).  Prints one JSON line with the card's name and power limit."""
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
    from nonrigid_nerf_b200 import _lib, run_nerf_helpers as H, train as T

    coarse, fine, bender = B.build_models(dev, H)
    torch.manual_seed(1)
    kw = dict(D=8, W=256, input_ch=63, output_ch=5, skips=[4], input_ch_views=27, use_viewdirs=True, ray_bender=bender,
              ray_bending_latent_size=32, approx_nonrigid_viewdirs=True)
    coarse_v = H.NeRF(num_ray_samples=64, **kw).to(dev)
    fine_v = H.NeRF(num_ray_samples=128, **kw).to(dev)
    Hh, Ww, focal = 378, 504, 252.6
    j, i = np.meshgrid(np.arange(Hh, dtype=np.float32), np.arange(Ww, dtype=np.float32), indexing="ij")
    dirs = np.stack([(i - Ww * 0.5) / focal, -(j - Hh * 0.5) / focal, -np.ones_like(i)], -1).reshape(-1, 3).astype(np.float32)
    rays_d = torch.from_numpy(dirs).to(dev)
    rays_o = torch.zeros_like(rays_d)
    lat = torch.from_numpy((np.random.RandomState(7).randn(32) * 0.1).astype(np.float32)).to(dev)
    sub = torch.from_numpy(np.random.RandomState(8).choice(rays_d.shape[0], 1024, replace=False)).to(dev)

    def render(views, ro, rd):
        c, f = (coarse_v, fine_v) if views else (coarse, fine)
        with torch.no_grad():
            return T.render(ro, rd, chunk=65536, near=0.0022, far=1.0024, use_viewdirs=views, ndc=False,
                            additional_pixel_information={"ray_bending_latents": lat[None].expand(ro.shape[0], 32)},
                            network_query_fn=None, perturb=0.0, N_importance=64, network_fine=f, N_samples=64, network_fn=c,
                            white_bkgd=False, raw_noise_std=0.0, lindisp=False)[0]

    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "steps": args.steps, "warmup": args.warmup}
    for name, ro, rd in (("frame_504x378", rays_o, rays_d), ("rays_1024", rays_o[sub], rays_d[sub])):
        for k in range(args.warmup):
            render(False, ro, rd)
            render(True, ro, rd)
        ms = {False: [], True: []}
        for k in range(args.steps):   # alternate, so drifting clocks hit both alike
            for views in (False, True):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                render(views, ro, rd)
                e1.record()
                torch.cuda.synchronize()
                ms[views].append(e0.elapsed_time(e1))
        n = ro.shape[0]
        med = {v: float(np.median(ms[v])) for v in ms}
        res[name] = {"rays": n, "ms_median": {"use_viewdirs=False": med[False], "use_viewdirs=True": med[True]},
                     "rays_per_sec": {"use_viewdirs=False": n / (med[False] * 1e-3), "use_viewdirs=True": n / (med[True] * 1e-3)},
                     "slowdown": med[True] / med[False]}
        kinds = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS
        per = {}
        for views in (False, True):
            torch.cuda.synchronize()
            _lib.timing_enable(True)
            render(views, ro, rd)
            t = _lib.timing_read(kinds)
            _lib.timing_enable(False)
            per["use_viewdirs=" + str(views)] = {k: round(v[0], 4) for k, v in t.items() if v[1]}
        res[name]["kernel_ms"] = per
    _lib.device_error_check()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
