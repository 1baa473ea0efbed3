#!/usr/bin/env python3
"""Rendering time and accuracy with baked per-frame deformation grids (render(..., baked=BakedScene(coarse, fine,
deformation))) beside the exact render and the radiance-only baked render, in one process.

    python scripts/bench_baked_deformation.py --steps 10 --warmup 3 [--out result.json]

Workload: scripts/bench_baked.py's -- a 504 x 378 full frame, fixed camera, one latent, 64 coarse + 64 importance
samples (128 fine), deterministic sampling, chunk = 65536, under torch.no_grad(), bench.py's models with a ray bender --
with the bender's two zero-initialised output layers re-drawn (oracle.make_bender_params(7, offset_std=0.1)), since an
untrained bender is the identity and its bake would measure nothing.  Radiance grids: 256^3 over the box of the exact
frame's bent sample points (padded by 0.01).  Deformation grids: one frame, 64^3, 128^3 and 256^3 over the box of the
exact frame's observation-space sample points (padded by 0.01), so that no ray falls back, and one 128^3 grid whose box
is cut in x at the 10th percentile of the far x of the rays towards +x, so that about half the rays leave the box
partway and fall back.  Reported per configuration: the median frame time (frames alternate between every configuration,
so drifting clocks hit all alike), one eager frame's per-kernel times from the library's timing, the bake time and bytes
per frame, PSNR against the exact frame and against the radiance-only baked frame, and the share of rays that fall back
in each pass.  The models are untrained.  Prints one JSON line with the card's name and power limit, read in the same
run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as B  # noqa: E402
import oracle.nrnerf_oracle as O  # noqa: E402
from scripts.bench_baked import power_limit_w  # noqa: E402

DEFORM_RESOLUTIONS = (64, 128, 256)
RADIANCE_RESOLUTION = 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from nonrigid_nerf_b200 import _lib, geometry as G, ops, run_nerf_helpers as H, train as T

    coarse, fine, bender = B.build_models(dev, H)
    bp = O.make_bender_params(7, offset_std=0.1)
    with torch.no_grad():
        bender.network[4].weight.copy_(bp["net_w"][4])
        bender.rigidity_network[2].weight.copy_(bp["rig_w"][2])
        bender.rigidity_network[2].bias.copy_(bp["rig_b"][2])
    ops.note_parameters_changed()
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

    def box(p):
        return ((p.min(0)[0].cpu().numpy() - np.float32(0.01)).astype(np.float32),
                (p.max(0)[0].cpu().numpy() + np.float32(0.01)).astype(np.float32))

    exact_full = render(None, detailed=True)
    exact = exact_full[0]
    ex = exact_full[3]
    rlo, rhi = box(torch.cat([ex["input_pts"].reshape(-1, 3), ex["fine_input_pts"].reshape(-1, 3)]))
    obs = torch.cat([ex["initial_input_pts"].reshape(-1, 3), ex["fine_initial_input_pts"].reshape(-1, 3)])
    dlo, dhi = box(obs)
    # the rays fan out from the camera at x = 0: cut at the 10th percentile of the last sample's x over the rays towards
    # +x, so the rays towards -x and the slowest tenth of the others lie inside, and the rest, about half of all rays,
    # start inside, leave the box partway and fall back
    far_x = ex["fine_initial_input_pts"][:, -1, 0]
    half_hi = dhi.copy()
    half_hi[0] = np.float32(float(torch.quantile(far_x[far_x > 0], 0.1)))
    del exact_full, ex, obs

    base = G.BakedScene(G.bake_radiance(coarse, rlo, rhi, RADIANCE_RESOLUTION), G.bake_radiance(fine, rlo, rhi, RADIANCE_RESOLUTION))
    G.bake_deformation(bender, lat, dlo, dhi, 32)   # warm-up
    scenes, bake_ms, grid_bytes = {"exact": None, "radiance_only": base}, {}, {}
    for name, res, hi in [(f"deformed_{r}", r, dhi) for r in DEFORM_RESOLUTIONS] + [("deformed_128_half_box", 128, half_hi)]:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        grid = G.bake_deformation(bender, lat, dlo, hi, res)
        torch.cuda.synchronize()
        bake_ms[name] = (time.perf_counter() - t0) * 1e3
        grid_bytes[name] = grid.values[0].numel() * grid.values.element_size()
        scenes[name] = G.BakedScene(base.coarse, base.fine, grid.frame(0))

    names = list(scenes)
    for _ in range(args.warmup):
        for c in names:
            render(scenes[c])
    ms = {c: [] for c in names}
    for _ in range(args.steps):
        for c in names:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            render(scenes[c])
            e1.record()
            torch.cuda.synchronize()
            ms[c].append(e0.elapsed_time(e1))

    def psnr(a, b):
        mse = float(((a - b).double() ** 2).mean())
        return -10.0 * np.log10(mse) if mse > 0 else float("inf")

    radiance_only = render(base)
    acc, fallback = {}, {}
    for c in names[1:]:
        full = render(scenes[c], detailed=True)
        acc[c] = {"psnr_vs_exact_db": psnr(full[0], exact), "psnr_vs_radiance_only_db": psnr(full[0], radiance_only)}
        d = scenes[c].deformation
        if d is not None:   # a ray falls back unless every sample is finite and inside the box
            lo_t, hi_t = torch.from_numpy(d.grid.min_point).to(dev), torch.from_numpy(d.grid.max_point).to(dev)
            share = lambda x: float((~((x >= lo_t) & (x <= hi_t)).all(-1).all(-1)).double().mean())
            fallback[c] = {"coarse": share(full[3]["initial_input_pts"]), "fine": share(full[3]["fine_initial_input_pts"])}
        del full

    kinds = (_lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + _lib.DET_KERNEL_KINDS
             + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + _lib.MESH_KERNEL_KINDS
             + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS + _lib.OCCUPANCY_KERNEL_KINDS + _lib.TERMINATION_KERNEL_KINDS
             + _lib.DEFORM_KERNEL_KINDS + _lib.NORMAL_KERNEL_KINDS + _lib.LPIPS_MAP_KERNEL_KINDS + _lib.BAKED_KERNEL_KINDS
             + _lib.DEFORMATION_KERNEL_KINDS)
    per = {}
    for c in names:
        torch.cuda.synchronize()
        _lib.timing_enable(True)
        render(scenes[c])
        t = _lib.timing_read(kinds)
        _lib.timing_enable(False)
        per[c] = {k: round(v[0], 4) for k, v in t.items() if v[1]}

    med = {c: float(np.median(ms[c])) for c in names}
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "steps": args.steps, "warmup": args.warmup,
           "workload": "504x378 frame, 64c+64 importance (128f), det sampling, chunk=65536, bench.py models, bender output layers "
                       "re-drawn (offset_std=0.1), radiance grids 256^3",
           "radiance_box": {"min": rlo.tolist(), "max": rhi.tolist()},
           "deformation_box": {"min": dlo.tolist(), "max": dhi.tolist(), "half_box_max_x": float(half_hi[0])},
           "ms_median": med,
           "ms_all": ms,
           "speedup_vs_radiance_only": {c: med["radiance_only"] / med[c] for c in names[2:]},
           "accuracy": acc,
           "fallback_ray_share": fallback,
           "bake_ms": bake_ms,
           "grid_bytes_per_frame": grid_bytes,
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
