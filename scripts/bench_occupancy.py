#!/usr/bin/env python3
"""Rendering time with an occupancy grid (render(..., occupancy=grid)) beside the same render without one, in one process.

    python scripts/bench_occupancy.py --steps 10 --warmup 3 [--out result.json]

Workload: scripts/bench_workloads.py's render workload -- a 504 x 378 full frame, fixed camera, one latent, 64 coarse + 64
importance samples (128 fine), deterministic sampling, chunk = 65536, under torch.no_grad() -- with the models bench.py
builds (create_nerf's default inits and one ray bender).  Those models are untrained, so their density says nothing about
which cells a trained scene leaves empty; the grids are synthetic instead: 128^3 cells over the box of the frame's
unbent sample points, each cell occupied with probability 1.0, 0.5, 0.2 or 0.05.  Reported per grid: the median frame
time (frames alternate between no grid and every grid, so drifting clocks hit all alike), the fraction of coarse samples
the grid keeps (looked up at the unbent points), whether the all-occupied grid reproduces the render without a grid bit
for bit, and one eager frame's per-kernel times from the library's timing.  Also the time of occupancy_grid() on the
coarse model at 128^3.  Prints one JSON line with the card's name and power limit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as B  # noqa: E402

FRACTIONS = (1.0, 0.5, 0.2, 0.05)
RES = 128


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
    from nonrigid_nerf_b200 import _lib, geometry as G, ops, run_nerf_helpers as H, train as T

    coarse, fine, bender = B.build_models(dev, H)
    Hh, Ww, focal = 378, 504, 252.6
    near, far = 0.0022, 1.0024
    j, i = np.meshgrid(np.arange(Hh, dtype=np.float32), np.arange(Ww, dtype=np.float32), indexing="ij")
    dirs = np.stack([(i - Ww * 0.5) / focal, -(j - Hh * 0.5) / focal, -np.ones_like(i)], -1).reshape(-1, 3).astype(np.float32)
    rays_d = torch.from_numpy(dirs).to(dev)
    rays_o = torch.zeros_like(rays_d)
    n = rays_d.shape[0]
    lat = torch.from_numpy((np.random.RandomState(7).randn(32) * 0.1).astype(np.float32)).to(dev)
    lo = np.minimum(dirs.min(0) * far, dirs.min(0) * near).astype(np.float32) - np.float32(0.05)
    hi = np.maximum(dirs.max(0) * far, dirs.max(0) * near).astype(np.float32) + np.float32(0.05)

    grids = {}
    rs = np.random.RandomState(3)
    for f in FRACTIONS:
        occ = rs.rand(RES, RES, RES) < f
        flat = np.zeros((occ.size + 31) // 32 * 32, bool)
        flat[:occ.size] = occ.reshape(-1)
        bits = torch.from_numpy(np.packbits(flat, bitorder="little").view("<i4").copy()).to(dev)
        grids[f] = G.OccupancyGrid(bits, lo, hi, (RES, RES, RES))

    def render(grid):
        kw = {} if grid is None else {"occupancy": grid}
        with torch.no_grad():
            return T.render(rays_o, rays_d, chunk=65536, near=near, far=far, use_viewdirs=False, ndc=False,
                            additional_pixel_information={"ray_bending_latents": lat[None].expand(n, 32)},
                            network_query_fn=None, perturb=0.0, N_importance=64, network_fine=fine, N_samples=64, network_fn=coarse,
                            white_bkgd=False, raw_noise_std=0.0, lindisp=False, **kw)[0]

    # fraction of coarse samples each grid keeps, looked up at the unbent points
    lib = _lib.load()
    rays8 = ops.pack_rays(rays_o, rays_d, near, far)
    z = ops.sample_coarse(rays8, 64, None, False)
    pts = (rays8[:, None, 0:3] + rays8[:, None, 3:6] * z[..., None]).reshape(-1, 3).contiguous()
    P = pts.shape[0]
    kept_frac = {}
    for f, g in grids.items():
        xyz = torch.empty(P, 3, device=dev)
        idx = torch.empty(P, dtype=torch.int32, device=dev)
        cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        ws = torch.empty(lib.nrn_occupancy_compact_workspace_bytes(P), dtype=torch.uint8, device=dev)
        cg = g.c_struct(dev)
        _lib.check(lib.nrn_occupancy_compact(C.byref(cg), pts.data_ptr(), P, 3, xyz.data_ptr(), idx.data_ptr(), cnt.data_ptr(),
                                             ws.data_ptr(), torch.cuda.current_stream().cuda_stream), "occupancy_compact")
        kept_frac[f] = int(cnt.item()) / P
    del pts, z

    configs = [None] + list(FRACTIONS)
    name = lambda c: "no_grid" if c is None else f"cells_{c:g}"
    for _ in range(args.warmup):
        for c in configs:
            render(None if c is None else grids[c])
    ms = {c: [] for c in configs}
    for _ in range(args.steps):
        for c in configs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            render(None if c is None else grids[c])
            e1.record()
            torch.cuda.synchronize()
            ms[c].append(e0.elapsed_time(e1))
    base = render(None)
    same = bool(torch.equal(base.view(torch.int32), render(grids[1.0]).view(torch.int32)))

    kinds = (_lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + _lib.DET_KERNEL_KINDS
             + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + _lib.MESH_KERNEL_KINDS
             + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS + _lib.OCCUPANCY_KERNEL_KINDS)
    per = {}
    for c in configs:
        torch.cuda.synchronize()
        _lib.timing_enable(True)
        render(None if c is None else grids[c])
        t = _lib.timing_read(kinds)
        _lib.timing_enable(False)
        per[name(c)] = {k: round(v[0], 4) for k, v in t.items() if v[1]}

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    G.occupancy_grid(coarse, lo, hi, RES, 10.0)   # warm-up
    e0.record()
    built = G.occupancy_grid(coarse, lo, hi, RES, 10.0)
    e1.record()
    torch.cuda.synchronize()

    med = {c: float(np.median(ms[c])) for c in configs}
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "steps": args.steps, "warmup": args.warmup,
           "workload": "504x378 frame, 64c+64 importance (128f), det sampling, chunk=65536, untrained bench.py models, ray bender on",
           "grid": f"{RES}^3 synthetic cells over the unbent samples' box",
           "ms_median": {name(c): med[c] for c in configs},
           "speedup_vs_no_grid": {name(c): med[None] / med[c] for c in configs if c is not None},
           "coarse_samples_kept": {name(c): kept_frac[c] for c in FRACTIONS},
           "all_occupied_equals_no_grid": same,
           "kernel_ms": per,
           "occupancy_grid_128_ms": e0.elapsed_time(e1), "occupancy_grid_128_fraction": built.occupied_fraction()}
    _lib.device_error_check()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
