#!/usr/bin/env python3
"""Rendering time with early ray termination (render(..., early_termination=t)) beside the same render without it, in one
process.

    python scripts/bench_termination.py --steps 6 --warmup 2 [--sweep 8,16,32,64] [--out result.json]

Workload: scripts/bench_workloads.py's render workload -- a 504 x 378 full frame, fixed camera, one latent, 64 coarse + 64
importance samples (128 fine), deterministic sampling, chunk = 65536, under torch.no_grad() -- with the models bench.py
builds (create_nerf's default inits and one ray bender).  Those models are untrained and almost transparent, so the
densities are synthetic: a constant is added to the sigma bias of both models so that a median ray's coarse
transmittance crosses 1e-4 at about 25, 50 or 75 % of [near, far].  For each level: median frame times, with frames
alternating between no termination and t = 1e-4, each also with a synthetic 128^3 grid of which 20 % of the cells are
occupied; the fraction of samples each pass evaluates (mean termination_index / S); one eager frame's per-kernel times from
the library's timing, with the bend pass's share of the frame; and whether t = 0 reproduces the render without
termination bit for bit.

--sweep K1,K2,...: for each segment size, copy the package to a temporary directory, rebuild it there with
-DNRN_TERM_SEGMENT=K (only c_abi.cu depends on it) and time the same frames in a child process.  --lib-root DIR imports
the package from DIR (what the sweep's children do).  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sweep", default="", help="comma-separated segment sizes to rebuild and time")
    ap.add_argument("--lib-root", default=None, help="import nonrigid_nerf_b200 from this directory")
    ap.add_argument("--timing-only", action="store_true", help="frame times only (the sweep's children)")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    return ap.parse_args()


args = _args()
sys.path.insert(0, ROOT)
if args.lib_root:
    sys.path.insert(0, os.path.abspath(args.lib_root))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nonrigid_nerf_b200  # noqa: E402,F401  (from --lib-root when given: bench.py below puts ROOT first on sys.path)
import bench as B  # noqa: E402

if args.lib_root:
    assert os.path.dirname(os.path.dirname(os.path.abspath(nonrigid_nerf_b200.__file__))) == os.path.abspath(args.lib_root)

CROSS = (0.25, 0.5, 0.75)
T_TERM = 1e-4
RES = 128


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:   # the number is informative only
        return None


def sweep(sizes, steps, warmup):
    """{K: the child's frame times} with one rebuild per segment size."""
    out = {}
    for K in sizes:
        tmp = tempfile.mkdtemp(prefix=f"nrn_term_k{K}_")
        try:
            shutil.copytree(os.path.join(ROOT, "nonrigid_nerf_b200"), os.path.join(tmp, "nonrigid_nerf_b200"), symlinks=True)
            shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
            csrc = os.path.join(tmp, "nonrigid_nerf_b200", "csrc")
            os.utime(os.path.join(csrc, "c_abi.cu"))   # newer than its object: the only file rebuilt
            subprocess.run(["make", "-C", csrc, f"EXTRA=-DNRN_TERM_SEGMENT={K}"], check=True, capture_output=True)
            res = subprocess.run([sys.executable, os.path.abspath(__file__), "--lib-root", tmp, "--timing-only", "--steps", str(steps),
                                  "--warmup", str(warmup)], check=True, capture_output=True, text=True)
            line = json.loads(res.stdout.strip().splitlines()[-1])
            assert line["segment"] == K, line
            out[K] = line["ms_median"]
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    return out


def main():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from nonrigid_nerf_b200 import _lib, geometry as G, run_nerf_helpers as H, train as T
    K = _lib.load().nrn_termination_segment()

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
    occ = np.random.RandomState(3).rand(RES, RES, RES) < 0.2
    flat = np.zeros((occ.size + 31) // 32 * 32, bool)
    flat[:occ.size] = occ.reshape(-1)
    grid = G.OccupancyGrid(torch.from_numpy(np.packbits(flat, bitorder="little").view("<i4").copy()).to(dev), lo, hi, (RES, RES, RES))
    dnorm = float(np.median(np.linalg.norm(dirs, axis=-1)))
    bias0 = (coarse.output_linear.bias.detach().clone(), fine.output_linear.bias.detach().clone())

    def set_density(cross):
        sigma = np.log(1e4) / (cross * (far - near) * dnorm)
        with torch.no_grad():
            for net, b0 in zip((coarse, fine), bias0):
                net.output_linear.bias.copy_(b0)
                net.output_linear.bias[3] += sigma

    def render(t=None, g=None, extras=False):
        kw = {}
        if t is not None:
            kw["early_termination"] = t
        if g is not None:
            kw["occupancy"] = g
        with torch.no_grad():
            out = T.render(rays_o, rays_d, chunk=65536, near=near, far=far, use_viewdirs=False, ndc=False,
                           additional_pixel_information={"ray_bending_latents": lat[None].expand(n, 32)},
                           network_query_fn=None, perturb=0.0, N_importance=64, network_fine=fine, N_samples=64, network_fn=coarse,
                           white_bkgd=False, raw_noise_std=0.0, lindisp=False, **kw)
        return out if extras else out[0]

    configs = [(None, None), (T_TERM, None), (None, grid), (T_TERM, grid)]
    name = lambda c: ("terminate_1e-4" if c[0] is not None else "no_termination") + ("_grid_20pct" if c[1] is not None else "")
    ms, evaluated, same_t0, kernel_ms, bend_share = {}, {}, {}, {}, {}
    for cross in CROSS:
        lvl = f"cross_{int(cross * 100)}pct"
        set_density(cross)
        for _ in range(args.warmup):
            for c in configs:
                render(*c)
        times = {name(c): [] for c in configs}
        for _ in range(args.steps):
            for c in configs:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                render(*c)
                e1.record()
                torch.cuda.synchronize()
                times[name(c)].append(e0.elapsed_time(e1))
        ms[lvl] = {k: float(np.median(v)) for k, v in times.items()}
        if args.timing_only:
            continue
        ex = render(T_TERM, None, True)[3]
        evaluated[lvl] = {"coarse": float(ex["termination_index0"].float().mean()) / 64,
                          "fine": float(ex["termination_index"].float().mean()) / 128}
        base, zero = render(None, None, True), render(0.0, None, True)
        same_t0[lvl] = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(base[:3], zero[:3]))
        kinds = (_lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + _lib.DET_KERNEL_KINDS
                 + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + _lib.MESH_KERNEL_KINDS
                 + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS + _lib.OCCUPANCY_KERNEL_KINDS + _lib.TERMINATION_KERNEL_KINDS)
        kernel_ms[lvl] = {}
        for c in configs:
            torch.cuda.synchronize()
            _lib.timing_enable(True)
            render(*c)
            tm = _lib.timing_read(kinds)
            _lib.timing_enable(False)
            kernel_ms[lvl][name(c)] = {k: round(v[0], 4) for k, v in tm.items() if v[1]}
        per = kernel_ms[lvl][name((T_TERM, None))]
        bend_share[lvl] = per.get("termination_bend", 0.0) / ms[lvl][name((T_TERM, None))]

    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "steps": args.steps, "warmup": args.warmup,
           "segment": K, "ms_median": ms}
    if not args.timing_only:
        res.update({
            "workload": "504x378 frame, 64c+64 importance (128f), det sampling, chunk=65536, bench.py models with a bender and a "
                        "synthetic sigma bias; t=1e-4",
            "grid": f"{RES}^3 synthetic cells over the unbent samples' box, 20 % occupied",
            "speedup_vs_no_termination": {lvl: {"no_grid": v["no_termination"] / v["terminate_1e-4"],
                                                "grid_20pct": v["no_termination_grid_20pct"] / v["terminate_1e-4_grid_20pct"]}
                                          for lvl, v in ms.items()},
            "samples_evaluated_fraction": evaluated,
            "t0_equals_no_termination": same_t0,
            "bend_pass_share_of_terminated_frame": bend_share,
            "kernel_ms": kernel_ms,
        })
        sizes = [int(s) for s in args.sweep.split(",") if s]
        if sizes:
            res["segment_sweep_ms_median"] = sweep(sizes, args.steps, args.warmup)
    _lib.device_error_check()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
