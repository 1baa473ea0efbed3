"""Mesh extraction on the GPU (geometry.extract_mesh) of a seeded model with a ray bender, at 256^3 and 512^3, split into
its three parts: the density grid (the fused field kernel, one z-plane per launch), marching cubes over that grid, and the
vertex attributes (colours and rigidity: one more point-mode pass over the vertices).  The numpy restatement
(tests/mesh_reference.py) runs on the host cores over the same 256^3 grid for comparison.

    python scripts/bench_mesh.py [--res 256 512] [--rounds 5] [--out DIR]

The parts are timed with CUDA events around each call: density_grid, marching_cubes of its grid, and extract_mesh with and
without attributes (attributes = the difference), taken in alternating order over several rounds, medians reported.  The
threshold is the median density of the 256^3 grid, so the surface is large.  Prints one JSON line per resolution, with the
card's name, power limit and maximum SM clock read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle.nrnerf_oracle as O  # noqa: E402
from nonrigid_nerf_b200 import geometry as G  # noqa: E402
from tests import helpers, mesh_reference as R  # noqa: E402

LO, HI = [-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh: no CUDA device; GPU timings cannot be taken here")
    net, _, _, _ = helpers.build_models(O, 2024, "cuda:0", True)
    lat = O.make_rays(2024, 2)["latents"][0].cuda()
    info = gpu_info()
    t = float(G.density_grid(net, LO, HI, 256, latent=lat).median())
    for n in args.res:
        calls = {
            "density": lambda: G.density_grid(net, LO, HI, n, latent=lat),
            "mesh_no_attributes": lambda: G.extract_mesh(net, LO, HI, n, t, latent=lat, colors=False, rigidity=False),
            "mesh": lambda: G.extract_mesh(net, LO, HI, n, t, latent=lat),
        }
        sigma = calls["density"]()
        calls["marching_cubes"] = lambda: G.marching_cubes(sigma, LO, HI, t)
        for fn in calls.values():   # warm-up of every shape
            fn()
        times = {k: [] for k in calls}
        for r in range(args.rounds):
            order = list(calls) if r % 2 == 0 else list(reversed(list(calls)))
            for k in order:
                ms, out = timed(calls[k])
                times[k].append(ms)
                if k == "mesh":
                    mesh = out
                del out
        med = {k: statistics.median(v) for k, v in times.items()}
        res = {"workload": f"extract_mesh {n}^3 (bender, one latent)", "gpu": info, "rounds": args.rounds, "threshold": round(t, 4),
               "vertices": int(mesh.vertices.shape[0]), "faces": int(mesh.faces.shape[0]),
               "density_ms": round(med["density"], 2), "marching_cubes_ms": round(med["marching_cubes"], 2),
               "attributes_ms": round(med["mesh"] - med["mesh_no_attributes"], 2),
               "extract_mesh_ms": round(med["mesh"], 2), "extract_mesh_no_attributes_ms": round(med["mesh_no_attributes"], 2),
               "density_ns_per_point": round(med["density"] * 1e6 / n ** 3, 3),
               "spread_ms": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()}}
        if n == 256:
            host = sigma.cpu().numpy()
            t0 = time.perf_counter()
            R.marching_cubes(host, LO, HI, np.float32(t))
            res["host_numpy_marching_cubes_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            res["host_threads"] = torch.get_num_threads()
        del sigma
        line = json.dumps(res)
        print(line)
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "bench_mesh.jsonl"), "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
