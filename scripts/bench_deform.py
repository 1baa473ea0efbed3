"""The inverse ray bender on the GPU (geometry.deform_points) against a torch fp32 Newton on the same GPU, the way a user
would invert the bender without this library (vmap(jacfwd) for J, torch.linalg.solve_ex, the same start, freezing rule
and iteration count).  Workload: 2 M canonical points in the example volume (about the vertex count of a 512^3 mesh) x
86 latents ~ N(0, 0.1^2) (the example sequence's frame count), benders of oracle.make_bender_params with offsets of
std 0.01 and 0.1.

    python scripts/bench_deform.py [--points 2000000] [--frames 86] [--torch-frames 1] [--reps 3] [--out DIR]

The two are alternated in one call: per repetition the kernel on all frames, then torch on --torch-frames frames.
Prints one JSON line: per bender the median time per frame of each and points*frames/s, the histogram of Newton steps to
convergence (from the converged counts of calls with 0..iterations steps: a point's result does not depend on how long
the others iterate), the achieved FLOP/s from the shape-derived operation count below, and the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle.nrnerf_oracle as O  # noqa: E402
from nonrigid_nerf_b200 import geometry as G, run_nerf_helpers as H  # noqa: E402
from tests import helpers  # noqa: E402

LO, HI = np.array([-1.2, -1.0, -1.4]), np.array([1.1, 1.0, 0.6])

# Operations of the bender network per point: multiply-adds x 2 of its layers (offset MLP 35-64-64-64-64-3, rigidity MLP
# 3-32-32-1).  One evaluation of b is all of them; one tangent J e_a skips the first layers (their tangent is a column of
# W0), so it is the rest.  A Newton step is one evaluation and three tangents.
NET_FLOP = 2 * (35 * 64 + 3 * 64 * 64 + 64 * 3 + 3 * 32 + 32 * 32 + 32)
TAN_FLOP = 2 * (3 * 64 * 64 + 64 * 3 + 32 * 32 + 32)


def gpu_info():
    try:
        name, limit = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                     capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(", ")
        return name, limit
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(), "unknown"


def torch_newton(bp32, c, z, iterations, tol):
    """The same iteration in torch fp32 for one latent z [32]: x [P, 3], converged [P]."""
    from torch.func import jacfwd, vmap
    zz = z.expand(c.shape[0], 32)

    def bend(x):
        return O.bender_forward(bp32, x, zz)["bent"]

    def one(xi, zi):
        return O.bender_forward(bp32, xi[None], zi[None])["bent"][0]

    jac = vmap(jacfwd(one, argnums=0))
    x = c - O.bender_forward(bp32, c, zz)["masked_offsets"]
    frozen = torch.zeros(c.shape[0], dtype=torch.bool, device=c.device)
    for it in range(iterations + 1):
        g = bend(x) - c
        frozen = frozen | (g.norm(dim=1) <= tol)
        if it == iterations:
            break
        st, info = torch.linalg.solve_ex(jac(x, zz), g)
        st = torch.where(((info == 0) & torch.isfinite(st).all(1)).unsqueeze(1), st, g)
        x = torch.where(frozen.unsqueeze(1), x, x - st)
    return x, frozen


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=2_000_000)
    ap.add_argument("--frames", type=int, default=86)
    ap.add_argument("--torch-frames", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iterations", type=int, default=G.DEFORM_ITERATIONS)
    ap.add_argument("--tol", type=float, default=G.DEFORM_TOL)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = "cuda:0"
    if not torch.cuda.is_available():
        raise SystemExit("bench_deform: no CUDA device")
    name, limit = gpu_info()
    embed_fn, ch = H.get_embedder(10, 0)
    c = torch.from_numpy(np.random.RandomState(1).uniform(LO, HI, size=(args.points, 3)).astype(np.float32)).to(dev)
    z = torch.from_numpy((np.random.RandomState(2).randn(args.frames, 32) * 0.1).astype(np.float32)).to(dev)
    res = {"gpu": name, "power_limit": limit, "points": args.points, "frames": args.frames, "iterations": args.iterations,
           "tol": args.tol, "benders": {}}
    for std in (0.01, 0.1):
        bp = O.make_bender_params(7, offset_std=std)
        bender = helpers.load_bender_module(H.ray_bending(ch, 32, "simple_neural", embed_fn), bp).to(dev)
        bp32 = {k: [t.to(dev) for t in v] for k, v in bp.items()}
        with torch.no_grad():
            G.deform_points(bender, c, z[:1], args.iterations, args.tol)          # warm-up: pack, module load
            torch_newton(bp32, c, z[0], args.iterations, args.tol)
            torch.cuda.synchronize()
            ker, tor = [], []
            for _ in range(args.reps):
                ms, d = timed(lambda: G.deform_points(bender, c, z, args.iterations, args.tol))
                ker.append(ms / args.frames)
                ms, (xt, ct) = timed(lambda: [torch_newton(bp32, c, z[f], args.iterations, args.tol)
                                              for f in range(args.torch_frames)][-1])
                tor.append(ms / args.torch_frames)
            f0 = args.torch_frames - 1
            agree = float(((xt - d.points[f0]).norm(dim=1)[ct & d.converged[f0]]).max())
            # steps to convergence over 8 frames: converged after k steps minus after k - 1 (bucket 1 also holds the points
            # whose start x_0 is already within tol)
            counts = [int(G.deform_points(bender, c, z[:8], k, args.tol).converged.sum()) for k in range(1, args.iterations + 1)]
        n8 = args.points * min(8, args.frames)
        hist = [counts[0]] + [counts[k] - counts[k - 1] for k in range(1, len(counts))]
        never = n8 - counts[-1]
        # a point frozen after k steps costs k + 2 evaluations (start, x_0 .. x_k) and 3 k tangents; bucket 1 counted as
        # k = 0 and the warpgroups' idle rows not at all, so this is a lower bound of the work done
        flop = sum(((k + 2) * NET_FLOP + 3 * k * TAN_FLOP) * n for k, n in enumerate(hist))
        flop += ((args.iterations + 2) * NET_FLOP + 3 * args.iterations * TAN_FLOP) * never
        ker_med, tor_med = statistics.median(ker), statistics.median(tor)
        res["benders"][str(std)] = {
            "kernel_ms_per_frame": ker_med, "torch_fp32_ms_per_frame": tor_med, "speedup": tor_med / ker_med,
            "kernel_points_frames_per_s": args.points / (ker_med * 1e-3),
            "torch_points_frames_per_s": args.points / (tor_med * 1e-3),
            "converged_fraction": float(d.converged.float().mean()),
            "steps_to_converge_hist_8_frames": {"<=1": hist[0], **{str(k + 1): n for k, n in enumerate(hist) if k},
                                                "never": never},
            "network_tflops_lower_bound": flop / min(8, args.frames) / (ker_med * 1e-3) / 1e12,
            "max_kernel_vs_torch_distance": agree,
            "kernel_ms_all": ker, "torch_ms_all": tor,
        }
        del d
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        tag = name.lower().replace("nvidia ", "").replace(" ", "-")
        watts = limit.split(" ")[0].split(".")[0]
        tag += f"_{watts}w" if watts.isdigit() else ""
        with open(os.path.join(args.out, f"r21_{tag}_bench_deform.jsonl"), "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
