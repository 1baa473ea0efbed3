"""Surface normals on the GPU (geometry.density_gradient / vertex_normals, render(..., surface_normals=True)) against torch
fp32 autograd of the same network (the oracle's nerf_mlp and bender_forward on the model's fp32 parameters) on the same GPU.

    python scripts/bench_normals.py [--res 256 512] [--rounds 5] [--out DIR]

Workloads: the vertex normals of bench_mesh.py's 256^3 and 512^3 meshes of a seeded model with a ray bender (the frame's
latent, its median-density surface), and the surface normals of one 504 x 378 frame (one point per pixel, the rays of
O.make_rays at mid depth, per-ray latents).  Each is timed with CUDA events, the two arms alternating over the rounds;
medians are reported with the card's name, power limit and maximum SM clock read in the same run, one JSON line each.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle.nrnerf_oracle as O  # noqa: E402
from nonrigid_nerf_b200 import geometry as G  # noqa: E402
from scripts.bench_mesh import HI, LO, gpu_info, timed  # noqa: E402
from tests import helpers, normals_reference as R  # noqa: E402

TORCH_CHUNK = 1 << 18   # points per autograd pass of the torch arm (bounds its activation memory)


def torch_gradient(npar, bp, x, z):
    """d raw[3] / d x by torch fp32 autograd, in chunks."""
    out = torch.empty_like(x)
    for c in range(0, x.shape[0], TORCH_CHUNK):
        xc = x[c:c + TORCH_CHUNK].detach().requires_grad_(True)
        zc = z.expand(xc.shape[0], -1) if z.dim() == 1 else z[c:c + TORCH_CHUNK]
        bent = O.bender_forward(bp, xc, zc)["bent"]
        r = O.nerf_mlp(npar, O.positional_encoding(bent))[:, 3]
        out[c:c + TORCH_CHUNK] = torch.autograd.grad(r.sum(), xc)[0]
    return out


def compare(name, fused, reference, rounds, info, extra):
    fused(), reference()   # warm-up
    t = {"fused": [], "torch_fp32_autograd": []}
    for r in range(rounds):
        order = list(t) if r % 2 == 0 else list(reversed(list(t)))
        for k in order:
            t[k].append(timed(fused if k == "fused" else reference)[0])
    g, ref = fused(), reference()
    rel = float(((g - ref).norm(dim=1) / ref.norm(dim=1).clamp_min(1e-6)).median())
    line = {"workload": name, **extra, **{f"{k}_ms": round(statistics.median(v), 3) for k, v in t.items()},
            "speedup": round(statistics.median(t["torch_fp32_autograd"]) / statistics.median(t["fused"]), 2),
            "median_rel_diff_vs_torch": rel, "gpu": info}
    print(json.dumps(line), flush=True)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_normals: no CUDA device; GPU timings cannot be taken here")
    net, _, _, _ = helpers.build_models(O, 2024, "cuda:0", True)
    lat = O.make_rays(2024, 2)["latents"][0].cuda()
    npar, bp = R.params(net, device="cuda:0")
    npar = {k: [t.float() for t in v] if isinstance(v, list) else v.float() for k, v in npar.items()}
    bp = {k: [t.float() for t in v] for k, v in bp.items()}
    info = gpu_info()
    lines = []
    t = float(G.density_grid(net, LO, HI, 256, latent=lat).median())
    for n in args.res:
        mesh = G.extract_mesh(net, LO, HI, n, t, latent=lat, colors=False, rigidity=False)
        v = mesh.vertices
        lines.append(compare(f"vertex_normals_{n}", lambda: G.density_gradient(net, v, lat), lambda: torch_gradient(npar, bp, v, lat),
                             args.rounds, info, {"vertices": int(v.shape[0])}))
        del mesh, v
    r = O.make_rays(7, 504 * 378)
    pts = (r["rays_o"] + r["rays_d"] * (0.5 * (r["near"] + r["far"]))).cuda()
    lats = r["latents"].cuda()
    lines.append(compare("surface_normals_504x378", lambda: G.density_gradient(net, pts, lats), lambda: torch_gradient(npar, bp, pts, lats),
                         args.rounds, info, {"points": int(pts.shape[0])}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_normals.jsonl"), "w") as fh:
            fh.writelines(json.dumps(x) + "\n" for x in lines)


if __name__ == "__main__":
    main()
