"""Frame correspondences on the GPU (correspondence.match_frames) against scipy's cKDTree on the host cores, the way a
user matches surface points without this library.  Frames are a wavy height field seen from above that drifts a little
from frame to frame (tests/test_match_gpu.py), 10 % of the pixels masked.  Workloads: 86 frames at 504 x 378 (the example
sequence) tracked from frame 0 (one query frame against 86 targets) and frame to next frame (85 pairs), each with and
without the round trip, and one pair at 1008 x 756.

    python scripts/bench_match.py [--reps 10] [--host-pairs 4] [--out DIR]

Prints one JSON line: per workload the median GPU time of match_frames and of its two timing kinds (grid builds,
queries; CUDA events, warmed up), the host cKDTree time per pair (build + query, all cores; the round trip adds a tree of
the query frame and a second query) and its estimate for all pairs, and the card's name and power limit.
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

from nonrigid_nerf_b200 import _lib, correspondence as M  # noqa: E402

ALL_KINDS = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + \
    _lib.DET_KERNEL_KINDS + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + \
    _lib.MESH_KERNEL_KINDS + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def time_gpu(fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def frames(f, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    v, u = torch.meshgrid(torch.linspace(-0.75, 0.75, h, device="cuda"), torch.linspace(-1, 1, w, device="cuda"), indexing="ij")
    shift = 0.01 * torch.arange(f, device="cuda")[:, None, None]
    uu = u[None] + shift
    z = 0.2 * torch.sin(3 * uu) * torch.cos(2 * v)[None]
    pts = torch.stack([uu, v[None].expand_as(uu), z], -1)
    pts = pts + 1e-3 * torch.randn(pts.shape, generator=g, device="cuda")
    mask = torch.rand((f, h, w), generator=g, device="cuda") > 0.1
    return pts.contiguous(), mask


def host_pair(spatial, q, qm, t, tm, round_trip):
    t0 = time.perf_counter()
    tv = t.reshape(-1, 3)[tm.reshape(-1)]
    qv = q.reshape(-1, 3)[qm.reshape(-1)]
    _, j = spatial.cKDTree(tv).query(qv, workers=-1)
    if round_trip:
        spatial.cKDTree(qv).query(tv[j], workers=-1)
    return (time.perf_counter() - t0) * 1e3


def workload(q, qm, t, tm, round_trip, reps, host_pairs, spatial):
    res = {"query_frames": q.shape[0], "target_frames": t.shape[0], "height": q.shape[1], "width": q.shape[2],
           "round_trip": round_trip}
    call = lambda: M.match_frames(q, t, qm, tm, round_trip=round_trip)
    ms = time_gpu(call, reps)
    res["gpu_ms"] = round(ms, 3)
    _lib.timing_enable(True)
    for _ in range(reps):
        call()
    tk = _lib.timing_read(ALL_KINDS)
    _lib.timing_enable(False)
    for k in _lib.MATCH_KERNEL_KINDS:
        res[f"{k}_ms"] = round(tk[k][0] / reps, 3)
    out = call()
    res["matched_fraction"] = round(float((out.index >= 0).float().mean()), 4)
    if round_trip:
        res["consistent_fraction"] = round(float(out.consistent.float().mean()), 4)
    pairs = max(q.shape[0], t.shape[0])
    if spatial is not None:
        n = min(host_pairs, pairs)
        qs, qms, ts, tms = (x.cpu().numpy().astype(np.float64) if x.dtype == torch.float32 else x.cpu().numpy()
                            for x in (q, qm, t, tm))
        sel = lambda a, k: a[0 if a.shape[0] == 1 else k]
        host_pair(spatial, sel(qs, 0), sel(qms, 0), sel(ts, 0), sel(tms, 0), round_trip)   # warm-up
        host = statistics.median(host_pair(spatial, sel(qs, k), sel(qms, k), sel(ts, k), sel(tms, k), round_trip)
                                 for k in range(n))
        res["host_ckdtree_ms_per_pair"] = round(host, 1)
        res["host_ckdtree_ms_all_pairs_estimated"] = round(host * pairs, 1)
        res["speedup_vs_host"] = round(host * pairs / ms, 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-pairs", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_match: no CUDA device; GPU timings cannot be taken here")
    try:
        import scipy.spatial as spatial
    except ImportError:
        spatial = None
    res = {"workload": "match_frames", "gpu": gpu_info(), "reps": args.reps, "host_threads": os.cpu_count()}
    pts, mask = frames(86, 378, 504, 0)
    for rt in (False, True):
        tag = "_round_trip" if rt else ""
        res["track_from_frame0_504x378" + tag] = workload(pts[:1], mask[:1], pts, mask, rt, args.reps, args.host_pairs, spatial)
        res["frame_to_next_504x378" + tag] = workload(pts[:-1], mask[:-1], pts[1:], mask[1:], rt, args.reps, args.host_pairs, spatial)
    big, bmask = frames(2, 756, 1008, 1)
    for rt in (False, True):
        res["pair_1008x756" + ("_round_trip" if rt else "")] = workload(big[:1], bmask[:1], big[1:], bmask[1:], rt, args.reps,
                                                                        args.host_pairs, spatial)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_match.jsonl"), "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
