"""The saved 8-bit images of a free-viewpoint run on the GPU (evaluation.frame_images: rgb, disp, the disparity video,
disp_jet, disp_phong, correspondences, rigidity, rigidity_jet) against the numpy path on the host cores, at 86 frames
(the example sequence's image count) of 1008 x 756.  The inputs are seeded random data on the device, as render(...,
surface_output=True) leaves them there; the host side copies the four fp32 inputs to host memory and runs the numpy
restatement in tests/frame_images_reference.py, and that copy is part of its time.

    python scripts/bench_frame_images.py [--frames 86] [--height 756] [--width 1008] [--reps 20] [--host-reps 2] [--out DIR]

Prints one JSON line: the median GPU time of the call (CUDA events around both launches, warmed up), the bytes it must
move at least and their rate against the 3.35 TB/s data-sheet HBM bandwidth, the host median, and the card's name and
power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nonrigid_nerf_b200 import evaluation as E  # noqa: E402
from tests import frame_images_reference as R  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=86)
    ap.add_argument("--height", type=int, default=756)
    ap.add_argument("--width", type=int, default=1008)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_images: no CUDA device; GPU timings cannot be taken here")
    f, h, w = args.frames, args.height, args.width
    g = torch.Generator(device="cuda").manual_seed(0)
    rgbs = torch.rand((f, h, w, 3), generator=g, device="cuda") * 1.2 - 0.1
    disps = torch.rand((f, h, w), generator=g, device="cuda") * (1.0 + torch.arange(f, device="cuda"))[:, None, None]
    pts = torch.rand((f, h * w, 3), generator=g, device="cuda") * 2.4 - 1.2
    rig = torch.rand((f, h * w), generator=g, device="cuda")
    lo, hi = [-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]

    call = lambda: E.frame_images(rgbs, disps, pts, rig, lo, hi)  # noqa: E731
    px = f * h * w
    # at least: the four inputs read once (12 + 4 + 12 + 4 bytes per pixel), the eight images written once (18 bytes)
    min_bytes = px * (12 + 4 + 12 + 4) + px * (3 + 1 + 1 + 3 + 3 + 3 + 1 + 3)
    res = {"workload": f"frame_images {f} x {w}x{h}", "gpu": gpu_info(), "reps": args.reps}
    ms = time_gpu(call, args.reps)
    res["gpu_ms"] = round(ms, 4)
    res["min_bytes"] = min_bytes
    res["GBps"] = round(min_bytes / (ms * 1e-3) / 1e9, 1)
    res["share_of_hbm_bound"] = round(min_bytes / HBM_BYTES_PER_S / (ms * 1e-3), 3)
    res["gpu_disps_only_ms"] = round(time_gpu(lambda: E.frame_images(disps=disps), args.reps), 4)   # the maxima + the disparity images

    host = []
    for _ in range(args.host_reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        hr, hd, hp, hg = (x.cpu().numpy() for x in (rgbs, disps, pts, rig))
        R.frame_images(hr, hd, hp, hg, lo, hi)
        host.append((time.perf_counter() - t) * 1e3)
    res["host_numpy_ms"] = round(statistics.median(host), 1)
    res["host_threads"] = torch.get_num_threads()
    res["speedup_vs_host"] = round(res["host_numpy_ms"] / ms, 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_frame_images.jsonl"), "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
