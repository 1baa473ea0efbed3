"""The whole evaluation of a free-viewpoint run on the GPU against the numpy / scipy path on the host cores: PSNR, SSIM
(with its map) and both error images of 37 test frames, jet and Blinn-Phong images of their disparity maps, and the
background-stability map, at 504 x 378 (the example sequence's resolution).  Frames are seeded random data already on
the device (the GPU side) or in host memory (the host side); the host side is the fp64 restatement in
tests/eval_reference.py (scipy.ndimage in place of scikit-image, which it restates).

    python scripts/bench_evaluation.py [--frames 37] [--height 378] [--width 504] [--reps 20] [--host-reps 3] [--out DIR]

Prints one JSON line: median GPU time per stage and in total (CUDA events, warmed up), the bytes each stage must move
and their rate, the host median, and the card's name and power limit.
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

from nonrigid_nerf_b200 import evaluation as E  # noqa: E402
from tests import eval_reference as R  # noqa: E402

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


def host_evaluation(gt, gen, disps):
    mask = R.mask_from(gt[0])
    lut8 = R.to8b(R.jet_lut())
    for i in range(gt.shape[0]):
        g, r = R.apply_mask(gt[i], gen[i], mask)
        R.psnr(g, r)
        _, S = R.ssim(g, r)
        lut8[R.lut_index(R.error_rgb_value(g, r))]
        lut8[R.lut_index(R.error_ssim_value(S))]
        R.jet_lut()[R.lut_index(disps[i])]
        R.phong(disps[i])
    R.std_image(gen)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=37)
    ap.add_argument("--height", type=int, default=378)
    ap.add_argument("--width", type=int, default=504)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluation: no CUDA device; GPU timings cannot be taken here")
    f, h, w = args.frames, args.height, args.width
    gt, gen = R.frames("masked", f, h, w, seed=0)
    disps = np.random.default_rng(1).random((f, h, w), dtype=np.float32) * np.float32(0.5) + np.float32(0.25)
    gt_d, gen_d, disps_d = (torch.from_numpy(x).cuda() for x in (gt, gen, disps))

    stages = {
        "image_scores": lambda: E.image_scores(gt_d, gen_d, error_maps=True, ssim_map=True),
        "disparity_images": lambda: E.disparity_images(disps_d),
        "background_stability": lambda: E.background_stability(gen_d),
    }
    px = f * h * w
    # bytes each stage must move at least: inputs read once, outputs written once
    min_bytes = {
        "image_scores": px * 3 * 4 * 2 + px * 3 * 4 + px * 3 * 2,       # gt + gen; S map; two uint8 error images
        "disparity_images": px * 4 + px * 3 * 4 * 2,                    # disparity; jet + Phong
        "background_stability": px * 3 * 4 + h * w * 3 * 4 * 2,        # frames; std + image
    }
    res = {"workload": f"evaluation {f} x {w}x{h}", "gpu": gpu_info(), "reps": args.reps}
    total = 0.0
    for name, fn in stages.items():
        ms = time_gpu(fn, args.reps)
        total += ms
        res[f"{name}_ms"] = round(ms, 4)
        res[f"{name}_min_bytes"] = min_bytes[name]
        res[f"{name}_GBps"] = round(min_bytes[name] / (ms * 1e-3) / 1e9, 1)
        res[f"{name}_share_of_hbm_bound"] = round(min_bytes[name] / HBM_BYTES_PER_S / (ms * 1e-3), 3)
    res["gpu_total_ms"] = round(total, 4)
    res["gpu_all_in_one_ms"] = round(time_gpu(lambda: [fn() for fn in stages.values()], args.reps), 4)
    host = []
    for _ in range(args.host_reps):
        t = time.perf_counter()
        host_evaluation(gt, gen, disps)
        host.append((time.perf_counter() - t) * 1e3)
    res["host_numpy_ms"] = round(statistics.median(host), 1)
    res["host_threads"] = torch.get_num_threads()
    res["speedup_vs_host"] = round(res["host_numpy_ms"] / res["gpu_all_in_one_ms"], 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_evaluation.jsonl"), "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
