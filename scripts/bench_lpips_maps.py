"""Spatial LPIPS maps on the GPU (evaluation.lpips_maps) against the scores alone (evaluation.lpips) and against the same
maps through torch.nn.functional in fp32 (F.conv2d AlexNet taps with TF32 off, the per-pixel distances, F.interpolate and
the tap-order sum).  Workload: F frames of 1008 x 756 (default 37), seeded weights and frames (tests/lpips_reference.py).

    python scripts/bench_lpips_maps.py [--frames 37] [--reps 10] [--out DIR]

The four ways run alternately, each rep timed with CUDA events after a warm-up of every way.  Prints one JSON line: the
median ms of each way, the upsample kernel's time (timing kind 44) and its bytes, the cost of the maps over the scores,
the largest difference of the map to the torch fp32 one, and the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nonrigid_nerf_b200 import _lib, evaluation as E  # noqa: E402
from tests import lpips_layout as L  # noqa: E402
from tests import lpips_reference as R  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def torch_maps(gt, gen, params):
    """map [F, H, W] through torch.nn.functional in fp32: lpips.LPIPS(net='alex', spatial=True)'s computation"""
    ws, bs, lins, shift, scale = params
    n, h, w, _ = gt.shape
    x = torch.cat([gt, gen]).permute(0, 3, 1, 2)
    x = ((2 * x - 1) - shift.view(1, 3, 1, 1)) / scale.view(1, 3, 1, 1)
    total = None
    for i, (_, _, _, _, s, p) in enumerate(R.CONVS):
        if i in (1, 2):
            x = F.max_pool2d(x, 3, 2)
        x = F.relu(F.conv2d(x, ws[i], bs[i], stride=s, padding=p))
        f = x / (torch.sqrt((x * x).sum(dim=1, keepdim=True)) + 1e-10)
        d = (lins[i].view(1, -1, 1, 1) * (f[:n] - f[n:]) ** 2).sum(dim=1, keepdim=True)
        up = F.interpolate(d, size=(h, w), mode="bilinear", align_corners=False)[:, 0]
        total = up if total is None else total + up
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=37)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips_maps: no CUDA device; GPU timings cannot be taken here")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    f, h, w = args.frames, 756, 1008
    sd = R.random_state_dict(0)
    wt = E.lpips_weights(sd)
    gt, gen = R.frames(7, f, h, w)
    g, r = torch.from_numpy(gt).cuda(), torch.from_numpy(gen).cuda()
    params = ([sd[k + ".weight"].cuda() for k, *_ in R.CONVS], [sd[k + ".bias"].cuda() for k, *_ in R.CONVS],
              [sd[f"lin{i}.model.1.weight"].reshape(-1).cuda() for i in range(5)],
              sd["scaling_layer.shift"].reshape(-1).cuda(), sd["scaling_layer.scale"].reshape(-1).cuda())
    # the torch path at 37 frames of 1008 x 756 holds every activation of both images at once: in slices of 8 frames
    step = 8
    ways = {
        "lpips": lambda: E.lpips(g, r, wt),
        "lpips_maps_map": lambda: E.lpips_maps(g, r, wt),
        "lpips_maps_all": lambda: E.lpips_maps(g, r, wt, per_layer=True, error_images=True),
        "torch_fp32_maps": lambda: [torch_maps(g[i:i + step], r[i:i + step], params) for i in range(0, f, step)],
    }
    for fn in ways.values():   # warm-up of every way and shape
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in ways}
    for _ in range(args.reps):
        for k, fn in ways.items():   # alternately
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    res = {"workload": "lpips maps alex", "gpu": gpu_info(), "frames": f, "width": w, "height": h, "reps": args.reps}
    for k, v in times.items():
        res[f"{k}_ms"] = round(statistics.median(v), 3)
        res[f"{k}_ms_min_max"] = [round(min(v), 3), round(max(v), 3)]
    kinds = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + \
        _lib.DET_KERNEL_KINDS + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + \
        _lib.MESH_KERNEL_KINDS + _lib.LPIPS_KERNEL_KINDS + _lib.MATCH_KERNEL_KINDS + _lib.OCCUPANCY_KERNEL_KINDS + \
        _lib.TERMINATION_KERNEL_KINDS + _lib.DEFORM_KERNEL_KINDS + _lib.NORMAL_KERNEL_KINDS + _lib.LPIPS_MAP_KERNEL_KINDS
    for name, fn in (("map", ways["lpips_maps_map"]), ("all", ways["lpips_maps_all"])):
        _lib.timing_enable(True)
        for _ in range(args.reps):
            fn()
        t = _lib.timing_read(kinds)
        _lib.timing_enable(False)
        for k in ("lpips_distance", "lpips_upsample"):
            res[f"{k}_ms_{name}"] = round(t[k][0] / args.reps, 3)
    tap_bytes = sum(L.px(h, w, s) for s in L.TAP_STAGES) * 4
    res["tap_map_bytes_per_frame"] = tap_bytes
    res["upsample_write_bytes_per_frame"] = {"map": h * w * 4, "all": h * w * (4 + 5 * 4 + 3)}
    for name, n_out in (("map", h * w * 4), ("all", h * w * 27)):
        ms = res[f"lpips_upsample_ms_{name}"]
        res[f"lpips_upsample_write_gbps_{name}"] = round(f * n_out / (ms * 1e-3) / 1e9, 1) if ms > 0 else None
    res["maps_over_scores_ms"] = {k: round(res[f"lpips_maps_{k}_ms"] - res["lpips_ms"], 3) for k in ("map", "all")}
    ours = E.lpips_maps(g, r, wt).map
    ref = torch.cat([torch_maps(g[i:i + step], r[i:i + step], params) for i in range(0, f, step)])
    res["max_abs_diff_map_vs_torch_fp32"] = float((ours.double() - ref.double()).abs().max())
    res["speedup_vs_torch_fp32"] = round(res["torch_fp32_maps_ms"] / res["lpips_maps_map_ms"], 2)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_lpips_maps.jsonl"), "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
