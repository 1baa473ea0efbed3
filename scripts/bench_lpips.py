"""LPIPS (v0.1, AlexNet) of rendered frames on the GPU (evaluation.lpips) against the same network run through
torch.nn.functional: on the GPU in fp32 with TF32 off, on the GPU in fp16 channels_last (cuDNN), and in fp32 on the host
cores, which is what free_viewpoint_rendering.py:788-849 runs.  Workloads: F frames at 504 x 378 (the example sequence)
and at 1008 x 756; weights and frames are seeded (tests/lpips_reference.py).

    python scripts/bench_lpips.py [--frames 37] [--reps 10] [--host-frames 2] [--out DIR]

Prints one JSON line: per workload the median GPU time of evaluation.lpips and of each timing kind (CUDA events, warmed
up), the tensor-core rate from the FLOP count, the torch.nn.functional times, the host time per frame, the largest
difference to the fp32 GPU result, and the card's name and power limit.
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
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nonrigid_nerf_b200 import _lib, evaluation as E  # noqa: E402
from tests import lpips_reference as R  # noqa: E402

PEAK_FP16_DENSE = 989e12   # H100 SXM data sheet, dense fp16 tensor


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


def conv_flops(h, w, padded=False):
    """multiply-adds x 2 of the five convolutions of one image (padded: conv1's 3 channels as the kernel runs them, 8)"""
    total, hh, ww = 0, h, w
    for i, (_, cout, cin, k, s, p) in enumerate(R.CONVS):
        if i in (1, 2):
            hh, ww = (hh - 3) // 2 + 1, (ww - 3) // 2 + 1
        hh, ww = (hh + 2 * p - k) // s + 1, (ww + 2 * p - k) // s + 1
        total += 2 * hh * ww * cout * (8 if padded and i == 0 else cin) * k * k
    return total


def torch_lpips(gt, gen, params, dtype, channels_last=False):
    """the restatement's network through torch.nn.functional on gt / gen [F, H, W, 3] (both images in one batch)"""
    ws, bs, lins, shift, scale = params
    x = torch.cat([gt, gen]).permute(0, 3, 1, 2)
    x = ((2 * x - 1) - shift.view(1, 3, 1, 1)) / scale.view(1, 3, 1, 1)
    x = x.to(dtype)
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    n = gt.shape[0]
    total = torch.zeros(n, dtype=torch.float32, device=gt.device)
    for i, (_, _, _, _, s, p) in enumerate(R.CONVS):
        if i in (1, 2):
            x = F.max_pool2d(x, 3, 2)
        x = F.relu(F.conv2d(x, ws[i], bs[i], stride=s, padding=p))
        f = x.float()
        f = f / (torch.sqrt((f * f).sum(dim=1, keepdim=True)) + 1e-10)
        total += (lins[i].view(1, -1, 1, 1) * (f[:n] - f[n:]) ** 2).sum(dim=1).mean(dim=(1, 2))
    return total


def params_on(sd, device, dtype, channels_last=False):
    ws = [sd[k + ".weight"].to(device, dtype) for k, *_ in R.CONVS]
    if channels_last:
        ws = [w.contiguous(memory_format=torch.channels_last) for w in ws]
    bs = [sd[k + ".bias"].to(device, dtype) for k, *_ in R.CONVS]
    lins = [sd[f"lin{i}.model.1.weight"].reshape(-1).to(device) for i in range(5)]
    return ws, bs, lins, sd["scaling_layer.shift"].reshape(-1).to(device), sd["scaling_layer.scale"].reshape(-1).to(device)


def workload(sd, wt, f, h, w, reps, host_frames):
    gt, gen = R.frames(7, f, h, w)
    g, r = torch.from_numpy(gt).cuda(), torch.from_numpy(gen).cuda()
    res = {"frames": f, "width": w, "height": h}
    ms = time_gpu(lambda: E.lpips(g, r, wt), reps)
    res["gpu_ms"] = round(ms, 3)
    kinds = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + \
        _lib.DET_KERNEL_KINDS + _lib.HELD_OUT_KERNEL_KINDS + _lib.EVAL_KERNEL_KINDS + _lib.FRAME_IMAGE_KERNEL_KINDS + \
        _lib.MESH_KERNEL_KINDS + _lib.LPIPS_KERNEL_KINDS
    _lib.timing_enable(True)
    for _ in range(reps):
        E.lpips(g, r, wt)
    t = _lib.timing_read(kinds)
    _lib.timing_enable(False)
    for k in _lib.LPIPS_KERNEL_KINDS:
        res[f"{k}_ms"] = round(t[k][0] / reps, 3)
    flops, flops_run = 2 * f * conv_flops(h, w), 2 * f * conv_flops(h, w, padded=True)
    res["conv_gflop"], res["conv_gflop_executed"] = round(flops / 1e9, 1), round(flops_run / 1e9, 1)
    res["conv_tflops"] = round(flops / (t["lpips_conv"][0] / reps * 1e-3) / 1e12, 1)
    res["conv_tflops_executed"] = round(flops_run / (t["lpips_conv"][0] / reps * 1e-3) / 1e12, 1)
    res["conv_share_of_fp16_peak"] = round(res["conv_tflops_executed"] * 1e12 / PEAK_FP16_DENSE, 3)
    ours = E.lpips(g, r, wt).double()

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    p32 = params_on(sd, "cuda", torch.float32)
    res["torch_fp32_no_tf32_ms"] = round(time_gpu(lambda: torch_lpips(g, r, p32, torch.float32), reps), 3)
    ref32 = torch_lpips(g, r, p32, torch.float32).double()
    p16 = params_on(sd, "cuda", torch.float16, channels_last=True)
    res["cudnn_fp16_channels_last_ms"] = round(time_gpu(lambda: torch_lpips(g, r, p16, torch.float16, True), reps), 3)
    ref16 = torch_lpips(g, r, p16, torch.float16, True).double()
    res["max_abs_diff_vs_torch_fp32"] = float((ours - ref32).abs().max())
    res["max_abs_diff_cudnn_fp16_vs_torch_fp32"] = float((ref16 - ref32).abs().max())
    res["speedup_vs_cudnn_fp16"] = round(res["cudnn_fp16_channels_last_ms"] / ms, 2)

    pc = params_on(sd, "cpu", torch.float32)
    n = min(host_frames, f)
    gc, rc = torch.from_numpy(gt[:n]), torch.from_numpy(gen[:n])
    with torch.no_grad():
        torch_lpips(gc[:1], rc[:1], pc, torch.float32)
        t0 = time.perf_counter()
        for i in range(n):   # frame by frame, as the reference scores them
            torch_lpips(gc[i:i + 1], rc[i:i + 1], pc, torch.float32)
        host = (time.perf_counter() - t0) * 1e3 / n
    res["host_fp32_ms_per_frame"] = round(host, 1)
    res["host_fp32_ms_all_frames_estimated"] = round(host * f, 1)
    res["speedup_vs_host"] = round(host * f / ms, 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=37)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-frames", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips: no CUDA device; GPU timings cannot be taken here")
    sd = R.random_state_dict(0)
    wt = E.lpips_weights(sd)
    res = {"workload": "lpips alex", "gpu": gpu_info(), "reps": args.reps, "host_threads": torch.get_num_threads()}
    for h, w in ((378, 504), (756, 1008)):
        res[f"{w}x{h}"] = workload(sd, wt, args.frames, h, w, args.reps, args.host_frames)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_lpips.jsonl"), "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
