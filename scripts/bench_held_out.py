"""Held-out rays: the example_sequence training step with 2/7 of the frames held out, timed as the reference loop runs it
(two backward passes, train.py:1595-1608) and as one backward with render(..., held_out=), alternating in one process.
Prints one JSON line per batch size with the medians, the card's name and its power limit.
    python scripts/bench_held_out.py [--steps 30] [--warmup 5] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nonrigid_nerf_b200 import _lib  # noqa: E402
from tests.test_held_out_gpu import DEV, _loss, _setup, _weights  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = _card()
    lines = []
    for n in (1024, 8192):
        coarse, fine, bender, r, rnd, latents, pix, test = _setup(2024 + n, n)
        named = _weights(coarse, fine, bender)
        train, testf = (~test).float(), test.float()

        def two_pass():
            loss = _loss(coarse, fine, bender, r, rnd, latents, pix)
            (testf * loss).mean().backward(retain_graph=True)
            for _, p in named:
                p.grad = None
            (train * loss).mean().backward()

        def one_pass():
            loss = _loss(coarse, fine, bender, r, rnd, latents, pix, held_out=test)
            ((train + testf) * loss).mean().backward()

        times = {"two_pass": [], "one_pass": []}
        for it in range(a.warmup + a.steps):
            for label, fn in (("two_pass", two_pass), ("one_pass", one_pass)) if it % 2 == 0 else (("one_pass", one_pass), ("two_pass", two_pass)):
                for _, p in named:
                    p.grad = None
                for l in latents:
                    l.grad = None
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                if it >= a.warmup:
                    times[label].append(e0.elapsed_time(e1))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        # per-kernel times of one extra step of each (CUDA events around every launch; separate from the timed steps)
        kinds = _lib.KERNEL_KINDS + _lib.TC_KERNEL_KINDS + _lib.VIEW_KERNEL_KINDS + _lib.VIEW_TRAIN_KERNEL_KINDS + \
            _lib.DET_KERNEL_KINDS + _lib.HELD_OUT_KERNEL_KINDS
        per_kernel = {}
        for label, fn in (("two_pass", two_pass), ("one_pass", one_pass)):
            _lib.timing_enable(True)
            fn()
            torch.cuda.synchronize()
            per_kernel[label] = {k: [round(ms, 4), c] for k, (ms, c) in _lib.timing_read(kinds).items() if c}
            _lib.timing_enable(False)
        line = {"workload": "example_sequence_held_out_2_of_7", "n_rand": n, "steps": a.steps, "gpu": name, "power_limit": power,
                "two_pass_ms_median": round(med["two_pass"], 3), "one_pass_ms_median": round(med["one_pass"], 3),
                "saving": round(1.0 - med["one_pass"] / med["two_pass"], 4),
                "kernel_ms_and_launches": per_kernel,
                "note": "eager forward + backward of training_wrapper_class (no optimizer step), CUDA events, alternating order"}
        print(json.dumps(line), flush=True)
        lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
