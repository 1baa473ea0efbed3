"""Bit-level dump and comparison of the fused field kernels' outputs: one training forward and one backward (DGRAD +
WGRAD) through the C ABI on seeded inputs, for checking that a kernel change leaves every byte where it was.

    python scripts/field_bits.py dump OUT_DIR [--tree TREE]   # writes OUT_DIR/<case>.pt for every case
    python scripts/field_bits.py compare REF_DIR OTHER_DIR...  # every OTHER_DIR against REF_DIR

--tree selects the checkout whose built library (and test harness) is used, default the one this script lives in, so a
parent build and a new build can be dumped side by side by one copy of the script.  The harness is the one of
tests/test_stage_parity_gpu.py: its Case inputs (seeded rays, samples, d_raw and both regulariser upstreams) and models
(tests/helpers.build_models, whose bender output layers are drawn non-zero so that rays bend).

A dump holds raw, the forward stash, the ReLU masks, the gradient stash, d_latents and the flat weight gradients.
compare reports, per case: byte-identity of raw, stash and masks; per gradient-stash image the number of tiles whose bytes
differ; and max |difference| of d_latents and the weight gradients, whose fp32 atomics add in no fixed order.
"""
import argparse
import os
import sys

CASES = {
    "bender_1024x128": dict(n=1024, s=128),                  # the benchmark's fine pass, bending, both upstreams
    "ragged_1023x100": dict(n=1023, s=100),                  # P = 102300, not a multiple of 128
    "nobender_1024x128": dict(n=1024, s=128, bender=False),
}
GRAD_IMAGE_NAMES = ["raw"] + [f"dY{l}" for l in range(8)] + ["dYb4", "dYb3", "dYb2", "dYb1", "dYb0"]


def dump(out_dir, tree):
    sys.path.insert(0, os.path.abspath(tree))
    import torch
    from tests import stash_layout as SL
    from tests import test_stage_parity_gpu as H

    os.makedirs(out_dir, exist_ok=True)
    for name, kw in CASES.items():
        cs = H.Case(**kw)
        o = H.run_forward(cs)
        b = H.run_backward(cs, o)
        torch.cuda.synchronize()
        T = cs.T
        rec = {
            "raw": o["raw"].cpu(),
            "stash": o["stash"][:T * SL.STASH_TILE].cpu(),
            "mask": o["mask"][:T * SL.MASK_TILE].cpu(),
            "gstash": b["gstash"][:T * SL.GRAD_TILE].cpu(),
            "nerf_grad": b["nerf_grad"].cpu(),
            "n_tiles": T,
        }
        if cs.bender:
            rec["d_lat"] = b["d_lat"].cpu()
            rec["bender_grad"] = b["bender_grad"].cpu()
        torch.save(rec, os.path.join(out_dir, f"{name}.pt"))
        print(f"{name}: P = {cs.P}, {T} tiles -> {out_dir}")


def compare(ref_dir, others):
    import torch

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from tests import stash_layout as SL

    ok = True
    for other in others:
        print(f"== {ref_dir} vs {other}")
        for name in CASES:
            a = torch.load(os.path.join(ref_dir, f"{name}.pt"))
            b = torch.load(os.path.join(other, f"{name}.pt"))
            T = a["n_tiles"]
            line = []
            for k in ("raw", "stash", "mask"):
                same = torch.equal(a[k].view(torch.uint8), b[k].view(torch.uint8))
                ok &= same
                line.append(f"{k} {'identical' if same else 'DIFFERS'}")
            print(f"  {name} ({T} tiles): " + ", ".join(line))
            ga = a["gstash"].view(T, SL.GRAD_TILE)
            gb = b["gstash"].view(T, SL.GRAD_TILE)
            parts = []
            for nm, (off, chunks) in zip(GRAD_IMAGE_NAMES, SL.GRAD_IMAGES):
                n_bad = int((ga[:, off:off + chunks * SL.CHUNK] != gb[:, off:off + chunks * SL.CHUNK]).any(1).sum())
                ok &= n_bad == 0
                parts.append(f"{nm} {n_bad}")
            print(f"    gradient stash, tiles that differ per image: {', '.join(parts)}"
                  f" -> {'all bytes identical' if torch.equal(ga, gb) else 'DIFFERS'}")
            for k in ("d_lat", "nerf_grad", "bender_grad"):
                if k in a:
                    d = float((a[k] - b[k]).abs().max())
                    print(f"    {k}: max |diff| {d:.3e} (max |ref| {float(a[k].abs().max()):.3e})")
    print("stash, masks, raw and gradient stash: " + ("all identical" if ok else "DIFFERENCES FOUND"))
    return ok


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    d = sub.add_parser("dump")
    d.add_argument("out_dir")
    d.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    c = sub.add_parser("compare")
    c.add_argument("ref_dir")
    c.add_argument("others", nargs="+")
    args = ap.parse_args()
    if args.cmd == "dump":
        dump(args.out_dir, args.tree)
    else:
        sys.exit(0 if compare(args.ref_dir, args.others) else 1)


if __name__ == "__main__":
    main()
