#!/usr/bin/env python3
"""Summarise an `ncu --page raw --csv` export of one training step:
    python scripts/ncu_summary.py ncu_out/h100_ncu_full_step_raw.csv ncu_out/h100
writes <prefix>_traffic.json (DRAM bytes per step and kernel kind) and
<prefix>_ncu_summary.md (one row per launch: duration, DRAM read / write, achieved DRAM GB/s, tensor-pipe and SM activity)."""
import csv
import json
import sys

UNIT = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12, "ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6, "%": 1.0, "": 1.0}


def main():
    src, prefix = sys.argv[1], sys.argv[2]
    rows = list(csv.reader(open(src)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}

    def val(r, name):
        if name not in col or r[col[name]] in ("", "no data", "n/a"):
            return None
        return float(r[col[name]].replace(",", "")) * UNIT.get(units[col[name]], 1.0)

    kinds = {"field_fwd": "field_fwd", "field_bwd": "field_dgrad", "wgrad_kernel": "wgrad", "wgrad_reduce": "wgrad", "div_fwd": "divergence",
             "div_bwd": "divergence", "div_G": "divergence"}
    traffic, lines = {}, []
    for r in data:
        name = r[col["Kernel Name"]]
        kind = next((v for k, v in kinds.items() if k in name), None)
        rd, wr = val(r, "dram__bytes_read.sum") or 0.0, val(r, "dram__bytes_write.sum") or 0.0
        us = val(r, "gpu__time_duration.sum") or 0.0
        if kind:
            traffic[kind] = traffic.get(kind, 0) + int(rd + wr)
        tens = val(r, "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed")
        sm_act = val(r, "sm__cycles_active.avg.pct_of_peak_sustained_elapsed") if "sm__cycles_active.avg.pct_of_peak_sustained_elapsed" in col else None
        thr = val(r, "sm__throughput.avg.pct_of_peak_sustained_elapsed")
        lines.append((name[:58], r[col["Grid Size"]], us, rd / 1e6, wr / 1e6, (rd + wr) / us / 1e3 if us else 0.0, tens, thr, sm_act))
    traffic["note"] = ("dram__bytes_read.sum + dram__bytes_write.sum per training step (all launches of the kind: coarse + fine; WGRAD includes the "
                       f"divergence launch and the split reductions), N_rand=1024, from {src.split('/')[-1]} (ncu --set full, cold caches, one launch at a time)")
    with open(prefix + "_traffic.json", "w") as f:
        json.dump(traffic, f, indent=1)
    with open(prefix + "_ncu_summary.md", "w") as f:
        f.write(f"# ncu --set full --clock-control none: one training step (N_rand = 1024), from {src.split('/')[-1]}\n\n")
        f.write("| kernel | grid | duration us | DRAM read MB | DRAM write MB | DRAM GB/s | tensor pipe active % of elapsed | SM throughput % | \n|---|---|---|---|---|---|---|---|\n")
        for n, g, us, rd, wr, gbs, tens, thr, _ in lines:
            f.write(f"| `{n}` | {g} | {us:.1f} | {rd:.1f} | {wr:.1f} | {gbs:.0f} | {'' if tens is None else f'{tens:.1f}'} | {'' if thr is None else f'{thr:.1f}'} |\n")
    print(json.dumps(traffic, indent=1))


if __name__ == "__main__":
    main()
