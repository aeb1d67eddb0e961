#!/usr/bin/env python
"""Summarise an .ncu-rep (captured with `ncu --set full`) into a small markdown table.
usage: python scripts/ncu_summary.py prof.ncu-rep > summary.md"""
import csv
import subprocess
import sys

WANT = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "DRAM % of peak"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 % of peak"),
    ("l1tex__throughput.avg.pct_of_peak_sustained_active", "L1TEX % of peak"),
    ("l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "L1TEX global-load sectors"),
    ("l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum", "L1TEX global-load requests"),
    ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "shared-memory wavefronts"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "shared bank conflicts"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate"),
    ("smsp__cycles_active.avg", "SMSP active cycles"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("launch__registers_per_thread", "registers / thread"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__shared_mem_per_block_static", "static smem / block"),
    ("launch__shared_mem_per_block_dynamic", "dynamic smem / block"),
]


def main():
    rep = sys.argv[1]
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    print(f"# ncu summary of `{rep}` (--set full --clock-control none; cold-cache replays: compare shares, not absolutes)\n")
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")].split("(")[0]
        print(f"## {name}\n\n| metric | value |\n|---|---|")
        for key, label in WANT:
            if key in hdr:
                i = hdr.index(key)
                print(f"| {label} (`{key}`) | {r[i]} {units[i]} |")
        if "dram__bytes_read.sum" in hdr:
            mult = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}  # ncu scales each cell itself
            tot = 0.0
            for key in ("dram__bytes_read.sum", "dram__bytes_write.sum"):
                i = hdr.index(key)
                tot += float(r[i].replace(",", "")) * mult.get(units[i], 1.0)
            print(f"| **traffic = DRAM read + write** | {tot / 1e6:.3f} Mbyte |")
        print()


if __name__ == "__main__":
    main()
