"""Condense an .ncu-rep (read with `ncu -i ... --page raw --csv`) into the table the docs cite.

    python tools/ncu_summary.py <report>.ncu-rep > <summary>.md
"""
import csv
import io
import subprocess
import sys

METRICS = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM % of peak"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe active %"),
    ("sm__inst_executed_pipe_tensor.sum", "tensor instructions"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
    ("smsp__issue_active.avg.pct", "issue active %"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("launch__registers_per_thread", "registers"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("lts__t_sector_hit_rate.pct", "L2 hit %"),
    ("l1tex__t_sector_hit_rate.pct", "L1 hit %"),
]


def main():
    path = sys.argv[1]
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    if len(rows) < 3:
        print("no kernels in", path)
        return
    header, units = rows[0], rows[1]
    col = {h: i for i, h in enumerate(header)}
    print(f"# `ncu --set full --clock-control none` summary of `{path.split('/')[-1]}`\n")
    print("| kernel | " + " | ".join(n for _, n in METRICS) + " |")
    print("|---|" + "---|" * len(METRICS))
    for r in rows[2:]:
        name = r[col["Kernel Name"]].split("(")[0][-60:]
        vals = []
        for m, _ in METRICS:
            if m in col:
                u = units[col[m]]
                vals.append(f"{r[col[m]]} {u}".strip())
            else:
                vals.append("-")
        print(f"| `{name}` | " + " | ".join(vals) + " |")


if __name__ == "__main__":
    main()
