"""Summarise an .ncu-rep (ncu --set full) as a markdown table: one row per captured launch.
    python tools/ncu_summary.py x.ncu-rep [more.ncu-rep ...]"""
import csv
import subprocess
import sys

COLS = [("gpu__time_duration.sum", "µs", 1e-3), ("launch__grid_size", "grid", 1), ("launch__registers_per_thread", "regs", 1),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "tensor %", 1),
        ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "FMA %", 1),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue %", 1),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps %", 1),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM %", 1),
        ("dram__bytes_read.sum", "DRAM rd MB", None), ("dram__bytes_write.sum", "DRAM wr MB", None),
        ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 %", 1),
        ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smem conflicts", 1)]


def to_mb(v, unit):
    f = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}.get(unit, None)
    return v * f if f else v


for rep in sys.argv[1:]:
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    h, units, data = rows[0], rows[1], rows[2:]
    ix = {k: i for i, k in enumerate(h)}
    print(f"### `{rep.split('/')[-1]}`\n")
    print("| kernel | " + " | ".join(c[1] for c in COLS) + " |")
    print("|---|" + "---|" * len(COLS))
    for r in data:
        name = r[ix["Kernel Name"]].split("(")[0].replace("void ", "").replace("l2h::", "")
        cells = []
        for key, _, sc in COLS:
            if key not in ix or r[ix[key]] == "":
                cells.append("–")
                continue
            v = float(r[ix[key]].replace(",", ""))
            if sc is None:
                v = to_mb(v, units[ix[key]])
            elif key == "gpu__time_duration.sum":
                v = v * {"ns": 1e-3, "nsecond": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "s": 1e6, "second": 1e6}.get(units[ix[key]], 1e-3)
            cells.append(f"{v:.1f}" if abs(v) < 1e6 else f"{v:.3g}")
        print(f"| `{name}` | " + " | ".join(cells) + " |")
    print()
