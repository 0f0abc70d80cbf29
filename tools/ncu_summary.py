"""Dev tool: compact markdown summary of an `ncu --set full` report (one row per captured launch).
Usage: python tools/ncu_summary.py x.ncu-rep > x_summary.md   (needs the ncu CLI; no GPU)"""
import csv
import io
import subprocess
import sys

COLS = [("gpu__time_duration.sum", "us", 1.0), ("dram__bytes_read.sum", "DRAM rd MB", 1.0), ("dram__bytes_write.sum", "DRAM wr MB", 1.0),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM %", 1.0),
        ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 %", 1.0),
        ("l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "L1/smem %", 1.0),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe %", 1.0),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue %", 1.0),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %", 1.0),
        ("launch__registers_per_thread", "regs", 1.0), ("launch__grid_size", "grid", 1.0), ("launch__block_size", "block", 1.0)]


def main():
    raw = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    ki = hdr.index("Kernel Name")
    print("| # | kernel | " + " | ".join(c[1] for c in COLS) + " |")
    print("|---|---|" + "---:|" * len(COLS))
    for n, d in enumerate(data):
        name = d[ki].split("(")[0].replace("void ", "").replace("masr::", "")
        vals = []
        for key, _, _ in COLS:
            if key in hdr:
                i = hdr.index(key)
                v = float(d[i].replace(",", "")) if d[i] not in ("", "n/a") else float("nan")
                u = units[i]
                if u in ("ns", "nsecond"): v /= 1e3
                if u in ("byte",): v /= 1e6
                if u == "Kbyte": v /= 1e3
                if u == "Gbyte": v *= 1e3
                vals.append(f"{v:.1f}" if abs(v) < 1e5 else f"{v:.0f}")
            else:
                vals.append("")
        print(f"| {n} | `{name}` | " + " | ".join(vals) + " |")


if __name__ == "__main__":
    main()
