"""Dev tool: per-kernel roofline table of the headline step from an ncu CSV (long format, one row per launch x metric):

    ncu --profile-from-start off --clock-control none --csv --log-file step_metrics.csv \\
        --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,\\
sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active,lts__t_sectors.sum python tools/profile_step.py
    python tools/kernel_roofline.py step_metrics.csv > kernel_roofline.md

Per kernel (aggregated over its launches in one step): mean duration, DRAM traffic per launch (ncu flushes caches between
kernels, so this is cold-cache traffic), achieved DRAM GB/s, the ALGORITHMIC bytes per launch (inputs read once + outputs
written once, DESIGN.md §4) / duration as a fraction of the measured HBM peak, and the tensor-pipe active share.
Durations under ncu are serialised and cold-cache: compare shares and fractions, not absolutes."""
import collections
import csv
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, F, T = 32, 998, 248
M = B * T
MB = 1e6
# algorithmic bytes per launch at the headline size (B=32 x 10 s): name substring -> bytes
ALGO = [
    ("wave_sumsq", B * 160000 * 4),
    ("wave_gain", B * 8),
    ("fbank_kernel", B * 160000 * 4 + B * F * 80 * 4),
    ("conv1_cmvn_relu", B * F * 80 * 4 + B * 498 * 39 * 256 * 4),
    ("layernorm_kernel<256, 1>", M * 256 * 4 + M * 256 * 4),
    ("layernorm_kernel<256, 0>", M * 256 * 4 + M * 256 * 4),
    ("dwconv_ln_silu", M * 256 * 4 + M * 256 * 4),
    ("relpos_attention_mma", M * 256 * 4 + 2 * M * 256 * 4 + M * 256 * 4),
    ("ctc_frame_argmax", M * 4240 * 4 + M * 8),
    ("ctc_greedy_collapse", M * 8 + B * T * 4),
]


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d["hbm_gbs"], d.get("bf16_tflops_sustained", d["bf16_tflops"])
    return 6650.0, 1400.0


def main():
    rows = [r for r in csv.reader(open(sys.argv[1])) if len(r) > 10]
    hdr = rows[0]
    ii, ki, mi, ui, vi = (hdr.index(k) for k in ("ID", "Kernel Name", "Metric Name", "Metric Unit", "Metric Value"))
    launches = collections.OrderedDict()
    for r in rows[1:]:
        name = r[ki].split("(")[0].replace("void ", "").replace("masr::", "")
        d = launches.setdefault(r[ii], {"name": name})
        v = float(r[vi].replace(",", ""))
        u = r[ui]
        if u in ("ns", "nsecond"): v /= 1e3
        elif u in ("ms", "msecond"): v *= 1e3
        elif u == "Kbyte": v *= 1e3
        elif u == "Mbyte": v *= 1e6
        elif u == "Gbyte": v *= 1e9
        d[r[mi]] = v
    agg = collections.OrderedDict()
    for d in launches.values():
        a = agg.setdefault(d["name"], collections.defaultdict(float))
        a["n"] += 1
        a["us"] += d.get("gpu__time_duration.sum", 0.0)
        a["dram"] += d.get("dram__bytes_read.sum", 0.0) + d.get("dram__bytes_write.sum", 0.0)
        a["tensor"] += d.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 0.0)
        a["l2"] += d.get("lts__t_sectors.sum", 0.0) * 32
    hbm, _ = peaks()
    tot = sum(a["us"] for a in agg.values())
    print(f"HBM peak (MEASURED_PEAKS.json): {hbm:.1f} GB/s; step under ncu: {tot / 1e3:.2f} ms, {len(launches)} launches\n")
    print("| kernel | launches | share | us / launch | DRAM MB / launch | DRAM GB/s | algorithmic MB | algorithmic GB/s | frac of HBM peak | L2 MB / launch | tensor pipe % |")
    print("|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|")
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1]["us"]):
        n = a["n"]
        us = a["us"] / n
        dram = a["dram"] / n
        algo = next((b for s, b in ALGO if s in k), None)
        ag = "" if algo is None else f"{algo / MB:.1f}"
        ab = "" if algo is None else f"{algo / us / 1e3:.0f}"
        fr = "" if algo is None else f"{algo / us / 1e3 / hbm:.3f}"
        print(f"| `{k}` | {int(n)} | {a['us'] / tot:.3f} | {us:.1f} | {dram / MB:.1f} | {dram / us / 1e3:.0f} | {ag} | {ab} | {fr} | "
              f"{a['l2'] / n / MB:.1f} | {a['tensor'] / n:.1f} |")


if __name__ == "__main__":
    main()
