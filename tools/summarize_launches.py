"""Dev tool: turn an `ncu --metrics gpu__time_duration.sum --csv` launch list into the markdown table
(kernel, launches, total us, share).  Usage: python tools/summarize_launches.py launches.csv [title]"""
import collections
import csv
import sys


def load(path):
    rows = [r for r in csv.reader(open(path)) if len(r) > 10]
    hdr = rows[0]
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    out = []
    for r in rows[1:]:
        v = float(r[vi].replace(",", ""))
        v = v / 1000 if r[ui] == "ns" else v * 1000 if r[ui] == "ms" else v
        out.append((r[ki].split("(")[0].replace("void ", "").replace("masr::", ""), v))
    return out


def main():
    seq = load(sys.argv[1])
    agg = collections.OrderedDict()
    for n, v in seq:
        c = agg.setdefault(n, [0, 0.0])
        c[0] += 1
        c[1] += v
    tot = sum(v[1] for v in agg.values())
    print("| kernel | launches | total us | share |\n|---|---:|---:|---:|")
    for k, v in sorted(agg.items(), key=lambda x: -x[1][1]):
        print(f"| `{k}` | {v[0]} | {v[1]:.1f} | {v[1] / tot:.3f} |")
    print(f"\nserialised step total under ncu: {tot / 1000:.2f} ms ({len(seq)} launches)")


if __name__ == "__main__":
    main()
