"""Summarise an ncu launch list (`--metrics gpu__time_duration.sum --csv`) of bench.py: one device step = the launches between
two consecutive k_scatter_cnt (the encode kernel that opens a step).  Usage:
    python tools/launch_list.py gpurun_out/launches.csv > profiles/rN_launches_bench_cfg2.md"""
import collections
import csv
import re
import sys

rows = [r for r in csv.reader(open(sys.argv[1], errors="replace")) if len(r) > 14 and r[0].isdigit()]
starts = [i for i, r in enumerate(rows) if "k_scatter_cnt" in r[4]]
# the encode of a step is preceded by two torch fills (the frame buffer); a step ends where the next one's fills begin
lo, hi = starts[-2], starts[-1]
step = rows[lo:hi]


def short(name):
    name = re.sub(r"^void ", "", name)
    name = name.replace("esr::", "")
    m = re.match(r"([\w:]+(<[^(]*>)?)", name)
    return m.group(1) if m else name


agg = collections.OrderedDict()
for r in step:
    k = short(r[4])
    n, t = agg.get(k, (0, 0.0))
    agg[k] = (n + 1, t + float(r[14].replace(",", "")) / 1e3)
tot = sum(t for _, t in agg.values())
print(f"launches {rows[lo][0]}..{rows[hi - 1][0]} of the capture = one step ({len(step)} launches, {tot:.1f} us under ncu)\n")
print("| kernel | launches | total µs | share |\n|---|---|---|---|")
for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"| `{k}` | {n} | {t:.1f} | {100 * t / tot:.1f} % |")
print(f"| **sum** | {len(step)} | {tot:.1f} | 100 % |")
tc = sum(t for k, (n, t) in agg.items() if k.startswith(("k_conv_tc", "k_dcn_fused")))
print(f"\nwgmma kernels (k_conv_tc* + k_dcn_fused): {100 * tc / tot:.1f} % of the step.")
