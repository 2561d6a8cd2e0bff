"""Summarise an `ncu --csv` launch list (long format: one row per metric per launch).

    python tools/ncu_launches.py launches.csv [--traffic-key resnet50_w4a4/512/nhwc]

Prints per-kernel launch counts, summed gpu__time_duration and the share of the total; with dram__bytes_* metrics present
also the DRAM traffic per launch of every fq_* kernel.  --traffic-key writes / updates profiles/ncu_traffic.json with the
average DRAM read + write bytes of the fused mode-D launches (three streaming phases), the figure bench.py reports as
`roofline.traffic`."""
import csv
import json
import os
import re
import sys
from collections import defaultdict

path = sys.argv[1]
key = sys.argv[sys.argv.index("--traffic-key") + 1] if "--traffic-key" in sys.argv else None
rows = [r for r in csv.reader(open(path, errors="replace")) if len(r) >= 15 and r[0].isdigit()]
launch = defaultdict(dict)
names = {}
for r in rows:
    lid = int(r[0])
    names[lid] = r[4]
    try:
        launch[lid][r[12]] = float(r[14].replace(",", ""))
    except ValueError:
        pass
    if r[13] and r[12] == "gpu__time_duration.sum":
        launch[lid]["_unit"] = r[13]


def short(n):
    n = re.sub(r"\(.*", "", n).replace("void ", "")
    return re.sub(r"^fqb::", "", n)[:70]


agg = defaultdict(lambda: [0, 0.0, 0.0])
for lid, m in launch.items():
    t = m.get("gpu__time_duration.sum", 0.0)
    if m.get("_unit", "ns") in ("usecond", "us"):
        t *= 1e3
    elif m.get("_unit") in ("msecond", "ms"):
        t *= 1e6
    a = agg[short(names[lid])]
    a[0] += 1
    a[1] += t
    a[2] += m.get("dram__bytes_read.sum", 0.0) + m.get("dram__bytes_write.sum", 0.0)
total = sum(a[1] for a in agg.values()) or 1.0
print("%-72s %6s %10s %6s %14s" % ("kernel", "n", "ms", "share", "DRAM MB/launch"))
for k, (n, t, b) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print("%-72s %6d %10.3f %5.1f%% %14.1f" % (k, n, t / 1e6, 100 * t / total, b / n / 1e6))
ours = sum(a[1] for k, a in agg.items() if k.startswith("fq_"))
print("fq_* kernels: %.1f %% of the summed kernel time (%.3f ms of %.3f ms)" % (100 * ours / total, ours / 1e6, total / 1e6))
if key:
    pat = r"fq_cl_kernel<\(int\)0, \(bool\)1|fq_cl_kernel<0, true|fq_cl_kernel<0, 1"
    if not key.endswith("/nhwc"):
        pat += r"|fq_fused_kernel<4, 0, true|fq_fused_kernel<4, 0, 1"
    fused = [(m.get("dram__bytes_read.sum", 0.0) + m.get("dram__bytes_write.sum", 0.0)) for lid, m in launch.items()
             if re.search(pat, names[lid])]
    if fused:
        out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles", "ncu_traffic.json")
        table = json.load(open(out)) if os.path.exists(out) else {}
        table[key] = {"bytes_per_launch": sum(fused) / len(fused), "launches": len(fused), "source": "profiles/" + os.path.basename(path)}
        json.dump(table, open(out, "w"), indent=1, sort_keys=True)
        print("traffic: %.1f MB per mode-D launch over %d launches -> %s" % (sum(fused) / len(fused) / 1e6, len(fused), out))
