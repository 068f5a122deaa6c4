"""Per-kernel totals of an `ncu --metrics gpu__time_duration.sum --csv` launch list:

    python tools/launch_summary.py launches.csv launch_summary.csv [first_id [last_id]]

Only launches with first_id <= ID <= last_id are counted (e.g. the steps with frames resident in HBM, leaving out
the chunked host-buffer runs that follow in the same bench.py process)."""
import csv
import re
import sys
from collections import OrderedDict

src, dst = sys.argv[1], sys.argv[2]
first = int(sys.argv[3]) if len(sys.argv) > 3 else 0
last = int(sys.argv[4]) if len(sys.argv) > 4 else 1 << 30
rows = [r for r in csv.reader(l for l in open(src) if l.startswith('"'))]
head = rows[0]
ki, vi, ui, ii = head.index("Kernel Name"), head.index("Metric Value"), head.index("Metric Unit"), head.index("ID")
tot = OrderedDict()
for r in rows[1:]:
    if not first <= int(r[ii]) <= last:
        continue
    name = re.sub(r"^void ", "", r[ki]).split("(")[0].split("<")[0].replace("sfe::", "")
    ms = float(r[vi].replace(",", "")) * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}[r[ui]]
    n, t = tot.get(name, (0, 0.0))
    tot[name] = (n + 1, t + ms)
total = sum(t for _, t in tot.values())
with open(dst, "w") as f:
    f.write("kernel,launches,total_ms,share\n")
    for name, (n, t) in sorted(tot.items(), key=lambda kv: -kv[1][1]):
        f.write(f"{name},{n},{t:.3f},{t / total:.4f}\n")
print(open(dst).read())
