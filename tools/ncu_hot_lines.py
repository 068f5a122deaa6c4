"""Hot source lines of one kernel from an `ncu --set full --import-source on` report (run where ncu is installed):

    python tools/ncu_hot_lines.py <report.ncu-rep> <kernel-substring> [cubin-or-.so] [top_n]

ncu's CSV export of the source page is per SASS instruction; this joins it with nvdisasm's line table of the same
cubin (the build must be the profiled one) and prints, per source line, the share of warp-stall samples and of
executed warp instructions, and the mean number of active threads."""
import csv
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict

rep, kern = os.path.abspath(sys.argv[1]), sys.argv[2]
kern, _, nth = kern.partition("#")   # "name#k": the k-th launch (0-based) whose kernel name contains `name`
nth = int(nth) if nth else 0
lib = sys.argv[3] if len(sys.argv) > 3 else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                         "sonar_slam_b200", "libsonarfe.so")
lib = os.path.abspath(lib)
top = int(sys.argv[4]) if len(sys.argv) > 4 else 25
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
# the export holds one table per kernel launch: take the first whose name matches
start = [i for i, r in enumerate(rows) if r and r[0] == "Kernel Name" and kern in r[1]][nth]
head = rows[start + 1]
body = []
for r in rows[start + 2:]:
    if not r or r[0] == "Kernel Name":
        break
    body.append(r)
ia, isrc, isamp, iinst, ithr = (head.index(k) for k in ("Address", "Source", "# Samples", "Instructions Executed",
                                                        "Thread Instructions Executed"))
base = int(body[0][ia], 16)
mangled = None
with tempfile.TemporaryDirectory() as td:
    cubins = [lib]
    if lib.endswith(".so"):
        subprocess.run(["cuobjdump", "-xelf", "all", lib], cwd=td, capture_output=True)
        cubins = [os.path.join(td, f) for f in os.listdir(td) if f.endswith(".cubin")]
    line_of = {}
    for cb in cubins:
        dis = subprocess.run(["nvdisasm", "-g", "-c", cb], capture_output=True, text=True).stdout
        cur_fn, cur_line, want = None, None, False
        for l in dis.splitlines():
            m = re.match(r"\s*\.text\.(\S+):", l)
            if m:
                cur_fn = m.group(1)
                want = all(t in cur_fn for t in re.findall(r"[A-Za-z_0-9]+", kern) if t != "int") and (mangled is None or cur_fn == mangled)
                if want and mangled is None and len(line_of) == 0:
                    mangled = cur_fn
                continue
            m = re.search(r'//## File "([^"]+)", line (\d+)', l)
            if m:
                cur_line = (os.path.basename(m.group(1)), int(m.group(2)))
                continue
            m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+\S", l)
            if m and want and cur_fn == mangled:
                line_of[int(m.group(1), 16)] = cur_line
        if line_of:
            break
tot_s = sum(int(r[isamp] or 0) for r in body) or 1
tot_i = sum(int(r[iinst] or 0) for r in body) or 1
agg = defaultdict(lambda: [0, 0, 0])
for r in body:
    off = int(r[ia], 16) - base
    key = line_of.get(off, ("?", 0))
    a = agg[key]
    a[0] += int(r[isamp] or 0)
    a[1] += int(r[iinst] or 0)
    a[2] += int(r[ithr] or 0)
print(f"kernel {kern}: {len(body)} SASS instructions, {tot_i} warp instructions executed, {tot_s} stall samples")
print(f"{'file:line':28s} {'samples%':>8s} {'inst%':>7s} {'thr/inst':>8s}")
for key, (sm, ins, thr) in sorted(agg.items(), key=lambda kv: -kv[1][0])[:top]:
    print(f"{key[0] + ':' + str(key[1]):28s} {100.0 * sm / tot_s:8.2f} {100.0 * ins / tot_i:7.2f} {thr / max(1, ins):8.1f}")
