"""Condense `ncu --set full` reports into one JSON file (run where ncu is installed):

    python tools/ncu_summary.py summaries.json name=path.ncu-rep[@kernel-substring] [...]

One entry per report (its first kernel): launch shape, duration, DRAM bytes, issue utilisation, divergence and the
warp-stall reasons per issued instruction."""
import csv
import json
import subprocess
import sys

KEEP = [
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "gpu__time_duration.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "launch__block_size", "launch__grid_size",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static", "lts__t_sector_hit_rate.pct",
    "sm__cycles_elapsed.avg", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__thread_inst_executed_per_inst_executed.ratio",
]


def summarise(path):
    """path or path@substring: the first launch whose kernel name contains the substring (default: first launch)"""
    path, _, want = path.partition("@")
    want, _, nth = want.partition("#")   # kernel-substring#k: the k-th such launch (0-based)
    nth = int(nth) if nth else 0
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(out.splitlines()))
    head, units = rows[0], rows[1]
    ki = head.index("Kernel Name")
    first = [r for r in rows[2:] if want in r[ki]][nth]
    d = dict(zip(head, first))
    u = dict(zip(head, units))
    res = {"kernel": d["Kernel Name"]}
    for k in KEEP:
        if k in d:
            res[k] = f"{d[k]} {u.get(k, '')}".strip()
    for k, v in d.items():
        if k.startswith("smsp__average_warps_issue_stalled_") and k.endswith("_per_issue_active.ratio"):
            try:
                x = float(v)
            except ValueError:
                continue
            if x >= 0.1:
                res["stall:" + k[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]] = round(x, 3)
    return res


if __name__ == "__main__":
    dst, items = sys.argv[1], sys.argv[2:]
    try:
        data = json.load(open(dst))
    except (OSError, ValueError):
        data = {}
    for it in items:
        name, path = it.split("=", 1)
        data[name] = summarise(path)
    json.dump(data, open(dst, "w"), indent=1, sort_keys=True)
    print("wrote", dst, sorted(data))
