"""Static resource table of every kernel in libsonarfe.so from the build's own `-Xptxas -v` log
(sonar_slam_b200/build/ptxas.log, written by sonar_slam_b200/build.py): registers, spills, stack, static shared
memory, barriers.  No GPU needed.

    python tools/ptxas_table.py
"""
import os
import re
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(REPO, "sonar_slam_b200", "build", "ptxas.log")


def demangle(names):
    try:
        out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
        return out.splitlines()
    except Exception:  # noqa: BLE001
        return names


def short(name):
    """sfe::icp_kernel<128, 7, false, false, false, false>(sfe::IcpBatch, sfe::MapArgs) -> icp_kernel<128, 7, false, false, false, false>"""
    name = re.sub(r"^void ", "", name).replace("(anonymous namespace)::", "")
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):  # drop the argument list: the first '(' outside template brackets
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    return name[:cut].replace("sfe::", "")


def main():
    if not os.path.exists(LOG):
        sys.exit(f"{LOG} not found: run `python -m sonar_slam_b200.build --force` first")
    rows, cur = [], None
    for line in open(LOG):
        m = re.search(r"Compiling entry function '(\S+)' for '(\S+)'", line)
        if m:
            cur = {"name": m.group(1), "arch": m.group(2), "stack": 0, "spill_st": 0, "spill_ld": 0, "regs": 0,
                   "bar": 0, "smem": 0}
            rows.append(cur)
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            cur["stack"], cur["spill_st"], cur["spill_ld"] = map(int, m.groups())
        m = re.search(r"Used (\d+) registers, used (\d+) barriers", line)
        if m:
            cur["regs"], cur["bar"] = int(m.group(1)), int(m.group(2))
            s = re.search(r"(\d+) bytes smem", line)
            cur["smem"] = int(s.group(1)) if s else 0
            cur = None
    names = [short(n) for n in demangle([r["name"] for r in rows])]
    print("# ptxas -v of the build that produced sonar_slam_b200/libsonarfe.so (nvcc -gencode arch=compute_90a,"
          "code=sm_90a -O3 -lineinfo); static shared memory only -- dynamic shared memory is chosen at launch")
    print(f"# {len(rows)} entry functions, {sum(1 for r in rows if r['spill_st'] or r['spill_ld'])} with register spills")
    print(f"{'kernel':<78} {'regs':>4} {'spill st/ld B':>13} {'stack B':>7} {'smem B':>7} {'bar':>3}")
    for r, n in sorted(zip(rows, names), key=lambda t: t[1]):
        print(f"{n[:78]:<78} {r['regs']:>4} {str(r['spill_st']) + '/' + str(r['spill_ld']):>13} {r['stack']:>7} "
              f"{r['smem']:>7} {r['bar']:>3}")


if __name__ == "__main__":
    main()
