"""What an OctreeGridDataPointsFilter in the ICP chain (SFE_ICP_DATA_OCTREE) costs and saves on the device.

Workloads:
  map2d    the README's 2-D map-to-map rows: sources of 20 k, 70 k and 200 k points against the 243 726-point map
           (tools/bench_icp_big_source.py's maps and problems), 1 and 30 guesses; without a filter, and with a
           reading octree filter of maxSizeByNode 0.2 m and 0.5 m for each sampler (0 first point, 2 centroid,
           3 medoid)
  wave     the config-3 wave (132-SM-sized batches of 2 000-point sources on 20 000-point targets, 8 waves per call,
           tools/bench_icp_filters.py's shape) without a filter and with a reference octree filter of 0.2 m per sampler
Shipped checkers (icp.yaml).  Per row:
  device_ms   ops.icp on device tensors between two CUDA events, median of 3 after a warm-up call (wave: ms per wave)
  octree_ms   torch.profiler kernel time of the data-filter stage of one call, in a separate pass: the compaction
              passes and the one-CTA and grid-wide down-sample kernels, with the CUB sort and scan kernels that start
              before the call's first map_build or ICP kernel (stage_kernels: how many kernels that is)
  cpu_ms      the CPU oracle (oracle/octree_filter_ref.c) on one host thread for one guess (wave: one problem)
  exact       the first three device results equal the oracle's bit for bit (status, iterations, inliers, T)
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/bench_icp_octree_filter.py [--out FILE] [--only map2d:200000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
F32 = np.float32
SAMPLERS = (0, 2, 3)
# the data-filter stage's own kernels; CUB's sort and scan count too when they start before the call's first
# map_build or ICP kernel (map_build sorts with CUB as well)
STAGE_KERNELS = ("icp_data_filter_kernel", "downsample_cta_kernel", "dsg_", "icp_keep_too_large_kernel")
AFTER_FILTERS = ("map_flag_kernel", "icp_kernel", "icp_classify_kernel")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in q.split(",")]
    except Exception:  # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def measure(name, srcs, tgts, guesses, src_id, tgt_id, filters, waves=1):
    """One ops.icp call over P = len(guesses) problems; problem p: srcs[src_id[p]] onto tgts[tgt_id[p]]."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from oracle import octree_filter_ref as ofr
    from oracle import oracle as orc
    from sonar_slam_b200 import _lib, ops

    def pack(cl):
        off = np.zeros(len(cl) + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in cl])
        return torch.from_numpy(np.concatenate(cl).astype(F32)).cuda(), torch.from_numpy(off).cuda()

    sp, so = pack(srcs)
    tp, to = pack(tgts)
    si = torch.tensor(src_id, dtype=torch.int32).cuda()
    ti = torch.tensor(tgt_id, dtype=torch.int32).cuda()
    g = torch.from_numpy(np.stack(guesses).astype(F32)).cuda()
    prm = _lib.IcpParams()
    flt = _lib.IcpFilters(**filters) if filters else None
    call = lambda: ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, src_id=si, tgt_id=ti,
                           filters=flt)
    res = call()
    torch.cuda.synchronize()
    dev = {k: v.cpu().numpy() for k, v in res.items()}
    oflt = ofr.IcpFilters(**filters) if filters else ofr.IcpFilters()
    exact = True
    for k in range(min(3, len(guesses))):
        w = ofr.icp(srcs[src_id[k]], tgts[tgt_id[k]], guesses[k], orc.IcpParams(), oflt)
        exact &= (int(dev["status"][k]) == w["status"] and int(dev["iterations"][k]) == w["iterations"] and
                  int(dev["inliers"][k]) == w["inliers"] and dev["T"][k].tobytes() == np.asarray(w["T"], F32).tobytes())
    ev = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        torch.cuda.synchronize()
        ev.append(a.elapsed_time(b))
    stage, n_stage = 0.0, 0
    if filters:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        kern = [e for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower() and
                "memset" not in e.name.lower()]
        end = min([e.time_range.start for e in kern if any(k in e.name for k in AFTER_FILTERS)], default=float("inf"))
        for e in kern:
            if any(k in e.name for k in STAGE_KERNELS) or ("cub" in e.name.lower() and e.time_range.start < end):
                us = getattr(e, "device_time_total", None)
                stage += us if us is not None else e.cuda_time_total
                n_stage += 1
    t = time.perf_counter()
    w = ofr.icp(srcs[src_id[0]], tgts[tgt_id[0]], guesses[0], orc.IcpParams(), oflt)
    cpu = (time.perf_counter() - t) * 1e3
    n_filtered = len(ofr.data_filters(srcs[src_id[0]], filters.get("reading", []))) if filters else len(srcs[src_id[0]])
    return dict(name=name, filters=filters, n_source=len(srcs[src_id[0]]), n_source_filtered=n_filtered,
                n_target=len(tgts[tgt_id[0]]), problems=len(guesses), status=[int(v) for v in dev["status"][:3]],
                iterations=[int(v) for v in dev["iterations"][:3]], oracle_iterations=w["iterations"],
                device_ms=round(float(np.median(ev)) / waves, 3), octree_ms=round(stage / 1e3 / waves, 3),
                stage_kernels=n_stage,
                cpu_ms=round(cpu, 1), exact=bool(exact))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default=None, help="the rows whose name:source points starts with this text")
    args = ap.parse_args()
    want = lambda key: args.only is None or key.startswith(args.only)
    import torch
    from bench_icp_big_source import maps, problem

    from sonar_slam_b200 import synth
    OCT = 3
    rows = []
    m2, _ = maps() if want("map2d") else (None, None)
    for n in (20000, 70000, 200000):
        if not want(f"map2d:{n}"):
            continue
        for k in (1, 30):
            src, gs = problem(m2, n, k, 8)
            chains = [None] + [dict(reading=[(OCT, s, size)]) for size in (0.2, 0.5) for s in SAMPLERS]
            for ch in chains:
                rows.append(measure("map2d", [src], [m2], gs, [0] * k, [0] * k, ch))
                print(json.dumps(rows[-1]), file=sys.stderr)
    if want("wave"):
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        waves = 8
        P = sms * waves
        pairs = [synth.make_icp_pair(1000 + k, n_source=2000, n_target=20000) for k in range(16)]
        ids = [k % 16 for k in range(P)]
        gs = [pairs[i][2].astype(F32) for i in ids]
        for ch in [None] + [dict(reference=[(OCT, s, 0.2)]) for s in SAMPLERS]:
            rows.append(measure("wave", [p[0] for p in pairs], [p[1] for p in pairs], gs, ids, ids, ch, waves=waves))
            print(json.dumps(rows[-1]), file=sys.stderr)
    name, power = card()
    line = json.dumps(dict(gpu=name, power_limit=power, checkers="shipped", rows=rows))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
