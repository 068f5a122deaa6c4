"""Whole-map outlier removal (pcl.remove_outlier on SLAM.get_points-sized clouds, mapping.py:392-398): device time of
sfe_remove_outlier_dev on resident data (CUDA events), pcl.remove_outlier end to end (copy in, kernels, copy out) and
the CPU oracle on one thread, every result checked against the oracle; then a sweep of single clouds from 4 k points to
the one-CTA limit with both paths (the map class from a build where every cloud takes it:
tools/build_map_class_variant.sh).  Prints one JSON line.

    python tools/bench_map_outlier.py [--out FILE] [--map-lib scratch/lib_mapclass.so]
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
PARAMS = ((1.0, 5), (5.0, 20))  # (1.0, 5): the front end's feature.yaml; (5.0, 20): mapping.yaml


def median(v):
    return float(np.median(np.asarray(v)))


def device_ms(pts_np, radius, min_points, reps=10):
    """sfe_remove_outlier_dev on one resident cloud (n_max = its size): median of `reps` event-timed calls."""
    import torch
    from sonar_slam_b200 import ops
    pts = torch.from_numpy(pts_np).cuda()
    off = torch.tensor([0, len(pts_np)], dtype=torch.int32, device="cuda")
    ctx = ops.context(0)
    for _ in range(2):
        out = ops.remove_outlier(pts, off, len(pts_np), radius, min_points, ctx=ctx)
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(torch.cuda.current_stream())
        out = ops.remove_outlier(pts, off, len(pts_np), radius, min_points, ctx=ctx)
        e1.record(torch.cuda.current_stream())
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return median(ts), out


def sweep(sizes):
    from sonar_slam_b200 import synth
    base = synth.make_map_cloud(max(sizes), seed=1)[0]
    return {f"{r}/{k}": {str(n): round(device_ms(np.ascontiguousarray(base[:n]), r, k)[0], 4) for n in sizes}
            for r, k in PARAMS}


def cta_limit(optin):
    """cloud.cu, remove_outlier_cta_limit: 8 bytes per point + a cell table of two cells per point (256..16384) + 16
    bytes within the opt-in shared memory less 4 KiB, at most 65 535 points."""
    def smem(n):
        mc = min(max(2 * n, 256), 16384)
        return 8 * n + 4 * ((mc + 2) // 2 + 1) + 16
    lo, hi = 0, 65535
    while lo < hi:
        mid = lo + (hi - lo + 1) // 2
        lo, hi = (mid, hi) if smem(mid) <= optin - 4096 else (lo, mid - 1)
    return lo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    ap.add_argument("--map-lib", default=os.path.join(REPO, "scratch", "lib_mapclass.so"),
                    help="library built with SFE_MAP_CLASS_ALL (every cloud in the map class)")
    ap.add_argument("--sweep", default=None, help=argparse.SUPPRESS)  # child mode: comma-separated sizes
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    if args.sweep:
        print(json.dumps(sweep([int(s) for s in args.sweep.split(",")])))
        return

    from oracle import oracle as orc
    from sonar_slam_b200 import synth
    from sonar_slam_b200.bruce_slam import pcl
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown", clouds={})
    rng = np.random.default_rng(2)
    m200 = synth.make_map_cloud(200000, seed=1)[0]
    clouds = {
        "map_200k": m200,
        "map_360k": synth.make_map_cloud(360000, seed=1)[0],
        "map_1M": synth.make_map_cloud(1000000, seed=1)[0],
        "uniform_1M": rng.uniform(0, 350, (1000000, 2)).astype(np.float32),
        "map_200k_xyz": np.c_[m200, rng.choice([0.0, 0.6, 3.0], len(m200)) +
                              0.05 * rng.standard_normal(len(m200))].astype(np.float32),
    }
    for name, pts in clouds.items():
        for radius, min_points in PARAMS:
            dev, out = device_ms(pts, radius, min_points)
            pcl.remove_outlier(pts, radius, min_points)
            e2e = []
            for _ in range(5):
                t0 = time.perf_counter()
                got = pcl.remove_outlier(pts, radius, min_points)
                e2e.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            want, keep = orc.remove_outlier(pts, radius, min_points)
            cpu = (time.perf_counter() - t0) * 1e3
            k = int(out["count"][0])
            exact = (np.array_equal(got, want) and k == len(want) and
                     np.array_equal(out["idx"][:k].cpu().numpy(), np.flatnonzero(keep)) and
                     np.array_equal(out["pts"][:k].cpu().numpy(), want))
            res["clouds"][f"{name} r={radius} k={min_points}"] = dict(
                points=len(pts), kept=len(want), device_ms=round(dev, 4), pcl_e2e_ms=round(median(e2e), 3),
                oracle_cpu_1thread_ms=round(cpu, 2), exact=exact)

    limit = cta_limit(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)
    sizes = [4096, 8192, 12288, 16384, 20480, limit]
    res["one_cta_limit"] = limit
    res["sweep_one_cta_ms"] = sweep(sizes)
    if os.path.exists(args.map_lib):
        env = dict(os.environ, SFE_LIB_PATH=os.path.abspath(args.map_lib))
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--sweep", ",".join(map(str, sizes))],
                           env=env, capture_output=True, text=True)
        res["sweep_map_ms"] = json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else p.stderr[-500:]
    else:
        res["sweep_map_ms"] = f"not measured ({args.map_lib} missing)"
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
