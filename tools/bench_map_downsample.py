"""Whole-map down-sampling (pcl.downsample on SLAM.get_points-sized clouds): device time of sfe_downsample_dev on
resident data (CUDA events), pcl.downsample end to end (copy in, kernels, copy out) and the CPU oracle on one thread,
every result checked against the oracle; then a sweep of single clouds either side of the one-CTA limit, as shipped
and from a build where every cloud takes the grid-wide path (tools/build_map_class_variant.sh).
Prints one JSON line.

    python tools/bench_map_downsample.py [--out FILE] [--grid-lib scratch/lib_mapclass.so]
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
RES = 0.5  # slam.yaml point_resolution


def median(v):
    return float(np.median(np.asarray(v)))


def device_ms(pts_np, reps=10):
    """sfe_downsample_dev on one resident cloud (n_max = its size): median of `reps` event-timed calls."""
    import torch
    from sonar_slam_b200 import ops
    pts = torch.from_numpy(pts_np).cuda()
    off = torch.tensor([0, len(pts_np)], dtype=torch.int32, device="cuda")
    ctx = ops.context(0)
    for _ in range(2):
        out = ops.downsample(pts, off, len(pts_np), RES, ctx=ctx)
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(torch.cuda.current_stream())
        out = ops.downsample(pts, off, len(pts_np), RES, ctx=ctx)
        e1.record(torch.cuda.current_stream())
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return median(ts), out


def sweep(sizes):
    from sonar_slam_b200 import synth
    base = synth.make_map_cloud(max(sizes), seed=1)[0]
    return {str(n): device_ms(np.ascontiguousarray(base[:n]))[0] for n in sizes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    ap.add_argument("--grid-lib", default=os.path.join(REPO, "scratch", "lib_mapclass.so"),
                    help="library built with SFE_MAP_CLASS_ALL (every cloud on the grid-wide path)")
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
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown", resolution=RES, clouds={})
    rng = np.random.default_rng(2)
    clouds = {
        "map_200k": synth.make_map_cloud(200000, seed=1)[0],
        "map_360k": synth.make_map_cloud(360000, seed=1)[0],
        "map_1M": synth.make_map_cloud(1000000, seed=1)[0],
        "uniform_1M": rng.uniform(0, 350, (1000000, 2)).astype(np.float32),
        "leaf_20k": rng.uniform(10.0, 10.5, (20000, 2)).astype(np.float32),
    }
    for name, pts in clouds.items():
        dev, out = device_ms(pts)
        pcl.downsample(pts, RES)
        e2e = []
        for _ in range(5):
            t0 = time.perf_counter()
            got = pcl.downsample(pts, RES)
            e2e.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        want, widx = orc.downsample(pts, RES)
        cpu = (time.perf_counter() - t0) * 1e3
        k = int(out["count"][0])
        exact = (np.array_equal(got, want) and k == len(want) and
                 np.array_equal(out["idx"][:k].cpu().numpy(), widx) and np.array_equal(out["pts"][:k].cpu().numpy(), want))
        res["clouds"][name] = dict(points=len(pts), kept=len(want), device_ms=round(dev, 4),
                                   pcl_e2e_ms=round(median(e2e), 3), oracle_cpu_1thread_ms=round(cpu, 2), exact=exact)

    # either side of the one-CTA limit (13 880 points on an H100: cloud.cu, downsample_cta_limit)
    sizes = [4096, 8192, 13000, 16384, 24576, 57084]
    res["sweep_ms"] = sweep(sizes)
    if os.path.exists(args.grid_lib):
        env = dict(os.environ, SFE_LIB_PATH=os.path.abspath(args.grid_lib))
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--sweep", ",".join(map(str, sizes))],
                           env=env, capture_output=True, text=True)
        res["sweep_grid_ms"] = json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else p.stderr[-500:]
    else:
        res["sweep_grid_ms"] = f"not measured ({args.grid_lib} missing)"
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
