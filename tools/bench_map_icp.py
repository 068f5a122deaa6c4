"""Loop-closure scan matching against whole maps: the 30-guess SLAM.compute_icp_with_cov on map targets of 25 k, 50 k,
100 k and ~245 k points (a 1 500-point source cut from the map).  Per size:
  build_ms / icp_ms  device time of the map-grid build (map_* kernels, CUB sort and scan) and of the scan-match launches
                     of one ICP.compute_batch call (kernel durations from torch.profiler, median of 10 calls)
  batch_ms           ICP.compute_batch end to end (copies in, kernels, copies out), median of 10
  cov_ms             SLAM.compute_icp_with_cov end to end (the batch plus scikit-learn's MinCovDet), median of 10
  cpu_ms             the CPU oracle's 30 ICP runs on one thread
every device result checked against the oracle.  Then one 16 k target that both layouts hold, through the shipped build
(in-CTA kernel) and through scratch/lib_mapclass.so (tools/build_map_class_variant.sh: every target in the map class): what
reading the target from a global-memory grid costs.  Prints one JSON line.

    python tools/bench_map_icp.py [--out FILE] [--map-lib scratch/lib_mapclass.so]
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
SIZES = (25000, 50000, 100000, 250000)


def median(v):
    return float(np.median(np.asarray(v)))


def big_map():
    from oracle import oracle as orc
    from sonar_slam_b200 import synth
    return orc.downsample(synth.make_map_cloud(1600000, seed=11)[0], 0.05)[0]


def problem(tgt, seed=1, n=1500):
    rng = np.random.default_rng(seed)
    centre = tgt[rng.integers(len(tgt))]
    near = tgt[np.linalg.norm(tgt - centre, axis=1) < 30.0]
    pts = near[rng.choice(len(near), min(n, len(near)), replace=False)]
    c, s = np.cos(0.7), np.sin(0.7)
    R = np.array([[c, -s], [s, c]])
    src = ((pts - centre) @ R).astype(np.float32)
    guesses = []
    for _ in range(30):
        th = 0.7 + rng.normal(0, 0.02)
        guesses.append((centre[0] + rng.normal(0, 0.2), centre[1] + rng.normal(0, 0.2), th))
    return src, guesses


def measure(tgt, src, guesses, cpu=True):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from oracle import oracle as orc
    from sonar_slam_b200.bruce_slam.slam import SLAM, Pose2
    slam = SLAM()
    slam.icp.loadFromYaml("/nonexistent")  # the shipped icp.yaml values
    poses = [Pose2(*g) for g in guesses]
    mats = [p.matrix() for p in poses]
    res = slam.icp.compute_batch(src, tgt, mats)  # warm-up (and the result checked below)
    for k, m in enumerate(mats):
        w = orc.icp(src, tgt, m.astype(np.float32))
        assert int(res["status"][k]) == w["status"] and np.array_equal(res["T"][k], w["T"]), k
    batch = []
    for _ in range(10):
        t = time.perf_counter()
        slam.icp.compute_batch(src, tgt, mats)
        batch.append((time.perf_counter() - t) * 1e3)
    cov = []
    for _ in range(10):
        t = time.perf_counter()
        slam.compute_icp_with_cov(src, tgt, poses)
        cov.append((time.perf_counter() - t) * 1e3)
    build, icp = [], []
    for _ in range(10):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            slam.icp.compute_batch(src, tgt, mats)
            torch.cuda.synchronize()
        b = i = 0.0
        for e in prof.events():
            if e.device_type.name != "CUDA" or "memcpy" in e.name.lower() or "memset" in e.name.lower():
                continue
            us = getattr(e, "device_time_total", None)
            us = us if us is not None else e.cuda_time_total
            if "icp_kernel" in e.name:  # both classes: icp_kernel<..., MAP, ...>
                i += us
            else:
                b += us
        build.append(b / 1e3)
        icp.append(i / 1e3)
    out = dict(n_target=len(tgt), n_source=len(src), build_ms=median(build), icp_ms=median(icp),
               batch_ms=median(batch), cov_ms=median(cov))
    if cpu:
        t = time.perf_counter()
        for m in mats:
            orc.icp(src, tgt, m.astype(np.float32))
        out["cpu_ms"] = (time.perf_counter() - t) * 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--map-lib", default=os.path.join(REPO, "scratch", "lib_mapclass.so"))
    ap.add_argument("--one", type=int, default=0, help=argparse.SUPPRESS)  # child: the 16 k target only
    args = ap.parse_args()
    import torch
    world = big_map()
    if args.one:
        tgt = world[: args.one]
        src, guesses = problem(tgt, seed=3)
        print(json.dumps(measure(tgt, src, guesses, cpu=False)))
        return
    rows = []
    for n in SIZES:
        tgt = world[:n]
        src, guesses = problem(tgt, seed=2)
        rows.append(measure(tgt, src, guesses))
    forced = {}
    for tag, lib in (("in_cta", None), ("map_class", args.map_lib)):
        env = dict(os.environ)
        if lib:
            if not os.path.exists(lib):
                forced[tag] = "not measured: build it with tools/build_map_class_variant.sh"
                continue
            env["SFE_LIB_PATH"] = lib
        out = subprocess.run([sys.executable, __file__, "--one", "16000"], env=env, capture_output=True, text=True)
        forced[tag] = json.loads(out.stdout.strip().splitlines()[-1]) if out.returncode == 0 else out.stderr[-400:]
    p = torch.cuda.get_device_properties(0)
    try:
        pw = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pw = None
    line = json.dumps(dict(gpu=p.name, power_limit_w=pw, guesses=30, sizes=rows, target_16k=forced))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
