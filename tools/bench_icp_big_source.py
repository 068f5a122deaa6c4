"""Scan matching with large sources (the global-source class): what crossing the class boundary costs, and 2-D / 3-D
map-to-map alignment with sources of 20 k, 70 k and 200 k points against ~245 k-point map targets.

Workloads (every target is the 1.6 M-point synth.make_map_cloud down-sampled at 0.05 m, 243 726 points; 3-D: the same
map over an undulating floor):
  boundary   sources of exactly ops.icp_source_limit points (the map class) and one more (the global-source class),
             2-D and 3-D, 30 guesses
  map2d      2-D sources of 20 k, 70 k and 200 k points, 1 and 30 guesses
  map3d      3-D sources of 20 k, 70 k and 200 k points, 1 and 30 guesses
Sources are map points with 2 cm of noise moved by a known rigid transform; guesses scatter 0.3 m / 0.03 rad around it.
Shipped checkers (icp.yaml).  Per row:
  device_ms        ops.icp on device tensors between two CUDA events, median of 5 (after a warm-up call)
  build_ms/icp_ms  torch.profiler kernel time of one call in a separate pass: the map-grid build (every kernel that is not
                   icp_kernel / icp3_*) and the ICP kernels
  batch_ms         pcl.ICP.compute_batch end to end (copies in, kernels, copies out), median of 3
  cpu_ms           the CPU oracle (oracle/icp_ref.c, icp3_ref.c) on one host thread for one guess
  exact            the first min(3, guesses) device results equal the oracle's bit for bit (status, iterations, inliers, T)
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/bench_icp_big_source.py [--out FILE] [--only map3d:200000:30]
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
F32 = np.float32


def median(v):
    return float(np.median(np.asarray(v)))


def maps():
    from oracle import oracle as orc
    from sonar_slam_b200 import synth
    m = orc.downsample(synth.make_map_cloud(1600000, seed=11)[0], 0.05)[0]
    md = m.astype(np.float64)
    z = 0.8 * np.sin(md[:, 0] / 9.0) * np.cos(md[:, 1] / 7.0) + np.random.default_rng(3).normal(0, 0.03, len(m))
    return m, np.c_[md, z].astype(F32)


def problem(tgt, n, k, seed):
    """n points of tgt with 2 cm of noise, moved by a rigid transform about the map's centre, and k guesses near it"""
    from sonar_slam_b200 import synth
    rng = np.random.default_rng(seed)
    dim = tgt.shape[1]
    pts = tgt[rng.permutation(len(tgt))[:n]].astype(np.float64)
    pts += np.random.default_rng(seed + 1).normal(0, 0.02, (len(tgt), dim))[:n]  # (n and n + 1: the same first n)
    rng = np.random.default_rng(seed + 2)  # (the transform and the guesses do not depend on n)
    c = tgt.mean(0).astype(np.float64)

    def rigid(t, angle, axis):
        if dim == 2:
            co, si = np.cos(angle), np.sin(angle)
            return np.array([[co, -si, t[0]], [si, co, t[1]], [0, 0, 1]])
        return synth.se3(t, axis, angle)

    T = rigid(c[:dim] + rng.normal(0, 2, dim), rng.uniform(-np.pi, np.pi), np.array([0.1, -0.2, 1.0]))
    src = ((pts - T[:dim, dim]) @ T[:dim, :dim]).astype(F32)
    guesses = [(rigid(rng.normal(0, 0.3, dim), rng.normal(0, 0.03), rng.normal(size=3)) @ T).astype(F32)
               for _ in range(k)]
    return src, guesses


def oracle(src, tgt, g):
    from oracle import icp3_ref as o3
    from oracle import oracle as orc
    return o3.icp3(src, tgt, g) if src.shape[1] == 3 else orc.icp(src, tgt, g)


def measure(name, src, tgt, guesses):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from sonar_slam_b200 import _lib, ops
    from sonar_slam_b200.bruce_slam import pcl
    icp = pcl.ICP()
    icp.loadFromYaml("/nonexistent")  # the shipped icp.yaml values
    dim = src.shape[1]
    sp = torch.from_numpy(src).cuda()
    tp = torch.from_numpy(tgt).cuda()
    so = torch.tensor([0, len(src)], dtype=torch.int32).cuda()
    to = torch.tensor([0, len(tgt)], dtype=torch.int32).cuda()
    zero = torch.zeros(len(guesses), dtype=torch.int32).cuda()
    g = torch.from_numpy(np.stack(guesses)).cuda()
    prm = _lib.IcpParams()
    call = lambda: ops.icp(sp, so, tp, to, g, len(src), len(tgt), prm, src_id=zero, tgt_id=zero)
    res = call()
    torch.cuda.synchronize()
    dev = {k: v.cpu().numpy() for k, v in res.items()}
    exact = True
    for k in range(min(3, len(guesses))):
        w = oracle(src, tgt, guesses[k])
        exact &= (int(dev["status"][k]) == w["status"] and int(dev["iterations"][k]) == w["iterations"] and
                  int(dev["inliers"][k]) == w["inliers"] and dev["T"][k].tobytes() == np.asarray(w["T"], F32).tobytes())
    ev = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        torch.cuda.synchronize()
        ev.append(a.elapsed_time(b))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    build = kern = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA" or "memcpy" in e.name.lower() or "memset" in e.name.lower():
            continue
        us = getattr(e, "device_time_total", None)
        us = us if us is not None else e.cuda_time_total
        if "icp_kernel" in e.name or "icp3_kernel" in e.name or "icp3_map_kernel" in e.name or "icp3_gsrc" in e.name:
            kern += us
        else:
            build += us
    icp.compute_batch(src, tgt, guesses)
    batch = []
    for _ in range(3):
        t = time.perf_counter()
        icp.compute_batch(src, tgt, guesses)
        batch.append((time.perf_counter() - t) * 1e3)
    t = time.perf_counter()
    oracle(src, tgt, guesses[0])
    cpu = (time.perf_counter() - t) * 1e3
    lim = ops.icp_source_limit(dim, prm)
    return dict(name=name, dim=dim, n_source=len(src), n_target=len(tgt), guesses=len(guesses),
                global_source=len(src) > lim, status=[int(v) for v in dev["status"][:3]],
                iterations=[int(v) for v in dev["iterations"][:3]],
                device_ms=round(median(ev), 3), build_ms=round(build / 1e3, 3), icp_ms=round(kern / 1e3, 3),
                batch_ms=round(median(batch), 3), cpu_ms=round(cpu, 1), exact=bool(exact))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default=None, help="the rows whose name:source points:guesses starts with this text")
    args = ap.parse_args()
    want = lambda name, n, k: args.only is None or f"{name}:{n}:{k}".startswith(args.only)
    import torch
    from sonar_slam_b200 import _lib, ops
    m2, m3 = maps()
    rows = []
    for dim, tgt in ((2, m2), (3, m3)):
        lim = ops.icp_source_limit(dim, _lib.IcpParams())
        for n in (lim, lim + 1):
            if not want(f"boundary{dim}d", n, 30):
                continue
            src, gs = problem(tgt, n, 30, 7)
            rows.append(measure(f"boundary{dim}d", src, tgt, gs))
            print(json.dumps(rows[-1]), file=sys.stderr)
    for dim, tgt in ((2, m2), (3, m3)):
        for n in (20000, 70000, 200000):
            for k in (1, 30):
                if not want(f"map{dim}d", n, k):
                    continue
                src, gs = problem(tgt, n, k, 8)
                rows.append(measure(f"map{dim}d", src, tgt, gs))
                print(json.dumps(rows[-1]), file=sys.stderr)
    p = torch.cuda.get_device_properties(0)
    try:
        pw = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pw = None
    line = json.dumps(dict(gpu=p.name, power_limit_w=pw, checkers="shipped", rows=rows))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
