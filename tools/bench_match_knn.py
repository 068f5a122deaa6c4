"""k-nearest-neighbour matching (`pcl.match_knn(ref, in, knn, max_dist)`) for knn 1, 5 and 16 on two workloads:
  config3  a 20 000-point reference (synth.make_icp_pair's target) and its 2 000-point source as queries: one CTA
  map      a 200 000-point whole map (synth.make_map_cloud) and 20 000 queries near it: the map class
Per (workload, knn):
  device_ms  ops.match on device-resident clouds, CUDA events around the call (median of 10): every kernel of the call,
             the map-grid build included
  pcl_ms     pcl.match_knn end to end (copies in, kernels, copies out; host clock, median of 10)
  ckdtree_ms scipy cKDTree build + query(k, distance_upper_bound) on one host thread (median of 3)
Every device result is checked bit for bit against the brute-force oracle (on the first 2 000 queries of the map
workload).  max_dist 10 (icp.yaml's maxDist).  Prints one JSON line with the card's name and power limit.

    python tools/bench_match_knn.py [--out FILE]
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
KNNS = (1, 5, 16)
MAX_DIST = 10.0


def median(v):
    return float(np.median(np.asarray(v)))


def workloads():
    from sonar_slam_b200 import synth
    src, tgt, _ = synth.make_icp_pair(3)
    world = synth.make_map_cloud(200000, seed=5)[0]
    rng = np.random.default_rng(6)
    q = (world[rng.integers(len(world), size=20000)] + rng.normal(0, 0.5, (20000, 2))).astype(np.float32)
    return {"config3": (tgt, src), "map": (world, q)}


def measure(ref, q, knn):
    import torch
    from scipy.spatial import cKDTree

    from oracle import knn_ref
    from sonar_slam_b200 import ops
    from sonar_slam_b200.bruce_slam import pcl
    rp = torch.from_numpy(ref).cuda()
    ip = torch.from_numpy(q).cuda()
    ro = torch.tensor([0, len(ref)], dtype=torch.int32, device="cuda")
    io = torch.tensor([0, len(q)], dtype=torch.int32, device="cuda")
    out = ops.match(rp, ro, ip, io, len(ref), MAX_DIST, knn=knn)  # warm-up, checked below
    torch.cuda.synchronize()
    n_chk = min(len(q), 2000)
    wi, wd = knn_ref.match_knn(ref, q[:n_chk], knn, MAX_DIST)
    assert np.array_equal(out["ids"][:, :n_chk].cpu().numpy(), wi), knn
    assert np.array_equal(out["dists"][:, :n_chk].cpu().numpy().view(np.uint32), wd.view(np.uint32)), knn
    dev = []
    for _ in range(10):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ops.match(rp, ro, ip, io, len(ref), MAX_DIST, knn=knn)
        b.record()
        b.synchronize()
        dev.append(a.elapsed_time(b))
    ids, _ = pcl.match_knn(ref, q, knn, MAX_DIST)
    assert np.array_equal(ids, out["ids"].cpu().numpy())
    host = []
    for _ in range(10):
        t = time.perf_counter()
        pcl.match_knn(ref, q, knn, MAX_DIST)
        host.append((time.perf_counter() - t) * 1e3)
    kd = []
    for _ in range(3):
        t = time.perf_counter()
        cKDTree(ref).query(q, k=knn, distance_upper_bound=MAX_DIST, workers=1)
        kd.append((time.perf_counter() - t) * 1e3)
    return dict(knn=knn, device_ms=median(dev), pcl_ms=median(host), ckdtree_ms=median(kd))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    rows = {}
    for name, (ref, q) in workloads().items():
        rows[name] = dict(n_ref=len(ref), n_query=len(q), runs=[measure(ref, q, k) for k in KNNS])
    p = torch.cuda.get_device_properties(0)
    try:
        pw = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pw = None
    line = json.dumps(dict(gpu=p.name, power_limit_w=pw, max_dist=MAX_DIST, workloads=rows))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
