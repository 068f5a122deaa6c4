"""3-D clouds through `pcl.downsample` and `pcl.match` / `pcl.match_knn`, next to the 2-D calls on the same xy points.
Clouds: synth.make_map_cloud's walls of 20 000, 200 000 and 1 000 000 points with z uniform over 4 m (the xy columns
are the 2-D clouds); 2 000 queries near each (xy + N(0, 0.2) per axis).  Per cloud and dim:
  downsample (resolution 0.5)
    device_ms  sfe_downsample_dev through ops.downsample on device-resident points, CUDA events around the call
               (median of 10)
    pcl_ms     pcl.downsample end to end (copies in, kernels, copies out; host clock, median of 5)
    oracle_ms  the CPU oracle (orc_downsample3 / orc_downsample) on one host thread (median of 3)
  match, knn 1, 5 and 16 (max_dist 2)
    device_ms  sfe_match_knn_dim_dev through ops.match (3-D) / sfe_match_dev, sfe_match_knn_dev (2-D), CUDA events
               (median of 10)
    pcl_ms     pcl.match (knn 1) / pcl.match_knn end to end (median of 5)
    ckdtree_ms scipy cKDTree build + query(k, distance_upper_bound) on one host thread (median of 3)
Every row's device result is compared with the CPU oracle (index for index, float32 bit for bit): `exact`.
Prints one JSON line with the card's name and power limit.

    python tools/bench_3d_clouds.py [--out FILE] [--sizes 20000,200000,1000000]
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
RES = 0.5
MAX_DIST = 2.0
N_QUERY = 2000


def median(v):
    return float(np.median(np.asarray(v)))


def host_ms(fn, reps):
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t) * 1e3)
    return median(out)


def device_ms(fn, reps=10):
    import torch
    fn()  # warm-up
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return median(out)


def cloud(n, seed):
    from sonar_slam_b200 import synth
    xy = synth.make_map_cloud(n, seed=seed)[0]
    rng = np.random.default_rng(seed + 1)
    pts = np.c_[xy, rng.uniform(0, 4, n)].astype(np.float32)
    q = (pts[rng.integers(n, size=N_QUERY)] + rng.normal(0, 0.2, (N_QUERY, 3))).astype(np.float32)
    return pts, q


def bench_downsample(pts):
    import torch

    from oracle import cloud3_ref as c3
    from oracle import oracle as orc
    from sonar_slam_b200 import ops
    from sonar_slam_b200.bruce_slam import pcl
    oracle = c3.downsample3 if pts.shape[1] == 3 else orc.downsample
    d = torch.from_numpy(pts).cuda()
    off = torch.tensor([0, len(pts)], dtype=torch.int32, device="cuda")
    dev = device_ms(lambda: ops.downsample(d, off, len(pts), RES))
    out = ops.downsample(d, off, len(pts), RES)
    torch.cuda.synchronize()
    want, widx = oracle(pts, RES)
    m = int(out["count"][0])
    exact = (m == len(widx) and np.array_equal(out["idx"][:m].cpu().numpy(), widx)
             and np.array_equal(out["pts"][:m].cpu().numpy().view(np.uint32), want.view(np.uint32))
             and np.array_equal(pcl.downsample(pts, RES), want))
    return dict(n_out=len(widx), device_ms=dev, pcl_ms=host_ms(lambda: pcl.downsample(pts, RES), 5),
                oracle_ms=host_ms(lambda: oracle(pts, RES), 3), exact=bool(exact))


def bench_match(ref, q, knn):
    import torch
    from scipy.spatial import cKDTree

    from oracle import cloud3_ref as c3
    from oracle import knn_ref
    from sonar_slam_b200 import ops
    from sonar_slam_b200.bruce_slam import pcl
    rp, ip = torch.from_numpy(ref).cuda(), torch.from_numpy(q).cuda()
    ro = torch.tensor([0, len(ref)], dtype=torch.int32, device="cuda")
    io = torch.tensor([0, len(q)], dtype=torch.int32, device="cuda")
    kk = None if knn == 1 else knn  # 2-D knn 1: sfe_match_dev, the call pcl.match makes
    dev = device_ms(lambda: ops.match(rp, ro, ip, io, len(ref), MAX_DIST, knn=kk))
    out = ops.match(rp, ro, ip, io, len(ref), MAX_DIST, knn=kk)
    torch.cuda.synchronize()
    wi, wd = (c3.match_knn3 if ref.shape[1] == 3 else knn_ref.match_knn)(ref, q, knn, MAX_DIST)

    def call():
        return pcl.match(ref, q, 1, MAX_DIST) if knn == 1 else pcl.match_knn(ref, q, knn, MAX_DIST)

    ids, d = call()
    exact = (np.array_equal(out["ids"].cpu().numpy().reshape(knn, -1), wi)
             and np.array_equal(out["dists"].cpu().numpy().reshape(knn, -1).view(np.uint32), wd.view(np.uint32))
             and np.array_equal(ids, wi) and np.array_equal(d.view(np.uint32), wd.view(np.uint32)))
    kd = host_ms(lambda: cKDTree(ref).query(q, k=knn, distance_upper_bound=MAX_DIST, workers=1), 3)
    return dict(knn=knn, device_ms=dev, pcl_ms=host_ms(call, 5), ckdtree_ms=kd, exact=bool(exact))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", default="20000,200000,1000000")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_3d_clouds.py measures on a GPU"
    from sonar_slam_b200 import ops
    rows = []
    for i, n in enumerate(int(s) for s in args.sizes.split(",")):
        pts, q = cloud(n, seed=10 + i)
        for dim in (3, 2):
            p, qq = np.ascontiguousarray(pts[:, :dim]), np.ascontiguousarray(q[:, :dim])
            rows.append(dict(n=n, dim=dim, downsample=bench_downsample(p),
                             match=[bench_match(p, qq, k) for k in KNNS]))
    p = torch.cuda.get_device_properties(0)
    try:
        pw = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pw = None
    line = json.dumps(dict(gpu=p.name, power_limit_w=pw, resolution=RES, max_dist=MAX_DIST, n_query=N_QUERY,
                           cta_limit_downsample={"2": ops.downsample_cta_limit(2), "3": ops.downsample_cta_limit(3)},
                           exact=all(r["downsample"]["exact"] and all(m["exact"] for m in r["match"]) for r in rows),
                           rows=rows))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
