"""Distribution of the scan-match problem sizes on bench.py's bag (CPU oracle chain, no GPU needed).

    python tools/icp_sizes.py [--frames 4096] [--procs N]

Per frame: ns = source points after the voxel and outlier filters, nt = window submap after the 0.5 m thinning (the
ICP target), and the submap before thinning.  Same seeded bag and parameters as bench.py (window 3, min_points 50).
Used to choose the front end's small ICP size class (pipeline.cu, FE_ICP_SMALL_*)."""
import argparse
import os
import re
import sys
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (the reference arm's per-frame cloud: bench._cpu_init / bench._cpu_cloud)


def small_class():
    """(FE_ICP_SMALL_SRC, FE_ICP_SMALL_TGT) as pipeline.cu defines them."""
    src = open(os.path.join(ROOT, "sonar_slam_b200", "csrc", "pipeline.cu")).read()
    m = re.search(r"FE_ICP_SMALL_SRC = (\d+), FE_ICP_SMALL_TGT = (\d+)", src)
    return int(m.group(1)), int(m.group(2))


def _target(parts):
    """bench._cpu_match's submap: the window's clouds in the previous frame's pose, thinned to 0.5 m."""
    from oracle import oracle as orc
    if not parts:
        return 0, 0
    tgt = np.concatenate(parts)
    thin, _ = orc.downsample(tgt, 0.5)
    return len(tgt), len(thin)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--procs", type=int, default=os.cpu_count())
    args = ap.parse_args()
    from oracle import pipeline_ref
    from sonar_slam_b200 import synth
    d = synth.make_trajectory_frames(args.frames, seed=0)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    with Pool(args.procs, initializer=bench._cpu_init, initargs=(d["bearings"],)) as pool:
        clouds = pool.map(bench._cpu_cloud, list(frames), chunksize=16)
        jobs = [[pipeline_ref.transform_points(clouds[k], pipeline_ref.between(poses[i - 1], poses[k]))
                 for k in range(max(0, i - 3), i)] for i in range(len(frames))]
        tg = pool.map(_target, jobs, chunksize=16)
    ns = np.array([len(c) for c in clouds])
    raw = np.array([t[0] for t in tg])
    nt = np.array([t[1] for t in tg])
    matched = (ns >= 50) & (nt >= 50)
    print(f"{args.frames} frames, {int(matched.sum())} matched (ns, nt >= 50)")
    print(f"{'per frame':34s} {'mean':>7s} {'p50':>6s} {'p90':>6s} {'p99':>6s} {'p99.9':>6s} {'max':>6s}")
    for name, v in (("source after filters (ns)", ns), ("window submap before thinning", raw),
                    ("submap after 0.5 m thinning (nt)", nt)):
        q = np.percentile(v, [50, 90, 99, 99.9])
        print(f"{name:34s} {v.mean():7.0f} {q[0]:6.0f} {q[1]:6.0f} {q[2]:6.0f} {q[3]:6.0f} {v.max():6d}")
    cs, ct = small_class()
    for name, (a, b) in (("pipeline.cu small class", (cs, ct)), ("former class", (640, 1536))):
        out = int((matched & ((ns > a) | (nt > b))).sum())
        print(f"{name} ns <= {a}, nt <= {b}: {out} matched frames outside (served by the capacity launch)")


if __name__ == "__main__":
    main()
