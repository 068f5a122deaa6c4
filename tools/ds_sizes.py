"""Input sizes of the front end's frame down-sample on bench.py's bag (CPU oracle chain, no GPU needed).

    python tools/ds_sizes.py [--frames 4096] [--procs N]

Per frame: the raw Cartesian points (CFAR -> remap -> nonzero, before any filter; the input of the per-frame voxel
filter) and, over all frames, the sizes of the 0.5 m quadtree leaves they fall into (members per leaf, the length of
the medoid sums).  The leaves are taken from the same tree as cloud.cu (ds_tree / ds_path_key), restated in numpy
float32.  Same seeded bag as bench.py.  Used to size the front end's frame class of the down-sample (pipeline.cu,
FE_DS_FRAME)."""
import argparse
import os
import re
import sys
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (the reference arm's geometry: bench._cpu_init)

RESOLUTION = 0.5


def frame_class():
    """FE_DS_FRAME as pipeline.cu defines it."""
    src = open(os.path.join(ROOT, "sonar_slam_b200", "csrc", "pipeline.cu")).read()
    return int(re.search(r"FE_DS_FRAME = (\d+)", src).group(1))


def leaf_sizes(pts, resolution=RESOLUTION):
    """Members per leaf of the down-sample's quadtree (cloud.cu: ds_tree + ds_path_key), depth-first order."""
    if len(pts) == 0:
        return np.zeros(0, np.int64), 0
    f = np.float32
    x, y = pts[:, 0].astype(f), pts[:, 1].astype(f)
    mn_x, mn_y, mx_x, mx_y = x.min(), y.min(), x.max(), y.max()
    rx, ry = f(mx_x - mn_x), f(mx_y - mn_y)
    cx0, cy0 = f(mn_x + f(rx * f(0.5))), f(mn_y + f(ry * f(0.5)))
    r = f(max(rx, ry) * f(0.5))
    D, rr = 0, r
    while not (float(rr) * 2.0 <= float(f(resolution))) and D < 15:
        rr, D = f(rr * f(0.5)), D + 1
    key = np.zeros(len(x), np.int64)
    cx, cy = np.full(len(x), cx0, f), np.full(len(x), cy0, f)
    rd = r
    for _ in range(D):
        bx, by = x > cx, y > cy
        key = (key << 2) | bx.astype(np.int64) | (by.astype(np.int64) << 1)
        rd = f(rd * f(0.5))
        cx = np.where(bx, cx + rd, cx - rd).astype(f)
        cy = np.where(by, cy + rd, cy - rd).astype(f)
    _, counts = np.unique(key, return_counts=True)
    return counts, D


def _raw(img):
    from oracle import pipeline_ref
    pts = pipeline_ref.frame_cloud(img, bench._W["geo"], tau=bench.TAU_SOCA, use_reference=True, resolution=0,
                                   min_points=1)
    sizes, D = leaf_sizes(pts)
    return len(pts), sizes, D


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--procs", type=int, default=os.cpu_count())
    args = ap.parse_args()
    from sonar_slam_b200 import synth
    d = synth.make_trajectory_frames(args.frames, seed=0)
    with Pool(args.procs, initializer=bench._cpu_init, initargs=(d["bearings"],)) as pool:
        res = pool.map(_raw, list(d["frames"].numpy()), chunksize=16)
    raw = np.array([r[0] for r in res])
    leaves = np.concatenate([r[1] for r in res])
    depth = np.bincount([r[2] for r in res])
    print(f"{args.frames} frames; tree depth D: " + ", ".join(f"{k}: {v}" for k, v in enumerate(depth) if v))
    print(f"{'':34s} {'mean':>7s} {'p50':>6s} {'p99':>6s} {'p99.9':>6s} {'max':>6s}")
    for name, v in (("raw points per frame", raw), ("members per 0.5 m leaf", leaves)):
        q = np.percentile(v, [50, 99, 99.9])
        print(f"{name:34s} {v.mean():7.1f} {q[0]:6.0f} {q[1]:6.0f} {q[2]:6.0f} {v.max():6d}")
    w = leaves.astype(np.float64)
    print(f"member-weighted mean leaf size (mean length of a member's sum): {(w * w).sum() / w.sum():.1f}")
    try:
        cls = frame_class()
        print(f"pipeline.cu frame class n <= {cls}: {int((raw > cls).sum())} frames outside (capacity launch)")
    except (AttributeError, OSError):
        pass


if __name__ == "__main__":
    main()
