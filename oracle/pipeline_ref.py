"""TEST INFRASTRUCTURE ONLY -- CPU oracle of the batched per-keyframe front end.

Chains the oracle pieces exactly as the reference chains its own calls:
  per frame    FeatureExtraction.callback, feature_extraction.py:220-249
               (CFAR -> `&= img > threshold` -> cv2.remap -> nonzero -> metres -> pcl.downsample ->
               pcl.remove_outlier; float32 where pybind converts)
  hand-over    publish_features sends xyz = [p0, 0, p1] as float32 (feature_extraction.py:182); the SLAM node
               reads `points = np.c_[x, -z]` = (p0, -p1) (slam_ros.py:169-170): the keyframe cloud is the
               feature cloud with its lateral coordinate negated (`slam_cloud`).
  per keyframe SLAM.initialize_sequential_scan_matching / add_sequential_scan_matching,
               slam.py:626-633,769-771: target = get_points(previous `window` frames, ref = previous
               frame) = Keyframe.transform_points (float32 `points @ R^T + t`, slam_objects.py:178-198)
               + concatenate + pcl.downsample; guess = between(pose[i-1], pose[i]); ICP.compute.
"""
import math
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import featx_ref, oracle as orc


def between(a, b):
    """gtsam Pose2.between(a, b).matrix().astype(float32) for poses (x, y, theta): rotation r_a^-1 * r_b formed
    from the (cos, sin) pairs like gtsam's Rot2 product, translation r_a.unrotate(t_b - t_a)."""
    ca, sa, cb, sb = math.cos(a[2]), math.sin(a[2]), math.cos(b[2]), math.sin(b[2])
    dx, dy = b[0] - a[0], b[1] - a[1]
    x, y = ca * dx + sa * dy, -sa * dx + ca * dy
    c, s = ca * cb + sa * sb, ca * sb - sa * cb
    return np.array([[c, -s, x], [s, c, y], [0, 0, 1]], np.float64).astype(np.float32)


def transform_points(points, T):
    """Keyframe.transform_points (slam_objects.py:178-198: `points.dot(T[:2,:2].T) + T[:2,2]`) with a float32 T.
    numpy's float32 dot evaluates fl32(fma(y, r01, fl32(x * r00))) on FMA hardware (checked point for point in
    tests/test_oracle_globalinit.py); spelled out here so the oracle does not depend on the host's BLAS kernel."""
    p = np.asarray(points, np.float32)
    x, y = p[:, 0], p[:, 1]

    def row(r0, r1, t):
        first = (x * r0).astype(np.float32)
        acc = (y.astype(np.float64) * np.float64(r1) + first.astype(np.float64)).astype(np.float32)
        return (acc + t).astype(np.float32)
    return np.stack([row(T[0, 0], T[0, 1], T[0, 2]), row(T[1, 0], T[1, 1], T[1, 2])], 1)


def frame_cloud(img, geo, alg="SOCA", train_hs=20, guard_hs=5, rank=10, tau=2.749063720096473, threshold=65,
                resolution=0.5, radius=1.0, min_points=5, use_reference=False, cap_points=None):
    return frame_cloud_raw(img, geo, alg, train_hs, guard_hs, rank, tau, threshold, resolution, radius, min_points,
                           use_reference, cap_points)[0]


def frame_cloud_raw(img, geo, alg="SOCA", train_hs=20, guard_hs=5, rank=10, tau=2.749063720096473, threshold=65,
                    resolution=0.5, radius=1.0, min_points=5, use_reference=False, cap_points=None):
    """(frame_cloud, the number of Cartesian points before the filters).  cap_points: the front end's per-frame
    capacity -- a frame with more points keeps its first cap_points (row-major order) before the filters."""
    if use_reference and orc.have_reference():  # the unmodified reference cfar.cpp (oracle/_ref)
        mask, _ = orc.cfar_reference(alg, img, train_hs, guard_hs, rank, tau)
        mask = np.ascontiguousarray(mask)
        mask &= img > threshold
    else:
        mask = orc.cfar_u8(alg, img, train_hs, guard_hs, rank, tau, threshold)
    _, pts = featx_ref.cart_points(mask, geo)
    raw = len(pts)
    pts = pts[:cap_points].astype(np.float32)  # pybind: points -> Eigen float matrix
    if len(pts) and resolution > 0:
        pts, _ = orc.downsample(pts, resolution)
    if min_points > 1 and len(pts) > 0:
        pts, _ = orc.remove_outlier(pts, radius, min_points)
    return pts, raw


def slam_cloud(points, flip_lateral=True):
    """feature_extraction.py:182 -> slam_ros.py:169-170: float32 xyz = [p0, 0, p1] on the wire, read back as
    (x, -z).  `flip_lateral=False` keeps FeatureExtraction.callback's own convention."""
    pts = np.asarray(points, np.float32)
    if not flip_lateral or len(pts) == 0:
        return pts
    xyz = np.c_[pts[:, 0], np.zeros(len(pts), np.float32), pts[:, 1]].astype(np.float32)
    return np.c_[xyz[:, 0], -1 * xyz[:, 2]].astype(np.float32)


def run(frames, poses, geo, window=3, submap_resolution=0.5, min_points=50, icp_params=None, flip_lateral=True,
        cap_points=None, cap_source=None, cap_target=None, icp_filters=None, threads=1, **feat_kw):
    """Returns (clouds, results); clouds = the keyframe clouds as SLAM holds them;
    results[i] = dict(status, T, iterations, inliers, n_target).
    The batched front end's limits (None: none): cap_points cuts every frame's Cartesian cloud (frame_cloud_raw),
    and a frame that overflowed it, or whose source / window submap exceeds cap_source / cap_target, is TOO_LARGE (8)
    before the min_points test.  icp_filters: a voxel_filter_ref.IcpFilters for the scan match (the min_points test
    counts the clouds before its data filters).  threads: host threads for the frames' clouds and the scan matches
    (the oracle's C calls release the GIL); the results do not depend on it."""
    prm = icp_params or orc.IcpParams()
    orc._load_port()  # (load, and build if need be, the oracle libraries before any thread calls them)
    if icp_filters is not None:
        from . import voxel_filter_ref
        voxel_filter_ref._load()
    pool = ThreadPoolExecutor(max(1, int(threads)))
    made = list(pool.map(lambda f: frame_cloud_raw(f, geo, cap_points=cap_points, **feat_kw), frames))
    clouds = [slam_cloud(c, flip_lateral) for c, _ in made]
    results = []
    for i in range(len(frames)):
        guess = between(poses[i - 1], poses[i]) if i > 0 else np.eye(3, dtype=np.float32)
        parts = [transform_points(clouds[k], between(poses[i - 1], poses[k])) for k in range(max(0, i - window), i)]
        tgt = np.concatenate(parts) if parts else np.zeros((0, 2), np.float32)
        if len(tgt) and submap_resolution > 0:
            tgt, _ = orc.downsample(tgt, submap_resolution)
        src = clouds[i]
        skip = dict(T=guess, iterations=0, inliers=0, n_target=len(tgt))
        if ((cap_points is not None and made[i][1] > cap_points) or (cap_source is not None and len(src) > cap_source)
                or (cap_target is not None and len(tgt) > cap_target)):
            results.append(dict(status=8, **skip))
            continue
        if len(src) < min_points or len(tgt) < min_points:
            results.append(dict(status=7, **skip))
            continue
        results.append(pool.submit(_match, src, tgt, guess, prm, icp_filters))
    results = [r.result() if not isinstance(r, dict) else r for r in results]
    pool.shutdown()
    return clouds, results


def _match(src, tgt, guess, prm, icp_filters):
    if icp_filters is None:
        r = orc.icp(src, tgt, guess, prm)
    else:
        from . import voxel_filter_ref
        r = voxel_filter_ref.icp(src, tgt, guess, prm, icp_filters)
    r["n_target"] = len(tgt)
    return r
