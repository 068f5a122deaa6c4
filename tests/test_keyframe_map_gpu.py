"""SLAM.get_points served from the device-resident keyframe map (sfe_keyframe_map, bruce_slam.slam.KeyframeList):
bit-exact against the host path on a plain list (numpy transform + pcl.downsample) and the oracle chain (numpy
transform_points + oracle.downsample)."""
import os
import types

import numpy as np
import pytest

from oracle import oracle as orc
from sonar_slam_b200 import _lib, synth
from sonar_slam_b200.bruce_slam import pcl
from sonar_slam_b200.bruce_slam.slam import SLAM, Pose2, transform_points
from sonar_slam_b200.keyframe_map import KeyframeMap

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "slam_host.npz")


def _kf(points, pose):
    return types.SimpleNamespace(points=points, pose=pose)


def _pair(kfs):
    """(resident, host): SLAM() with the keyframes appended, and one with a plain list of the same keyframes."""
    res = SLAM()
    res.keyframes.extend(kfs)
    host = SLAM()
    host.keyframes = list(kfs)
    return res, host


def _same(a, b):
    if isinstance(a, tuple):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


def _oracle(kfs, frames, ref_pose, keys, res=0.5):
    """slam.py:229-292 restated: numpy transform_points, concatenation, the oracle's down-sample."""
    parts = [np.zeros((0, 3), np.float64)]
    for k in frames:
        kf = kfs[k]
        pts = transform_points(kf.points, ref_pose.between(kf.pose) if ref_pose is not None else kf.pose)
        parts.append(np.c_[pts, k * np.ones((len(pts), 1))])
    allp = np.concatenate(parts)
    if len(allp) == 0:
        e = np.zeros((0, 2), np.float32)
        return (e, np.zeros((0, 1), np.float32)) if keys else e
    out, idx = orc.downsample(np.ascontiguousarray(allp[:, :2], np.float32), res)
    return (out, allp[idx][:, (2,)].astype(np.float32)) if keys else out


def test_golden_fixture_through_the_resident_path(gpu_ctx):
    g = np.load(GOLD)
    res, _ = _pair([_kf(g[f"kf{k}_points"], Pose2(*g[f"kf{k}_pose"])) for k in range(4)])
    assert _same(res.get_points(), g["points_all"])
    assert _same(res.get_points([0, 1, 2], 3), g["points_ref_idx"])
    assert _same(res.get_points([1, 3], Pose2(1.0, 0.5, -0.2)), g["points_ref_pose"])
    pts, keys = res.get_points([0, 2, 3], 1, True)
    assert _same(pts, g["points_keys_pts"]) and np.array_equal(keys, g["points_keys_keys"])
    assert keys.dtype == np.float32 and keys.shape == (len(pts), 1)
    assert res.keyframes.map.size == (4, sum(len(g[f"kf{k}_points"]) for k in range(4)))


def _random_keyframes(n, total, seed):
    """n keyframes of random sizes (a few empty, some of 3 points, one of 7 000) summing to about `total` points, on
    walls seen from poses along a loop."""
    rng = np.random.default_rng(seed)
    sizes = rng.integers(0, 2 * total // n, n)
    sizes[:3] = [0, 3, 7000 if total > 20000 else 3]
    kfs = []
    for k, m in enumerate(sizes):
        pose = Pose2(*(rng.uniform(-1, 1, 3) * [40, 40, 3.1]))
        local = rng.normal(0, 8, (int(m), 2)) + rng.normal(0, 3, 2)
        kfs.append(_kf(np.round(local / 0.05).astype(np.float32) * np.float32(0.05), pose))
    rng.shuffle(kfs)
    return kfs


@pytest.fixture(scope="module")
def map_keyframes():
    world, kf, poses = synth.make_map_cloud(216000, seed=10)
    kfs = []
    for k, (x, y, t) in enumerate(poses):
        c, s = np.cos(t), np.sin(t)
        kfs.append(_kf(((world[kf == k] - [x, y]) @ np.array([[c, -s], [s, c]])).astype(np.float32), Pose2(x, y, t)))
    kfs[5].points = np.zeros((0, 2), np.float32)
    return kfs


def _selections(n):
    return {"all": None, "ascending": list(range(0, n, 3)), "descending": list(range(n - 1, -1, -2)),
            "repeated": [1, 1, 0, n - 1, 1, 0], "negative": [-1, -n, 2, -3], "empty": [], "empty_clouds": [0, 0],
            "thousands": list(np.random.default_rng(n).integers(-n, n, 2000))}


@pytest.mark.parametrize("size", ["below_cta", "above_cta", "map"])
def test_random_sets_equal_host_path(gpu_ctx, size, map_keyframes):
    """Totals below and above the one-CTA down-sample limit (13 880 points) and at map size; ref_frame None / int /
    Pose2; keys on and off; every kind of selection."""
    if size == "map":
        kfs = map_keyframes
    else:
        kfs = _random_keyframes(40, 6000 if size == "below_cta" else 60000, seed=len(size))
    res, host = _pair(kfs)
    n = len(kfs)
    empty = next(i for i, k in enumerate(kfs) if len(k.points) == 0)
    for name, frames in _selections(n).items():
        if name == "empty_clouds":
            frames = [empty, empty - n]
        for ref in (None, n // 2, Pose2(3.0, -2.0, 0.7)):
            for keys in (False, True):
                got = res.get_points(frames, ref, keys)
                assert _same(got, host.get_points(frames, ref, keys)), (size, name, ref, keys)
    # the oracle chain on two calls (it is the slow side at map size)
    ref_pose = kfs[-1].pose
    assert _same(res.get_points(None, n - 1, True), _oracle(kfs, range(n), ref_pose, True))
    assert _same(res.get_points(_selections(n)["negative"], None), _oracle(kfs, _selections(n)["negative"], None, False))
    assert res.keyframes.map.size == (n, sum(len(k.points) for k in kfs))


def test_pose_updates_follow_without_upload(gpu_ctx, map_keyframes):
    kfs = [_kf(k.points, k.pose) for k in map_keyframes]
    res, host = _pair(kfs)
    first = res.get_points(None, None, True)
    size = res.keyframes.map.size
    rng = np.random.default_rng(4)
    for kf in kfs:   # an ISAM2 update moves every pose a little
        kf.pose = kf.pose.compose(Pose2(*(rng.normal(0, 1, 3) * [0.05, 0.05, 0.002])))
    n = len(kfs)
    for frames, ref in ((None, None), (list(range(n - 8)), n - 1), (list(range(n - 1, n - 6, -1)), n - 2)):
        got = res.get_points(frames, ref, True)
        assert _same(got, host.get_points(frames, ref, True))
    assert not np.array_equal(res.get_points(None, None, True)[0][:100], first[0][:100])
    assert res.keyframes.map.size == size       # nothing was uploaded again


def test_appends_across_calls_grow_the_arena(gpu_ctx):
    kfs = _random_keyframes(60, 9000, seed=21)
    res = SLAM()
    host = SLAM()
    host.keyframes = []
    res.keyframes.map = KeyframeMap(_lib.default_context(), capacity=1000)   # a small first arena: several doublings
    for i in range(0, 60, 7):
        for kf in kfs[i:i + 7]:
            res.keyframes.append(kf)
            host.keyframes.append(kf)
        n = len(res.keyframes)
        assert _same(res.get_points(None, None, True), host.get_points(None, None, True)), i
        assert _same(res.get_points(range(n - 1, -1, -1), 0), host.get_points(range(n - 1, -1, -1), 0)), i
    assert res.keyframes.map.size == (60, sum(len(k.points) for k in kfs))
    # a replaced .points array is picked up (new slot), the old contents no longer used
    res.keyframes[4].points = res.keyframes[4].points[::2] + np.float32(1.0)
    assert _same(res.get_points(None, 2, True), host.get_points(None, 2, True))
    assert res.keyframes.map.size[0] == 61


def test_append_from_front_end_equals_host_copies(gpu_ctx):
    from oracle import featx_ref
    from sonar_slam_b200 import pipeline
    d = synth.make_trajectory_frames(12, seed=3)
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(gpu_ctx, maps, max_frames=16, min_points=30)
    fe.run_host(d["frames"].numpy(), d["poses_odom"])
    r = fe.results_dev()
    n, stride = 12, r["cloud_stride"]
    xy = gpu_ctx.to_host(r["cloud_xy"], (n, stride, 2), np.float32)
    cnt = gpu_ctx.to_host(r["cloud_count"], (n,), np.int32)
    assert cnt.min() > 0
    a, b = KeyframeMap(gpu_ctx), KeyframeMap(gpu_ctx)
    sa = a.append_dev(r["cloud_xy"], r["cloud_count"], stride, n)
    sb = b.append([xy[i, :cnt[i]] for i in range(n)])
    assert np.array_equal(sa, np.arange(n)) and np.array_equal(sb, sa) and np.array_equal(a.counts, cnt)
    assert a.size == b.size == (n, int(cnt.sum()))
    rng = np.random.default_rng(5)
    slots = np.r_[np.arange(n), rng.integers(0, n, 20)]
    poses = [Pose2(*p) for p in rng.uniform(-1, 1, (len(slots), 3)) * [20, 20, 3]]
    tf = np.array([[T[0, 0], T[0, 1], T[1, 0], T[1, 1], T[0, 2], T[1, 2]]
                   for T in (p.matrix().astype(np.float32) for p in poses)], np.float32)
    keys = rng.normal(0, 100, len(slots)).astype(np.float32)
    pa, ka = a.assemble(slots, keys, tf, 0.5, True)
    pb, kb = b.assemble(slots, keys, tf, 0.5, True)
    assert len(pa) > 100 and np.array_equal(pa, pb) and np.array_equal(ka, kb)
    want = _oracle({i: _kf(xy[s, :cnt[s]], p) for i, (s, p) in enumerate(zip(slots, poses))}, range(len(slots)), None,
                   True)
    assert np.array_equal(pa, want[0])
    a.close()
    b.close()


def test_device_flavour_feeds_match(gpu_ctx, map_keyframes):
    import torch
    from sonar_slam_b200 import ops
    kfs = map_keyframes
    res, host = _pair(kfs)
    n = len(kfs)
    frames = list(range(n - 8))
    km = res.keyframes.map = KeyframeMap(_lib.default_context())
    slots = res.keyframes.slots([kfs[i].points for i in frames])
    ref = kfs[-1].pose
    tf = np.array([[T[0, 0], T[0, 1], T[1, 0], T[1, 1], T[0, 2], T[1, 2]]
                   for T in (ref.between(kfs[i].pose).matrix().astype(np.float32) for i in frames)], np.float32)
    pts_d, keys_d = km.assemble(slots, np.array(frames, np.float32), tf, 0.5, True, device=True)
    want_pts, want_keys = host.get_points(frames, n - 1, True)
    assert pts_d.is_cuda and np.array_equal(pts_d.cpu().numpy(), want_pts)
    assert np.array_equal(keys_d.cpu().numpy(), want_keys[:, 0])
    src = transform_points(kfs[-1].points, Pose2())
    ids, dists = pcl.match(want_pts, src, 1, 0.5)
    dev = pts_d.device
    got = ops.match(pts_d, torch.tensor([0, len(pts_d)], dtype=torch.int32, device=dev),
                    torch.from_numpy(np.ascontiguousarray(src)).to(dev),
                    torch.tensor([0, len(src)], dtype=torch.int32, device=dev), len(pts_d), 0.5)
    torch.cuda.synchronize()
    assert (ids >= 0).sum() > 100
    assert np.array_equal(got["ids"].cpu().numpy(), ids[0]) and np.array_equal(got["dists"].cpu().numpy(), dists[0])


def test_argument_errors_before_any_launch(gpu_ctx):
    ctx = _lib.default_context()
    km = KeyframeMap(ctx)
    km.append([np.ones((10, 2), np.float32), np.zeros((4, 2), np.float32)])
    lib = ctx.lib
    launches = ctx.launches
    tf = np.tile(np.array([1, 0, 0, 1, 0, 0], np.float32), (2, 1))
    out = np.empty((14, 2), np.float32)
    m = np.zeros(1, np.int32)

    def assemble(slots, res=0.5, cap=14):
        slots = np.array(slots, np.int32)
        return lib.sfe_keyframe_map_assemble_host(km.handle, _lib.ptr(slots), None, _lib.ptr(tf), len(slots),
                                                  float(res), cap, _lib.ptr(out), None, _lib.ptr(m))

    assert assemble([0, 2]) == -1 and "slot 2" in lib.sfe_last_error().decode()
    assert assemble([-1, 0]) == -1
    assert assemble([0, 1], res=0.0) == -1 and assemble([0, 1], res=-0.5) == -1
    assert assemble([0, 1], res=float("nan")) == -1
    assert assemble([0, 1], cap=13) == -3
    counts = np.array([3, -1], np.int32)
    pts = np.zeros((3, 2), np.float32)
    assert lib.sfe_keyframe_map_append_host(km.handle, _lib.ptr(pts), _lib.ptr(counts), 2, None) == -1
    assert ctx.launches == launches and km.size == (2, 14)
    with pytest.raises(IndexError):
        km.assemble([0, 5], None, tf, 0.5, False)
    with pytest.raises(_lib.SonarFEError, match="resolution"):
        km.assemble([0, 1], None, tf, 0.0, False)
    with pytest.raises(ValueError):
        km.append([np.zeros((3, 3), np.float32)])
    assert ctx.launches == launches
    assert assemble([0, 1]) == 0 and m[0] == 2 and ctx.launches > launches
    km.close()
