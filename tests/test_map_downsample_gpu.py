"""GPU: pcl.downsample / ops.downsample on whole-map clouds -- sizes above what one CTA's shared memory holds run on
the grid-wide path -- compared exactly (indices, order, float32 points, counts) with the CPU oracle."""
import functools

import numpy as np
import pytest

from oracle import oracle as orc
from sonar_slam_b200 import synth

pytestmark = pytest.mark.gpu

RESOLUTIONS = (0.5, 0.13, 7.0)


DSF_STATIC_SMEM = 8624  # static shared memory of cloud.cu's downsample_cta_kernel<512, false> (tools/ptxas_table.py)


def _cta_limit():
    """Largest cloud the one-CTA kernel lays out in shared memory (cloud.cu, downsample_cta_limit): the largest n
    whose layout (dsf_layout: two 16-bit index lists, 32-bit keys, head bits and float2 points, each array 16-byte
    aligned) fits the device's opt-in shared memory less the kernel's static shared memory."""
    import torch
    budget = torch.cuda.get_device_properties(0).shared_memory_per_block_optin - DSF_STATIC_SMEM

    def a16(x):
        return (x + 15) // 16 * 16

    def total(n):
        return a16(4 * n) + a16(4 * n) + a16(4 * (n // 32 + 1)) + 8 * n

    n = min(budget * 8 // 129, 32 * 512 - 1)
    while n > 0 and total(n) > budget:
        n -= 1
    return n


@functools.lru_cache(maxsize=None)
def _map(n, seed=1):
    return synth.make_map_cloud(n, seed=seed)[0]


def _check(pts, res):
    from sonar_slam_b200.bruce_slam import pcl
    keys = np.arange(len(pts), dtype=np.float32)[:, None]
    got, gk = pcl.downsample(pts, keys, res)
    want, widx = orc.downsample(pts, res)
    assert len(got) == len(want), (len(pts), res)
    assert np.array_equal(gk[:, 0].astype(np.int64), widx), (len(pts), res)
    assert got.dtype == np.float32 and np.array_equal(got, want), (len(pts), res)
    assert np.array_equal(pcl.downsample(pts, res), want)


def _uniform(n, seed=2):
    return np.random.default_rng(seed).uniform(0, 350, (n, 2)).astype(np.float32)


def _single_leaf(n=20000, seed=3):
    return np.random.default_rng(seed).uniform(10.0, 10.5, (n, 2)).astype(np.float32)


def _lattice():
    """Every point on a node centre of some level: a 0.25 m lattice over [0, 64]^2 (exact binary fractions), a
    bounding square of radius 32 whose centres are multiples of 0.25 down to depth 7 -- the `x > cx` boundary."""
    g = np.arange(257, dtype=np.float32) * 0.25
    x, y = np.meshgrid(g, g)
    return np.c_[x.ravel(), y.ravel()].astype(np.float32)


def _deep(res, seed=4):
    """Two dense blobs (20 leaves wide) 0.75 * res * 2^15 apart: the tree is 15 levels deep, the most the device path
    builds."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(0, 20 * res, (60000, 2))
    b = rng.uniform(0, 20 * res, (60000, 2)) + 0.75 * res * 2 ** 15
    return np.concatenate([a, b]).astype(np.float32)


CLOUDS = {
    "map_200k": lambda res: _map(200000),
    "map_1M": lambda res: _map(1000000, seed=5),
    "uniform_1M": lambda res: _uniform(1000000),
    "leaf_20k": lambda res: _single_leaf(),
    "node_centres": lambda res: _lattice(),
    "depth_15": _deep,
}


@pytest.mark.parametrize("res", RESOLUTIONS)
@pytest.mark.parametrize("name", list(CLOUDS))
def test_single_cloud_equals_oracle(gpu_ctx, name, res):
    _check(CLOUDS[name](res), res)


def test_one_point_repeated_is_one_leaf(gpu_ctx):
    from sonar_slam_b200.bruce_slam import pcl
    pts = np.repeat(np.float32([[3.25, -7.5]]), 100000, 0)
    keys = np.arange(len(pts), dtype=np.float32)[:, None]
    for res in RESOLUTIONS:
        got, gk = pcl.downsample(pts, keys, res)
        assert np.array_equal(got, pts[:1]) and np.array_equal(gk, keys[:1])


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_sizes_around_the_shared_memory_limit(gpu_ctx, delta):
    """limit - 1 and limit run in the one-CTA kernel with its layout in shared memory (1 launch), limit + 1 on the
    grid-wide path (the one-CTA launch for the small class plus 8); all three equal the oracle."""
    from sonar_slam_b200 import _lib
    ctx = _lib.default_context()
    pts = _map(200000)[: _cta_limit() + delta]
    for res in RESOLUTIONS:
        n0 = ctx.launches
        _check(pts, res)
        per_call = (ctx.launches - n0) // 2  # _check calls pcl.downsample twice
        assert per_call == (9 if delta > 0 else 1), (delta, per_call)


def test_keyed_overload_returns_the_kept_keys(gpu_ctx):
    from sonar_slam_b200.bruce_slam import pcl
    pts, kf, _ = synth.make_map_cloud(200000, seed=6)
    keys = kf.astype(np.float64)[:, None]
    got, gk = pcl.downsample(pts, keys, 0.5)
    want, widx = orc.downsample(pts, 0.5)
    assert np.array_equal(got, want) and np.array_equal(gk, keys[widx].astype(np.float32))


def test_mixed_batch_small_and_map_sized_clouds(gpu_ctx):
    """30 small clouds and clouds of 100 k and 300 k points in one sfe_downsample_dev call (n_max = 300 k): each
    equals the oracle at its own offset, and the small ones equal a batch of only the small clouds (one-CTA path)."""
    import torch
    from sonar_slam_b200 import ops
    rng = np.random.default_rng(7)
    small = [synth.sample_walls(rng, synth.make_walls(rng, 6, 40.0), int(n), 0.05).astype(np.float32)
             for n in rng.integers(1, 1500, 30)]
    big = [_map(100000, seed=8), _map(300000, seed=9)]
    clouds = small[:12] + [big[0]] + small[12:25] + [big[1]] + small[25:]
    n_max = max(len(c) for c in clouds)
    assert n_max == 300000

    def pack(cl):
        off = np.zeros(len(cl) + 1, np.int64)
        off[1:] = np.cumsum([len(c) for c in cl])
        return (torch.from_numpy(np.concatenate(cl)).cuda(), torch.from_numpy(off.astype(np.int32)).cuda(), off)

    pts, off, off_h = pack(clouds)
    spts, soff, soff_h = pack(small)
    for res in (0.5, 0.13):
        out = ops.downsample(pts, off, n_max, res)
        alone = ops.downsample(spts, soff, max(len(c) for c in small), res)
        torch.cuda.synchronize()
        cnt, idx, opts = out["count"].cpu().numpy(), out["idx"].cpu().numpy(), out["pts"].cpu().numpy()
        scnt, sidx, sopts = alone["count"].cpu().numpy(), alone["idx"].cpu().numpy(), alone["pts"].cpu().numpy()
        si = 0
        for c, cl in enumerate(clouds):
            want, widx = orc.downsample(cl, res)
            s = off_h[c]
            assert cnt[c] == len(want), (c, res)
            assert np.array_equal(idx[s:s + cnt[c]], widx) and np.array_equal(opts[s:s + cnt[c]], want), (c, res)
            if len(cl) < 100000:
                t = soff_h[si]
                assert scnt[si] == cnt[c]
                assert np.array_equal(sidx[t:t + cnt[c]], idx[s:s + cnt[c]])
                assert np.array_equal(sopts[t:t + cnt[c]], opts[s:s + cnt[c]])
                si += 1


def test_slam_get_points_at_map_size(gpu_ctx):
    """SLAM.get_points over ~600 keyframes (> 200 k points), against the reference's lines (slam.py:229-292)
    restated with numpy and the oracle's down-sample."""
    from sonar_slam_b200.bruce_slam.slam import SLAM, Pose2, transform_points
    world, kf, poses = synth.make_map_cloud(216000, seed=10)

    class KF:  # the two Keyframe fields get_points reads
        def __init__(self, points, pose):
            self.points, self.pose = points, pose

    slam = SLAM()
    for k, (x, y, t) in enumerate(poses):
        c, s = np.cos(t), np.sin(t)
        local = (world[kf == k] - [x, y]) @ np.array([[c, -s], [s, c]])  # R^T (p - t), row vectors
        slam.keyframes.append(KF(local.astype(np.float32), Pose2(x, y, t)))
    assert len(slam.keyframes) == 600
    # get_points(None, None, True): every keyframe in world coordinates, with its key
    parts = [np.c_[transform_points(k.points, k.pose), i * np.ones((len(k.points), 1))]
             for i, k in enumerate(slam.keyframes)]
    allp = np.concatenate(parts)
    want, widx = orc.downsample(np.ascontiguousarray(allp[:, :2], np.float32), slam.point_resolution)
    got, keys = slam.get_points(None, None, True)
    assert np.array_equal(got, want) and np.array_equal(keys[:, 0], allp[widx, 2].astype(np.float32))
    # get_points(frames, ref_frame): all but the last 8 keyframes, relative to the last one
    frames = list(range(len(slam.keyframes) - 8))
    ref = slam.keyframes[-1].pose
    want2, _ = orc.downsample(np.concatenate([transform_points(slam.keyframes[i].points, ref.between(slam.keyframes[i].pose))
                                              for i in frames]).astype(np.float32), slam.point_resolution)
    assert np.array_equal(slam.get_points(frames, len(slam.keyframes) - 1), want2)
