"""GPU: pcl.remove_outlier / ops.remove_outlier on whole-map clouds -- sizes above what one CTA's shared memory holds
run in the map class (the map grid of pcl.match in global memory) -- compared exactly (kept count, kept indices,
float32 points) with the CPU oracle."""
import functools

import numpy as np
import pytest

from oracle import oracle as orc
from sonar_slam_b200 import synth

pytestmark = pytest.mark.gpu

PARAMS = ((1.0, 5), (5.0, 20), (0.3, 1))
MAP_LAUNCHES = 13  # the one-CTA launch for the small class, map_build's 9, the count kernel, the scan, the output


def _cta_limit():
    """Largest cloud remove_outlier_kernel lays out: 8 bytes per point, a 16-bit cell table of two cells per point
    (256 to 16 384 cells, two per 32-bit word, plus one word) and 16 bytes, within the device's opt-in shared memory less
    4 KiB (cloud.cu, remove_outlier_cta_smem), and at most 65 535 points."""
    import torch
    budget = torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 4096

    def smem(n):
        mc = min(max(2 * n, 256), 16384)
        return 8 * n + 4 * ((mc + 2) // 2 + 1) + 16

    lo, hi = 0, 65535
    while lo < hi:
        mid = lo + (hi - lo + 1) // 2
        lo, hi = (mid, hi) if smem(mid) <= budget else (lo, mid - 1)
    return lo


@functools.lru_cache(maxsize=None)
def _map(n, seed=1):
    return synth.make_map_cloud(n, seed=seed)[0]


def _host(pts, radius, min_points):
    """sfe_remove_outlier_host, the entry point pcl.remove_outlier calls, with the kept indices too."""
    from sonar_slam_b200 import _lib
    ctx = _lib.default_context()
    pts = np.ascontiguousarray(pts, np.float32)
    out = np.empty_like(pts)
    idx = np.empty(len(pts), np.int32)
    m = np.zeros(1, np.int32)
    _lib.check(ctx.lib.sfe_remove_outlier_host(ctx.handle, _lib.ptr(pts), len(pts), pts.shape[1], float(radius),
                                               int(min_points), _lib.ptr(out), _lib.ptr(idx), _lib.ptr(m)),
               "remove_outlier")
    k = int(m[0])
    return out[:k], idx[:k]


def _check(pts, radius, min_points, want=None):
    from sonar_slam_b200.bruce_slam import pcl
    want, keep = want if want is not None else orc.remove_outlier(pts, radius, min_points)
    got, idx = _host(pts, radius, min_points)
    assert len(got) == len(want), (len(pts), radius, min_points, len(got), len(want))
    assert np.array_equal(idx, np.flatnonzero(keep)), (len(pts), radius, min_points)
    assert got.dtype == np.float32 and np.array_equal(got, want), (len(pts), radius, min_points)
    assert np.array_equal(pcl.remove_outlier(pts, radius, min_points), want)
    return want, keep


def _uniform(n, seed=2):
    return np.random.default_rng(seed).uniform(0, 350, (n, 2)).astype(np.float32)


def _blob(n=25600, seed=3):
    """One dense blob (0.5 m across, just above the one-CTA limit): at 1 m and 5 m every point has every other point
    as a neighbour, so the device stops counting early everywhere while the oracle counts all n."""
    return np.random.default_rng(seed).uniform(10.0, 10.5, (n, 2)).astype(np.float32)


def _sparse(seed=4):
    """Isolated points on a 2 m lattice (no neighbour within 1 m) plus a few dense clusters."""
    rng = np.random.default_rng(seed)
    g = np.arange(200, dtype=np.float32) * 2.0
    x, y = np.meshgrid(g, g)
    lattice = np.c_[x.ravel(), y.ravel()]
    clusters = [rng.normal(c, 0.2, (2000, 2)) for c in rng.uniform(0, 400, (5, 2))]
    pts = np.concatenate([lattice] + clusters).astype(np.float32)
    return pts[rng.permutation(len(pts))]


def _line(n=30000, seed=5):
    """A 16 km line: the map grid's cell table cap and a very elongated bounding box."""
    rng = np.random.default_rng(seed)
    x = np.sort(rng.uniform(0, 16000, n))
    return np.c_[x, 0.01 * rng.standard_normal(n) - 250.0].astype(np.float32)


# The oracle counts every neighbour of every point (about 250 per 0.5 m cell on the walls of a synth map), so the
# clouds shrink as the radius grows to keep its time to seconds: the names give the size at the smallest radius.
CLOUDS = {
    "map_200k": lambda r: _map(200000 if r <= 1.0 else 60000),
    "map_1M": lambda r: _map({0.3: 1000000, 1.0: 400000}.get(r, 100000), seed=5),
    "uniform_1M": lambda r: (_uniform(1000000) * (1.0 if r <= 1.0 else 3.0)).astype(np.float32),
    "blob": lambda r: _blob(),
    "sparse_lattice_clusters": lambda r: _sparse(),
    "line_16km": lambda r: _line(),
}


@functools.lru_cache(maxsize=None)
def _oracle(name, radius, min_points):
    if name == "blob" and radius > 1.0:  # every pair is within 0.71 m: the same counts (all n) as at 1 m
        return _oracle(name, 1.0, 5)
    return orc.remove_outlier(CLOUDS[name](radius), radius, min_points)


@pytest.mark.parametrize("radius,min_points", PARAMS)
@pytest.mark.parametrize("name", list(CLOUDS))
def test_single_cloud_equals_oracle(gpu_ctx, name, radius, min_points):
    pts = CLOUDS[name](radius)
    assert len(pts) > _cta_limit()
    _check(pts, radius, min_points, _oracle(name, radius, min_points))


def test_exact_radius_ties(gpu_ctx):
    """A 0.25 m lattice (exact binary fractions): many distances equal the radius exactly, and `<=` decides.  An
    interior point has 5, 13 and 29 points (itself included) within 0.25, 0.5 and 0.75 m, 4 of them at exactly that
    distance: min_points 4, 12 and 28 keep the interior only through the ties, 5, 13 and 29 keep nothing."""
    g = np.arange(240, dtype=np.float32) * 0.25
    x, y = np.meshgrid(g, g)
    pts = np.c_[x.ravel(), y.ravel()].astype(np.float32)
    assert len(pts) > _cta_limit()
    for radius, min_points in ((0.5, 12), (0.5, 13), (0.25, 4), (0.25, 5), (0.75, 28), (0.75, 29)):
        want, keep = _check(pts, radius, min_points)
        # the ties matter: the same call with a radius a hair smaller keeps fewer points
        if keep.any():
            assert orc.remove_outlier(pts, np.nextafter(radius, 0), min_points)[1].sum() < keep.sum()


def test_min_points_edge_values(gpu_ctx):
    pts = _map(200000)
    for min_points in (0, 1, 10 ** 6):
        want, keep = _check(pts, 1.0, min_points)
        if min_points == 0:
            assert keep.all()
        if min_points == 10 ** 6:
            assert not keep.any()


def test_three_column_map(gpu_ctx):
    """Map points spread over 20 m in z: at 1 m and 40 points the z spread decides which survive (a few thousand
    fewer than the 2-column call keeps); with z = 0 the same cloud equals the 2-column call."""
    rng = np.random.default_rng(6)
    xy = _map(200000, seed=7)
    p3 = np.c_[xy, rng.uniform(0, 20.0, len(xy))].astype(np.float32)
    want3, keep3 = _check(p3, 1.0, 40)
    _, keep2 = orc.remove_outlier(xy, 1.0, 40)
    assert keep3.sum() < keep2.sum()  # the z spread removes points the 2-column call keeps
    flat = np.c_[xy, np.zeros(len(xy))].astype(np.float32)
    got_flat, idx_flat = _host(flat, 1.0, 40)
    got2, idx2 = _host(xy, 1.0, 40)
    assert np.array_equal(idx_flat, idx2) and np.array_equal(got_flat[:, :2], got2)
    assert np.array_equal(idx2, np.flatnonzero(keep2))


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_sizes_around_the_one_cta_limit(gpu_ctx, delta):
    """limit - 1 and limit run in remove_outlier_kernel (1 launch), limit + 1 in the map class; all equal the oracle."""
    from sonar_slam_b200 import _lib
    ctx = _lib.default_context()
    pts = _map(200000)[: _cta_limit() + delta]
    for radius, min_points in PARAMS:
        want = orc.remove_outlier(pts, radius, min_points)
        n0 = ctx.launches
        got, idx = _host(pts, radius, min_points)
        assert ctx.launches - n0 == (MAP_LAUNCHES if delta > 0 else 1), (delta, ctx.launches - n0)
        assert np.array_equal(got, want[0]) and np.array_equal(idx, np.flatnonzero(want[1])), (delta, radius)


def test_mixed_batch_small_and_map_sized_clouds(gpu_ctx):
    """About 30 small clouds, map clouds of 100 k and 300 k points and an empty cloud in one sfe_remove_outlier_dev call
    (n_max = 300 k): each equals the oracle at its own offset, and the small ones equal a batch of only the small clouds
    (one-CTA path)."""
    import torch
    from sonar_slam_b200 import ops
    rng = np.random.default_rng(8)
    small = [synth.sample_walls(rng, synth.make_walls(rng, 6, 40.0), int(n), 0.05).astype(np.float32)
             for n in rng.integers(1, 1500, 30)]
    big = [_map(100000, seed=8), _map(300000, seed=9)]
    empty = np.zeros((0, 2), np.float32)
    clouds = small[:12] + [big[0]] + small[12:20] + [empty] + small[20:25] + [big[1]] + small[25:]
    n_max = max(len(c) for c in clouds)
    assert n_max == 300000

    def pack(cl):
        off = np.zeros(len(cl) + 1, np.int64)
        off[1:] = np.cumsum([len(c) for c in cl])
        return (torch.from_numpy(np.concatenate(cl)).cuda(), torch.from_numpy(off.astype(np.int32)).cuda(), off)

    pts, off, off_h = pack(clouds)
    spts, soff, soff_h = pack(small)
    for radius, min_points in ((1.0, 5), (0.3, 1)):  # (5 m: the oracle would take most of a minute here)
        out = ops.remove_outlier(pts, off, n_max, radius, min_points)
        alone = ops.remove_outlier(spts, soff, max(len(c) for c in small), radius, min_points)
        torch.cuda.synchronize()
        cnt, idx, opts = out["count"].cpu().numpy(), out["idx"].cpu().numpy(), out["pts"].cpu().numpy()
        scnt, sidx, sopts = alone["count"].cpu().numpy(), alone["idx"].cpu().numpy(), alone["pts"].cpu().numpy()
        si = 0
        for c, cl in enumerate(clouds):
            s = off_h[c]
            if len(cl) == 0:
                assert cnt[c] == 0
                continue
            want, keep = orc.remove_outlier(cl, radius, min_points)
            assert cnt[c] == len(want), (c, radius)
            assert np.array_equal(idx[s:s + cnt[c]], np.flatnonzero(keep)), (c, radius)
            assert np.array_equal(opts[s:s + cnt[c]], want), (c, radius)
            if len(cl) < 100000:
                t = soff_h[si]
                assert scnt[si] == cnt[c]
                assert np.array_equal(sidx[t:t + cnt[c]], idx[s:s + cnt[c]])
                assert np.array_equal(sopts[t:t + cnt[c]], opts[s:s + cnt[c]])
                si += 1


def test_mapping_occupancy_grid_call(gpu_ctx):
    """The reference's map clean-up (mapping.py:365-372 and :392-398): a keyed map cloud [x, y, z, key], the points of
    all frames or of a frame subset, then pcl.remove_outlier(points[:, :2], 5.0, 20)."""
    from sonar_slam_b200.bruce_slam import pcl
    world, kf, _ = synth.make_map_cloud(100000, seed=10)
    point_cloud = np.c_[world, np.zeros(len(world)), kf].astype(np.float32)
    keys = np.uint32(point_cloud[:, 3])
    subsets = {"all": None, "every_third": range(0, int(keys.max()) + 1, 3)}
    for name, frames in subsets.items():
        points = point_cloud[:, :2]
        if frames is not None:
            points = np.concatenate([np.zeros((0, 2))] + [point_cloud[keys == k, :2] for k in frames])
        assert len(points) > _cta_limit()
        want, _ = orc.remove_outlier(np.ascontiguousarray(points[:, :2], np.float32), 5.0, 20)
        assert np.array_equal(pcl.remove_outlier(points[:, :2], 5.0, 20), want), name
