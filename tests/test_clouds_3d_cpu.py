"""CPU-only: the 3-D cloud oracles (oracle/cloud3_ref.c orc_downsample3 / orc_match_brute3 /
orc_match_knn3) against independent restatements, the z = 0 equivalence with the 2-D oracles, and the argument checks
`bruce_slam.pcl` / `ops` make on [N,3] clouds before any device work."""
import numpy as np
import pytest

from oracle import cloud3_ref as c3
from oracle.cloud3_ref import octree_literal
from oracle import knn_ref
from oracle import oracle as orc

F = np.float32


def _random(n, seed, spread=(20.0, 20.0, 5.0)):
    return (np.random.default_rng(seed).uniform(0, 1, (n, 3)) * np.asarray(spread)).astype(F)


def _lattice():
    g = np.arange(9, dtype=F) * F(0.5)  # exact binary fractions on node centres: the `x > cx` boundaries
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    return np.c_[x.ravel(), y.ravel(), z.ravel()].astype(F)


CASES = {
    "random": (_random(1500, 1), 1.0),
    "random_fine": (_random(800, 2, (3.0, 2.0, 4.0)), 0.1),
    "lattice_ties": (_lattice(), 0.5),
    "lattice_coarse": (_lattice(), 1.3),
    "z_line": (np.c_[np.full(300, 1.5), np.full(300, -2.0), np.linspace(0, 30, 300)].astype(F), 0.7),
    "coincident": (np.tile(F([[3.25, -1.0, 7.5]]), (150, 1)), 0.5),
    "single": (F([[1.0, 2.0, 3.0]]), 0.5),
    "duplicates": (np.repeat(_random(200, 3), 3, axis=0), 0.8),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_octree_oracle_equals_literal_recursive_octree(name):
    pts, res = CASES[name]
    got_pts, got_idx = c3.downsample3(pts, res)
    want = octree_literal(pts, res)
    assert np.array_equal(got_idx.astype(np.int64), want), name
    assert np.array_equal(got_pts, pts[want])
    if name == "coincident":
        assert len(got_idx) == 1 and got_idx[0] == 0  # one leaf at the root, first minimum wins
    if name == "z_line":  # only bit 2 ever splits: leaves come out in ascending z
        assert np.all(np.diff(pts[got_idx, 2]) > 0)


def test_octree_oracle_empty_input():
    got_pts, got_idx = c3.downsample3(np.zeros((0, 3), F), 0.5)
    assert got_pts.shape == (0, 3) and len(got_idx) == 0


def test_octree_depth_cap_changes_only_clouds_deeper_than_it():
    pts, res = CASES["random"]
    assert np.array_equal(octree_literal(pts, res, max_depth=15), octree_literal(pts, res))
    # two clusters 2^17 resolutions apart: 18 levels uncapped; the cut at 15 merges what lies below it
    rng = np.random.default_rng(9)
    deep = np.concatenate([rng.uniform(0, 4, (60, 3)), rng.uniform(0, 4, (60, 3)) + 2.0 ** 17]).astype(F)
    assert not np.array_equal(octree_literal(deep, 1.0, max_depth=15), octree_literal(deep, 1.0))
    assert np.array_equal(c3.downsample3(deep, 1.0)[1].astype(np.int64), octree_literal(deep, 1.0))


@pytest.mark.parametrize("name", ["random", "random_fine", "lattice_ties", "duplicates"])
def test_octree_with_z_zero_equals_the_quadtree(name):
    pts, res = CASES[name]
    flat = pts.copy()
    flat[:, 2] = 0
    _, i3 = c3.downsample3(flat, res)
    _, i2 = orc.downsample(flat[:, :2], res)
    assert np.array_equal(i3, i2)


def _brute_knn3(ref, q, knn, max_dist):
    """numpy statement of the 3-D kNN rule: float32 (dx*dx + dy*dy) + dz*dz, d <= max_dist^2, ties -> lower index."""
    ref, q = np.asarray(ref, F), np.asarray(q, F)
    d = q[:, None, :] - ref[None, :, :]
    d2 = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(F)
    md2 = F(F(max_dist) * F(max_dist))
    ids = np.full((knn, len(q)), -1, np.int32)
    out = np.full((knn, len(q)), np.inf, F)
    for i in range(len(q)):
        ok = np.nonzero(d2[i] <= md2)[0]
        order = ok[np.lexsort((ok, d2[i, ok]))][:knn]
        ids[:len(order), i] = order
        out[:len(order), i] = d2[i, order]
    return ids, out


@pytest.mark.parametrize("knn", [1, 2, 5, 16])
def test_knn3_oracle_equals_ckdtree_on_distinct_distances(knn):
    spatial = pytest.importorskip("scipy.spatial")
    rng = np.random.default_rng(knn)
    ref = rng.uniform(0, 10, (3000, 3)).astype(F)
    q = rng.uniform(-1, 11, (400, 3)).astype(F)
    ids, d = c3.match_knn3(ref, q, knn, 1.5)
    dd, ii = spatial.cKDTree(ref.astype(np.float64)).query(q.astype(np.float64), k=knn, distance_upper_bound=1.5)
    dd, ii = dd.reshape(len(q), knn).T, ii.reshape(len(q), knn).T
    found = np.isfinite(dd)
    # float32 and float64 distances may disagree on the radius only within rounding; keep queries away from it
    clear = np.all(np.abs(dd - 1.5) > 1e-4, axis=0) & np.all(np.abs(np.sqrt(d.astype(np.float64)) - 1.5) > 1e-4, axis=0)
    assert clear.sum() > 300
    assert np.array_equal(np.where(found, ii, -1)[:, clear], ids[:, clear])
    np.testing.assert_allclose(np.sqrt(d[found & (ids >= 0)]), dd[found & (ids >= 0)], rtol=1e-5)


@pytest.mark.parametrize("knn", [1, 2, 5, 16])
def test_knn3_oracle_equals_brute_force_with_ties(knn):
    g = np.arange(4, dtype=F)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    ref = np.concatenate([np.c_[x.ravel(), y.ravel(), z.ravel()]] * 2).astype(F)  # every point twice: exact ties
    q = np.concatenate([ref[:20] + F(0.5), ref[:10], F([[9, 9, 9], [1.5, 1.5, -1.0]])]).astype(F)
    for md in (1.0, 0.8660254, 2.0, 0.0):  # 0.866...: exactly at distance sqrt(0.75) from the half-offset queries
        ids, d = c3.match_knn3(ref, q, knn, md)
        wi, wd = _brute_knn3(ref, q, knn, md)
        assert np.array_equal(ids, wi) and np.array_equal(d, wd), (knn, md)
        one, d1 = c3.match3(ref, q, md)
        assert np.array_equal(one[0], ids[0]) and np.array_equal(d1[0], d[0])


@pytest.mark.parametrize("knn", [1, 3, 16])
def test_knn3_with_z_zero_equals_2d(knn):
    rng = np.random.default_rng(7)
    ref = np.c_[rng.uniform(0, 5, (500, 2)), np.zeros(500)].astype(F)
    q = np.c_[rng.uniform(0, 5, (100, 2)), np.zeros(100)].astype(F)
    i3, d3 = c3.match_knn3(ref, q, knn, 0.7)
    i2, d2 = knn_ref.match_knn(ref[:, :2], q[:, :2], knn, 0.7)
    assert np.array_equal(i3, i2) and np.array_equal(d3, d2)
    m3, e3 = c3.match3(ref, q, 0.7)
    m2, e2 = orc.match(ref[:, :2], q[:, :2], 0.7, brute=True)
    assert np.array_equal(m3, m2) and np.array_equal(e3, e2)


def test_3d_argument_checks_happen_before_any_device_work():
    from sonar_slam_b200.bruce_slam import pcl
    p3, p2 = np.zeros((4, 3), F), np.zeros((3, 2), F)
    for fn in (lambda r, q: pcl.match(r, q, 1, 0.5), lambda r, q: pcl.match_knn(r, q, 3, 0.5)):
        with pytest.raises(TypeError):
            fn(p3, p2)  # libnabo rejects a query whose dimension is not the tree's
        with pytest.raises(TypeError):
            fn(p2, np.zeros((3, 3), F))
        with pytest.raises(TypeError):
            fn(np.zeros((4, 4), F), np.zeros((3, 4), F))
    with pytest.raises(TypeError):
        pcl.downsample(np.zeros((4, 4), F), 0.5)
    with pytest.raises(TypeError):
        pcl.downsample(p3, np.zeros((5, 2), F), 0.5)  # one descriptor row per point
    assert pcl.downsample(np.zeros((0, 3), F), 0.5).shape == (0, 3)
    pe, de = pcl.downsample(np.zeros((0, 3), F), np.zeros((0, 4), F), 0.5)
    assert pe.shape == (0, 3) and de.shape == (0, 4)
    ids, d = pcl.match(p3, np.zeros((0, 3), F), 1, 0.5)
    assert ids.shape == (1, 0) and d.shape == (1, 0)
    ids, d = pcl.match_knn(p3, np.zeros((0, 3), F), 7, 0.5)
    assert ids.shape == (7, 0) and ids.dtype == np.int32 and d.dtype == np.float32


def test_ops_match_rejects_mismatched_columns_before_any_device_work():
    import torch
    from sonar_slam_b200 import ops
    off = torch.tensor([0, 2], dtype=torch.int32)
    with pytest.raises(ValueError, match="2 or 3 columns"):
        ops.match(torch.zeros(2, 3), off, torch.zeros(2, 2), off, 2, 0.5)
    with pytest.raises(ValueError, match="2 or 3 columns"):
        ops.match(torch.zeros(2, 4), off, torch.zeros(2, 4), off, 2, 0.5, knn=2)
